// The plane fit of the point-cloud normals (point-cloud-utils_b200/csrc/plane_fit.h) built for the CPU, so
// tests/test_normals_conditioning.py can check it without a GPU.  The kernels feed it offsets the same way:
// scaled by pow2_scale of the largest |component|, pass after pass in one order.
// stdin: int64 rows, then per row int64 m and m * 3 float64 offsets; stdout: rows * 3 float64 normals.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "plane_fit.h"

int main() {
    int64_t rows = 0;
    if (fread(&rows, sizeof rows, 1, stdin) != 1) return 1;
    std::vector<double> off;
    for (int64_t r = 0; r < rows; ++r) {
        int64_t m = 0;
        if (fread(&m, sizeof m, 1, stdin) != 1) return 1;
        off.resize((size_t)(3 * m));
        if (m > 0 && fread(off.data(), sizeof(double), off.size(), stdin) != off.size()) return 1;
        double big = 0.0;
        for (double x : off) big = std::fmax(big, std::fabs(x));
        pcu::PlaneFit fit(pcu::pow2_scale(big));
        do {
            for (int64_t j = 0; j < m; ++j) fit.add(off[3 * j], off[3 * j + 1], off[3 * j + 2]);
        } while (fit.solve());
        double n[3];
        fit.normal(m, n);
        if (fwrite(n, sizeof(double), 3, stdout) != 3) return 1;
    }
    return 0;
}

// The reference's triangle-box test (src/common/tribox.h, included from the reference tree, not copied) behind a C
// entry point, driven by this file's own face / candidate loop: voxelize_triangle_mesh's test without its bindings.
// Built by oracle/voxelize_ref.py's build() into oracle/_ref/libpcu_ref_voxelize.so with the reference's flags
// (-O3 -msse3 -ffp-contract=off).
//
// full_x = 0: x runs over [inix, inix], the reference's loop (src/voxelize_triangle_mesh.cpp:40).
// full_x = 1: x runs over [inix, inox], as y and z do: what voxelize_triangle_mesh computes here.
// Voxel (i, j, k) is the box centred at origin + (i, j, k) * size with half-size size / 2 (:14, :42-44).
#include <algorithm>
#include <cmath>
#include <cstdint>

#include "common/tribox.h"

extern "C" {

// v: (nv, 3) fp64, f: (nf, 3) int64 (in range; the caller checks).  Writes up to `cap` accepted (i, j, k) triples to
// out (face by face, x, y, z loops as the reference nests them) and returns their total number.
int64_t pcu_ref_voxelize(const double* v, int64_t nv, const int64_t* f, int64_t nf, const double* origin, const double* size, int full_x,
                         int32_t* out, int64_t cap) {
    (void)nv;
    double half[3] = {size[0] / 2, size[1] / 2, size[2] / 2};
    int64_t count = 0;
    for (int64_t fi = 0; fi < nf; ++fi) {
        double c[3][3];
        for (int k = 0; k < 3; ++k)
            for (int a = 0; a < 3; ++a) c[k][a] = v[3 * f[3 * fi + k] + a];
        int ini[3], ino[3];
        for (int a = 0; a < 3; ++a) {
            const double mn = std::min(c[0][a], std::min(c[1][a], c[2][a]));
            const double mx = std::max(c[0][a], std::max(c[1][a], c[2][a]));
            ini[a] = static_cast<int>(std::floor((mn - origin[a]) / size[a]));
            ino[a] = static_cast<int>(std::ceil((mx - origin[a]) / size[a]));
        }
        const int x_end = full_x ? ino[0] : ini[0];
        for (int x = ini[0]; x <= x_end; ++x)
            for (int y = ini[1]; y <= ino[1]; ++y)
                for (int z = ini[2]; z <= ino[2]; ++z) {
                    const double pos[3] = {(double)x * size[0], (double)y * size[1], (double)z * size[2]};
                    double center[3] = {origin[0] + pos[0], origin[1] + pos[1], origin[2] + pos[2]};
                    double* tri[3] = {c[0], c[1], c[2]};
                    if (triBoxOverlap(center, half, tri)) {
                        if (count < cap) { out[3 * count] = x; out[3 * count + 1] = y; out[3 * count + 2] = z; }
                        ++count;
                    }
                }
    }
    return count;
}

}  // extern "C"

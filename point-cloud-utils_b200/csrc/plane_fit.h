// plane_fit.h -- the plane fit of the point-cloud normals (normals.cuh, row N1): the right singular vector of the
// smallest singular value of the (m, 3) matrix X whose rows are a neighbourhood's offsets.  Plain C++ that nvcc
// compiles for the device and any host compiler for the CPU, so the routine can be tested without a GPU.
//
// The caller feeds the offsets pass by pass, in the same order every pass:
//     PlaneFit f(scale);
//     do { for every offset: f.add(x, y, z); } while (f.solve());
//     f.normal(m, n);
// `scale` is a power of two with |scale * component| <= 1 for every offset (pow2_scale below): multiplying by it is
// exact, so the result does not depend on the cloud's scale and no square over- or underflows unless the offsets of
// one neighbourhood span more than ~2^500.
//
// Pass 1 accumulates S = (sX)^T (sX) and diagonalises it by cyclic Jacobi rotations, giving a basis V.  That basis is
// only as good as the squared condition number allows: S carries an error of ~u s1^2 in every entry, so the normal
// is off by ~u s1^2 / (s2^2 - s3^2) (s1 >= s2 >= s3 the singular values of X, u = 2^-53).  Every further pass rotates
// the offsets into V's basis, Y = sXV, and diagonalises Y^T Y, which is diagonal but for the rounding of the last
// pass: its entry (i, j) now carries an error of ~u s_i s_j instead of ~u s1^2, so the refined basis V W is as
// accurate as an SVD of X, ~u s1 / (s2 - s3).  Passes end when one turns the basis by less than 2^-26 (it started
// close enough that its own result is at that floor), after at most kMaxPasses.
//
// Rules where the fit is not defined:
//  - fewer than 3 offsets (k = 1 or 2): the zero vector, the oracle's choice of padding the thin V with zeros;
//  - X = 0 (a point duplicated at least k times): (0, 0, 1), the third column of the V = I that numpy's SVD returns;
//  - s2 = s3 exactly (e.g. an axis-aligned line): the first such axis of the basis -- any unit vector of that plane is
//    a right singular vector.
#pragma once
#include <cmath>

#ifdef __CUDACC__
#define PCU_HD __host__ __device__ __forceinline__
#else
#define PCU_HD inline
#endif

namespace pcu {

// 2^-e, where big = f 2^e with f in [0.5, 1): |scale * x| < 1 for |x| <= big.  big = 0 gives 1.
PCU_HD double pow2_scale(double big) {
    int e = 0;
    frexp(big, &e);
    return ldexp(1.0, -(e < -1021 ? -1021 : e));
}

// One Jacobi rotation annihilating a[p][q] of the symmetric 3 x 3 matrix a; w accumulates the rotations.  A pair is
// left alone once |a_pq| <= 2^-53 sqrt(a_pp a_qq): what remains turns its eigenvectors by at most
// u sqrt(a_pp a_qq) / |a_pp - a_qq| <= u s1 / (s2 - s3) / 2.  The test is relative, so a matrix scaled by any power
// of two takes the same rotations.  Returns whether it rotated.
template <int P, int Q>
PCU_HD bool jacobi_rotate(double (&a)[3][3], double (&w)[3][3]) {
    const double apq = a[P][Q];
    if (apq == 0.0 || apq * apq <= 0x1p-106 * (a[P][P] * a[Q][Q])) return false;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
    constexpr int R = 3 - P - Q;   // the third index
    const double app = a[P][P], aqq = a[Q][Q], arp = a[R][P], arq = a[R][Q];
    a[P][P] = app - t * apq;
    a[Q][Q] = aqq + t * apq;
    a[P][Q] = a[Q][P] = 0.0;
    a[R][P] = a[P][R] = c * arp - s * arq;
    a[R][Q] = a[Q][R] = s * arp + c * arq;
    for (int i = 0; i < 3; ++i) {
        const double wip = w[i][P], wiq = w[i][Q];
        w[i][P] = c * wip - s * wiq;
        w[i][Q] = s * wip + c * wiq;
    }
    return true;
}

struct PlaneFit {
    static constexpr int kMaxPasses = 4;
    double scale;
    double v[3][3];        // the basis so far (columns)
    double a[3][3];        // the last pass's diagonalised matrix
    double s00, s01, s02, s11, s12, s22;   // this pass's sums
    int pass;
    bool zero;             // X = 0

    PCU_HD explicit PlaneFit(double scale_) : scale(scale_), pass(0), zero(false) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) v[i][j] = a[i][j] = i == j ? 1.0 : 0.0;
        reset();
    }
    PCU_HD void reset() { s00 = s01 = s02 = s11 = s12 = s22 = 0.0; }

    // One offset: scaled, rotated into the basis (exactly the scaled offset in pass 1, where V = I), accumulated.
    PCU_HD void add(double x, double y, double z) {
        x *= scale; y *= scale; z *= scale;
        const double y0 = v[0][0] * x + v[1][0] * y + v[2][0] * z;
        const double y1 = v[0][1] * x + v[1][1] * y + v[2][1] * z;
        const double y2 = v[0][2] * x + v[1][2] * y + v[2][2] * z;
        s00 += y0 * y0; s01 += y0 * y1; s02 += y0 * y2; s11 += y1 * y1; s12 += y1 * y2; s22 += y2 * y2;
    }

    // Ends a pass: diagonalises its sums and turns the basis.  True when another pass is wanted.
    PCU_HD bool solve() {
        ++pass;
        if (pass == 1 && s00 + s11 + s22 == 0.0) { zero = true; return false; }
        a[0][0] = s00; a[0][1] = a[1][0] = s01; a[0][2] = a[2][0] = s02;
        a[1][1] = s11; a[1][2] = a[2][1] = s12; a[2][2] = s22;
        double w[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
        for (int sweep = 0; sweep < 16; ++sweep) {
            bool rotated = jacobi_rotate<0, 1>(a, w);
            rotated = jacobi_rotate<0, 2>(a, w) || rotated;
            rotated = jacobi_rotate<1, 2>(a, w) || rotated;
            if (!rotated) break;
        }
        double nv[3][3];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) nv[i][j] = v[i][0] * w[0][j] + v[i][1] * w[1][j] + v[i][2] * w[2][j];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) v[i][j] = nv[i][j];
        reset();
        const double turn = fmax(fabs(w[0][1]), fmax(fabs(w[0][2]), fabs(w[1][2])));
        return pass == 1 || (turn > 0x1p-26 && pass < kMaxPasses);
    }

    // The column of the basis v that is the normal when the fit is defined: the first smallest diagonal entry.  The other
    // two columns span the fitted plane.
    PCU_HD int normal_axis() const {
        const double e0 = a[0][0], e1 = a[1][1], e2 = a[2][2];
        return (e0 <= e1 && e0 <= e2) ? 0 : (e1 <= e2 ? 1 : 2);
    }

    // The unit normal of m offsets (see the rules above).
    PCU_HD void normal(long long m, double (&n)[3]) const {
        if (m < 3) { n[0] = n[1] = n[2] = 0.0; return; }
        if (zero) { n[0] = 0.0; n[1] = 0.0; n[2] = 1.0; return; }
        const int c = normal_axis();
        const double nx = v[0][c], ny = v[1][c], nz = v[2][c];
        const double len = sqrt(nx * nx + ny * ny + nz * nz);
        n[0] = nx / len; n[1] = ny / len; n[2] = nz / len;
    }
};

}  // namespace pcu

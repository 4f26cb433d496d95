// laplacian.cuh -- Laplacian smoothing of a triangle mesh (the reference's src/smooth.cpp): the cotangent Laplacian in
// CSR form, a three-column sparse product and a Jacobi-preconditioned conjugate-gradient solve with deterministic
// reductions.  Results defined in DESIGN.md §3.
//
// Assembly, once per call, from the input vertices (fp64):
//   mg_face_kernel      half the cotangent of every corner (0 for a face with dblA = 0)
//   lap_edge_kernel     six directed-edge records per face: the edge opposite corner k joins a = f[k+1] and b = f[k+2];
//                       records 6t + 2k and 6t + 2k + 1 are (a, b) and (b, a), key (row << bits) | column
//   radix sort (sort.cuh), stable: each run of equal keys lists its contributions in ascending face order
//   mc_heads_kernel (runtime.cu), keep_count / keep_offsets (compact.cuh): one entry per run, nnz
//   lap_entries_kernel  each run head sums its run in order: L_ij = sum of cot / 2, as int32 columns and fp64 values
//   mg_rows_kernel      row pointers of the entries (rows = vertices)
//   lap_diag_kernel     L_ii = -sum_j L_ij in ascending column order; `lone` marks the rows without a non-zero weight
// Every iteration: (cotan mode) the mass M_ii = sum over i's corners of dblA / 6 of the current u, through the corner
// CSR of mesh_geometry.cuh; then CG on (M - h L) u' = M u, three columns at once, from u:
//   lap_cg_init_kernel     r = M u - S u, z = r / diag(S), p = z; r.z, r.r and b.b per column
//   lap_cg_spmv_kernel     q = S p = M p - h (L p), p.q  -> alpha
//   lap_cg_update_kernel   x += alpha p, r -= alpha q, z = r / diag(S); r.r and r.z -> convergence, beta
//   lap_cg_direction_kernel p = z + beta p
// The host reads CgState once per window of iterations; a launch after convergence returns at once.  The dot products
// are reduce_grid sums over at most kMgBlocks CTAs: no floating-point atomics, so two calls give the same bits.
// (cotan mode) after each solve, mg_face_kernel's partials give the area and its centroid, and lap_rescale_kernel
// moves u about the centroid and scales it by 1 / sqrt(area).
#pragma once
#include "common.cuh"
#include "compact.cuh"
#include "mesh_geometry.cuh"

namespace pcu {

constexpr double kCgTol2 = 1e-24;   // a column stops when |r|^2 <= kCgTol2 |b|^2, i.e. |r| <= 1e-12 |b|

// The conjugate-gradient state of the current solve, per column (zeroed by the host before each solve).
struct CgState {
    double rz[3], rr[3], bb[3], alpha[3], beta[3];
    int active[3];
    int done;           // no active column left, or the iteration cap was reached
    int iters;          // iterations of this solve
    unsigned ticket;    // arrivals of the current reduce_grid
    int pad;
};

// The whole record the host reads during a smoothing call.
struct LapRecord {
    MgRecord mesh;
    CgState cg;
};

// The system S = M - h L, in CSR form with a separate diagonal; mass == nullptr means M = I.
struct LapSystem {
    const int* rowptr;
    const int* col;
    const double* val;
    const double* diag;
    const double* mass;
    double h;
    long long n;
};

__device__ __forceinline__ bool lap_halted(const LapRecord* rec) { return rec->cg.done || rec->mesh.zero_area; }

__device__ __forceinline__ double lap_mass(const LapSystem& s, long long i) { return s.mass ? __ldg(s.mass + i) : 1.0; }

// The Jacobi preconditioner: diag(S), or 1 where that is not positive.
__device__ __forceinline__ double lap_precond(const LapSystem& s, long long i) {
    const double d = lap_mass(s, i) - s.h * __ldg(s.diag + i);
    return d > 0.0 ? d : 1.0;
}

// q = (S p)_i for the three columns of row i.
__device__ __forceinline__ void lap_apply(const LapSystem& s, long long i, const double* __restrict__ p, double q[3]) {
    double lp[3];
    const double di = __ldg(s.diag + i);
#pragma unroll
    for (int c = 0; c < 3; ++c) lp[c] = di * p[3 * i + c];
    for (int e = __ldg(s.rowptr + i), end = __ldg(s.rowptr + i + 1); e < end; ++e) {
        const long long j = __ldg(s.col + e);
        const double w = __ldg(s.val + e);
#pragma unroll
        for (int c = 0; c < 3; ++c) lp[c] += w * p[3 * j + c];
    }
    const double m = lap_mass(s, i);
#pragma unroll
    for (int c = 0; c < 3; ++c) q[c] = m * p[3 * i + c] - s.h * lp[c];
}

// u = v in fp64; the coordinates that are not finite are counted.
template <typename T>
__global__ void __launch_bounds__(kThreads) lap_load_kernel(const T* __restrict__ v, long long count, double* __restrict__ u,
                                                            MgRecord* __restrict__ rec) {
    const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool bad = false;
    if (e < count) {
        const double x = (double)v[e];
        u[e] = x;
        bad = !(fabs(x) <= 1.7976931348623157e308);
    }
    const int nbad = __syncthreads_count(bad);
    if (threadIdx.x == 0 && nbad) atomicAdd(&rec->nonfinite, (unsigned long long)nbad);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) lap_store_kernel(const double* __restrict__ u, long long count, T* __restrict__ out) {
    const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (e < count) out[e] = (T)u[e];
}

// Six directed-edge records per face (see the top of the file); idx = 6 t + 2 k + direction, so idx >> 1 is the
// corner whose half cotangent the record carries.  A face with a corner outside [0, nv) gives (0, 0) records (the call
// fails).
__global__ void __launch_bounds__(kThreads) lap_edge_kernel(const void* __restrict__ f, int fkind, long long m, long long nv, int bits,
                                                            MgRec* __restrict__ recs) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    long long c[3];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c[k] = load_index(f, 3 * t + k, fkind, nv, false);
        bad = bad || c[k] < 0;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned long long a = bad ? 0ull : (unsigned long long)c[(k + 1) % 3], b = bad ? 0ull : (unsigned long long)c[(k + 2) % 3];
        MgRec r;
        r.key[0] = a << bits | b;
        r.idx = (unsigned long long)(6 * t + 2 * k);
        store_rec(recs + 6 * t + 2 * k, r);
        r.key[0] = b << bits | a;
        r.idx += 1ull;
        store_rec(recs + 6 * t + 2 * k + 1, r);
    }
}

// After keep_count / keep_offsets over the run heads: entry e of every run, its row (for mg_rows_kernel's key), column
// and value, the run's half cotangents added in order.
__global__ void __launch_bounds__(kThreads) lap_entries_kernel(const MgRec* __restrict__ sorted, long long n, const unsigned char* __restrict__ head,
                                                               const unsigned* __restrict__ block_offset, const double* __restrict__ halfcot,
                                                               int bits, MgRec* __restrict__ rows, int* __restrict__ col,
                                                               double* __restrict__ val) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const bool mine = i < n && head[i];
    const unsigned e = keep_rank(mine, block_offset);
    if (!mine) return;
    const unsigned long long key = sorted[i].key[0];
    double s = __ldg(halfcot + (sorted[i].idx >> 1));
    for (long long j = i + 1; j < n && sorted[j].key[0] == key; ++j) s = __dadd_rn(s, __ldg(halfcot + (sorted[j].idx >> 1)));
    MgRec r;
    r.key[0] = key >> bits;
    r.idx = e;
    store_rec(rows + e, r);
    col[e] = (int)(key & ((1ull << bits) - 1ull));
    val[e] = s;
}

// L_ii = -sum_j L_ij (ascending j); lone[i] = the row has no non-zero weight.
__global__ void __launch_bounds__(kThreads) lap_diag_kernel(const int* __restrict__ rowptr, const double* __restrict__ val, long long n,
                                                            double* __restrict__ diag, unsigned char* __restrict__ lone) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    bool any = false;
    for (int e = rowptr[i], end = rowptr[i + 1]; e < end; ++e) {
        const double w = val[e];
        s = __dadd_rn(s, w);
        any = any || w != 0.0;
    }
    diag[i] = -s;
    lone[i] = !any;
}

// M_ii = sum over i's corners (ascending) of dblA / 6; 1 for a row with neither mass nor weight (the identity).
__global__ void __launch_bounds__(kThreads) lap_mass_kernel(const int* __restrict__ first, const int* __restrict__ corner, long long n,
                                                            const double* __restrict__ dbla, const unsigned char* __restrict__ lone,
                                                            double* __restrict__ mass) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int j = first[i], e = first[i + 1]; j < e; ++j) s = __dadd_rn(s, __ddiv_rn(__ldg(dbla + __ldg(corner + j) / 3), 6.0));
    mass[i] = s == 0.0 && lone[i] ? 1.0 : s;
}

// r = M x - S x, z = r / diag(S), p = z; sets up the columns (the state was zeroed by the host).
__global__ void __launch_bounds__(kThreads) lap_cg_init_kernel(LapSystem s, const double* __restrict__ x, double* __restrict__ r,
                                                               double* __restrict__ z, double* __restrict__ p, double* __restrict__ partial,
                                                               LapRecord* rec) {
    if (lap_halted(rec)) return;
    double acc[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // r.z, r.r, b.b per column
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < s.n; i += (long long)gridDim.x * kThreads) {
        double q[3];
        lap_apply(s, i, x, q);
        const double m = lap_mass(s, i), d = lap_precond(s, i);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double b = m * x[3 * i + c], ri = b - q[c], zi = ri / d;
            r[3 * i + c] = ri;
            z[3 * i + c] = zi;
            p[3 * i + c] = zi;
            acc[c] += ri * zi;
            acc[3 + c] += ri * ri;
            acc[6 + c] += b * b;
        }
    }
    if (reduce_grid<9>(acc, partial, &rec->cg.ticket) && threadIdx.x == 0) {
        CgState& st = rec->cg;
        bool any = false;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            st.rz[c] = acc[c];
            st.rr[c] = acc[3 + c];
            st.bb[c] = acc[6 + c];
            st.active[c] = !(acc[3 + c] <= kCgTol2 * acc[6 + c]);
            any = any || st.active[c];
        }
        st.done = !any;
    }
}

__global__ void __launch_bounds__(kThreads) lap_cg_spmv_kernel(LapSystem s, const double* __restrict__ p, double* __restrict__ q,
                                                               double* __restrict__ partial, LapRecord* rec) {
    if (lap_halted(rec)) return;
    double acc[3] = {0.0, 0.0, 0.0};
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < s.n; i += (long long)gridDim.x * kThreads) {
        double qi[3];
        lap_apply(s, i, p, qi);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            q[3 * i + c] = qi[c];
            acc[c] += p[3 * i + c] * qi[c];
        }
    }
    if (reduce_grid<3>(acc, partial, &rec->cg.ticket) && threadIdx.x == 0) {
        CgState& st = rec->cg;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (st.active[c] && !(acc[c] > 0.0)) st.active[c] = 0;   // S is not positive definite along p: stop the column
            st.alpha[c] = st.active[c] ? st.rz[c] / acc[c] : 0.0;
        }
    }
}

__global__ void __launch_bounds__(kThreads) lap_cg_update_kernel(LapSystem s, double* __restrict__ x, double* __restrict__ r, double* __restrict__ z,
                                                                 const double* __restrict__ p, const double* __restrict__ q,
                                                                 double* __restrict__ partial, int max_iters, LapRecord* rec) {
    if (lap_halted(rec)) return;
    const CgState& st = rec->cg;
    const double alpha[3] = {st.alpha[0], st.alpha[1], st.alpha[2]};
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // r.r, r.z per column
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < s.n; i += (long long)gridDim.x * kThreads) {
        const double d = lap_precond(s, i);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const long long e = 3 * i + c;
            double ri = r[e];
            if (alpha[c] != 0.0) {
                x[e] += alpha[c] * p[e];
                ri -= alpha[c] * q[e];
                r[e] = ri;
            }
            const double zi = ri / d;
            z[e] = zi;
            acc[c] += ri * ri;
            acc[3 + c] += ri * zi;
        }
    }
    if (reduce_grid<6>(acc, partial, &rec->cg.ticket) && threadIdx.x == 0) {
        CgState& w = rec->cg;
        bool any = false;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (!w.active[c]) continue;
            w.rr[c] = acc[c];
            if (acc[c] <= kCgTol2 * w.bb[c]) {
                w.active[c] = 0;
                continue;
            }
            w.beta[c] = acc[3 + c] / w.rz[c];
            w.rz[c] = acc[3 + c];
            any = true;
        }
        w.iters += 1;
        w.done = !any || w.iters >= max_iters;
    }
}

__global__ void __launch_bounds__(kThreads) lap_cg_direction_kernel(long long n, const double* __restrict__ z, double* __restrict__ p,
                                                                    const LapRecord* rec) {
    if (lap_halted(rec)) return;
    const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (e >= 3 * n) return;
    const int c = (int)(e % 3);
    if (rec->cg.active[c]) p[e] = z[e] + rec->cg.beta[c] * p[e];
}

// u = (u - c) / sqrt(area) + c, area = sum dblA / 2, c = sum dblA barycentre / sum dblA (MgRecord::sums of the face
// pass just before); nothing when that area was 0 or not finite (the call fails).
__global__ void __launch_bounds__(kThreads) lap_rescale_kernel(double* __restrict__ u, long long n, const MgRecord* __restrict__ rec) {
    if (rec->zero_area) return;
    const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (e >= 3 * n) return;
    const double total = rec->sums[0];
    const double c = __ddiv_rn(rec->sums[1 + e % 3], total), scale = __dsqrt_rn(__dmul_rn(0.5, total));
    u[e] = __dadd_rn(__ddiv_rn(__dsub_rn(u[e], c), scale), c);
}

}  // namespace pcu

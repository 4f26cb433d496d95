// sinkhorn.cuh -- dense pairwise distances and the log-domain Sinkhorn iteration (SURVEY.md 8f, row N4).
//
// Replaces the numpy code of /root/reference/point_cloud_utils/_sinkhorn.py: pairwise_distances (:4-34),
// sinkhorn (:37-126; the iteration :104-118, the plan :120-122) and what earth_movers_distance (:129-156) adds on
// top, (P * M).sum().  Floating point:
// - pairwise distances for p = 2, 1, inf, -inf and 0 are bit-exact: the same rounded operations, the sums in numpy's
//   pairwise order (np_pairwise_sum), NaN propagated as numpy does.  General p calls pow in fp64 where numpy calls it
//   in the arrays' precision: within a few ulp (tests/test_dense_metrics.py derives the bound).
// - Sinkhorn evaluates every element-wise expression in the arrays' precision in the reference's order -- (-M + v) /
//   eps, x - max, exp, log, eps * (log a - lse) -- and accumulates the two reductions (the sum of the exponentials, the
//   L1 change of the iterates) in fp64 instead of numpy's pairwise sum in the arrays' precision, so the plan agrees to
//   rounding, not bit for bit (the tests state the tolerance).  The stopping test is the reference's, NaN included.
#pragma once
#include "common.cuh"

namespace pcu {

// p-norm selector of np.linalg.norm(x, ord=p, axis=-1) for vectors
constexpr int kNorm2 = 0, kNorm1 = 1, kNormInf = 2, kNormNegInf = 3, kNorm0 = 4, kNormP = 5;

// numpy's add.reduce over a contiguous axis of at most 128 elements (pairwise_sum in numpy's loops_utils.h.src):
// below 8 terms a plain sequential sum from 0; otherwise eight strided partial sums, combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the remainder added one by one.
template <typename T, typename F>
__device__ __forceinline__ T np_block_sum(const F& term, int off, int n) {
    using R = Real<T>;
    if (n < 8) {
        T s = (T)0;
        for (int c = 0; c < n; ++c) s = R::add(s, term(off + c));
        return s;
    }
    T r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = term(off + k);
    int c = 8;
    for (; c < n - n % 8; c += 8) {
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] = R::add(r[k], term(off + c + k));
    }
    T s = R::add(R::add(R::add(r[0], r[1]), R::add(r[2], r[3])), R::add(R::add(r[4], r[5]), R::add(r[6], r[7])));
    for (; c < n; ++c) s = R::add(s, term(off + c));
    return s;
}

// The whole of numpy's pairwise summation of term(0 .. n-1): a range of more than 128 terms splits at
// h = n / 2 - (n / 2) % 8 into [0, h) + [h, n), recursively.  The recursion is walked in post-order without a call
// stack: bit k of `path` says whether the walk is in the right half at depth k, and left[k] holds that level's
// finished left half until the right half is done.  Depth stays below 32 for any int n (each split at least halves
// the range, less 8).
template <typename T, typename F>
__device__ __forceinline__ T np_pairwise_sum(const F& term, int n) {
    if (n <= 128) return np_block_sum<T>(term, 0, n);
    T left[32];
    unsigned path = 0;
    int depth = 0, off = 0, len = n;
    for (;;) {
        for (; len > 128; ++depth) { len = len / 2 - (len / 2) % 8; path &= ~(1u << depth); }
        T s = np_block_sum<T>(term, off, len);
        for (; depth > 0 && (path >> (depth - 1) & 1u); --depth) s = Real<T>::add(left[depth - 1], s);
        if (depth == 0) return s;
        left[depth - 1] = s;
        path |= 1u << (depth - 1);
        off = 0; len = n;                 // descend from the root to the right half just entered
        for (int k = 0; k < depth; ++k) {
            const int h = len / 2 - (len / 2) % 8;
            if (path >> k & 1u) { off += h; len -= h; } else len = h;
        }
    }
}

template <typename T> __device__ __forceinline__ T abs_t(T x);
template <> __device__ __forceinline__ float abs_t<float>(float x) { return fabsf(x); }
template <> __device__ __forceinline__ double abs_t<double>(double x) { return fabs(x); }

// out[b, i, j] = || a[b, i, :] - b[b, j, :] ||_p ; a: (nb, n, d), b: (nb, m, d).  grid (ceil(m / 256), n, nb); the
// host offsets the pointers to launch more than 65535 rows or batches in chunks (n and m stay the full strides).
// np.linalg.norm(axis=-1) of the difference, operation for operation: p = 2 sums the rounded squares, p = 1 the
// absolute values and general p the rounded |x|^p, all in numpy's pairwise order (np_pairwise_sum), so p = 2, 1,
// inf, -inf and 0 are bit-exact.  inf / -inf are max / min of |x| and propagate NaN.  General p rounds p and its
// reciprocal to T and evaluates each pow in fp64, where numpy calls pow in T: within a few ulp of numpy.
template <typename T>
__global__ void __launch_bounds__(kThreads) pairwise_kernel(const T* __restrict__ a, const T* __restrict__ b, long long n,
                                                            long long m, int d, int kind, double p, T* __restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y, bt = blockIdx.z;
    if (j >= m) return;
    const T* pa = a + (bt * n + i) * d;
    const T* pb = b + (bt * m + j) * d;
    using R = Real<T>;
    T acc;
    if (kind == kNormInf || kind == kNormNegInf) {
        acc = kind == kNormNegInf ? R::inf() : (T)0;
        for (int c = 0; c < d; ++c) {
            const T ad = abs_t(R::sub(pa[c], pb[c]));
            const bool take = kind == kNormInf ? ad > acc : ad < acc;
            if (take || ad != ad) acc = ad;                  // once acc is NaN no comparison replaces it
        }
    } else if (kind == kNorm0) {
        acc = (T)0;                                          // a count of ones: exact in any order
        for (int c = 0; c < d; ++c) acc += R::sub(pa[c], pb[c]) != (T)0 ? (T)1 : (T)0;
    } else if (kind == kNorm2) {
        // no contraction: numpy rounds the product and the sum
        acc = R::root(np_pairwise_sum<T>([&](int c) { const T x = R::sub(pa[c], pb[c]); return R::mul(x, x); }, d));
    } else if (kind == kNorm1) {
        acc = np_pairwise_sum<T>([&](int c) { return abs_t(R::sub(pa[c], pb[c])); }, d);
    } else {
        const double pt = (double)(T)p;
        acc = np_pairwise_sum<T>([&](int c) { return (T)pow((double)abs_t(R::sub(pa[c], pb[c])), pt); }, d);
        acc = (T)pow((double)acc, (double)((T)1 / (T)p));
    }
    out[(bt * n + i) * m + j] = acc;
}

template <typename T> __device__ __forceinline__ T exp_t(T x);
template <> __device__ __forceinline__ float exp_t<float>(float x) { return expf(x); }
template <> __device__ __forceinline__ double exp_t<double>(double x) { return exp(x); }
template <typename T> __device__ __forceinline__ T log_t(T x);
template <> __device__ __forceinline__ float log_t<float>(float x) { return logf(x); }
template <> __device__ __forceinline__ double log_t<double>(double x) { return log(x); }

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];   // fixed order
    __syncthreads();
    return t;
}
template <typename T>
__device__ __forceinline__ T block_max(T v, T* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const T u = __shfl_xor_sync(0xffffffffu, v, o); v = u > v ? u : v; }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = red[0];
    for (int w = 1; w < kThreads / 32; ++w) t = red[w] > t ? red[w] : t;
    __syncthreads();
    return t;
}

// One half-iteration (_sinkhorn.py:108-112): for every row r of the (nb, R, C) matrix view
//   pot_out[b, r] = eps * (log(w[b, r]) - logsumexp_c((-M[b, r, c] + pot_in[b, c]) / eps))
// and err[b] += |pot_out_old - pot_out_new|.  kTranspose: the row of the VIEW is a column of M (the v update walks
// M^T): a block then owns 32 consecutive view rows and reads M row-major, coalesced, each warp taking a slice of the
// c range.  Skipped entirely when *done != 0 (converged: the remaining launches of the call are no-ops).
// grid (R or ceil(R / 32), nb)
template <typename T, bool kTranspose>
__global__ void __launch_bounds__(kThreads) sinkhorn_half_kernel(const T* __restrict__ M, const T* __restrict__ w,
                                                                 const T* __restrict__ pot_in, T* __restrict__ pot_out,
                                                                 long long R, long long C, T eps, double* __restrict__ err,
                                                                 const int* __restrict__ done) {
    if (*done) return;
    const long long bt = blockIdx.y;
    __shared__ double red_d[kThreads / 32];
    __shared__ T red_t[kThreads / 32];
    if (!kTranspose) {
        const long long r = blockIdx.x;
        const T* row = M + (bt * R + r) * C;
        const T* pin = pot_in + bt * C;
        T mx = -Real<T>::inf();
        for (long long c = threadIdx.x; c < C; c += blockDim.x) {
            const T x = (-row[c] + pin[c]) / eps;
            mx = x > mx ? x : mx;
        }
        mx = block_max<T>(mx, red_t);
        double sum = 0.0;
        for (long long c = threadIdx.x; c < C; c += blockDim.x) {
            const T x = (-row[c] + pin[c]) / eps;
            sum += (double)exp_t<T>(x - mx);
        }
        sum = block_sum(sum, red_d);
        if (threadIdx.x == 0) {
            const T lse = log_t<T>((T)sum) + mx;
            const T nu = eps * (log_t<T>(w[bt * R + r]) - lse);
            const T old = pot_out[bt * R + r];
            pot_out[bt * R + r] = nu;
            const T diff = old - nu;
            atomicAdd(err + bt, (double)(diff < (T)0 ? -diff : diff));
        }
    } else {
        // 32 view rows (columns of M) per block; lane = column, warp w walks M rows w, w + 8, ...
        __shared__ T part_mx[kThreads / 32][32];
        __shared__ double part_sum[kThreads / 32][32];
        const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
        const long long r = (long long)blockIdx.x * 32 + lane;     // view row = column of M
        const bool ok = r < R;
        const T* base = M + bt * C * R;                            // M is (C, R) row-major here: C rows of length R
        const T* pin = pot_in + bt * C;
        T mx = -Real<T>::inf();
        for (long long c = wp; c < C; c += kThreads / 32) {
            if (ok) { const T x = (-base[c * R + r] + pin[c]) / eps; mx = x > mx ? x : mx; }
        }
        part_mx[wp][lane] = mx;
        __syncthreads();
        mx = part_mx[0][lane];
        for (int k = 1; k < kThreads / 32; ++k) mx = part_mx[k][lane] > mx ? part_mx[k][lane] : mx;
        double sum = 0.0;
        for (long long c = wp; c < C; c += kThreads / 32) {
            if (ok) { const T x = (-base[c * R + r] + pin[c]) / eps; sum += (double)exp_t<T>(x - mx); }
        }
        part_sum[wp][lane] = sum;
        __syncthreads();
        if (wp == 0 && ok) {
            double tot = 0.0;
            for (int k = 0; k < kThreads / 32; ++k) tot += part_sum[k][lane];
            const T lse = log_t<T>((T)tot) + mx;
            const T nu = eps * (log_t<T>(w[bt * R + r]) - lse);
            const T old = pot_out[bt * R + r];
            pot_out[bt * R + r] = nu;
            const T diff = old - nu;
            atomicAdd(err + bt, (double)(diff < (T)0 ? -diff : diff));
        }
    }
}

// End of an iteration (_sinkhorn.py:114-118): err_u = max_b sum_i |du|, err_v likewise; converged when both are
// below stop_thresh.  Also counts the iterations done and clears the accumulators.  One block.  The maximum propagates
// NaN as numpy's .max() does: a zero weight makes its potential -inf and its change -inf - -inf = NaN, and a NaN error
// never counts as converged, so such a problem runs all max_iters as in the reference.
__device__ __forceinline__ double max_nan(double x, double y) { return x > y || x != x ? x : y; }
__global__ void sinkhorn_check_kernel(double* __restrict__ err_u, double* __restrict__ err_v, long long nb, double stop_thresh,
                                      int* __restrict__ done, int* __restrict__ iters) {
    if (*done) return;
    __shared__ double su[kThreads], sv[kThreads];
    double mu = 0.0, mv = 0.0;
    for (long long b = threadIdx.x; b < nb; b += blockDim.x) {
        mu = max_nan(mu, err_u[b]); mv = max_nan(mv, err_v[b]);
        err_u[b] = 0.0; err_v[b] = 0.0;
    }
    su[threadIdx.x] = mu; sv[threadIdx.x] = mv;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { su[threadIdx.x] = max_nan(su[threadIdx.x], su[threadIdx.x + o]); sv[threadIdx.x] = max_nan(sv[threadIdx.x], sv[threadIdx.x + o]); }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *iters += 1;
        if (su[0] < stop_thresh && sv[0] < stop_thresh) *done = 1;
    }
}

// P[b, i, j] = exp((-M[b, i, j] + u[b, i] + v[b, j]) / eps)  (:120-122); optionally cost[b] += sum_ij P * M (fp64).
// grid (ceil(m / 256), n, nb)
template <typename T>
__global__ void __launch_bounds__(kThreads) sinkhorn_plan_kernel(const T* __restrict__ M, const T* __restrict__ u,
                                                                 const T* __restrict__ v, long long n, long long m, T eps,
                                                                 T* __restrict__ P, double* __restrict__ cost) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y, bt = blockIdx.z;
    double mine = 0.0;
    if (j < m) {
        const long long at = (bt * n + i) * m + j;
        const T val = exp_t<T>(((-M[at] + u[bt * n + i]) + v[bt * m + j]) / eps);
        P[at] = val;
        mine = (double)(T)(val * M[at]);
    }
    if (cost != nullptr) {
        __shared__ double red[kThreads / 32];
        const double tot = block_sum(mine, red);
        if (threadIdx.x == 0 && tot != 0.0) atomicAdd(cost + bt, tot);
    }
}

}  // namespace pcu

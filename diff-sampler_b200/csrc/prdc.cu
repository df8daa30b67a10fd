// Precision, recall, density and coverage: the CUDA-core ops after the distance GEMMs (ops.h, DESIGN.md 4.12).
//
//   GEMM (rows mode): K-slice partials of sq st q_b.t_i -> prdc_kth (k-NN radii of a set against itself) or prdc_count (real-fake
//   neighbourhood counts and realism).  Both run one CTA per query row: the approximate squared distance of every pair from the
//   partials and the float64 norms, a per-pair bound on its error, and an exact float64 recomputation (one warp per pair) of every
//   pair the bound cannot decide.  The recomputed pairs are compacted in index order into a shared list that is flushed whenever it
//   could overflow, so their number has no cap.
//
// Counts are integer sums and the realism a maximum, the ranks of the radius candidates are total orders, and nothing uses atomics: two
// calls on the same input are bit-identical.
#include "ops.h"
#include "block.cuh"
#include <math.h>

namespace dsb {

static constexpr int kPrdcThreads = 512;
static constexpr int kPrdcWarps = kPrdcThreads / 32;

static int prdc_ok() { return cudaGetLastError() == cudaSuccess ? 0 : -1; }

// Bound on |approximate d2 - exact d2| for rows of squared norms qn2, tn2 (DESIGN.md 4.12): the GEMM's 2 eps ||q|| ||t|| with the
// float64 -> fp32 narrowing of the operands (2^-15 covers both), the fp16 subnormal floor of the lo planes, and the rounding of the
// float64 norms, of the exact sum and of the fp32 copy prdc_kth keeps.
__device__ __forceinline__ double d2_bound(double qn2, double tn2, double sq, double st, int D) {
    const double qn = sqrt(qn2), tn = sqrt(tn2);
    return ldexp(qn * tn, -15) + ldexp(sqrt((double)D), -24) * (tn / sq + qn / st) +
           (ldexp(1.0, -21) + ldexp((double)D + 4.0, -51)) * (qn2 + tn2);
}

// qn2 + tn2 - 2 q.t from the slice partials (added in order in fp64).
__device__ __forceinline__ double approx_d2(const float* p, long long sstride, int nslice, double qn2, double tn2, double inv) {
    double acc = 0.0;
    for (int s = 0; s < nslice; ++s) acc += (double)p[s * sstride];
    return qn2 + tn2 - 2.0 * acc * inv;
}

// 1: d < tau for certain, 0: d >= tau for certain, -1: undecided.  T = tau^2 up to an ulp; the relative slack of 2^-48 keeps the
// sqrt of a decided d2 off tau (DESIGN.md 4.12).
__device__ __forceinline__ int classify(double a, double B, double T) {
    const double s = ldexp(T, -48);
    if (a + B < T - s) return 1;
    if (a - B > T + s) return 0;
    return -1;
}

// ||x - y||^2 by one warp in float64: differences, squares and sums in a fixed order (lane-strided fma, then a butterfly).
__device__ __forceinline__ double warp_exact_d2(const double* __restrict__ x, const double* __restrict__ y, int D) {
    double s = 0.0;
    for (int k = threadIdx.x & 31; k < D; k += 32) {
        const double t = x[k] - y[k];
        s = fma(t, t, s);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

// The realism maximum takes fmax, not MaxOp: fmax drops a nan operand wherever it stands, so the maximum covers the ratios that are
// numbers whatever the order; a nan ratio is counted in nan_seen and wins there, as in numpy.
struct FmaxOp {
    __device__ double operator()(double a, double b) const { return fmax(a, b); }
};

// The list is flushed once it holds more than this, so one more tile always fits.
static constexpr int kFlushAt = DS_PRDC_LIST - kPrdcThreads;

__global__ void __launch_bounds__(kPrdcThreads) prdc_kth_kernel(ds_prdc_kth_desc d) {
    __shared__ float shf[kPrdcWarps];
    __shared__ int shi[kPrdcWarps];
    __shared__ int list[DS_PRDC_LIST];
    __shared__ double ld2[DS_PRDC_LIST];
    __shared__ int bidx[DS_PRDC_KMAX + 1], nidx[DS_PRDC_KMAX + 1];
    __shared__ double bd2[DS_PRDC_KMAX + 1], nd2[DS_PRDC_KMAX + 1];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int N = d.N, D = d.D, kk = d.k + 1;
    const long long sstride = (long long)d.B * d.ldp;
    float* a = d.part + (long long)b * d.ldp;
    const double qn2 = d.qn2[b], inv = 1.0 / (d.sq * d.st);
    const double* q = d.q + (long long)b * D;
    for (int i = tid; i < N; i += kPrdcThreads) a[i] = (float)approx_d2(a + i, sstride, d.nslice, qn2, d.tn2[i], inv);
    __syncthreads();
    // the k+1 smallest approximate d2, each taken out of the row (+inf) once chosen; hi bounds the exact d2 of all of them, so the
    // (k+1)-th exact distance is at most sqrt(hi), and a row whose d2 may be below hi is a candidate
    double hi = -INFINITY;
    for (int c = 0; c < kk; ++c) {
        float v = INFINITY;
        int idx = 0x7fffffff;
        for (int i = tid; i < N; i += kPrdcThreads) {
            const float t = a[i];
            if (t < v || (t == v && i < idx)) { v = t; idx = i; }
        }
        block_argbest<kPrdcWarps, false>(v, idx, shf, shi);
        hi = fmax(hi, (double)v + d2_bound(qn2, d.tn2[idx], d.sq, d.st, D));
        if (tid == 0) { bidx[c] = idx; a[idx] = INFINITY; }
        __syncthreads();
    }
    for (int j = w; j < kk; j += kPrdcWarps) {
        const double e = warp_exact_d2(q, d.t + (long long)bidx[j] * D, D);
        if (lane == 0) bd2[j] = e;
    }
    int n = 0, rescored = kk;
    for (int base = 0; base < N; base += kPrdcThreads) {
        const int i = base + tid;
        n = block_compact<kPrdcWarps>(i < N && (double)a[i] - d2_bound(qn2, d.tn2[i], d.sq, d.st, D) <= hi, i, list, n, shi);
        const bool last = base + kPrdcThreads >= N;
        if (n <= kFlushAt && !last) continue;                 // block-uniform
        __syncthreads();
        for (int j = w; j < n; j += kPrdcWarps) {
            const double e = warp_exact_d2(q, d.t + (long long)list[j] * D, D);
            if (lane == 0) ld2[j] = e;
        }
        __syncthreads();
        // the k+1 smallest of (best so far) + (list) by (d2, index): ranks are distinct because the indices are
        for (int j = tid; j < kk + n; j += kPrdcThreads) {
            const double dj = j < kk ? bd2[j] : ld2[j - kk];
            const int ij = j < kk ? bidx[j] : list[j - kk];
            int r = 0;
            for (int t = 0; t < kk + n && r < kk; ++t) {
                const double dt = t < kk ? bd2[t] : ld2[t - kk];
                const int it = t < kk ? bidx[t] : list[t - kk];
                r += (dt < dj || (dt == dj && it < ij)) ? 1 : 0;
            }
            if (r < kk) { nd2[r] = dj; nidx[r] = ij; }
        }
        __syncthreads();
        if (tid < kk) { bd2[tid] = nd2[tid]; bidx[tid] = nidx[tid]; }
        __syncthreads();
        rescored += n;
        n = 0;
    }
    if (tid == 0) {
        const double e = bd2[kk - 1];
        d.rad2[b] = e;
        d.rad[b] = sqrt(e);
        if (d.nres) d.nres[b] = rescored;
    }
}

__global__ void __launch_bounds__(kPrdcThreads) prdc_count_kernel(ds_prdc_count_desc d) {
    __shared__ int shi[kPrdcWarps];
    __shared__ double shd[kPrdcWarps];
    __shared__ int list[DS_PRDC_LIST];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int N = d.N, D = d.D;
    const long long sstride = (long long)d.B * d.ldp;
    const float* p = d.part + (long long)b * d.ldp;
    const double qn2 = d.qn2[b], inv = 1.0 / (d.sq * d.st);
    const double* q = d.q + (long long)b * D;
    const bool own = d.rho != nullptr, real = d.realism != nullptr;
    const double rho = own ? d.rho[b] : 0.0, rho2 = own ? d.rho2[b] : 0.0;
    int ct = 0, co = 0, rescored = 0;                         // per thread; a recomputed pair is counted by its warp's lane 0
    double lo_best = 0.0;                                     // largest lower bound of a realism ratio
    int n = 0;
    for (int base = 0; base < N; base += kPrdcThreads) {
        const int i = base + tid;
        bool und = false;
        if (i < N) {
            const double tn2 = d.tn2[i];
            const double a = approx_d2(p + i, sstride, d.nslice, qn2, tn2, inv);
            const double B = d2_bound(qn2, tn2, d.sq, d.st, D);
            const int c1 = classify(a, B, d.tau2[i]);
            const int c2 = own ? classify(a, B, rho2) : 0;
            und = c1 < 0 || c2 < 0;
            if (!und) { ct += c1; co += c2; }                  // an undecided pair is counted only from its exact distance
            if (real && d.tau[i] < d.med && a + B > 0.0)
                lo_best = fmax(lo_best, d.tau[i] / sqrt(a + B) * (1.0 - 0x1p-40));
        }
        n = block_compact<kPrdcWarps>(und, i, list, n, shi);
        if (n <= kFlushAt && base + kPrdcThreads < N) continue;
        __syncthreads();
        for (int j = w; j < n; j += kPrdcWarps) {
            const int ii = list[j];
            const double dist = sqrt(warp_exact_d2(q, d.t + (long long)ii * D, D));
            if (lane == 0) {
                ct += dist < d.tau[ii] ? 1 : 0;
                co += own && dist < rho ? 1 : 0;
                ++rescored;
            }
        }
        __syncthreads();
        n = 0;
    }
    ct = block_reduce<kPrdcWarps>(ct, SumOp(), shi);
    co = block_reduce<kPrdcWarps>(co, SumOp(), shi);
    if (real) {
        // every masked pair whose ratio could reach the best lower bound is recomputed; the others cannot hold the maximum
        lo_best = block_reduce<kPrdcWarps>(lo_best, FmaxOp(), shd);
        double best = -INFINITY;
        int nan_seen = 0;
        for (int base = 0; base < N; base += kPrdcThreads) {
            const int i = base + tid;
            bool cand = false;
            if (i < N && d.tau[i] < d.med) {
                const double tn2 = d.tn2[i];
                const double a = approx_d2(p + i, sstride, d.nslice, qn2, tn2, inv);
                const double lo = a - d2_bound(qn2, tn2, d.sq, d.st, D);
                cand = !(lo > 0.0) || d.tau[i] / sqrt(lo) * (1.0 + 0x1p-40) >= lo_best;
            }
            n = block_compact<kPrdcWarps>(cand, i, list, n, shi);
            if (n <= kFlushAt && base + kPrdcThreads < N) continue;
            __syncthreads();
            for (int j = w; j < n; j += kPrdcWarps) {
                const int ii = list[j];
                const double r = d.tau[ii] / sqrt(warp_exact_d2(q, d.t + (long long)ii * D, D));
                if (lane == 0) {
                    if (r != r) nan_seen = 1;
                    else best = fmax(best, r);
                    ++rescored;
                }
            }
            __syncthreads();
            n = 0;
        }
        best = block_reduce<kPrdcWarps>(best, FmaxOp(), shd);
        nan_seen = block_reduce<kPrdcWarps>(nan_seen, SumOp(), shi);
        if (tid == 0) d.realism[b] = nan_seen ? NAN : best;
    }
    rescored = block_reduce<kPrdcWarps>(rescored, SumOp(), shi);
    if (tid == 0) {
        d.cnt_t[b] = ct;
        if (own) d.cnt_own[b] = co;
        if (d.nres) d.nres[b] = rescored;
    }
}

}  // namespace dsb

dsb::OpCheck dsb::prdc_kth_check(const ds_prdc_kth_desc& d) {
    if (d.B <= 0 || d.N <= 0 || d.D <= 0 || d.nslice <= 0 || d.ldp < d.N) return {-1, "prdc_kth: shape"};
    if (d.k < 1 || d.k > DS_PRDC_KMAX || d.k >= d.N) return {-1, "prdc_kth: k"};
    if (!(d.sq > 0.0) || !(d.st > 0.0)) return {-1, "prdc_kth: scale"};
    if (!d.part || !d.q || !d.t || !d.qn2 || !d.tn2 || !d.rad || !d.rad2) return {-1, "prdc_kth: operands"};
    return {0, nullptr};
}

extern "C" int ds_prdc_kth_launch(const ds_prdc_kth_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::prdc_kth_check(*d).rc) return rc;
    dsb::prdc_kth_kernel<<<d->B, dsb::kPrdcThreads, 0, stream>>>(*d);
    return dsb::prdc_ok();
}

dsb::OpCheck dsb::prdc_count_check(const ds_prdc_count_desc& d) {
    if (d.B <= 0 || d.N <= 0 || d.D <= 0 || d.nslice <= 0 || d.ldp < d.N) return {-1, "prdc_count: shape"};
    if (!(d.sq > 0.0) || !(d.st > 0.0)) return {-1, "prdc_count: scale"};
    if (!d.part || !d.q || !d.t || !d.qn2 || !d.tn2 || !d.tau || !d.tau2 || !d.cnt_t) return {-1, "prdc_count: operands"};
    if (!d.rho != !d.rho2 || !d.rho != !d.cnt_own) return {-1, "prdc_count: own"};
    return {0, nullptr};
}

extern "C" int ds_prdc_count_launch(const ds_prdc_count_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::prdc_count_check(*d).rc) return rc;
    dsb::prdc_count_kernel<<<d->B, dsb::kPrdcThreads, 0, stream>>>(*d);
    return dsb::prdc_ok();
}

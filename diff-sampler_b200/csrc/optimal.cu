// Optimal (empirical-Bayes) denoiser: the CUDA-core ops around the two tensor-core contractions (ops.h, DESIGN.md 4.9).
//
//   x -> fp16 hi/lo planes (opt_prep) -> GEMM: K-slice partials of x.y_i -> opt_softmax (slices added in fixed order, 0.5||y||^2
//   subtracted, band rescoring, P = softmax as fp16 planes) -> GEMM: split-K partials of P.Y -> opt_reduce (fixed-order sum).
//
// Every reduction is a fixed tree (warp shuffles, then the warp totals in warp order) and nothing uses atomics, so two calls on the
// same input are bit-identical.
#include "ops.h"
#include "block.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace dsb {

static constexpr int kOptThreads = 512;
static constexpr int kOptWarps = kOptThreads / 32;

static int opt_ok() { return cudaGetLastError() == cudaSuccess ? 0 : -1; }

// ||x - y||^2 by one warp: fp32 differences, squares and sums in fp64 (the squares of fp32 values are exact in fp64).
__device__ __forceinline__ double warp_dist2(const float* __restrict__ x, const float* __restrict__ y, int D) {
    double s = 0.0;
    for (int k = threadIdx.x & 31; k < D; k += 32) {
        const double t = (double)__fsub_rn(x[k], y[k]);
        s = fma(t, t, s);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

// u_i = sum_s part[s][b][i] - 0.5 ||y_i||^2 (fp64, slices in order), stored as fp32 over slice 0.  Returns max_i u_i * inv (fp32).
__device__ __forceinline__ float row_u(float* part, const double* __restrict__ hy2, long long ldp, long long sstride, int nslice,
                                       int N, int b, float inv, float* shf) {
    float* u = part + (long long)b * ldp;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < N; i += kOptThreads) {
        double acc = 0.0;
        for (int s = 0; s < nslice; ++s) acc += (double)u[s * sstride + i];
        const float uf = (float)(acc - hy2[i]);
        u[i] = uf;
        m = fmaxf(m, uf * inv);
    }
    return block_reduce<kOptWarps>(m, MaxOp(), shf);
}

// Bound on |computed u_i - exact u_i| per unit of 1 / sigma^2:  (||x|| + Y) (eps Y + 2^-25 sqrt(D))   (DESIGN.md 4.9).
__device__ __forceinline__ double u_error(double xn2, float ymax, int D) {
    return (sqrt(xn2) + (double)ymax) * (DS_OPT_EPS * (double)ymax + ldexp(sqrt((double)D), -25));
}

__device__ __forceinline__ void store_p(__half* hi, __half* lo, long long i, float p) {
    const __half h = __float2half_rn(p);
    hi[i] = h;
    lo[i] = __float2half_rn(p - __half2float(h));
}

__global__ void __launch_bounds__(256) opt_prep_kernel(ds_opt_prep_desc d) {
    __shared__ double shd[8];
    const int b = blockIdx.x;
    const float* x = d.x + (long long)b * d.D;
    __half* hi = static_cast<__half*>(d.planes) + (long long)b * d.pitch;
    __half* lo = hi + (long long)d.B * d.pitch;
    double s = 0.0;
    for (int c = threadIdx.x; c < d.pitch; c += 256) {
        const float v = c < d.D ? x[c] : 0.f;
        store_p(hi, lo, c, v);
        s = fma((double)v, (double)v, s);
    }
    s = block_reduce<8>(s, SumOp(), shd);
    if (threadIdx.x == 0) d.xn2[b] = s;
}

__global__ void __launch_bounds__(kOptThreads) opt_softmax_kernel(ds_opt_softmax_desc d) {
    __shared__ double shd[kOptWarps];
    __shared__ float shf[kOptWarps];
    __shared__ int shi[kOptWarps];
    __shared__ int band[DS_OPT_CAP];
    __shared__ double bl[DS_OPT_CAP];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int N = d.N;
    const float sg = d.sigma[d.nsig > 1 ? b : 0];
    const double s2 = (double)sg * (double)sg;
    const float inv = (float)(1.0 / s2);
    float* u = d.part + (long long)b * d.ldp;
    const float m = row_u(d.part, d.hy2, d.ldp, (long long)d.B * d.ldp, d.nslice, N, b, inv, shf);
    const double E = u_error(d.xn2[b], d.ymax, d.D) / s2;
    __half* phi = static_cast<__half*>(d.P) + (long long)b * d.ldP;
    __half* plo = phi + (long long)d.B * d.ldP;
    const float pscale = (float)(1 << DS_OPT_P_SHIFT);
    int status = DS_OPT_PLAIN;
    if (E > (double)DS_OPT_TAU) {
        // band: computed logit >= max - (2 E + 40); order-preserving compaction with warp ballots, one 512-key tile at a time
        const double thr = (double)m - (2.0 * E + (double)DS_OPT_BAND_NATS);
        int total = 0;
        for (int base = 0; base < N; base += kOptThreads) {
            const int i = base + tid;
            total = block_compact<kOptWarps, DS_OPT_CAP>(i < N && (double)(u[i] * inv) >= thr, i, band, total, shi);
            if (total > DS_OPT_CAP) break;                 // block-uniform
        }
        __syncthreads();
        if (total > DS_OPT_CAP || total == 0) {
            status = DS_OPT_UNREFINED;
        } else {
            status = DS_OPT_RESCORED;
            const float* x = d.x + (long long)b * d.D;
            for (int j = w; j < total; j += kOptWarps) {
                const double d2 = warp_dist2(x, d.y + (long long)band[j] * d.D, d.D);
                if (lane == 0) bl[j] = -0.5 * d2 / s2;
            }
            __syncthreads();
            double mx = -INFINITY;
            for (int j = tid; j < total; j += kOptThreads) mx = fmax(mx, bl[j]);
            mx = block_reduce<kOptWarps>(mx, MaxOp(), shd);
            double l = 0.0;
            for (int j = tid; j < total; j += kOptThreads) l += exp(bl[j] - mx);
            l = block_reduce<kOptWarps>(l, SumOp(), shd);
            for (long long i = tid; i < d.ldP; i += kOptThreads) { phi[i] = __float2half_rn(0.f); plo[i] = __float2half_rn(0.f); }
            __syncthreads();
            for (int j = tid; j < total; j += kOptThreads) store_p(phi, plo, band[j], (float)(exp(bl[j] - mx) / l) * pscale);
        }
    }
    if (status != DS_OPT_RESCORED) {
        double l = 0.0;
        for (int i = tid; i < N; i += kOptThreads) l += (double)expf(u[i] * inv - m);
        l = block_reduce<kOptWarps>(l, SumOp(), shd);
        const double rl = 1.0 / l;
        for (long long i = tid; i < d.ldP; i += kOptThreads)
            store_p(phi, plo, i, i < N ? (float)((double)expf(u[i] * inv - m) * rl) * pscale : 0.f);
    }
    if (tid == 0 && d.status) d.status[b] = status;
}

__global__ void __launch_bounds__(256) opt_reduce_kernel(ds_opt_reduce_desc d) {
    const long long n = d.rows * d.cols, sstride = d.rows * d.ld;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / d.cols;
        const float* p = d.part + r * d.ld + (e - r * d.cols);
        float a = p[0];
        for (int s = 1; s < d.nsplit; ++s) a += p[s * sstride];
        d.out[e] = a * d.scale;
    }
}

__global__ void __launch_bounds__(kOptThreads) opt_knn_kernel(ds_opt_knn_desc d) {
    __shared__ float shf[kOptWarps];
    __shared__ int shi[kOptWarps];
    __shared__ int cand[DS_KNN_CAND];
    __shared__ double cd2[DS_KNN_CAND];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    float* u = d.part + (long long)b * d.ldp;
    row_u(d.part, d.hy2, d.ldp, (long long)d.B * d.ldp, d.nslice, d.N, b, 1.f, shf);
    // the k largest u, then every further key within twice the u error bound of the k-th (it may be nearer in exact arithmetic)
    const double err = u_error(d.xn2[b], d.ymax, d.D);
    int cnt = 0;
    double kth = 0.0;
    while (cnt < DS_KNN_CAND && cnt < d.N) {
        float v = -INFINITY;
        int idx = 0x7fffffff;
        for (int i = tid; i < d.N; i += kOptThreads) {
            const float t = u[i];
            if (t > v || (t == v && i < idx)) { v = t; idx = i; }
        }
        block_argbest<kOptWarps, true>(v, idx, shf, shi);
        if (idx == 0x7fffffff) break;
        if (cnt >= d.k && (double)v < kth - 2.0 * err) break;
        if (tid == 0) { cand[cnt] = idx; u[idx] = -INFINITY; }
        if (cnt == d.k - 1) kth = (double)v;
        ++cnt;
        __syncthreads();
    }
    __syncthreads();
    const float* x = d.x + (long long)b * d.D;
    for (int j = w; j < cnt; j += kOptWarps) {
        const double d2 = warp_dist2(x, d.y + (long long)cand[j] * d.D, d.D);
        if (lane == 0) cd2[j] = d2;
    }
    __syncthreads();
    // rank sort of (distance, index): ranks are distinct because the indices are
    for (int j = tid; j < cnt; j += kOptThreads) {
        const double dj = cd2[j];
        const int ij = cand[j];
        int r = 0;
        for (int t = 0; t < cnt; ++t) r += (cd2[t] < dj || (cd2[t] == dj && cand[t] < ij)) ? 1 : 0;
        if (r < d.k) {
            d.dist[(long long)b * d.k + r] = (float)sqrt(dj);
            d.idx[(long long)b * d.k + r] = ij;
        }
    }
}

}  // namespace dsb

dsb::OpCheck dsb::opt_prep_check(const ds_opt_prep_desc& d) {
    if (d.B <= 0 || d.D <= 0 || d.pitch < d.D || (d.pitch & 7)) return {-1, "opt_prep: shape"};
    return {0, nullptr};
}

extern "C" int ds_opt_prep_launch(const ds_opt_prep_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::opt_prep_check(*d).rc) return rc;
    dsb::opt_prep_kernel<<<d->B, 256, 0, stream>>>(*d);
    return dsb::opt_ok();
}

dsb::OpCheck dsb::opt_softmax_check(const ds_opt_softmax_desc& d) {
    if (d.B <= 0 || d.N <= 0 || d.nslice <= 0 || d.ldp < d.N || d.ldP < d.N) return {-1, "opt_softmax: shape"};
    if (d.nsig != 1 && d.nsig != d.B) return {-1, "opt_softmax: nsig"};
    return {0, nullptr};
}

extern "C" int ds_opt_softmax_launch(const ds_opt_softmax_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::opt_softmax_check(*d).rc) return rc;
    dsb::opt_softmax_kernel<<<d->B, dsb::kOptThreads, 0, stream>>>(*d);
    return dsb::opt_ok();
}

dsb::OpCheck dsb::opt_reduce_check(const ds_opt_reduce_desc& d) {
    if (d.rows <= 0 || d.cols <= 0 || d.ld < d.cols || d.nsplit <= 0) return {-1, "opt_reduce: shape"};
    return {0, nullptr};
}

extern "C" int ds_opt_reduce_launch(const ds_opt_reduce_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::opt_reduce_check(*d).rc) return rc;
    long long blocks = (d->rows * d->cols + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    dsb::opt_reduce_kernel<<<(unsigned)blocks, 256, 0, stream>>>(*d);
    return dsb::opt_ok();
}

dsb::OpCheck dsb::opt_knn_check(const ds_opt_knn_desc& d) {
    if (d.B <= 0 || d.N <= 0 || d.ldp < d.N) return {-1, "opt_knn: shape"};
    if (d.k <= 0 || d.k > DS_KNN_MAX || d.k > d.N) return {-1, "opt_knn: k"};
    return {0, nullptr};
}

extern "C" int ds_opt_knn_launch(const ds_opt_knn_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::opt_knn_check(*d).rc) return rc;
    dsb::opt_knn_kernel<<<d->B, dsb::kOptThreads, 0, stream>>>(*d);
    return dsb::opt_ok();
}

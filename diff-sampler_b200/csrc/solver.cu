// Solver-side kernels: the fused sigma-scaled update (one HBM pass per step) and the exact
// per-sample 0.995-quantile used by dynamic thresholding.
#include "ops.h"
#include <math.h>

namespace dsb {

__device__ __forceinline__ float4 ld4(const float* p, long long i4) { return __ldcs(reinterpret_cast<const float4*>(p) + i4); }
__device__ __forceinline__ void st4(float* p, long long i4, float4 v) { __stcs(reinterpret_cast<float4*>(p) + i4, v); }

__device__ __forceinline__ int b_of(long long i4, long long n4_per_sample) { return (int)(i4 / n4_per_sample); }

// (v * 127.5 + 128).clip(0, 255).to(uint8) as sample.py:311 evaluates it in fp32: the product and the sum are rounded separately.
// A contracted FFMA rounds once and truncates to one less for inputs within an ulp of a boundary (N - 128) / 127.5;
// __fmul_rn / __fadd_rn are never contracted.  NaN maps to 0: fmaxf returns the non-NaN operand.
__device__ __forceinline__ unsigned char image_u8(float v) {
    return (unsigned char)fminf(fmaxf(__fadd_rn(__fmul_rn(v, 127.5f), 128.0f), 0.0f), 255.0f);
}

template <int NH, int MODE>
__global__ void __launch_bounds__(256) update_kernel(ds_update_desc d, long long n4_total, long long n4_per_sample) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4_total; i += stride) {
        float cx = d.coef[0], c0 = d.coef[1], c1 = d.coef[2], c2 = d.coef[3], c3 = d.coef[4], c4 = d.coef[5];
        float t = d.t;
        int b = 0;
        if (d.coef_dev || d.t_dev || d.thr) b = (int)(i / n4_per_sample);
        if (d.coef_dev) {
            cx = d.coef_dev[0 * d.B + b]; c0 = d.coef_dev[1 * d.B + b]; c1 = d.coef_dev[2 * d.B + b];
            c2 = d.coef_dev[3 * d.B + b]; c3 = d.coef_dev[4 * d.B + b]; c4 = d.coef_dev[5 * d.B + b];
        }
        if (d.t_dev) t = d.t_dev[b];
        const float4 xb = ld4(d.xb, i);
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
        if (MODE == DS_M_X0) {
            m = ld4(d.D, i);
            if (d.thr) {
                const float s = d.thr[b];
                m.x = fminf(fmaxf(m.x, -s), s) / s; m.y = fminf(fmaxf(m.y, -s), s) / s;
                m.z = fminf(fmaxf(m.z, -s), s) / s; m.w = fminf(fmaxf(m.w, -s), s) / s;
            }
        } else if (MODE == DS_M_EPS) {
            const float4 xs = d.xs ? ld4(d.xs, i) : xb;
            const float4 D = ld4(d.D, i);
            m.x = (xs.x - D.x) / t; m.y = (xs.y - D.y) / t; m.z = (xs.z - D.z) / t; m.w = (xs.w - D.w) / t;
        } else if (MODE == DS_M_DIV) {
            const float4 xs = d.xs ? ld4(d.xs, i) : xb;
            m.x = xs.x / t; m.y = xs.y / t; m.z = xs.z / t; m.w = xs.w / t;
        }
        float4 o;
        o.x = cx * xb.x + c0 * m.x; o.y = cx * xb.y + c0 * m.y; o.z = cx * xb.z + c0 * m.z; o.w = cx * xb.w + c0 * m.w;
        if (NH >= 1) { const float4 h = ld4(d.h[0], i); o.x += c1 * h.x; o.y += c1 * h.y; o.z += c1 * h.z; o.w += c1 * h.w; }
        if (NH >= 2) { const float4 h = ld4(d.h[1], i); o.x += c2 * h.x; o.y += c2 * h.y; o.z += c2 * h.z; o.w += c2 * h.w; }
        if (NH >= 3) { const float4 h = ld4(d.h[2], i); o.x += c3 * h.x; o.y += c3 * h.y; o.z += c3 * h.z; o.w += c3 * h.w; }
        if (NH >= 4) { const float4 h = ld4(d.h[3], i); o.x += c4 * h.x; o.y += c4 * h.y; o.z += c4 * h.z; o.w += c4 * h.w; }
        if (d.out_x) st4(d.out_x, i, o);
        if (d.out_m) st4(d.out_m, i, m);
        if (d.out_u8) {
            // the four values are consecutive pixels of one channel plane (HW % 4 == 0): scatter them into the NHWC byte image
            const long long e = (i - (long long)b_of(i, n4_per_sample) * n4_per_sample) * 4;     // element offset inside the sample
            const int c = (int)(e / d.u8_HW), p = (int)(e - (long long)c * d.u8_HW);
            unsigned char* dst = d.out_u8 + ((long long)b_of(i, n4_per_sample) * d.u8_HW + p) * d.u8_C + c;
            const float v[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) dst[(long long)k * d.u8_C] = image_u8(v[k]);
        }
    }
}

template <int NH>
static int launch_update_nh(const ds_update_desc& d, long long n4, long long n4ps, int grid, cudaStream_t s) {
    switch (d.mode) {
        case DS_M_X0: update_kernel<NH, DS_M_X0><<<grid, 256, 0, s>>>(d, n4, n4ps); break;
        case DS_M_EPS: update_kernel<NH, DS_M_EPS><<<grid, 256, 0, s>>>(d, n4, n4ps); break;
        case DS_M_DIV: update_kernel<NH, DS_M_DIV><<<grid, 256, 0, s>>>(d, n4, n4ps); break;
        case DS_M_NONE: update_kernel<NH, DS_M_NONE><<<grid, 256, 0, s>>>(d, n4, n4ps); break;
        default: return -2;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------ quantile
// One CTA per sample.  |x| bit patterns are monotone as uint32, so an MSB-first 8-bit radix select
// finds the exact k-th order statistic; the (k+1)-th is either equal or the minimum of the larger keys.
// KEYS_IN_SMEM = false: rows too long for shared memory (> 50 K elements, e.g. 3x256x256 pixel models) re-read |x| from global memory
// (L2-resident after the first pass) in each of the five passes instead of staging the keys.
template <bool KEYS_IN_SMEM>
__global__ void __launch_bounds__(256) threshold_kernel(ds_threshold_desc d) {
    extern __shared__ uint32_t keys_smem[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_prefix, s_k, s_less;
    __shared__ uint32_t s_min_above;
    const int b = blockIdx.x;
    const int n = d.row_len;
    const float* x = d.x0 + (long long)b * n;
    auto key_at = [&](int i) -> uint32_t { return KEYS_IN_SMEM ? keys_smem[i] : __float_as_uint(fabsf(__ldg(x + i))); };
    if (KEYS_IN_SMEM)
        for (int i = threadIdx.x; i < n; i += blockDim.x) keys_smem[i] = __float_as_uint(fabsf(x[i]));
    // rank arithmetic in fp32, as torch.quantile does for an fp32 input
    const float rank = d.q * (float)(n - 1);
    const float below = floorf(rank);
    const float w = rank - below;
    const uint32_t k = (uint32_t)below;
    if (threadIdx.x == 0) { s_prefix = 0; s_k = k; s_less = 0; s_min_above = 0xFFFFFFFFu; }
    __syncthreads();
    uint32_t mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        hist[threadIdx.x] = 0;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t key = key_at(i);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xFF], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t kk = s_k, acc = 0;
            int bin = 0;
            for (; bin < 256; ++bin) {
                if (acc + hist[bin] > kk) break;
                acc += hist[bin];
            }
            s_k = kk - acc;
            s_less += acc;
            s_prefix = prefix | ((uint32_t)bin << shift);
        }
        mask |= 0xFFu << shift;
        __syncthreads();
    }
    const uint32_t vk = s_prefix;       // exact k-th smallest key
    // count of keys == vk and min of keys > vk
    uint32_t my_eq = 0, my_min = 0xFFFFFFFFu;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t key = key_at(i);
        if (key == vk) ++my_eq;
        else if (key > vk && key < my_min) my_min = key;
    }
    __syncthreads();
    hist[threadIdx.x] = my_eq;
    atomicMin(&s_min_above, my_min);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t eq = 0;
        for (int i = 0; i < 256; ++i) eq += hist[i];
        const float lo = __uint_as_float(vk);
        float hi = lo;
        if ((uint32_t)(k + 1) < (uint32_t)n && !(s_less + eq > k + 1)) hi = __uint_as_float(s_min_above);
        // torch lerp: a + w*(b-a) for w < 0.5, else b - (b-a)*(1-w)
        const float diff = hi - lo;
        const float qv = (w < 0.5f) ? (lo + w * diff) : (hi - diff * (1.0f - w));
        d.thr[b] = fmaxf(qv, d.floor_val);
    }
}

// ------------------------------------------------------------------------------------------ GITS cost
// grid (pairs, B); pair p -> (i, j), i < j.  One pass over 5 streams (traj[i], eps[i], traj[j], traj[0], traj[N-1]).
__global__ void __launch_bounds__(256) gits_cost_kernel(ds_gits_cost_desc d) {
    // decode the pair index
    int p = blockIdx.x, i = 0;
    while (p >= d.N - 1 - i) { p -= d.N - 1 - i; ++i; }
    const int j = i + 1 + p;
    const int b = blockIdx.y;
    const float h = d.t[j] - d.t[i];
    const long long n4 = d.n / 4;
    const long long stride = (long long)d.B * d.n;
    const float4* xi = reinterpret_cast<const float4*>(d.traj + (long long)i * stride + (long long)b * d.n);
    const float4* di = reinterpret_cast<const float4*>(d.eps + (long long)i * stride + (long long)b * d.n);
    const float4* xj = reinterpret_cast<const float4*>(d.traj + (long long)j * stride + (long long)b * d.n);
    const float4* x0 = reinterpret_cast<const float4*>(d.traj + (long long)b * d.n);
    const float4* xc = reinterpret_cast<const float4*>(d.traj + (long long)(d.N - 1) * stride + (long long)b * d.n);
    double s1 = 0, s2 = 0, s3 = 0, s4 = 0;
    for (long long k = threadIdx.x; k < n4; k += blockDim.x) {
        const float4 a = xi[k], dd = di[k], r = xj[k], b0 = x0[k], c = xc[k];
        const float xs[4] = {a.x + h * dd.x, a.y + h * dd.y, a.z + h * dd.z, a.w + h * dd.w};
        const float rr[4] = {r.x, r.y, r.z, r.w};
        const float bb[4] = {b0.x, b0.y, b0.z, b0.w};
        const float cc[4] = {c.x, c.y, c.z, c.w};
        float l1 = 0.f, l2 = 0.f, q1 = 0.f, q2 = 0.f;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const float e = xs[m] - rr[m];
            l1 += fabsf(e);
            l2 += e * e;
            const float ca = cc[m] - xs[m];
            q1 += ca * ca;
            q2 += ca * (cc[m] - bb[m]);
        }
        s1 += l1; s2 += l2; s3 += q1; s4 += q2;
    }
    __shared__ double red[4][8];
    double v[4] = {s1, s2, s3, s4};
#pragma unroll
    for (int m = 0; m < 4; ++m) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[m] += __shfl_xor_sync(0xffffffffu, v[m], o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][warp] = v[0]; red[1][warp] = v[1]; red[2][warp] = v[2]; red[3][warp] = v[3]; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double acc = 0;
        for (int w = 0; w < 8; ++w) acc += red[threadIdx.x][w];
        d.out[(((long long)i * d.N + j) * d.B + b) * 4 + threadIdx.x] = acc;
    }
}

// ------------------------------------------------------------------------------------------ AMED predictor
// The whole predictor (amed-solver-main/training/networks.py:121-155) for one sample per CTA: time embeddings of t_cur and t_next
// (PositionalEmbedding(8, endpoint=True) with the sin/cos swap, map_layer0, SiLU), bottleneck MLP (in -> hidden -> z, SiLU between),
// the sigmoid heads, and the geometric intermediate time t_mid = t_next^r * t_cur^(1-r) (solvers_amed.py:119).  Replaces ~25 ATen
// launches per sampling step.  Weights: one packed fp32 buffer (amed_predictor.pack): map_layer0 W[nc][nc], b[nc]; enc_layer0 W[hid][in],
// b[hid]; enc_layer1 W[z][hid], b[z]; fc_r W[z + 2 nc], b; then fc_scale_dir and fc_scale_time (W, b each) if present.
struct AmedDims { int in_dim, hid, z, nc, has_dir, has_time; };

__global__ void __launch_bounds__(256) amed_predict_kernel(const float* __restrict__ w, AmedDims dm, const float* __restrict__ bott,
                                                           const float* __restrict__ t_cur_p, const float* __restrict__ t_next_p,
                                                           float scale_dir, float scale_time, float* __restrict__ out, int B) {
    __shared__ float s_x[256], s_h[256], s_feat[64];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int nc = dm.nc, half = nc / 2;
    const float* w_map = w;
    const float* b_map = w_map + nc * nc;
    const float* w0 = b_map + nc;
    const float* b0 = w0 + dm.hid * dm.in_dim;
    const float* w1 = b0 + dm.hid;
    const float* b1 = w1 + dm.z * dm.hid;
    const int nf = dm.z + 2 * nc;
    const float* w_r = b1 + dm.z;
    const float t_cur = *t_cur_p, t_next = *t_next_p;
    if (tid < dm.in_dim) s_x[tid] = bott ? bott[(long long)b * dm.in_dim + tid] : 0.f;
    // time embeddings: e = [sin(t f_i) | cos(t f_i)], f_i = (1/10000)^(i / (half - 1)); feat[z + k] (t_cur), feat[z + nc + k] (t_next)
    if (tid < 2 * nc) {
        const int which = tid / nc, k = tid % nc;
        const float t = which ? t_next : t_cur;
        float acc = b_map[k];
        for (int i = 0; i < nc; ++i) {
            const int fi = i % half;
            const float f = powf(1.0f / 10000.0f, (float)fi / (float)(half - 1));
            const float e = (i < half) ? sinf(t * f) : cosf(t * f);
            acc = fmaf(w_map[k * nc + i], e, acc);
        }
        s_feat[dm.z + which * nc + k] = acc / (1.0f + expf(-acc));
    }
    __syncthreads();
    if (tid < dm.hid) {
        float acc = b0[tid];
        const float* row = w0 + (long long)tid * dm.in_dim;
        for (int i = 0; i < dm.in_dim; ++i) acc = fmaf(row[i], s_x[i], acc);
        s_h[tid] = acc / (1.0f + expf(-acc));
    }
    __syncthreads();
    if (tid < dm.z) {
        float acc = b1[tid];
        const float* row = w1 + (long long)tid * dm.hid;
        for (int j = 0; j < dm.hid; ++j) acc = fmaf(row[j], s_h[j], acc);
        s_feat[tid] = acc;
    }
    __syncthreads();
    if (tid == 0) {
        auto head = [&](const float* wh) {
            float acc = wh[nf];
            for (int i = 0; i < nf; ++i) acc = fmaf(wh[i], s_feat[i], acc);
            return 1.0f / (1.0f + expf(-acc));
        };
        const float r = head(w_r);
        const float* wn = w_r + nf + 1;
        float sd = 1.0f, st = 1.0f;
        if (dm.has_dir) { sd = head(wn) / (1.0f / (2.0f * scale_dir)) + (1.0f - scale_dir); wn += nf + 1; }
        if (dm.has_time) st = head(wn) / (1.0f / (2.0f * scale_time)) + (1.0f - scale_time);
        out[0 * B + b] = r;
        out[1 * B + b] = sd;
        out[2 * B + b] = st;
        out[3 * B + b] = powf(t_next, r) * powf(t_cur, 1.0f - r);
    }
}

// ------------------------------------------------------------------------------------------ image epilogue
// (x * 127.5 + 128).clip(0, 255) -> uint8, NCHW -> NHWC  (sample.py:311): one pass instead of five ATen launches.
__global__ void to_uint8_nhwc_kernel(const float* x, unsigned char* out, int B, int Cc, int HW) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;       // one thread per (n, pixel)
    if (idx >= (long long)B * HW) return;
    const int n = (int)(idx / HW), p = (int)(idx - (long long)n * HW);
    for (int c = 0; c < Cc; ++c) out[idx * Cc + c] = image_u8(x[((long long)n * Cc + c) * HW + p]);
}

}  // namespace dsb

using namespace dsb;

extern "C" int ds_amed_predict_launch(const float* w, const int* dims6, const float* bott, const float* t_cur, const float* t_next,
                                      float scale_dir, float scale_time, float* out, int B, cudaStream_t stream) {
    AmedDims dm = {dims6[0], dims6[1], dims6[2], dims6[3], dims6[4], dims6[5]};
    if (dm.in_dim <= 0 || dm.in_dim > 256 || dm.hid <= 0 || dm.hid > 256 || dm.z <= 0 || dm.nc < 4 || dm.nc % 2 || dm.z + 2 * dm.nc > 64 || B <= 0)
        return -2;
    amed_predict_kernel<<<B, 256, 0, stream>>>(w, dm, bott, t_cur, t_next, scale_dir, scale_time, out, B);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int ds_to_uint8_launch(const float* x, unsigned char* out, int B, int Cc, int HW, cudaStream_t stream) {
    const long long total = (long long)B * HW;
    to_uint8_nhwc_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, out, B, Cc, HW);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int ds_gits_cost_launch(const ds_gits_cost_desc* d, cudaStream_t stream) {
    if (d->n % 4 || d->N < 2) return -2;
    const int pairs = d->N * (d->N - 1) / 2;
    gits_cost_kernel<<<dim3(pairs, d->B), 256, 0, stream>>>(*d);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int ds_update_launch(const ds_update_desc* dp, cudaStream_t stream) {
    const ds_update_desc& d = *dp;
    if (d.n_per_sample % 4) return -2;
    const long long n4ps = d.n_per_sample / 4;
    const long long n4 = n4ps * d.B;
    if (n4 == 0) return 0;
    if (d.out_u8 && (d.u8_HW % 4 || (long long)d.u8_C * d.u8_HW != d.n_per_sample)) return -2;
    long long blocks = (n4 + 255) / 256;
    static int sms[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
    const long long cap = (long long)(sms[dev] > 0 ? sms[dev] : 132) * 16;
    const int grid = (int)(blocks < cap ? blocks : cap);
    int rc;
    switch (d.nhist) {
        case 0: rc = launch_update_nh<0>(d, n4, n4ps, grid, stream); break;
        case 1: rc = launch_update_nh<1>(d, n4, n4ps, grid, stream); break;
        case 2: rc = launch_update_nh<2>(d, n4, n4ps, grid, stream); break;
        case 3: rc = launch_update_nh<3>(d, n4, n4ps, grid, stream); break;
        case 4: rc = launch_update_nh<4>(d, n4, n4ps, grid, stream); break;
        default: return -2;
    }
    if (rc) return rc;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int ds_threshold_launch(const ds_threshold_desc* d, cudaStream_t stream) {
    if (d->B <= 0 || d->row_len <= 0) return -2;
    const size_t smem = (size_t)d->row_len * sizeof(uint32_t);
    if (smem > 200 * 1024) {                       // long rows: keys stay in global memory / L2
        threshold_kernel<false><<<d->B, 256, 0, stream>>>(*d);
        return cudaGetLastError() == cudaSuccess ? 0 : -1;
    }
    if (smem > 40 * 1024) {      // dynamic + ~1.1 KB static must stay under the 48 KB default, else opt in
        // the opt-in shared-memory limit is a per-device function attribute: set it on every device this process uses
        static bool attr_set[64] = {};
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64 || !attr_set[dev]) {
            if (cudaFuncSetAttribute(threshold_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) return -3;
            if (dev >= 0 && dev < 64) attr_set[dev] = true;
        }
    }
    threshold_kernel<true><<<d->B, 256, smem, stream>>>(*d);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

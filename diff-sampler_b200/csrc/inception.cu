// The ops of the Inception-v3 FID feature extractor that are not convolutions (inception_plan.py; DESIGN.md 4.10): the TF1 legacy
// bilinear input resize, im2col for the k > 1 convolutions that run on the GEMM kernel in rows mode, and max / average / global-mean
// pooling.  All are memory bound; one thread per output element group, no shared memory.
#include "ops.h"
#include <cuda_fp16.h>
#include <math.h>

namespace dsb {

static int ok() { return cudaGetLastError() == cudaSuccess ? 0 : -1; }

static unsigned grid_of(long long threads, int block) { return (unsigned)((threads + block - 1) / block); }

// ------------------------------------------------------------------------------------------ input stage
// One thread per output pixel (n, i, j).  TF1 ResizeBilinear without half-pixel centres: source row i H / Ho (computed in fp64 from the
// exact integer product), neighbours floor and floor + 1 (clamped), then (v - 128) / 128.
__global__ void img_input_kernel(const ds_img_input_desc d) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)d.B * d.Ho * d.Wo;
    if (t >= total) return;
    const int j = (int)(t % d.Wo);
    const int i = (int)((t / d.Wo) % d.Ho);
    const int n = (int)(t / ((long long)d.Wo * d.Ho));
    const double fy = (double)((long long)i * d.H) / d.Ho, fx = (double)((long long)j * d.W) / d.Wo;
    const int y0 = (int)floor(fy), x0 = (int)floor(fx);
    const int y1 = min(y0 + 1, d.H - 1), x1 = min(x0 + 1, d.W - 1);
    const double dy = fy - y0, dx = fx - x0;
    const unsigned char* s = d.src + n * d.sn;
    float* o = d.out + t * d.C;
    for (int c = 0; c < d.C; ++c) {
        const unsigned char* sc = s + c * d.sc;
        const double tl = sc[y0 * d.sy + x0 * d.sx], tr = sc[y0 * d.sy + x1 * d.sx];
        const double bl = sc[y1 * d.sy + x0 * d.sx], br = sc[y1 * d.sy + x1 * d.sx];
        const double top = tl + (tr - tl) * dx, bot = bl + (br - bl) * dx;
        o[c] = (float)((top + (bot - top) * dy - 128.0) / 128.0);
    }
}

OpCheck img_input_check(const ds_img_input_desc& d) {
    if (d.B < 1 || d.C < 1 || d.H < 1 || d.W < 1 || d.Ho < 1 || d.Wo < 1) return {-2, "img_input: shape"};
    return {0, nullptr};
}

// ------------------------------------------------------------------------------------------ im2col
__device__ __forceinline__ void store8(__half* hi, __half* lo, const float* v) {
    __align__(16) __half h[8];
    __align__(16) __half l[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        h[k] = __float2half_rn(v[k]);
        l[k] = __float2half_rn(v[k] - __half2float(h[k]));
    }
    *reinterpret_cast<uint4*>(hi) = *reinterpret_cast<const uint4*>(h);
    if (lo) *reinterpret_cast<uint4*>(lo) = *reinterpret_cast<const uint4*>(l);
}

// One thread per 8 consecutive columns of one row.  VEC (C, pitch and channel base multiples of 8 and 4): the 8 columns are 8 channels
// of one tap, two float4 loads; otherwise each column is located on its own (the 3-channel stem).
template <bool VEC>
__global__ void im2col_kernel(const ds_im2col_desc d, const int Ho, const int Wo) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int groups = d.K64 / 8;
    const long long rows = (long long)d.B * Ho * Wo;
    if (t >= rows * groups) return;
    const long long r = t / groups;
    const int k0 = (int)(t - r * groups) * 8;
    const int ox = (int)(r % Wo);
    const int oy = (int)((r / Wo) % Ho);
    const int n = (int)(r / ((long long)Wo * Ho));
    const int kvalid = d.kh * d.kw * d.C;
    float v[8];
    if (VEC) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = 0.f;
        if (k0 < kvalid) {
            const int tap = k0 / d.C, c = k0 - tap * d.C;
            const int iy = oy * d.sh - d.ph + tap / d.kw, ix = ox * d.sw - d.pw + tap % d.kw;
            if (iy >= 0 && iy < d.H && ix >= 0 && ix < d.W) {
                const float* s = d.src + (((long long)n * d.H + iy) * d.W + ix) * d.src_pitch + d.src_c0 + c;
                const float4 a = __ldg(reinterpret_cast<const float4*>(s)), b = __ldg(reinterpret_cast<const float4*>(s + 4));
                v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int kk = k0 + k;
            v[k] = 0.f;
            if (kk < kvalid) {
                const int tap = kk / d.C, c = kk - tap * d.C;
                const int iy = oy * d.sh - d.ph + tap / d.kw, ix = ox * d.sw - d.pw + tap % d.kw;
                if (iy >= 0 && iy < d.H && ix >= 0 && ix < d.W)
                    v[k] = __ldg(d.src + (((long long)n * d.H + iy) * d.W + ix) * d.src_pitch + d.src_c0 + c);
            }
        }
    }
    __half* hi = static_cast<__half*>(d.out) + r * d.K64 + k0;
    store8(hi, d.nplanes == 2 ? hi + rows * d.K64 : nullptr, v);
}

OpCheck im2col_check(const ds_im2col_desc& d) {
    if (d.B < 1 || d.H < 1 || d.W < 1 || d.C < 1 || d.kh < 1 || d.kw < 1 || d.sh < 1 || d.sw < 1 || d.ph < 0 || d.pw < 0 ||
        d.H + 2 * d.ph < d.kh || d.W + 2 * d.pw < d.kw)
        return {-2, "im2col: shape"};
    if (d.K64 % 64 != 0 || d.K64 < d.kh * d.kw * d.C) return {-2, "im2col: K64"};
    if (d.src_c0 < 0 || d.src_c0 + d.C > d.src_pitch) return {-2, "im2col: channels"};
    if (d.nplanes != 1 && d.nplanes != 2) return {-2, "im2col: nplanes"};
    return {0, nullptr};
}

// ------------------------------------------------------------------------------------------ pooling
// Modes 0 / 1: one thread per (output pixel, 4 channels).
__global__ void pool_kernel(const ds_pool_desc d, const int Ho, const int Wo) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int q = d.C / 4;
    const long long rows = (long long)d.B * Ho * Wo;
    if (t >= rows * q) return;
    const long long r = t / q;
    const int c = (int)(t - r * q) * 4;
    const int ox = (int)(r % Wo);
    const int oy = (int)((r / Wo) % Ho);
    const int n = (int)(r / ((long long)Wo * Ho));
    const bool is_max = d.mode == DS_POOL_MAX;
    float4 acc = is_max ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    const int y0 = oy * d.stride - d.pad, x0 = ox * d.stride - d.pad;
    for (int i = max(y0, 0); i < min(y0 + d.k, d.H); ++i)
        for (int j = max(x0, 0); j < min(x0 + d.k, d.W); ++j) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(d.src + (((long long)n * d.H + i) * d.W + j) * d.src_pitch + d.src_c0 + c));
            if (is_max) {
                acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w);
            } else {
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            ++cnt;
        }
    if (!is_max) {
        const float inv = (float)cnt;
        acc.x /= inv; acc.y /= inv; acc.z /= inv; acc.w /= inv;
    }
    const long long o = r * d.out_pitch + d.out_c0 + c;
    if (d.out_f32) *reinterpret_cast<float4*>(d.out_f32 + o) = acc;
    if (d.out_h16) {
        const float a[4] = {acc.x, acc.y, acc.z, acc.w};
        __align__(8) __half h[4];
        __align__(8) __half l[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            h[k] = __float2half_rn(a[k]);
            l[k] = __float2half_rn(a[k] - __half2float(h[k]));
        }
        __half* oh = static_cast<__half*>(d.out_h16) + o;
        *reinterpret_cast<uint2*>(oh) = *reinterpret_cast<const uint2*>(h);
        if (d.nplanes == 2) *reinterpret_cast<uint2*>(oh + rows * d.out_pitch) = *reinterpret_cast<const uint2*>(l);
    }
}

// Mode 2: one thread per (sample, channel), the H x W pixels added in order in fp64.
__global__ void pool_mean_kernel(const ds_pool_desc d) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)d.B * d.C) return;
    const int n = (int)(t / d.C), c = (int)(t - (long long)n * d.C);
    const int hw = d.H * d.W;
    const float* s = d.src + (long long)n * hw * d.src_pitch + d.src_c0 + c;
    double acc = 0.0;
    for (int p = 0; p < hw; ++p) acc += __ldg(s + (long long)p * d.src_pitch);
    d.out_f32[(long long)n * d.out_pitch + d.out_c0 + c] = (float)(acc / hw);
}

OpCheck pool_check(const ds_pool_desc& d) {
    if (d.mode < DS_POOL_MAX || d.mode > DS_POOL_MEAN) return {-2, "pool: mode"};
    if (d.B < 1 || d.H < 1 || d.W < 1 || d.C < 1) return {-2, "pool: shape"};
    // every window holds an in-image pixel when pad < k
    if (d.mode != DS_POOL_MEAN && (d.k < 1 || d.stride < 1 || d.pad < 0 || d.pad >= d.k || d.H + 2 * d.pad < d.k || d.W + 2 * d.pad < d.k))
        return {-2, "pool: window"};
    if (d.src_c0 < 0 || d.src_c0 + d.C > d.src_pitch || d.out_c0 < 0 || d.out_c0 + d.C > d.out_pitch) return {-2, "pool: channels"};
    // float4 loads and stores, 4-half fp16 stores
    if (d.mode != DS_POOL_MEAN && (d.C % 4 || d.src_pitch % 4 || d.src_c0 % 4 || d.out_pitch % 4 || d.out_c0 % 4))
        return {-2, "pool: alignment"};
    if (d.mode == DS_POOL_MEAN ? (!d.out_f32 || d.out_h16) : (!d.out_f32 && !d.out_h16)) return {-2, "pool: outputs"};
    if (d.out_h16 && d.nplanes != 1 && d.nplanes != 2) return {-2, "pool: nplanes"};
    return {0, nullptr};
}

}  // namespace dsb

extern "C" int ds_img_input_launch(const ds_img_input_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::img_input_check(*d).rc) return rc;
    dsb::img_input_kernel<<<dsb::grid_of((long long)d->B * d->Ho * d->Wo, 256), 256, 0, stream>>>(*d);
    return dsb::ok();
}

extern "C" int ds_im2col_launch(const ds_im2col_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::im2col_check(*d).rc) return rc;
    const int Ho = (d->H + 2 * d->ph - d->kh) / d->sh + 1, Wo = (d->W + 2 * d->pw - d->kw) / d->sw + 1;
    const unsigned grid = dsb::grid_of((long long)d->B * Ho * Wo * (d->K64 / 8), 256);
    if (d->C % 8 == 0 && d->src_pitch % 4 == 0 && d->src_c0 % 4 == 0) dsb::im2col_kernel<true><<<grid, 256, 0, stream>>>(*d, Ho, Wo);
    else dsb::im2col_kernel<false><<<grid, 256, 0, stream>>>(*d, Ho, Wo);
    return dsb::ok();
}

extern "C" int ds_pool_launch(const ds_pool_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::pool_check(*d).rc) return rc;
    if (d->mode == DS_POOL_MEAN) {
        dsb::pool_mean_kernel<<<dsb::grid_of((long long)d->B * d->C, 256), 256, 0, stream>>>(*d);
        return dsb::ok();
    }
    const int Ho = (d->H + 2 * d->pad - d->k) / d->stride + 1, Wo = (d->W + 2 * d->pad - d->k) / d->stride + 1;
    dsb::pool_kernel<<<dsb::grid_of((long long)d->B * Ho * Wo * (d->C / 4), 256), 256, 0, stream>>>(*d, Ho, Wo);
    return dsb::ok();
}

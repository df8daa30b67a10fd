// The ops of the CLIP score that are not transformer layers (openclip_plan.py; DESIGN.md 4.11): the image preprocessing of open_clip's
// ViT-g-14 transform (Pillow bicubic resize, centre crop, ToTensor, Normalize) and the pooled heads (row gather, L2 normalisation,
// score).  Both are memory bound; no shared memory.
#include "ops.h"
#include <math.h>

namespace dsb {

static int ok() { return cudaGetLastError() == cudaSuccess ? 0 : -1; }

static constexpr int kPrecisionBits = 22;           // Pillow's PRECISION_BITS (32 - 8 - 2) of the 8-bit resample passes

// Pillow's clip8: the fixed-point sum (rounding bias included) -> uint8
__device__ __forceinline__ int clip8(int v) {
    if (v >= (1 << kPrecisionBits << 8)) return 255;
    if (v <= 0) return 0;
    return v >> kPrecisionBits;
}

// ------------------------------------------------------------------------------------------ image input
// One thread per output pixel (n, i, j).  The horizontal pass is evaluated for each source row the vertical pass reads and rounded to
// uint8 as Pillow's intermediate image is; the two int32 sums are those of ImagingResampleHorizontal_8bpc / ImagingResampleVertical_8bpc.
__global__ void clip_input_kernel(const ds_clip_input_desc d) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)d.B * d.S * d.S;
    if (t >= total) return;
    const int j = (int)(t % d.S);
    const int i = (int)((t / d.S) % d.S);
    const int n = (int)(t / ((long long)d.S * d.S));
    const int32_t* y0 = d.tab;
    const int32_t* ny = y0 + d.S;
    const int32_t* x0 = ny + d.S;
    const int32_t* nx = x0 + d.S;
    const int32_t* wy = nx + d.S + (long long)i * d.ky;
    const int32_t* wx = nx + d.S + (long long)d.S * d.ky + (long long)j * d.kx;
    const int ys = __ldg(y0 + i), yn = __ldg(ny + i), xs = __ldg(x0 + j), xn = __ldg(nx + j);
    const unsigned char* s = d.src + n * d.sn + xs * d.sx;
    int acc[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
    for (int y = 0; y < yn; ++y) {
        const unsigned char* row = s + (long long)(ys + y) * d.sy;
        const int ky = __ldg(wy + y);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const unsigned char* px = row + c * d.sc;
            int h = 1 << (kPrecisionBits - 1);
            for (int x = 0; x < xn; ++x) h += (int)px[x * d.sx] * __ldg(wx + x);
            acc[c] += clip8(h) * ky;
        }
    }
    float* o = d.out + t * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = ((float)clip8(acc[c]) / 255.0f - d.mean[c]) / d.std[c];
}

OpCheck clip_input_check(const ds_clip_input_desc& d) {
    if (d.B < 1 || d.H < 1 || d.W < 1 || d.S < 1) return {-2, "clip_input: shape"};
    // every output row / column reads at least one source sample and at most Pillow's ksize, 2 ceil(2 max(scale, 1)) + 1, where the
    // scale (input over resized size) is at most input / S
    const int ky_max = 2 * max((2 * d.H + d.S - 1) / d.S, 2) + 1, kx_max = 2 * max((2 * d.W + d.S - 1) / d.S, 2) + 1;
    if (d.ky < 1 || d.kx < 1 || d.ky > ky_max || d.kx > kx_max) return {-2, "clip_input: taps"};
    if (!d.tab) return {-2, "clip_input: tables"};
    for (int c = 0; c < 3; ++c) if (!(d.std[c] > 0.f)) return {-2, "clip_input: std"};
    return {0, nullptr};
}

// ------------------------------------------------------------------------------------------ pooled heads
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int k = 0; k < nw; ++k) s += red[k];        // the same order in every thread
    return s;
}

__global__ void clip_head_kernel(const ds_clip_head_desc d) {
    __shared__ double red[32];
    __shared__ int s_row;
    const int n = blockIdx.x;
    if (d.mode == DS_CLIP_GATHER) {
        if (threadIdx.x == 0) {
            int r = d.row;
            if (d.ids) {
                const int32_t* id = d.ids + (long long)n * d.T;
                r = 0;
                for (int t = 1; t < d.T; ++t) if (id[t] > id[r]) r = t;
            }
            s_row = r;
        }
        __syncthreads();
        const float* s = d.src + n * d.src_stride + (long long)s_row * d.C;
        float* o = d.out + n * d.out_stride;
        for (int c = threadIdx.x; c < d.C; c += blockDim.x) o[c] = s[c];
        return;
    }
    const float* a = d.src + (long long)n * d.C;
    if (d.mode == DS_CLIP_L2NORM) {
        double ss = 0.0;
        for (int c = threadIdx.x; c < d.C; c += blockDim.x) ss += (double)a[c] * a[c];
        const double nrm = fmax(sqrt(block_sum(ss, red)), 1e-12);
        for (int c = threadIdx.x; c < d.C; c += blockDim.x) d.out[(long long)n * d.C + c] = (float)(a[c] / nrm);
        return;
    }
    const float* b = d.src2 + (long long)n * d.C;
    double dot = 0.0;
    for (int c = threadIdx.x; c < d.C; c += blockDim.x) dot += (double)a[c] * b[c];
    dot = block_sum(dot, red);
    if (threadIdx.x == 0) d.out[n] = (float)(d.scale * dot);
}

OpCheck clip_head_check(const ds_clip_head_desc& d) {
    if (d.mode < DS_CLIP_GATHER || d.mode > DS_CLIP_SCORE) return {-2, "clip_head: mode"};
    if (d.B < 1 || d.C < 1) return {-2, "clip_head: shape"};
    if (d.mode == DS_CLIP_GATHER && (d.ids ? d.T < 1 : d.row < 0)) return {-2, "clip_head: row"};
    if (!d.src || !d.out || (d.mode == DS_CLIP_SCORE && !d.src2)) return {-2, "clip_head: operands"};
    return {0, nullptr};
}

}  // namespace dsb

extern "C" int ds_clip_input_launch(const ds_clip_input_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::clip_input_check(*d).rc) return rc;
    const long long total = (long long)d->B * d->S * d->S;
    dsb::clip_input_kernel<<<(unsigned)((total + 127) / 128), 128, 0, stream>>>(*d);
    return dsb::ok();
}

extern "C" int ds_clip_head_launch(const ds_clip_head_desc* d, cudaStream_t stream) {
    if (const int rc = dsb::clip_head_check(*d).rc) return rc;
    dsb::clip_head_kernel<<<d->B, 256, 0, stream>>>(*d);
    return dsb::ok();
}

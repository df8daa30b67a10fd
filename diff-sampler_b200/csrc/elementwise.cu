// HBM-bound companions of the tensor-core kernels: GroupNorm statistics / apply (+SiLU, +resample),
// row softmax, timestep embedding, small dense layers, input preparation.  All NHWC, 128-bit accesses.
#include "ops.h"
#include "operand.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace dsb {

__device__ __forceinline__ float silu_f(float v) { return __fdividef(v, 1.0f + __expf(-v)); }

// ------------------------------------------------------------------------------------------ GN stats
// grid (chunks, B); block (ncol4 <= 384, rows).  Thread (tx, ty) owns float4 column tx.
__global__ void gn_stats_kernel(ds_gn_stats_desc d, int pix_per_cta) {
    __shared__ double s_sum[64];
    __shared__ double s_sq[64];
    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    if (tid < 64) { s_sum[tid] = 0.0; s_sq[tid] = 0.0; }
    __syncthreads();
    const int C = d.C0 + d.C1;
    const int cpg = C / d.groups;
    const int n = blockIdx.y;
    const int ncol4 = C / 4;
    const int p_begin = blockIdx.x * pix_per_cta;
    int p_end = p_begin + pix_per_cta;
    if (p_end > d.HW) p_end = d.HW;
    for (int col = threadIdx.x; col < ncol4; col += blockDim.x) {
        const int c = col * 4;
        const float* base;
        int pitch, cc;
        if (c < d.C0) { base = d.src0; pitch = d.C0; cc = c; }
        else { base = d.src1; pitch = d.C1; cc = c - d.C0; }
        const int gA = c / cpg;
        const int gB = (c + 3) / cpg;
        const int nA = (gA == gB) ? 4 : ((gA + 1) * cpg - c);   // channels of this float4 that belong to group A
        float sA = 0.f, qA = 0.f, sB = 0.f, qB = 0.f;
#pragma unroll 8
        for (int p = p_begin + threadIdx.y; p < p_end; p += blockDim.y) {
            const float4 v = __ldcs(reinterpret_cast<const float4*>(base + ((long long)n * d.HW + p) * pitch + cc));
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < nA) { sA += e[j]; qA += e[j] * e[j]; }
                else { sB += e[j]; qB += e[j] * e[j]; }
            }
        }
        atomicAdd(&s_sum[gA], (double)sA);
        atomicAdd(&s_sq[gA], (double)qA);
        if (gB != gA) {
            atomicAdd(&s_sum[gB], (double)sB);
            atomicAdd(&s_sq[gB], (double)qB);
        }
    }
    __syncthreads();
    if (tid < d.groups) {
        atomicAdd(&d.sums[((long long)n * d.groups + tid) * 2 + 0], s_sum[tid]);
        atomicAdd(&d.sums[((long long)n * d.groups + tid) * 2 + 1], s_sq[tid]);
    }
}

// ------------------------------------------------------------------------------------------ GN coefficients
// {mean, 1 / sqrt(var + eps)} of group g of sample n, from its fp64 {sum, sum of squares} over cnt values (D: the apply or finalize
// descriptor).
template <class D>
__device__ __forceinline__ float2 gn_group_stats(const D& d, int n, int g, double cnt) {
    const double s = d.sums[((long long)n * d.groups + g) * 2 + 0];
    const double q = d.sums[((long long)n * d.groups + g) * 2 + 1];
    const double mu = s / cnt;
    double var = q / cnt - mu * mu;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + (double)d.eps));
    return make_float2((float)mu, rstd);
}

// Channel c + j of sample n normalises as y = (x - mean) * a + b: a = rstd * gamma * (1 + ada_scale), b = beta * (1 + ada_scale) +
// ada_shift.
template <class D>
__device__ __forceinline__ void gn_channel_coef(const D& d, int n, int C, int c, int j, float rstd, float& a, float& b) {
    float aa = rstd * __ldg(d.gamma + c + j);
    float bb = __ldg(d.beta + c + j);
    if (d.ada) {
        const float sc = d.ada[(long long)n * d.ada_stride + c + j] + 1.0f;
        const float sh = d.ada[(long long)n * d.ada_stride + C + c + j];
        aa *= sc;
        bb = bb * sc + sh;
    }
    a = aa;
    b = bb;
}

// ------------------------------------------------------------------------------------------ GN statistics from quad partials
// One CTA per sample.  Step 1: thread t owns the (quad, sum|sumsq) column t of the concatenated partial row (C/2 columns) and adds
// it over the sample's slabs in fp64 (coalesced along t).  Step 2: thread j < 2*groups adds the cpg/4 quads of its group.
__global__ void __launch_bounds__(1024) gn_finalize_kernel(ds_gn_finalize_desc d) {
    extern __shared__ double s_cols[];                    // [cols] column sums, then [SG][cols] partials
    __shared__ float s_mu[64], s_rstd[64];
    const int n = blockIdx.x;
    const int C = d.C0 + d.C1;
    if (d.quads0) {
        // partial rows: {sum, sumsq} per unit of u0 / u1 channels (4 = quads, 2 = pairs) -> w floats per 32-row slab.
        // Thread (column, slab group): the 1024 threads split the sample's slabs SG ways (one thread per column walking all HW / 32
        // slabs alone is slow at 64 x 64); the SG partials of a column are added in a fixed order (deterministic).
        const int u0 = d.unit0 == 2 ? 2 : 4, u1 = d.unit1 == 2 ? 2 : 4;
        const int w0 = d.C0 / u0 * 2, w1 = d.C1 / u1 * 2;
        const int cols = w0 + w1;
        int SG = blockDim.x / cols;
        if (SG < 1) SG = 1;
        if (SG > d.slabs_per_sample) SG = d.slabs_per_sample;
        double* part = s_cols + cols;
        for (int idx = threadIdx.x; idx < cols * SG; idx += blockDim.x) {
            const int t = idx % cols, sg = idx / cols;
            const float* src = (t < w0) ? d.quads0 + (long long)n * d.slabs_per_sample * w0 + t
                                        : d.quads1 + (long long)n * d.slabs_per_sample * w1 + (t - w0);
            const int pitch = (t < w0) ? w0 : w1;
            double acc = 0.0;
#pragma unroll 4
            for (int sl = sg; sl < d.slabs_per_sample; sl += SG) acc += (double)__ldg(src + (long long)sl * pitch);
            part[(long long)sg * cols + t] = acc;
        }
        __syncthreads();
        for (int t = threadIdx.x; t < cols; t += blockDim.x) {
            double acc = 0.0;
            for (int sg = 0; sg < SG; ++sg) acc += part[(long long)sg * cols + t];
            s_cols[t] = acc;
        }
        __syncthreads();
        const int cpg = C / d.groups;
        for (int j = threadIdx.x; j < 2 * d.groups; j += blockDim.x) {
            const int g = j >> 1, k = j & 1;
            // channels [g * cpg, (g + 1) * cpg): whole units of source 0, then of source 1 (group boundaries fall on unit boundaries,
            // and C0 is a multiple of cpg or the group straddles the two sources at a unit boundary of each)
            double acc = 0.0;
            int c = g * cpg;
            const int c_end = c + cpg;
            while (c < c_end) {
                if (c < d.C0) { acc += s_cols[(c / u0) * 2 + k]; c += u0; }
                else { acc += s_cols[w0 + ((c - d.C0) / u1) * 2 + k]; c += u1; }
            }
            d.sums[((long long)n * d.groups + g) * 2 + k] = acc;
        }
        __syncthreads();
    }
    if (!d.coef) return;
    // second product: y = x * a + b per (sample, channel), so that gn_apply starts streaming without an fp64 prologue per thread
    const double cnt = (double)(C / d.groups) * d.HW;
    for (int g = threadIdx.x; g < d.groups; g += blockDim.x) {
        const float2 st = gn_group_stats(d, n, g, cnt);
        s_mu[g] = st.x;
        s_rstd[g] = st.y;
    }
    __syncthreads();
    const int cpg = C / d.groups;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        float aa, bb;
        gn_channel_coef(d, n, C, c, 0, s_rstd[g], aa, bb);
        reinterpret_cast<float2*>(d.coef)[(long long)n * C + c] = make_float2(aa, fmaf(-s_mu[g], aa, bb));
    }
}

// ------------------------------------------------------------------------------------------ GN apply
// grid (chunks, B); block = nc8 * rows threads.  Thread (c8, prow) owns 8 fixed channels: its normalisation coefficients
// live in registers (mean, a = rstd*gamma*(1+ada_scale), b = beta*(1+ada_scale)+ada_shift) and it streams over output pixels.
// RESAMPLE 1 (2x2 mean), 2 (nearest x2), 3 (space-to-depth) or 4 (space-to-depth at phase pitch pad0); resample 0 runs
// gn_apply_v2_kernel / gn_apply_v3_kernel below.
template <int RESAMPLE>
__global__ void __launch_bounds__(512) gn_apply_kernel(ds_gn_apply_desc d, int pix_per_cta, int nc8, int rows) {
    const int C = d.C0 + d.C1;
    const int n = blockIdx.y;
    const int c8 = threadIdx.x % nc8;
    const int prow = threadIdx.x / nc8;
    const int c = c8 * 8;
    const bool norm = d.sums != nullptr;
    float mean[8], a[8], b[8];
    if (norm) {
        const int cpg = C / d.groups;
        const double cnt = (double)cpg * d.H * d.W;
        int g_prev = -1;
        float mu_f = 0.f, rstd = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int g = (c + j) / cpg;
            if (g != g_prev) {                 // at most a few distinct groups per 8 channels
                const float2 st = gn_group_stats(d, n, g, cnt);
                mu_f = st.x;
                rstd = st.y;
                g_prev = g;
            }
            gn_channel_coef(d, n, C, c, j, rstd, a[j], b[j]);
            mean[j] = mu_f;
        }
    }
    const int Ho = RESAMPLE == 1 ? d.H / 2 : (RESAMPLE == 2 ? d.H * 2 : d.H);
    const int Wo = RESAMPLE == 1 ? d.W / 2 : (RESAMPLE == 2 ? d.W * 2 : d.W);
    const int npix = Ho * Wo;              // RESAMPLE >= 3 iterates over INPUT pixels and scatters them into the phase layout
    // RESAMPLE == 4: space-to-depth with each phase at a pitch of d.pad0 >= C channels (whole 64-channel GEMM K blocks)
    const int cp = RESAMPLE == 4 ? d.pad0 : C;
    const long long plane = (long long)d.B * npix * cp;
    const float* base;
    int pitch, cc;
    if (c < d.C0) { base = d.src0; pitch = d.C0; cc = c; }
    else { base = d.src1; pitch = d.C1; cc = c - d.C0; }
    base += (long long)n * d.H * d.W * pitch + cc;
    __half* oact = reinterpret_cast<__half*>(d.out_act);
    __half* oraw = reinterpret_cast<__half*>(d.out_raw);
    const int p_begin = blockIdx.x * pix_per_cta;
    int p_end = p_begin + pix_per_cta;
    if (p_end > npix) p_end = npix;
    for (int po = p_begin + prow; po < p_end; po += rows) {
        const int ho = po / Wo, wo = po - ho * Wo;
        float act[8], raw[8];
        if (RESAMPLE == 1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { act[j] = 0.f; raw[j] = 0.f; }
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float* src = base + (long long)((ho * 2 + (t >> 1)) * d.W + wo * 2 + (t & 1)) * pitch;
                const float4 v0 = __ldcs(reinterpret_cast<const float4*>(src));
                const float4 v1 = __ldcs(reinterpret_cast<const float4*>(src) + 1);
                const float e[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    raw[j] += 0.25f * e[j];
                    if (norm) {
                        float y = (e[j] - mean[j]) * a[j] + b[j];
                        if (d.silu) y = silu_f(y);
                        act[j] += 0.25f * y;
                    }
                }
            }
        } else {
            const int hi_ = RESAMPLE == 2 ? (ho >> 1) : ho;
            const int wi_ = RESAMPLE == 2 ? (wo >> 1) : wo;
            const float* src = base + (long long)(hi_ * d.W + wi_) * pitch;
            const float4 v0 = __ldcs(reinterpret_cast<const float4*>(src));
            const float4 v1 = __ldcs(reinterpret_cast<const float4*>(src) + 1);
            const float e[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                raw[j] = e[j];
                float y = 0.f;
                if (norm) {
                    y = (e[j] - mean[j]) * a[j] + b[j];
                    if (d.silu) y = silu_f(y);
                }
                act[j] = y;
            }
        }
        long long o = ((long long)n * npix + po) * C + c;
        if (RESAMPLE >= 3) {
            // space-to-depth: input pixel (ho, wo) -> output pixel (ho/2, wo/2), channel block ((ho&1)*2 + (wo&1))*cp
            const int h2 = ho >> 1, w2 = wo >> 1, ph = ((ho & 1) << 1) | (wo & 1);
            o = (((long long)n * (d.H / 2) + h2) * (d.W / 2) + w2) * (4LL * cp) + (long long)ph * cp + c;
        }
        if (oact) store_operand<8>(oact, plane, o, act, d.nplanes, d.fmt);
        if (oraw) store_operand<8>(oraw, plane, o, raw, d.nplanes, d.fmt);
        if (RESAMPLE == 4 && c + 8 == C) {
            // the phase's channels C .. cp: the GEMM's last K box of the phase reads them, so they must be zero
            const float zero[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int cz = 8; c + cz < cp; cz += 8) {
                if (oact) store_operand<8>(oact, plane, o + cz, zero, d.nplanes, d.fmt);
                if (oraw) store_operand<8>(oraw, plane, o + cz, zero, d.nplanes, d.fmt);
            }
        }
        if (d.out_raw_f32) {
            *reinterpret_cast<float4*>(d.out_raw_f32 + o) = make_float4(raw[0], raw[1], raw[2], raw[3]);
            *reinterpret_cast<float4*>(d.out_raw_f32 + o + 4) = make_float4(raw[4], raw[5], raw[6], raw[7]);
        }
    }
}

// Resample 0: the normalisation is folded to one FMA per element, y = x * a + b' with b' = b - mean * a (16 instead of 24 live
// coefficient registers), and four pixels are processed per iteration so that eight 16-byte loads are in flight per thread (two pixels
// keep ~49 KB per SM in flight, about the minimum HBM needs).
template <int NP>
__device__ __forceinline__ void gn_v2_pixels(const ds_gn_apply_desc& d, const float* base, int pitch, long long n, int npix, int C, int c,
                                             long long plane, int po, int rows, bool norm, const float* a, const float* b, __half* oact,
                                             __half* oraw) {
    float4 v[NP][2];
#pragma unroll
    for (int k = 0; k < NP; ++k) {
        const float4* s = reinterpret_cast<const float4*>(base + (long long)(po + k * rows) * pitch);
        v[k][0] = __ldcs(s);
        v[k][1] = __ldcs(s + 1);
    }
#pragma unroll
    for (int k = 0; k < NP; ++k) {
        const float e[8] = {v[k][0].x, v[k][0].y, v[k][0].z, v[k][0].w, v[k][1].x, v[k][1].y, v[k][1].z, v[k][1].w};
        const long long o = ((long long)n * npix + po + k * rows) * C + c;
        if (oact) {
            float y[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float u = 0.f;
                if (norm) {
                    u = fmaf(e[j], a[j], b[j]);
                    if (d.silu) u = silu_f(u);
                }
                y[j] = u;
            }
            store_operand<8>(oact, plane, o, y, d.nplanes, d.fmt);
        }
        if (oraw) store_operand<8>(oraw, plane, o, e, d.nplanes, d.fmt);
        if (d.out_raw_f32) {
            *reinterpret_cast<float4*>(d.out_raw_f32 + o) = v[k][0];
            *reinterpret_cast<float4*>(d.out_raw_f32 + o + 4) = v[k][1];
        }
    }
}

__global__ void __launch_bounds__(512) gn_apply_v2_kernel(ds_gn_apply_desc d, int pix_per_cta, int nc8, int rows) {
    const int C = d.C0 + d.C1;
    const int n = blockIdx.y;
    const int c8 = threadIdx.x % nc8;
    const int prow = threadIdx.x / nc8;
    const int c = c8 * 8;
    const bool norm = d.sums != nullptr;
    float a[8], b[8];
    if (norm) {
        const int cpg = C / d.groups;
        const double cnt = (double)cpg * d.H * d.W;
        int g_prev = -1;
        float mu_f = 0.f, rstd = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int g = (c + j) / cpg;
            if (g != g_prev) {
                const float2 st = gn_group_stats(d, n, g, cnt);
                mu_f = st.x;
                rstd = st.y;
                g_prev = g;
            }
            float bb;
            gn_channel_coef(d, n, C, c, j, rstd, a[j], bb);
            b[j] = fmaf(-mu_f, a[j], bb);
        }
    }
    const int npix = d.H * d.W;
    const long long plane = (long long)d.B * npix * C;
    const float* base;
    int pitch, cc;
    if (c < d.C0) { base = d.src0; pitch = d.C0; cc = c; }
    else { base = d.src1; pitch = d.C1; cc = c - d.C0; }
    base += (long long)n * npix * pitch + cc;
    __half* oact = reinterpret_cast<__half*>(d.out_act);
    __half* oraw = reinterpret_cast<__half*>(d.out_raw);
    const int p_begin = blockIdx.x * pix_per_cta;
    int p_end = p_begin + pix_per_cta;
    if (p_end > npix) p_end = npix;
    int po = p_begin + prow;
    for (; po + 3 * rows < p_end; po += 4 * rows) gn_v2_pixels<4>(d, base, pitch, n, npix, C, c, plane, po, rows, norm, a, b, oact, oraw);
    for (; po < p_end; po += rows) gn_v2_pixels<1>(d, base, pitch, n, npix, C, c, plane, po, rows, norm, a, b, oact, oraw);
}

// resample == 0 with precomputed coefficients (ds_gn_apply_desc.coef): the v2 inner loop inside a PERSISTENT, EVENLY SPLIT grid.
// v2 launches one CTA per (sample, 16-pixels-per-thread chunk): a partial last wave, and each thread pays an fp64 mean / rsqrt
// prologue for 16 pixels of work.  Here the (sample, pixel
// row) space is cut into gridDim.x equal ranges (+-1 row), the grid is exactly the number of co-resident CTAs, and a thread fetches its
// 16 coefficients (4 x 16 B, L2-resident table written by gn_finalize) only when its range crosses into another sample.
__global__ void __launch_bounds__(256, 3) gn_apply_v3_kernel(ds_gn_apply_desc d, int nc8, int rows, int units_per_sample, long long total_units) {
    const int C = d.C0 + d.C1;
    const int c8 = threadIdx.x % nc8;
    const int prow = threadIdx.x / nc8;
    const int c = c8 * 8;
    const int npix = d.H * d.W;
    const long long plane = (long long)d.B * npix * C;
    const float* base0;
    int pitch, cc;
    if (c < d.C0) { base0 = d.src0; pitch = d.C0; cc = c; }
    else { base0 = d.src1; pitch = d.C1; cc = c - d.C0; }
    __half* oact = reinterpret_cast<__half*>(d.out_act);
    __half* oraw = reinterpret_cast<__half*>(d.out_raw);
    // With one contiguous range per CTA every CTA would stream through its own distant pages (2 sources + up to 5 output planes each),
    // which slows the large concat layers.  Instead the grid sweeps the tensor together: chunks of kChunk units (>= 8 pixel rows, never crossing a sample) are dealt
    // round-robin, so at any time all CTAs work inside one ~30 MB window per stream; the coefficients are refetched only when the sample
    // changes.
    constexpr int kChunk = 8;
    const int chunks_per_sample = (units_per_sample + kChunk - 1) / kChunk;
    const long long total_chunks = (long long)chunks_per_sample * d.B;
    float a[8], b[8];
    int n_prev = -1;
    for (long long ch = blockIdx.x; ch < total_chunks; ch += gridDim.x) {
        const int n = (int)(ch / chunks_per_sample);
        const int uin = ((int)(ch - (long long)n * chunks_per_sample)) * kChunk;
        const int nun = min(kChunk, units_per_sample - uin);
        if (n != n_prev) {
            const float4* cf = reinterpret_cast<const float4*>(d.coef + ((long long)n * C + c) * 2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 t = __ldg(cf + j);
                a[2 * j] = t.x; b[2 * j] = t.y; a[2 * j + 1] = t.z; b[2 * j + 1] = t.w;
            }
            n_prev = n;
        }
        const float* base = base0 + (long long)n * npix * pitch + cc;
        int po = uin * rows + prow;                      // pixel of this thread in the first unit of the chunk
        int k = 0;
        // whole units only: the last unit of a sample may be partial when rows does not divide H*W
        const int full = ((uin + nun) * rows <= npix) ? nun : nun - 1;
        for (; k + 4 <= full; k += 4, po += 4 * rows) gn_v2_pixels<4>(d, base, pitch, n, npix, C, c, plane, po, rows, true, a, b, oact, oraw);
        for (; k < full; ++k, po += rows) gn_v2_pixels<1>(d, base, pitch, n, npix, C, c, plane, po, rows, true, a, b, oact, oraw);
        if (k < nun && po < npix) gn_v2_pixels<1>(d, base, pitch, n, npix, C, c, plane, po, rows, true, a, b, oact, oraw);
    }
}

// ------------------------------------------------------------------------------------------ softmax
// Single-read softmax: the row is held in registers (NV float4 per thread), one HBM read + one write per score.
//   ROWS_PER_CTA = 8 warps, one warp per row  (L <= 32*4*NV)         -- short rows
//   ROWS_PER_CTA = 1, 256 threads per row      (L <= 256*4*NV)        -- long rows (4096 keys of the 64x64 SD self-attention)
template <int NV, bool CTA_ROW>
__global__ void __launch_bounds__(256) softmax_reg_kernel(ds_softmax_desc d) {
    __shared__ float red[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row = CTA_ROW ? (long long)blockIdx.x : (long long)blockIdx.x * 8 + warp;
    if (row >= d.rows) return;                      // whole warp (or CTA) exits together
    const int tid = CTA_ROW ? threadIdx.x : lane;
    const int nthr = CTA_ROW ? 256 : 32;
    const float* s = d.S + row * d.L;
    float4 v[NV];
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int j = (tid + k * nthr) * 4;
        if (j < d.L) {
            v[k] = __ldcs(reinterpret_cast<const float4*>(s + j));
            m = fmaxf(m, fmaxf(fmaxf(v[k].x, v[k].y), fmaxf(v[k].z, v[k].w)));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (CTA_ROW) {
        if (lane == 0) red[warp] = m;
        __syncthreads();
        m = red[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        __syncthreads();
    }
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int j = (tid + k * nthr) * 4;
        if (j < d.L) {
            v[k].x = expf(v[k].x - m); v[k].y = expf(v[k].y - m); v[k].z = expf(v[k].z - m); v[k].w = expf(v[k].w - m);
            sum += v[k].x + v[k].y + v[k].z + v[k].w;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (CTA_ROW) {
        if (lane == 0) red[warp] = sum;
        __syncthreads();
        sum = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) sum += red[w];
    }
    const float inv = 1.0f / sum;
    __half* P = reinterpret_cast<__half*>(d.P);
    const long long plane = d.rows * d.L;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int j = (tid + k * nthr) * 4;
        if (j < d.L) {
            const float e[4] = {v[k].x * inv, v[k].y * inv, v[k].z * inv, v[k].w * inv};
            store_planes<4>(P, plane, row * d.L + j, e, d.nplanes);
        }
    }
}

// one warp per row
__global__ void softmax_kernel(ds_softmax_desc d) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= d.rows) return;
    const int lane = threadIdx.x & 31;
    const int pin = d.pitch_in ? d.pitch_in : d.L;
    const int pout = d.pitch_out ? d.pitch_out : d.L;
    const float* s = d.S + row * pin;
    __half* P = reinterpret_cast<__half*>(d.P);
    const long long plane = d.rows * pout;
    if ((d.L & 3) == 0 && (pin & 3) == 0 && (pout & 3) == 0) {
        float m = -INFINITY;
        for (int j = lane * 4; j < d.L; j += 128) {
            const float4 v = *reinterpret_cast<const float4*>(s + j);
            m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float sum = 0.f;
        for (int j = lane * 4; j < d.L; j += 128) {
            const float4 v = *reinterpret_cast<const float4*>(s + j);
            sum += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float inv = 1.0f / sum;
        for (int j = lane * 4; j < d.L; j += 128) {
            const float4 v = *reinterpret_cast<const float4*>(s + j);
            const float e[4] = {expf(v.x - m) * inv, expf(v.y - m) * inv, expf(v.z - m) * inv, expf(v.w - m) * inv};
            store_planes<4>(P, plane, row * pout + j, e, d.nplanes);
        }
        return;
    }
    // generic row length (e.g. 77 context tokens): scalar accesses
    float m = -INFINITY;
    for (int j = lane; j < d.L; j += 32) m = fmaxf(m, s[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int j = lane; j < d.L; j += 32) sum += expf(s[j] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    for (int j = lane; j < d.L; j += 32) {
        __half hi, lo;
        split_h16(expf(s[j] - m) * inv, hi, lo);
        P[row * pout + j] = hi;
        if (d.nplanes > 1) P[plane + row * pout + j] = lo;
    }
}

// ------------------------------------------------------------------------------------------ embedding
__global__ void posemb_kernel(ds_posemb_desc d) {
    const int n = blockIdx.x;
    if (d.mode == 1) {
        // LDM timestep_embedding (util.py:151-171): freqs = exp(-ln(10000) * i / half), [cos | sin]
        const float t = d.sigma[n];
        const int half = d.num_channels / 2;
        for (int i = threadIdx.x; i < half; i += blockDim.x) {
            const float freq = expf(-logf(10000.0f) * (float)i / (float)half);
            const float a = t * freq;
            d.emb[n * d.num_channels + i] = cosf(a);
            d.emb[n * d.num_channels + half + i] = sinf(a);
        }
        return;
    }
    const float sigma = d.sigma[n];
    const float sd = d.sigma_data;
    const float s2 = sigma * sigma + sd * sd;
    const float c_noise = logf(sigma) / 4.0f;
    if (threadIdx.x == 0) {
        d.coef[n * 4 + 0] = sd * sd / s2;
        d.coef[n * 4 + 1] = sigma * sd / sqrtf(s2);
        d.coef[n * 4 + 2] = 1.0f / sqrtf(s2);
        d.coef[n * 4 + 3] = c_noise;
    }
    // CMPrecond feeds 1000 * c_noise to its U-Net's timestep_embedding (networks_edm.py:539-540)
    const float t_emb = d.noise_scale != 0.0f ? d.noise_scale * c_noise : c_noise;
    const int half = d.num_channels / 2;
    for (int i = threadIdx.x; i < half; i += blockDim.x) {
        // freqs = (1/10000) ** (i / (half - endpoint))   (networks_edm.py:193-195)
        const float fr = (float)i / (float)(half - (d.endpoint ? 1 : 0));
        const float freq = powf(1.0f / 10000.0f, fr);
        const float a = t_emb * freq;
        const float cs = cosf(a), sn = sinf(a);
        // reference layout is [cos | sin]; SongUNet then swaps the halves to [sin | cos]
        if (d.swap_sincos) { d.emb[n * d.num_channels + i] = sn; d.emb[n * d.num_channels + half + i] = cs; }
        else { d.emb[n * d.num_channels + i] = cs; d.emb[n * d.num_channels + half + i] = sn; }
    }
}

// one warp per output feature; loops over rows re-using the weight row held in registers
template <int MAXF>
__global__ void linear_kernel(ds_linear_desc d) {
    const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (o >= d.out_f) return;
    const int lane = threadIdx.x & 31;
    float w[MAXF / 32];
#pragma unroll
    for (int k = 0; k < MAXF / 32; ++k) {
        const int i = lane + 32 * k;
        w[k] = (i < d.in_f) ? d.W[(long long)o * d.in_f + i] : 0.f;
    }
    const float bias = d.b ? d.b[o] : 0.f;
    for (int n = blockIdx.y; n < d.n_rows; n += gridDim.y) {
        const float* x = d.in + (long long)n * d.in_stride;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < MAXF / 32; ++k) {
            const int i = lane + 32 * k;
            if (i < d.in_f) acc += w[k] * (d.in_scale * x[i]);
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) {
            float v = acc + bias;
            if (d.add) v += d.add[(long long)n * d.add_stride + o];
            if (d.act == 1) v = silu_f(v);
            d.out[(long long)n * d.out_f + o] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------ input prep
__global__ void prep_input_kernel(ds_prep_input_desc d) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per (n, pixel, 8-ch group)
    const long long total = (long long)d.B * d.HW * 8;
    if (idx >= total) return;
    const int c8 = (int)(idx & 7);
    const long long px = idx >> 3;
    const int n = (int)(px / d.HW);
    const int hw = (int)(px - (long long)n * d.HW);
    const int xb = d.x_batch > 0 ? d.x_batch : d.B;
    const int nx = n % xb;
    const float cin = d.coef[nx * d.coef_stride + 2];
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = c8 * 8 + j;
        v[j] = c < d.C ? cin * d.x[((long long)nx * d.C + c) * d.HW + hw] : 0.f;
    }
    store_planes<8>(reinterpret_cast<__half*>(d.out), (long long)d.B * d.HW * 64, px * 64 + c8 * 8, v, d.nplanes);
}

// Vector-quantized input: one thread per pixel holds v = c_in * x (channels zero-padded to CP) and streams the codebook through shared
// memory in chunks of VQ_CHUNK rows; the padded channels are zero on both sides, so they add exactly 0 to every distance.  A strict
// '<' over ascending rows keeps the lowest index among equal distances (torch.argmin).  The chosen row is then written, split hi/lo,
// into the 64-column planes prep_input_kernel writes.
constexpr int VQ_CHUNK = 1024;

template <int CP>
__global__ void __launch_bounds__(256) vq_prep_input_kernel(ds_prep_input_desc d) {
    __shared__ float4 s_code[VQ_CHUNK * (CP / 4)];
    const long long px = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)d.B * d.HW;
    const bool live = px < total;
    const int n = live ? (int)(px / d.HW) : 0;
    const int hw = live ? (int)(px - (long long)n * d.HW) : 0;
    const int xb = d.x_batch > 0 ? d.x_batch : d.B;
    const int nx = n % xb;
    float v[CP];
    if (live) {
        const float cin = d.coef[nx * d.coef_stride + 2];
#pragma unroll
        for (int c = 0; c < CP; ++c) v[c] = c < d.C ? cin * d.x[((long long)nx * d.C + c) * d.HW + hw] : 0.f;
    }
    float best = INFINITY;
    int bi = 0;
    float* sc = reinterpret_cast<float*>(s_code);
    for (int base = 0; base < d.n_embed; base += VQ_CHUNK) {
        const int cnt = min(VQ_CHUNK, d.n_embed - base);
        __syncthreads();
        for (int i = threadIdx.x; i < cnt * CP; i += blockDim.x) {
            const int j = i / CP, c = i - j * CP;
            sc[i] = c < d.C ? d.codebook[(long long)(base + j) * d.C + c] : 0.f;
        }
        __syncthreads();
        if (!live) continue;
        for (int j = 0; j < cnt; ++j) {
            float dist = 0.f;
#pragma unroll
            for (int q = 0; q < CP / 4; ++q) {
                const float4 e = s_code[j * (CP / 4) + q];
                const float d0 = v[4 * q] - e.x, d1 = v[4 * q + 1] - e.y, d2 = v[4 * q + 2] - e.z, d3 = v[4 * q + 3] - e.w;
                dist = fmaf(d0, d0, dist);
                dist = fmaf(d1, d1, dist);
                dist = fmaf(d2, d2, dist);
                dist = fmaf(d3, d3, dist);
            }
            if (dist < best) { best = dist; bi = base + j; }
        }
    }
    if (!live) return;
    if (d.idx) d.idx[px] = bi;
    __half* o = reinterpret_cast<__half*>(d.out);
    const long long plane = total * 64;
#pragma unroll
    for (int c8 = 0; c8 < 8; ++c8) {
        float e[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = c8 * 8 + j;
            e[j] = c < d.C ? d.codebook[(long long)bi * d.C + c] : 0.f;
        }
        store_planes<8>(o, plane, px * 64 + c8 * 8, e, d.nplanes);
    }
}

// one warp per token row; the row lives in registers (C <= 2048), two-pass mean / variance like torch's layer_norm.
// FMT (ds_layernorm_desc.fmt): 0 fp16 planes, 1 f8 image (operand.cuh), 2 fp32 [rows][C] (the last LayerNorm of the CLIP text encoder).
template <int FMT>
__global__ void layernorm_kernel(ds_layernorm_desc d) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= d.rows) return;
    const int lane = threadIdx.x & 31;
    const float* x = d.src + row * d.C;
    constexpr int MAXV = 16;                                   // float4 per lane: C <= 32*4*16 = 2048
    float4 v[MAXV];
    const int nv = d.C / 4;
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int j = lane + 32 * k;
        if (j < nv) {
            v[k] = *reinterpret_cast<const float4*>(x + 4 * j);
            sum += v[k].x + v[k].y + v[k].z + v[k].w;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)d.C;
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int j = lane + 32 * k;
        if (j < nv) {
            const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, e = v[k].w - mean;
            sq += a * a + b * b + c * c + e * e;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / (float)d.C + d.eps);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int j = lane + 32 * k;
        if (j < nv) {
            const float4 g = *reinterpret_cast<const float4*>(d.gamma + 4 * j);
            const float4 b = *reinterpret_cast<const float4*>(d.beta + 4 * j);
            const float y[4] = {(v[k].x - mean) * rstd * g.x + b.x, (v[k].y - mean) * rstd * g.y + b.y,
                                (v[k].z - mean) * rstd * g.z + b.z, (v[k].w - mean) * rstd * g.w + b.w};
            if (FMT == 2) *reinterpret_cast<float4*>(reinterpret_cast<float*>(d.out) + row * d.C + 4 * j) = make_float4(y[0], y[1], y[2], y[3]);
            else store_operand<4>(reinterpret_cast<__half*>(d.out), d.rows * d.C, row * d.C + 4 * j, y, d.nplanes, FMT);
        }
    }
}

// token + position embedding (ds_embed_desc): one thread per 4 channels of one row
__global__ void embed_kernel(ds_embed_desc d) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int c4 = d.C / 4;
    if (idx >= d.rows * c4) return;
    const long long row = idx / c4;
    const int j = (int)(idx - row * c4) * 4;
    int id = d.ids[row];
    id = id < 0 ? 0 : (id >= d.vocab ? d.vocab - 1 : id);
    const float4 t = *reinterpret_cast<const float4*>(d.tok + (long long)id * d.C + j);
    const float4 p = *reinterpret_cast<const float4*>(d.pos + (long long)(row % d.T) * d.C + j);
    *reinterpret_cast<float4*>(d.out + row * d.C + j) = make_float4(t.x + p.x, t.y + p.y, t.z + p.z, t.w + p.w);
}

// Gated activations (ds_geglu_desc), one thread per 4 outputs of [rows][I], written in format FMT (operand.cuh):
//   MODE 0, GEGLU: out = x[:, :I] * gelu(x[:, I:]) on fp32 [rows][2I], exact erf GELU.
//   MODE 1, quick-GELU: out = x * sigmoid(1.702 x) on fp32 [rows][I] (CLIP MLP activation).
//   MODE 2, exact GELU: out = gelu(x) on fp32 [rows][I] (open_clip ViT-g-14 MLP activation), the erf form of MODE 0.
template <int MODE, int FMT>
__global__ void gate_kernel(ds_geglu_desc d) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int i4 = d.I / 4;
    if (idx >= d.rows * i4) return;
    float y[4];
    if (MODE == 0) {
        const long long row = idx / i4;
        const int j = (int)(idx - row * i4) * 4;
        const float4 a = *reinterpret_cast<const float4*>(d.src + row * 2 * d.I + j);
        const float4 g = *reinterpret_cast<const float4*>(d.src + row * 2 * d.I + d.I + j);
        const float av[4] = {a.x, a.y, a.z, a.w}, gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) y[q] = av[q] * (0.5f * gv[q] * (1.0f + erff(gv[q] * 0.70710678118654752f)));
    } else if (MODE == 1) {
        const float4 a = *reinterpret_cast<const float4*>(d.src + idx * 4);
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) y[q] = av[q] / (1.0f + expf(-1.702f * av[q]));
    } else {
        const float4 a = *reinterpret_cast<const float4*>(d.src + idx * 4);
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) y[q] = 0.5f * av[q] * (1.0f + erff(av[q] * 0.70710678118654752f));
    }
    store_operand<4>(reinterpret_cast<__half*>(d.out), d.rows * d.I, idx * 4, y, d.nplanes, FMT);
}

__global__ void chanmean_kernel(ds_chanmean_desc d) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= d.rows) return;
    const int lane = threadIdx.x & 31;
    float s = 0.f;
    for (int c = lane; c < d.C; c += 32) s += d.src[row * d.C + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) d.out[row] = s / (float)d.C;
}

static inline int ok() { return cudaGetLastError() == cudaSuccess ? 0 : -1; }

}  // namespace dsb

using namespace dsb;

OpCheck dsb::gn_stats_check(const ds_gn_stats_desc& d) {
    const int C = d.C0 + d.C1;
    if (C % 4 || d.groups <= 0 || d.groups > 64 || C % d.groups || (d.C0 % 4)) return {-2, "gn_stats: channels"};
    // gn_stats_kernel splits a float4 column between at most two groups (gA / gB): groups of one channel would be summed into the wrong group
    if (C / d.groups < 2) return {-2, "gn_stats: one-channel groups"};
    return {0, nullptr};
}

extern "C" int ds_gn_stats_launch(const ds_gn_stats_desc* d, cudaStream_t stream) {
    if (const int rc = gn_stats_check(*d).rc) return rc;
    const int C = d->C0 + d->C1;
    const int ncol4 = C / 4;
    int bx = ncol4 < 256 ? ncol4 : 256;
    // keep bx a divisor-friendly size; columns loop with stride bx anyway
    int by = 256 / bx; if (by < 1) by = 1;
    int pix_per_cta = 8 * by;                  // 8 loads in flight per thread
    if (pix_per_cta < 64) pix_per_cta = 64;
    // small batches (latent diffusion: 16 samples): shorter pixel runs per CTA so that the grid still covers the SMs
    const int min_pix = by > 8 ? by : 8;
    while (pix_per_cta > min_pix && (long long)((d->HW + pix_per_cta - 1) / pix_per_cta) * d->B < 132 * 4) pix_per_cta /= 2;
    const int chunks = (d->HW + pix_per_cta - 1) / pix_per_cta;
    gn_stats_kernel<<<dim3(chunks, d->B), dim3(bx, by), 0, stream>>>(*d, pix_per_cta);
    return ok();
}

// Block size and dynamic shared memory of gn_finalize_kernel.  threads: enough for (columns x slab groups), at most 1024; shared memory:
// [cols] + [SG][cols] doubles, cols <= C, SG * cols <= max(cols, threads)
static size_t gn_finalize_shape(const ds_gn_finalize_desc& d, int* threads) {
    *threads = 256;
    if (!d.quads0) return (size_t)(d.C0 + d.C1 + 2) * sizeof(double);
    const int u0 = d.unit0 == 2 ? 2 : 4, u1 = d.unit1 == 2 ? 2 : 4;
    const int cols = d.C0 / u0 * 2 + d.C1 / u1 * 2;
    *threads = 1024;
    const int sg = cols >= *threads ? 1 : *threads / cols;
    return (size_t)(cols + (size_t)sg * cols + 2) * sizeof(double);
}

OpCheck dsb::gn_finalize_check(const ds_gn_finalize_desc& d) {
    const int C = d.C0 + d.C1;
    if (d.groups <= 0 || d.groups > 64 || C % d.groups) return {-2, "gn_finalize: groups"};
    if (d.quads0) {
        const int u0 = d.unit0 == 2 ? 2 : 4, u1 = d.unit1 == 2 ? 2 : 4;
        const int cpg = C / d.groups;
        if (d.C0 % u0 || d.C1 % u1 || (d.C1 > 0 && !d.quads1)) return {-2, "gn_finalize: source units"};
        // every group must be a union of whole partial units of the sources it covers
        const int rem = d.C0 % cpg;                     // channels of a group that straddles the two sources, on the source-0 side
        if (cpg % u0 || rem % u0) return {-2, "gn_finalize: group units"};
        if (d.C1 > 0 && (cpg % u1 || (rem ? (cpg - rem) % u1 : 0))) return {-2, "gn_finalize: group units"};
    }
    if (!d.quads0 && !d.coef) return {-2, "gn_finalize: nothing to do"};
    if (d.coef && (!d.gamma || !d.beta || d.HW <= 0)) return {-2, "gn_finalize: coef inputs"};
    // the launch keeps the default 48 KiB limit of dynamic shared memory
    int threads;
    if (gn_finalize_shape(d, &threads) > 48 * 1024) return {-2, "gn_finalize: shared memory"};
    return {0, nullptr};
}

extern "C" int ds_gn_finalize_launch(const ds_gn_finalize_desc* d, cudaStream_t stream) {
    if (const int rc = gn_finalize_check(*d).rc) return rc;
    int threads;
    const size_t smem = gn_finalize_shape(*d, &threads);
    gn_finalize_kernel<<<d->B, threads, smem, stream>>>(*d);
    return ok();
}

OpCheck dsb::gn_apply_check(const ds_gn_apply_desc& d) {
    const int C = d.C0 + d.C1;
    if (C % 8 || (d.C0 % 8)) return {-2, "gn_apply: channels"};
    // the f8 layout reuses the two-plane footprint
    if (d.fmt != 0 && (d.fmt != 1 || d.resample == 3 || d.nplanes != 2)) return {-2, "gn_apply: fmt"};
    // the coefficient table is read by the resample-0 kernel only; the resampling kernels normalise from the sums
    if (d.coef && d.resample != 0) return {-2, "gn_apply: coef with resample"};
    if (d.out_act && !d.sums && !d.coef) return {-2, "gn_apply: statistics"};          // a normalised output needs statistics
    // 2x2 pooling and space-to-depth take whole 2x2 blocks: an odd row or column has no output pixel
    if ((d.resample == 1 || d.resample == 3) && (d.H % 2 || d.W % 2)) return {-2, "gn_apply: resample parity"};
    // pad0: phase pitch of the space-to-depth output (0 = C), a multiple of 8 channels; the f32 raw output has no pitch
    if (d.pad0 && (d.resample != 3 || d.pad0 < C || d.pad0 % 8 || d.out_raw_f32)) return {-2, "gn_apply: phase pitch"};
    const int nc8 = C / 8;
    if (nc8 > 512) return {-2, "gn_apply: width"};                                   // at most 4096 channels
    // the persistent kernel takes at most 256 threads (2048 channels); wider tensors use the sums path
    if (d.coef && d.resample == 0 && d.sums == nullptr && nc8 > 256) return {-2, "gn_apply: coef width"};
    return {0, nullptr};
}

extern "C" int ds_gn_apply_launch(const ds_gn_apply_desc* d, cudaStream_t stream) {
    if (const int rc = gn_apply_check(*d).rc) return rc;
    const int C = d->C0 + d->C1;
    const int nc8 = C / 8;
    int rows = 256 / nc8;
    if (rows < 1) rows = 1;
    const int threads = nc8 * rows;
    const int Ho = d->resample == 1 ? d->H / 2 : (d->resample == 2 ? d->H * 2 : d->H);
    const int Wo = d->resample == 1 ? d->W / 2 : (d->resample == 2 ? d->W * 2 : d->W);
    const int npix = Ho * Wo;
    // ~16 pixels per thread amortise the per-thread coefficient set-up; keep at least ~4 CTAs per SM in flight overall
    int pix_per_cta = rows * 16;
    while (pix_per_cta > rows && (long long)((npix + pix_per_cta - 1) / pix_per_cta) * d->B < 132 * 4) pix_per_cta /= 2;
    const int chunks = (npix + pix_per_cta - 1) / pix_per_cta;
    dim3 grid(chunks, d->B);
    if (d->coef && d->resample == 0 && d->sums == nullptr) {
        // persistent variant: grid = co-resident CTAs (occupancy query per block size and device, cached)
        static int occ[64][17] = {};
        static int sms[64] = {};
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64) dev = 0;
        const int slot = threads / 32;
        if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
        if (!occ[dev][slot]) {
            int nb = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, gn_apply_v3_kernel, threads, 0) != cudaSuccess || nb < 1) nb = 1;
            occ[dev][slot] = nb;
        }
        const int ups = (npix + rows - 1) / rows;
        const long long total_units = (long long)ups * d->B;
        long long g3 = (long long)sms[dev] * occ[dev][slot];
        const long long total_chunks = (long long)((ups + 7) / 8) * d->B;        // kChunk = 8 units per chunk (gn_apply_v3_kernel)
        if (g3 > total_chunks) g3 = total_chunks;
        if (g3 < 1) g3 = 1;
        gn_apply_v3_kernel<<<(unsigned)g3, threads, 0, stream>>>(*d, nc8, rows, ups, total_units);
        return ok();
    }
    if (d->resample == 1) gn_apply_kernel<1><<<grid, threads, 0, stream>>>(*d, pix_per_cta, nc8, rows);
    else if (d->resample == 3 && d->pad0 && d->pad0 != C) gn_apply_kernel<4><<<grid, threads, 0, stream>>>(*d, pix_per_cta, nc8, rows);
    else if (d->resample == 3) gn_apply_kernel<3><<<grid, threads, 0, stream>>>(*d, pix_per_cta, nc8, rows);
    else if (d->resample == 2) gn_apply_kernel<2><<<grid, threads, 0, stream>>>(*d, pix_per_cta, nc8, rows);
    else gn_apply_v2_kernel<<<grid, threads, 0, stream>>>(*d, pix_per_cta, nc8, rows);
    return ok();
}

OpCheck dsb::embed_check(const ds_embed_desc& d) {
    if (d.C % 4 || d.rows <= 0 || d.T <= 0 || d.vocab <= 0) return {-2, "embed: shape"};
    return {0, nullptr};
}

extern "C" int ds_embed_launch(const ds_embed_desc* d, cudaStream_t stream) {
    if (const int rc = embed_check(*d).rc) return rc;
    const long long total = d->rows * (d->C / 4);
    embed_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(*d);
    return ok();
}

OpCheck dsb::layernorm_check(const ds_layernorm_desc& d) {
    if (d.C % 4 || d.C > 2048) return {-2, "layernorm: C"};
    if (d.fmt == 1 && d.nplanes != 2) return {-2, "layernorm: f8 planes"};
    return {0, nullptr};
}

extern "C" int ds_layernorm_launch(const ds_layernorm_desc* d, cudaStream_t stream) {
    if (const int rc = layernorm_check(*d).rc) return rc;
    const int wpb = 8;
    const unsigned blocks = (unsigned)((d->rows + wpb - 1) / wpb);
    if (d->fmt == 1) {
        layernorm_kernel<1><<<blocks, wpb * 32, 0, stream>>>(*d);
    } else if (d->fmt == 2) {
        layernorm_kernel<2><<<blocks, wpb * 32, 0, stream>>>(*d);
    } else {
        layernorm_kernel<0><<<blocks, wpb * 32, 0, stream>>>(*d);
    }
    return ok();
}

OpCheck dsb::geglu_check(const ds_geglu_desc& d) {
    if (d.I % 4) return {-2, "geglu: I"};
    if (d.mode < 0 || d.mode > 2) return {-2, "geglu: mode"};
    if (d.mode == 1 && d.fmt != 0) return {-2, "geglu: quick-GELU fmt"};
    if (d.mode == 2 && d.fmt != 0) return {-2, "geglu: GELU fmt"};
    if (d.mode != 1 && d.fmt == 1 && d.nplanes != 2) return {-2, "geglu: f8 planes"};
    return {0, nullptr};
}

extern "C" int ds_geglu_launch(const ds_geglu_desc* d, cudaStream_t stream) {
    if (const int rc = geglu_check(*d).rc) return rc;
    const unsigned blocks = (unsigned)((d->rows * (d->I / 4) + 255) / 256);
    if (d->mode == 1) {
        gate_kernel<1, 0><<<blocks, 256, 0, stream>>>(*d);
    } else if (d->mode == 2) {
        gate_kernel<2, 0><<<blocks, 256, 0, stream>>>(*d);
    } else if (d->fmt == 1) {
        gate_kernel<0, 1><<<blocks, 256, 0, stream>>>(*d);
    } else {
        gate_kernel<0, 0><<<blocks, 256, 0, stream>>>(*d);
    }
    return ok();
}

extern "C" int ds_softmax_launch(const ds_softmax_desc* d, cudaStream_t stream) {
    const bool dense = (d->pitch_in == 0 || d->pitch_in == d->L) && (d->pitch_out == 0 || d->pitch_out == d->L) && (d->L % 4 == 0);
    if (dense && d->L <= 1024) {
        const unsigned blocks = (unsigned)((d->rows + 7) / 8);
        if (d->L <= 256) softmax_reg_kernel<2, false><<<blocks, 256, 0, stream>>>(*d);
        else softmax_reg_kernel<8, false><<<blocks, 256, 0, stream>>>(*d);
        return ok();
    }
    if (dense && d->L <= 8192) {
        if (d->L <= 4096) softmax_reg_kernel<4, true><<<(unsigned)d->rows, 256, 0, stream>>>(*d);
        else softmax_reg_kernel<8, true><<<(unsigned)d->rows, 256, 0, stream>>>(*d);
        return ok();
    }
    const int wpb = 8;
    const long long blocks = (d->rows + wpb - 1) / wpb;
    softmax_kernel<<<(unsigned)blocks, wpb * 32, 0, stream>>>(*d);
    return ok();
}

extern "C" int ds_posemb_launch(const ds_posemb_desc* d, cudaStream_t stream) {
    posemb_kernel<<<d->nsig, 128, 0, stream>>>(*d);
    return ok();
}

OpCheck dsb::linear_check(const ds_linear_desc& d) {
    if (d.in_f > 2048) return {-2, "linear: in_f"};            // the widest kernel holds 2048 weights of a row in registers
    return {0, nullptr};
}

extern "C" int ds_linear_launch(const ds_linear_desc* d, cudaStream_t stream) {
    if (const int rc = linear_check(*d).rc) return rc;
    const int wpb = 4;
    const int bx = (d->out_f + wpb - 1) / wpb;
    int by = d->n_rows < 16 ? d->n_rows : 16;
    if (by < 1) by = 1;
    if (d->in_f <= 256) linear_kernel<256><<<dim3(bx, by), wpb * 32, 0, stream>>>(*d);
    else if (d->in_f <= 512) linear_kernel<512><<<dim3(bx, by), wpb * 32, 0, stream>>>(*d);
    else if (d->in_f <= 1024) linear_kernel<1024><<<dim3(bx, by), wpb * 32, 0, stream>>>(*d);
    else linear_kernel<2048><<<dim3(bx, by), wpb * 32, 0, stream>>>(*d);
    return ok();
}

OpCheck dsb::prep_input_check(const ds_prep_input_desc& d) {
    if (d.C > 64) return {-2, "prep_input: C"};
    if (d.codebook && (d.C > 8 || d.n_embed < 1)) return {-2, "prep_input: codebook"};
    return {0, nullptr};
}

extern "C" int ds_prep_input_launch(const ds_prep_input_desc* d, cudaStream_t stream) {
    if (const int rc = prep_input_check(*d).rc) return rc;
    if (d->codebook) {
        const unsigned blocks = (unsigned)(((long long)d->B * d->HW + 255) / 256);
        if (d->C <= 4) vq_prep_input_kernel<4><<<blocks, 256, 0, stream>>>(*d);
        else vq_prep_input_kernel<8><<<blocks, 256, 0, stream>>>(*d);
        return ok();
    }
    const long long total = (long long)d->B * d->HW * 8;
    prep_input_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(*d);
    return ok();
}

extern "C" int ds_chanmean_launch(const ds_chanmean_desc* d, cudaStream_t stream) {
    const int wpb = 8;
    chanmean_kernel<<<(unsigned)((d->rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(*d);
    return ok();
}

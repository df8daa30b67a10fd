// Fused softmax attention for sm_90a (head dim padded to 64; 32-wide heads in pairs: attn_pair_kernel; 72..128-wide heads:
// attn_wide_kernel): O = softmax(scale * Q K^T) V
// without materialising the L x Lk score matrix in HBM.  Reference: diff-solvers-main/models/networks_edm.py:105-118 (AttentionOp) / :174-178 (UNetBlock attention),
// models/ldm/modules/attention.py:152-196 (CrossAttention.forward).
//
// One CTA per (sample, head, 128-query tile); keys/values stream through in blocks of 64:
//
//   warpgroup 0      TMA producer (warp 0)  Q tile once; K_j [64 keys x 64] and V_j^T [64 x 64 keys] (fp16 hi/lo planes) into a ring
//   warpgroups 1, 2  queries 0..63 / 64..127 of the tile, each on its own:
//                    S_j = Q K_j^T   (3 split-precision passes of 64 x 64 x 16 wgmma, A and B from shared memory)
//                    online softmax in registers (running max / sum per row, p = exp2(s * scale * log2 e - m))
//                    O   = alpha O + P_j V_j   (3 passes of 64 x 64 x 16 wgmma with P as the register A operand: the accumulator
//                                     fragment of S is the A fragment of the next product, so P never leaves registers; each key
//                                     block's product has its own accumulator and is added to O with fp32 FMAs)
//
// Same split-precision contract as the GEMM kernel: Q, K, V and P are fp16 hi + lo planes, products are hi*hi + lo*hi + hi*lo in fp32.
#include "ops.h"
#include "operand.cuh"
#include "ptx.cuh"
#include <cuda_fp16.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

namespace dsb {

int encode_map(CUtensorMap* m, const void* ptr, int rank, const int64_t* dims, const int64_t* strides_bytes, const int32_t* box);

static constexpr int kAttnThreads = 384;            // warpgroup 0: producer (warp 0), 1 and 2: 64 queries each
static constexpr int kAttnStages = 4;
static constexpr int kQBytes = 2 * 16384;          // Q hi, lo: 128 rows x 64 fp16 each
static constexpr int kKBytes = 2 * 8192;           // K hi, lo: 64 keys x 64 fp16
static constexpr int kVBytes = 2 * 8192;           // V^T hi, lo: 64 d-rows x 64 keys fp16
static constexpr int kStageBytes = kKBytes + kVBytes;
static constexpr int kOffKV = kQBytes;
static constexpr int kOffCtl = kOffKV + kAttnStages * kStageBytes;
static constexpr size_t kAttnSmem = kOffCtl + 256 + 1024;

struct alignas(64) AttnKernelParams {
    CUtensorMap tmQ, tmK, tmV;
    int B, nh, L, Lk, q_c0, k_c0, q_tiles;
    float scale_log2e;
    __half* out;
    long long o_plane;
    int o_pitch;
    int causal;                 // query l sees keys <= l
    int pair;                   // attn_pair_kernel: 32-wide heads, nh counts head pairs
    int hd;                     // attn_wide_kernel: the head width (72 .. 128); 0 for the other kernels
};

struct AttnCtl {
    uint64_t q_full;
    uint64_t kv_full[kAttnStages], kv_empty[kAttnStages];
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Where a CTA works and its shared memory, the same for the three kernels.
struct AttnCta {
    uint8_t* smem;              // dynamic shared memory, aligned to 1024 bytes
    AttnCtl* ctl;
    int wg;                     // warpgroup: 0 producer, 1 and 2 queries
    int qt, h, b;               // query tile, head (head pair in attn_pair_kernel), sample
    int nkv;                    // key blocks the tile reads
};

// Prologue of every kernel: decodes (query tile, head, sample) from blockIdx.x and counts the key blocks (kCausal: the kernel applies
// p.causal); thread 0 prefetches the tensor maps and initialises the barriers of a kStages-deep ring in the control block at kOffCtl.
template <int kStages, int kOffCtl, bool kCausal>
__device__ __forceinline__ AttnCta attn_prologue(const AttnKernelParams& p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    AttnCta cta;
    cta.smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    cta.ctl = reinterpret_cast<AttnCtl*>(cta.smem + kOffCtl);
    cta.wg = threadIdx.x >> 7;
    cta.qt = blockIdx.x % p.q_tiles;
    const int z = blockIdx.x / p.q_tiles;
    cta.h = z % p.nh;
    cta.b = z / p.nh;
    // causal: the tile's last query sees keys up to qt * 128 + 127
    const int lk_eff = kCausal && p.causal ? min(p.Lk, cta.qt * 128 + 128) : p.Lk;
    cta.nkv = (lk_eff + 63) >> 6;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tmQ);
        tma_prefetch_desc(&p.tmK);
        tma_prefetch_desc(&p.tmV);
        mbar_init(&cta.ctl->q_full, 1);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&cta.ctl->kv_full[s], 1);
            mbar_init(&cta.ctl->kv_empty[s], 2);                            // one arrival per query warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    return cta;
}

// TMA producer of attn_kernel and attn_pair_kernel (thread 0): the Q tile once, then K_j and V_j^T of the CTA's 64 channels (a head or
// a head pair) for key blocks 0 .. nkv - 1 into the ring, hi and lo plane each.
__device__ __forceinline__ void attn_produce(const AttnKernelParams& p, const AttnCta& cta) {
    mbar_arrive_expect_tx(&cta.ctl->q_full, kQBytes);
    tma_load_3d(&p.tmQ, &cta.ctl->q_full, cta.smem, p.q_c0 + cta.h * 64, cta.qt * 128, cta.b);
    tma_load_3d(&p.tmQ, &cta.ctl->q_full, cta.smem + 16384, p.q_c0 + cta.h * 64, cta.qt * 128, p.B + cta.b);
    for (int j = 0; j < cta.nkv; ++j) {
        const int s = j % kAttnStages;
        const uint32_t ph = (j / kAttnStages) & 1;
        mbar_wait(&cta.ctl->kv_empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&cta.ctl->kv_full[s], kStageBytes);
        uint8_t* sk = cta.smem + kOffKV + s * kStageBytes;
        tma_load_3d(&p.tmK, &cta.ctl->kv_full[s], sk, p.k_c0 + cta.h * 64, j * 64, cta.b);
        tma_load_3d(&p.tmK, &cta.ctl->kv_full[s], sk + 8192, p.k_c0 + cta.h * 64, j * 64, p.B + cta.b);
        tma_load_3d(&p.tmV, &cta.ctl->kv_full[s], sk + kKBytes, j * 64, cta.h * 64, cta.b);
        tma_load_3d(&p.tmV, &cta.ctl->kv_full[s], sk + kKBytes + 8192, j * 64, cta.h * 64, p.B + cta.b);
    }
}

// Online softmax of one key block on the thread's S fragment: S[4 g + e] is row r0 + 8 (e >> 1), key 8 g + 2 (lane & 3) + (e & 1) of
// the block, and column c of row half hr is valid iff c < kv[hr].  Updates the running max m (of scale_log2e * s) and sum l of each row
// and returns alpha, the factor for what was accumulated before this block, and P = exp2(scale_log2e * s - m) as the fp16 hi / lo A
// operand.  The first block's alpha has two forms, equal in value but compiled differently: kScaleInPlace for attn_wide_kernel, which
// scales O by alpha in place, and the other for the kernels that fold a per-block accumulator.  scale_log2e refers to the kernel
// parameter, so it is read where it is used; held in a register across the block it costs attn_kernel one more register.
template <bool kScaleInPlace>
__device__ __forceinline__ void attn_softmax_step(const float (&S)[32], const int (&kv)[2], const float& scale_log2e, float (&m)[2],
                                                  float (&l)[2], float (&alpha)[2], uint32_t (&Ph)[16], uint32_t (&Pl)[16]) {
    const int lane = threadIdx.x & 31;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        const int hr = (i >> 1) & 1;
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (col < kv[hr]) mx[hr] = fmaxf(mx[hr], S[i]);
    }
    float mn[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
        mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
        mn[hr] = fmaxf(m[hr], mx[hr] * scale_log2e);
        if (kScaleInPlace)
            alpha[hr] = m[hr] == -INFINITY ? 0.f : ex2_approx(m[hr] - mn[hr]);     // O and l are still zero before the first block
        else    // a row that has seen no key yet keeps m = -inf: its weights are all zero (masked), nothing to rescale
            alpha[hr] = mn[hr] == -INFINITY ? 1.f : ex2_approx(m[hr] - mn[hr]);
    }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
        const int hr = (i >> 1) & 1;
        const int col = 8 * (i >> 2) + 2 * (lane & 3);
        const float p0 = col < kv[hr] ? ex2_approx(fmaf(S[i], scale_log2e, -mn[hr])) : 0.f;
        const float p1 = col + 1 < kv[hr] ? ex2_approx(fmaf(S[i + 1], scale_log2e, -mn[hr])) : 0.f;
        ls[hr] += p0 + p1;
        split_h16_pair(p0, p1, Ph[i >> 1], Pl[i >> 1]);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        l[hr] = l[hr] * alpha[hr] + ls[hr];
        m[hr] = mn[hr];
    }
}

// End of a query warpgroup: quad-reduces the row sums l, then stores O / l of query rows q0 and q0 + 8 (those below L) as fp16 planes:
// NG groups of 8 columns from output column c0, of which those at or past ncols are skipped.  O[4 g + 2 hr], O[4 g + 2 hr + 1] are
// columns 8 g + 2 (lane & 3), + 1 of row q0 + 8 hr.
template <int NG>
__device__ __forceinline__ void attn_store_rows(const AttnKernelParams& p, const float* O, float (&l)[2], int b, int q0, int c0,
                                                int ncols) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 1);
        l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 2);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int grow = q0 + 8 * hr;
        if (grow >= p.L) continue;
        const float inv = 1.f / l[hr];
        __half* o = p.out + ((long long)b * p.L + grow) * p.o_pitch + c0 + 2 * (lane & 3);
#pragma unroll
        for (int g = 0; g < NG; ++g) {
            const float v[2] = {O[4 * g + 2 * hr] * inv, O[4 * g + 2 * hr + 1] * inv};
            if (8 * g < ncols) store_planes<2>(o, p.o_plane, 8 * g, v, 2);
        }
    }
}

__global__ void __launch_bounds__(kAttnThreads, 1) attn_kernel(const __grid_constant__ AttnKernelParams p) {
    const AttnCta cta = attn_prologue<kAttnStages, kOffCtl, true>(p);
    if (cta.wg == 0) {
        if (threadIdx.x == 0) attn_produce(p, cta);
        return;
    }

    // ---------------------------------------------------------------------- query warpgroups
    const int cw = cta.wg - 1;
    const int lane = threadIdx.x & 31;
    const int w = (threadIdx.x >> 5) & 3;
    const int r0 = cw * 64 + 16 * w + (lane >> 2);          // query rows r0 and r0 + 8 of the tile
    const int q0 = cta.qt * 128 + r0;
    const uint32_t sq = smem_u32(cta.smem) + cw * 64 * 128;
    float O[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) O[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    mbar_wait(&cta.ctl->q_full, 0);
    for (int j = 0; j < cta.nkv; ++j) {
        const int s = j % kAttnStages;
        mbar_wait(&cta.ctl->kv_full[s], (j / kAttnStages) & 1);
        const uint32_t sk = smem_u32(cta.smem + kOffKV + s * kStageBytes);
        const uint32_t sv = sk + kKBytes;
        float S[32];
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint64_t da = wgmma_desc_sw128(sq + (pass == 1 ? 16384 : 0));
            const uint64_t db = wgmma_desc_sw128(sk + (pass == 2 ? 8192 : 0));
#pragma unroll
            for (int k = 0; k < 4; ++k) Wgmma<64>::f16(S, da + 2 * k, db + 2 * k, (pass > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(S);

        int kv[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            int lim = p.Lk - j * 64;
            if (p.causal) lim = min(lim, q0 + 8 * hr - j * 64 + 1);
            kv[hr] = lim;                                     // keys of this block the row may see
        }
        float alpha[2];
        uint32_t Ph[16], Pl[16];
        attn_softmax_step<false>(S, kv, p.scale_log2e, m, l, alpha, Ph, Pl);

        // Ob = P V of this key block: k-chunk kc (keys 16 kc .. +15) of P is S registers 8 kc .. 8 kc + 7, i.e. Ph / Pl [4 kc .. 4 kc + 3];
        // the two correction passes (Pl V_hi, Ph V_lo) first.  The block's product gets its own accumulator and is folded into O below
        // with round-to-nearest FMAs.  In one accumulator over all Lk / 16 wgmma steps, the tensor cores' fp32 accumulation error grows
        // linearly with Lk (3.4e-5 of max |O| at Lk = 4096, the SD 64x64 self-attention, on an H100 80GB HBM3), while l is summed with
        // ordinary adds; per block it stays at the level of 64 keys.  Measured with per-block accumulators on an H100 80GB HBM3 (700 W),
        // values of mean 1 (max |O| about 1) at 4096 and 4097 keys: at most 9.4e-7 for 64-wide heads, 1.2e-6 for 40-wide heads padded
        // to 64 and 8.8e-7 in attn_pair_kernel, against 2e-5 allowed (tests/test_gpu_attention.py).
        float Ob[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) Ob[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t* A = pass == 0 ? Pl : Ph;
            const uint64_t db = wgmma_desc_sw128(sv + (pass == 1 ? 8192 : 0));
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) wgmma_f16_rs_n64(Ob, A + 4 * kc, db + 2 * kc);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(Ob);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&cta.ctl->kv_empty[s]);
#pragma unroll
        for (int i = 0; i < 32; ++i) O[i] = fmaf(O[i], alpha[(i >> 1) & 1], Ob[i]);
    }
    attn_store_rows<8>(p, O, l, cta.b, q0, cta.h * 64, 64);
}

// Heads of width 32, two per CTA (ds_attn_desc.pad0 == 32).  The loads are those of attn_kernel with a head PAIR in place of a
// head: the 64-channel Q / K boxes hold heads 2 hp (channels 0..31) and 2 hp + 1 (32..63) of the pair, the V^T box both heads'
// 32 d-rows.  Per key block each query warpgroup runs the two heads one after the other:
//   S_e = Q_e K_e^T   k16 steps 2 e, 2 e + 1 of the swizzled Q / K tiles (3 split-precision passes, as attn_kernel)
//   online softmax of S_e with its own running max / sum
//   O_e = alpha_e O_e + P_e V_e   m64n32k16 with B at V^T rows 32 e .. 32 e + 31 (4096 B: whole 1024-byte swizzle atoms)
// Against 64-wide zero-padded heads this halves the MMAs, the K / V^T bytes and the q/k/v/out GEMM widths.
__global__ void __launch_bounds__(kAttnThreads, 1) attn_pair_kernel(const __grid_constant__ AttnKernelParams p) {
    const AttnCta cta = attn_prologue<kAttnStages, kOffCtl, true>(p);    // cta.h: the head pair
    if (cta.wg == 0) {
        if (threadIdx.x == 0) attn_produce(p, cta);
        return;
    }

    const int cw = cta.wg - 1;
    const int lane = threadIdx.x & 31;
    const int w = (threadIdx.x >> 5) & 3;
    const int r0 = cw * 64 + 16 * w + (lane >> 2);
    const int q0 = cta.qt * 128 + r0;
    const uint32_t sq = smem_u32(cta.smem) + cw * 64 * 128;
    float O[2][16];
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int i = 0; i < 16; ++i) O[e][i] = 0.f;
    float m[2][2] = {{-INFINITY, -INFINITY}, {-INFINITY, -INFINITY}}, l[2][2] = {{0.f, 0.f}, {0.f, 0.f}};

    mbar_wait(&cta.ctl->q_full, 0);
    for (int j = 0; j < cta.nkv; ++j) {
        const int s = j % kAttnStages;
        mbar_wait(&cta.ctl->kv_full[s], (j / kAttnStages) & 1);
        const uint32_t sk = smem_u32(cta.smem + kOffKV + s * kStageBytes);
        const uint32_t sv = sk + kKBytes;
        int kv[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            int lim = p.Lk - j * 64;
            if (p.causal) lim = min(lim, q0 + 8 * hr - j * 64 + 1);
            kv[hr] = lim;
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            // Q descriptors are rebuilt per head and block rather than hoisted out of the key loop: kept live, they would be spilled
            uint32_t sqe = sq;
            asm volatile("" : "+r"(sqe));
            float S[32];
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint64_t da = wgmma_desc_sw128(sqe + (pass == 1 ? 16384 : 0));
                const uint64_t db = wgmma_desc_sw128(sk + (pass == 2 ? 8192 : 0));
#pragma unroll
                for (int k = 0; k < 2; ++k)
                    Wgmma<64>::f16(S, da + 2 * (2 * e + k), db + 2 * (2 * e + k), (pass > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(S);

            float alpha[2];
            uint32_t Ph[16], Pl[16];
            attn_softmax_step<false>(S, kv, p.scale_log2e, m[e], l[e], alpha, Ph, Pl);
            // per-block accumulator folded into O with fp32 FMAs, as in attn_kernel
            float Ob[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) Ob[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t* A = pass == 0 ? Pl : Ph;
                const uint64_t db = wgmma_desc_sw128(sv + e * 4096 + (pass == 1 ? 8192 : 0));
#pragma unroll
                for (int kc = 0; kc < 4; ++kc) wgmma_f16_rs_n32(Ob, A + 4 * kc, db + 2 * kc);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(Ob);
#pragma unroll
            for (int i = 0; i < 16; ++i) O[e][i] = fmaf(O[e][i], alpha[(i >> 1) & 1], Ob[i]);
        }
        if ((threadIdx.x & 127) == 0) mbar_arrive(&cta.ctl->kv_empty[s]);
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) attn_store_rows<4>(p, O[e], l[e], cta.b, q0, cta.h * 64 + e * 32, 32);
}

// Heads of width hd = 72 .. 128, a multiple of 8 (ds_attn_desc.pad0 = hd; open_clip ViT-g-14: 16 heads of 88).  One head per CTA as
// attn_kernel, with every head-width extent read as 128 channels through 4-D tensor maps that carry the head as its own dimension:
//   Q, K   {hd, nh, L | Lk, 2B}, boxes {64, 1, rows, 1} at channels 0 and 64 of the head: two 64-channel swizzle atoms per row
//   V^T    {keys, hd, nh, 2B}, box {64 keys, 128 d-rows, 1, 1}
// TMA zero-fills channels (V^T rows) hd .. 127, so no GEMM pads its output to 128 and the zero channels add nothing to S or O.  S takes
// ceil(hd / 16) k16 steps per pass; O is two m64n64k16 accumulators (d-rows 0..63, 64..127), of which the store keeps columns < hd.
// Q is 64 KB and a K + V^T stage 64 KB, so the ring has 2 stages.  O[64] accumulates in the wgmma itself (alpha-scaled first, no
// per-block accumulator as in attn_kernel): that keeps S, P and O within the 168 registers of a 384-thread CTA without a stack frame.
// The tensor cores' accumulation error then grows with the key count: measured on an H100 80GB HBM3, 3.6e-6 of max |O| at 257 keys,
// 7.0e-6 at 730 and 8.9e-6 at 1025 with values of mean 1 (tests/test_gpu_openclip.py), against 2e-5 allowed.
static constexpr int kWideStages = 2;
static constexpr int kWideQBytes = 4 * 16384;      // Q hi, lo: 2 channel blocks x 128 rows x 64 fp16 each
static constexpr int kWideKBytes = 4 * 8192;       // K hi, lo: 2 channel blocks x 64 keys x 64
static constexpr int kWideVBytes = 2 * 16384;      // V^T hi, lo: 128 d-rows x 64 keys
static constexpr int kWideStageBytes = kWideKBytes + kWideVBytes;
static constexpr int kWideOffCtl = kWideQBytes + kWideStages * kWideStageBytes;
static constexpr size_t kWideSmem = kWideOffCtl + 256 + 1024;
static_assert(kWideSmem <= 227 * 1024, "attn_wide_kernel shared memory");

__global__ void __launch_bounds__(kAttnThreads, 1) attn_wide_kernel(const __grid_constant__ AttnKernelParams p) {
    const AttnCta cta = attn_prologue<kWideStages, kWideOffCtl, false>(p);
    if (cta.wg == 0) {
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(&cta.ctl->q_full, kWideQBytes);
            for (int pl = 0; pl < 2; ++pl)
                for (int cb = 0; cb < 2; ++cb)
                    tma_load_4d(&p.tmQ, &cta.ctl->q_full, cta.smem + pl * 32768 + cb * 16384, cb * 64, cta.h, cta.qt * 128, pl * p.B + cta.b);
            for (int j = 0; j < cta.nkv; ++j) {
                const int s = j % kWideStages;
                mbar_wait(&cta.ctl->kv_empty[s], ((j / kWideStages) & 1) ^ 1);
                mbar_arrive_expect_tx(&cta.ctl->kv_full[s], kWideStageBytes);
                uint8_t* sk = cta.smem + kWideQBytes + s * kWideStageBytes;
                for (int pl = 0; pl < 2; ++pl) {
                    for (int cb = 0; cb < 2; ++cb)
                        tma_load_4d(&p.tmK, &cta.ctl->kv_full[s], sk + pl * 16384 + cb * 8192, cb * 64, cta.h, j * 64, pl * p.B + cta.b);
                    tma_load_4d(&p.tmV, &cta.ctl->kv_full[s], sk + kWideKBytes + pl * 16384, j * 64, 0, cta.h, pl * p.B + cta.b);
                }
            }
        }
        return;
    }

    const int cw = cta.wg - 1;
    const int lane = threadIdx.x & 31;
    const int w = (threadIdx.x >> 5) & 3;
    const int r0 = cw * 64 + 16 * w + (lane >> 2);
    const int q0 = cta.qt * 128 + r0;
    const uint32_t sq = smem_u32(cta.smem) + cw * 64 * 128;
    float O[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) O[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    mbar_wait(&cta.ctl->q_full, 0);
    for (int j = 0; j < cta.nkv; ++j) {
        const int s = j % kWideStages;
        mbar_wait(&cta.ctl->kv_full[s], (j / kWideStages) & 1);
        const uint32_t sk = smem_u32(cta.smem + kWideQBytes + s * kWideStageBytes);
        const uint32_t sv = sk + kWideKBytes;
        // Q descriptors are rebuilt per block rather than hoisted out of the key loop: kept live, they would be spilled
        uint32_t sqj = sq;
        asm volatile("" : "+r"(sqj));
        float S[32];
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
#pragma unroll
            for (int cb = 0; cb < 2; ++cb) {
                const uint64_t da = wgmma_desc_sw128(sqj + (pass == 1 ? 32768 : 0) + cb * 16384);
                const uint64_t db = wgmma_desc_sw128(sk + (pass == 2 ? 16384 : 0) + cb * 8192);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    Wgmma<64>::f16(S, da + 2 * k, db + 2 * k, (pass > 0 || cb > 0 || k > 0) ? 1u : 0u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(S);

        const int kv[2] = {p.Lk - j * 64, p.Lk - j * 64};      // keys of this block, the same for both row halves: no causal mask
        float alpha[2];
        uint32_t Ph[16], Pl[16];
        attn_softmax_step<true>(S, kv, p.scale_log2e, m, l, alpha, Ph, Pl);
#pragma unroll
        for (int i = 0; i < 64; ++i) O[i] *= alpha[(i >> 1) & 1];
        // O += P V: the two correction passes (Pl V_hi, Ph V_lo) first; d-rows 64 c .. 64 c + 63 of V^T are 8 KB into the tile
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t* A = pass == 0 ? Pl : Ph;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const uint64_t db = wgmma_desc_sw128(sv + (pass == 1 ? 16384 : 0) + c * 8192);
#pragma unroll
                for (int kc = 0; kc < 4; ++kc) wgmma_f16_rs_n64(O + 32 * c, A + 4 * kc, db + 2 * kc);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(O);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&cta.ctl->kv_empty[s]);
    }
    // O[32 c + 4 g ..] is group 8 c + g: columns 64 c + 8 g of the head; hd % 8 == 0, so the groups below hd are whole
    attn_store_rows<16>(p, O, l, cta.b, q0, cta.h * p.hd, p.hd);
}

// ------------------------------------------------------------------------------------------ host
// Width of each head: pad0 of the descriptor (0 = 64).
static int attn_head_dim(const ds_attn_desc& d) { return d.pad0 == 0 ? 64 : d.pad0; }
static bool attn_wide(int hd) { return hd >= 72 && hd <= 128 && hd % 8 == 0; }

OpCheck attn_check(const ds_attn_desc& d) {
    if (d.nplanes != 2 || d.B <= 0 || d.nh <= 0 || d.L <= 0 || d.Lk <= 0 || !(d.scale > 0.f)) return {-30, "attn: args"};
    if (d.q_pitch % 8 || d.k_pitch % 8 || d.vt_pitch % 8 || d.o_pitch % 8 || d.q_c0 % 8 || d.k_c0 % 8) return {-31, "attn: pitch"};
    const int hd = attn_head_dim(d);
    if (hd != 64 && hd != 32 && !attn_wide(hd)) return {-41, "attn: head_dim"};
    if (attn_wide(hd) && d.causal) return {-43, "attn: wide causal"};     // the wide kernel has no causal mask (CLIP text heads are 64 wide)
    // 32-wide heads run in pairs (one 64-channel box): an odd head count is padded with a zero head by the plan
    if (hd == 32 && d.nh % 2) return {-42, "attn: pair head count"};
    if (d.q_c0 + d.nh * hd > d.q_pitch || d.k_c0 + d.nh * hd > d.k_pitch || d.nh * hd > d.o_pitch || d.Lk > d.vt_pitch)
        return {-32, "attn: extent"};
    if (d.causal && d.L != d.Lk) return {-40, "attn: causal"};        // the causal mask is defined for self-attention only
    return {0, nullptr};
}

int attn_build(const ds_attn_desc* d, AttnKernelParams* kp) {
    if (const int rc = attn_check(*d).rc) return rc;
    const int hd = attn_head_dim(*d);
    kp->hd = attn_wide(hd) ? hd : 0;
    if (kp->hd) {
        const int64_t qdims[4] = {hd, d->nh, d->L, (int64_t)2 * d->B};
        const int64_t qstr[3] = {(int64_t)hd * 2, (int64_t)d->q_pitch * 2, (int64_t)d->L * d->q_pitch * 2};
        const int32_t qbox[4] = {64, 1, 128, 1};
        if (encode_map(&kp->tmQ, static_cast<const __half*>(d->q) + d->q_c0, 4, qdims, qstr, qbox)) return -33;
        const int64_t kdims[4] = {hd, d->nh, d->Lk, (int64_t)2 * d->B};
        const int64_t kstr[3] = {(int64_t)hd * 2, (int64_t)d->k_pitch * 2, (int64_t)d->Lk * d->k_pitch * 2};
        const int32_t kbox[4] = {64, 1, 64, 1};
        if (encode_map(&kp->tmK, static_cast<const __half*>(d->k) + d->k_c0, 4, kdims, kstr, kbox)) return -34;
        const int64_t vdims[4] = {d->Lk, hd, d->nh, (int64_t)2 * d->B};
        const int64_t vstr[3] = {(int64_t)d->vt_pitch * 2, (int64_t)hd * d->vt_pitch * 2, (int64_t)d->nh * hd * d->vt_pitch * 2};
        const int32_t vbox[4] = {64, 128, 1, 1};
        if (encode_map(&kp->tmV, d->vt, 4, vdims, vstr, vbox)) return -35;
    } else {
        {
            const int64_t dims[3] = {d->q_pitch, d->L, (int64_t)2 * d->B};
            const int64_t str[2] = {(int64_t)d->q_pitch * 2, (int64_t)d->L * d->q_pitch * 2};
            const int32_t box[3] = {64, 128, 1};
            if (encode_map(&kp->tmQ, d->q, 3, dims, str, box)) return -33;
        }
        {
            const int64_t dims[3] = {d->k_pitch, d->Lk, (int64_t)2 * d->B};
            const int64_t str[2] = {(int64_t)d->k_pitch * 2, (int64_t)d->Lk * d->k_pitch * 2};
            const int32_t box[3] = {64, 64, 1};
            if (encode_map(&kp->tmK, d->k, 3, dims, str, box)) return -34;
        }
        {
            const int64_t rows = (int64_t)d->nh * attn_head_dim(*d);
            const int64_t dims[3] = {d->Lk, rows, (int64_t)2 * d->B};
            const int64_t str[2] = {(int64_t)d->vt_pitch * 2, rows * d->vt_pitch * 2};
            const int32_t box[3] = {64, 64, 1};
            if (encode_map(&kp->tmV, d->vt, 3, dims, str, box)) return -35;
        }
    }
    kp->pair = attn_head_dim(*d) == 32 ? 1 : 0;
    kp->B = d->B; kp->nh = kp->pair ? d->nh / 2 : d->nh; kp->L = d->L; kp->Lk = d->Lk; kp->q_c0 = d->q_c0; kp->k_c0 = d->k_c0;
    kp->q_tiles = (d->L + 127) / 128;
    kp->scale_log2e = d->scale * 1.4426950408889634f;
    kp->out = reinterpret_cast<__half*>(d->out);
    kp->o_plane = (long long)d->B * d->L * d->o_pitch;
    kp->o_pitch = d->o_pitch;
    kp->causal = d->causal ? 1 : 0;
    return 0;
}

size_t attn_params_size() { return sizeof(AttnKernelParams); }

int attn_run(const AttnKernelParams* kp, cudaStream_t stream) {
    static bool attr_set[64][3] = {};               // per device (cudaFuncSetAttribute is a per-device setting) and kernel
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return -39;
    const int kind = kp->hd ? 2 : (kp->pair ? 1 : 0);
    const size_t smem = kind == 2 ? kWideSmem : kAttnSmem;
    if (!attr_set[dev][kind]) {
        const void* fn = kind == 2 ? (const void*)attn_wide_kernel : (kind == 1 ? (const void*)attn_pair_kernel : (const void*)attn_kernel);
        if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -36;
        attr_set[dev][kind] = true;
    }
    const long long grid = (long long)kp->B * kp->nh * kp->q_tiles;
    if (grid <= 0 || grid > 0x7fffffffLL) return -37;
    if (kind == 2) attn_wide_kernel<<<(unsigned)grid, kAttnThreads, kWideSmem, stream>>>(*kp);
    else if (kind == 1) attn_pair_kernel<<<(unsigned)grid, kAttnThreads, kAttnSmem, stream>>>(*kp);
    else attn_kernel<<<(unsigned)grid, kAttnThreads, kAttnSmem, stream>>>(*kp);
    return cudaGetLastError() == cudaSuccess ? 0 : -38;
}

}  // namespace dsb

extern "C" int ds_attn_launch(const ds_attn_desc* d, cudaStream_t stream) {
    dsb::AttnKernelParams kp;
    int rc = dsb::attn_build(d, &kp);
    if (rc) return rc;
    return dsb::attn_run(&kp, stream);
}

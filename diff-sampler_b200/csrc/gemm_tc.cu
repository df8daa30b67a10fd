// wgmma implicit-GEMM convolution / GEMM for sm_90a.
//
// One persistent, warp-specialised kernel serves every contraction of the denoiser U-Net
// (reference: diff-solvers-main/models/networks_edm.py:60-82 Conv2d, :105-118 AttentionOp,
//  :174-178 qkv/proj): 3x3 and 1x1 convolutions over NHWC fp16 activations, the 1x1 skip
// projection appended along K, and the batched Q.K^T / P.V products of self-attention.
//
//   warpgroup 0   TMA producer  (warp 0: cp.async.bulk.tensor 4-D boxes for A = shifted pixel tiles, 3-D for B)
//   warpgroups 1, 2  consumers  (rows 0..63 / 64..127 of the 128-row tile: wgmma 64 x BN x 16 fp16, fp32 accumulators in registers;
//                                in f8 mode the two split-precision correction products are e4m3 wgmmas, 64 x BN x 32, into the
//                                same accumulators), then the epilogue: accumulators -> shared-memory staging in 64-column chunks ->
//                                one row per thread: bias / embedding / residual / scale / GroupNorm partial sums -> fp32 and/or
//                                fp16 hi/lo
//
// Pipeline: a ring of shared-memory stages (one 64-channel fp16 or 128-channel e4m3 K block of A and B each; full / empty mbarriers)
// between the producer and the consumers.  The producer runs ahead into the next tile while the consumers drain the current one.
#include "ops.h"
#include "ptx.cuh"
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace dsb {

static constexpr int kMaxStages = 8;
static constexpr int kATileBytes = 128 * 128;   // 128 rows x 64 fp16 (or 128 e4m3)
static constexpr int kThreads = 384;           // warpgroup 0: producer (warp 0), 1 and 2: consumers
static constexpr int kStgPitch = 64;           // floats per row of the epilogue staging buffer (16-byte chunks XOR-swizzled: stg_swz)
static constexpr int kStgBytes = 2 * 64 * kStgPitch * 4;
static constexpr int kSmemLimit = 227 * 1024;

struct alignas(64) GemmKernelParams {
    CUtensorMap tmA, tmA2, tmB;
    CUtensorMap tmA8, tmA2_8, tmB8;      // f8 mode: e4m3 planes of the same operands (uint8 maps, 128-channel boxes)
    int f8, cpb8, nkb8_main, nkb8_aux, a8_plane_n;
    float acc_scale;
    int BN, m_tiles, n_tiles, num_z, nh;
    int taps, cpb, nkb_main, nkb_aux, npass;
    int a_mode, conv_H, conv_W, a_bn_dummy;
    int a_plane_n, a2_plane_n, b_plane_batch;
    int a_c_per_zh, a_n_per_zb, a_n_per_zh;
    int b_k0, b_k_per_zh, b_row_per_zh, b_z_per_zb, b_z_per_zh;
    int m_valid, n_valid;
    int num_stages;
    float* out_f32;
    __half* out_h16;
    long long o_zb, o_zh, ldo, o_plane;
    const float* bias_n;
    const float* bias_m;
    const float* rowvec;
    long long rowvec_stride;
    int rows_per_sample;
    const float* residual;
    long long ldr;
    float scale;
    int edm_out;
    const float* edm_x;
    const float* edm_coef;
    int edm_coef_stride;
    int edm_C;
    float* edm_D;
    // fused GroupNorm statistics of the tensor being written (up to two consumers with their own channel grouping):
    // per 32-row slab partial {sum, sumsq} per group, plain stores (no atomics); the consumer adds the slabs of a sample.
    float* st_quads;
    int st_unit;                         // 4 (quads) or 2 (pairs)
    int tap_dh[9], tap_dw[9], tap_cb[9];
    int f8_last_steps;                   // e4m3 MMAs (K = 32) of the last 128-channel block of a tap: 2 when only its first 64 channels exist
                                         // (C = 64, 192, 576: the other two would multiply TMA zero fill with zero-padded weights), else 4
    int relu;
};

struct SmemCtl {
    uint64_t full[kMaxStages];
    uint64_t empty[kMaxStages];
};

// Sum NV per-lane values over the 32 lanes of a warp with NV-ish shuffles instead of 5*NV: at every butterfly level each lane
// keeps one half of its values and hands the other half to its partner, so the value count halves while the lane span doubles.
// On return v[0] of lane L is the full sum of value index (L >> (5 - log2 NV)) (NV = 16: L >> 1; NV = 8: L >> 2).
// The levels recurse on a template count: with a runtime count (n >>= 1) the level loop stays rolled, v[i + n] becomes a dynamic
// index and the whole array moves to the stack.
template <int N>
__device__ __forceinline__ void warp_sum_levels(float* v, int lane, int off) {
    if constexpr (N >= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const float send = up ? v[i] : v[i + N];
            const float keep = up ? v[i + N] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
        warp_sum_levels<N / 2>(v, lane, off >> 1);
    } else {
        for (; off >= 1; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
    }
}
template <int NV>
__device__ __forceinline__ void warp_sum_multi(float (&v)[NV], int lane) {
    static_assert(NV == 32 || NV == 16 || NV == 8, "NV");
    warp_sum_levels<NV / 2>(v, lane, 16);
}

template <int W>
__device__ __forceinline__ void epilogue_chunk(const GemmKernelParams& p, const float* v, long long grow_in_z, int col0, bool row_ok,
                                               int zb, int zh) {
    // v[W]: accumulators of this thread's row, columns col0 .. col0+W-1 (col0 is the global column)
    const bool warp_rows_ok = __all_sync(0xffffffffu, row_ok);      // every lane has a valid row: the paired stores below may shuffle
    if (!row_ok) return;                                   // warp-uniform whenever statistics are fused (m_valid % 32 == 0)
    float r[W];
#pragma unroll
    for (int j = 0; j < W; ++j) r[j] = v[j] * p.acc_scale;     // 1 unless the operands carry power-of-two scales (f8 mode): exact
    const bool full = (col0 + W <= p.n_valid);
    if (p.bias_n) {
        if (full) {
#pragma unroll
            for (int j = 0; j < W; j += 4) {
                const float4 t = __ldg(reinterpret_cast<const float4*>(p.bias_n + col0 + j));
                r[j] += t.x; r[j + 1] += t.y; r[j + 2] += t.z; r[j + 3] += t.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (col0 + j < p.n_valid) r[j] += __ldg(p.bias_n + col0 + j);
        }
    }
    if (p.bias_m) {
        const float bm = __ldg(p.bias_m + grow_in_z);
#pragma unroll
        for (int j = 0; j < W; ++j) r[j] += bm;
    }
    if (p.rowvec) {
        const long long s = (p.rowvec_stride == 0) ? 0 : (grow_in_z / p.rows_per_sample) * p.rowvec_stride;
        const float* rv = p.rowvec + s + col0;
        if (full) {
#pragma unroll
            for (int j = 0; j < W; j += 4) {
                const float4 t = __ldg(reinterpret_cast<const float4*>(rv + j));
                r[j] += t.x; r[j + 1] += t.y; r[j + 2] += t.z; r[j + 3] += t.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (col0 + j < p.n_valid) r[j] += __ldg(rv + j);
        }
    }
    if (p.residual) {
        const float* rs = p.residual + grow_in_z * p.ldr + col0;
        if (full) {
#pragma unroll
            for (int j = 0; j < W; j += 4) {
                const float4 t = *reinterpret_cast<const float4*>(rs + j);
                r[j] += t.x; r[j + 1] += t.y; r[j + 2] += t.z; r[j + 3] += t.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (col0 + j < p.n_valid) r[j] += rs[j];
        }
    }
#pragma unroll
    for (int j = 0; j < W; ++j) r[j] *= p.scale;
    if (p.relu) {
#pragma unroll
        for (int j = 0; j < W; ++j) r[j] = r[j] > 0.f ? r[j] : 0.f;
    }

    if (p.st_quads) {
        const int lane = threadIdx.x & 31;
        if (p.st_unit == 2) {
            // per channel PAIR {sum, sumsq} (consumers whose groups are even but not multiples of four channels)
            float q[W];
#pragma unroll
            for (int j = 0; j < W; j += 2) {
                q[j] = r[j] + r[j + 1];
                q[j + 1] = fmaf(r[j], r[j], r[j + 1] * r[j + 1]);
            }
            warp_sum_multi<W>(q, lane);
            constexpr int kShift = (W == 32) ? 0 : 1;        // lane L holds value L >> kShift = 2 * pair + {0: sum, 1: sumsq}
            const int vi = lane >> kShift;
            if ((lane & ((1 << kShift) - 1)) == 0 && col0 + 2 * (vi >> 1) < p.n_valid)
                p.st_quads[(grow_in_z >> 5) * (long long)p.n_valid + col0 + vi] = q[0];
        } else {
            // GroupNorm partials of this 32-row slab: per channel quad {sum, sumsq}, reduced over the warp's 32 rows
            float q[W / 2];
#pragma unroll
            for (int j = 0; j < W; j += 4) {
                q[j / 2] = (r[j] + r[j + 1]) + (r[j + 2] + r[j + 3]);
                q[j / 2 + 1] = fmaf(r[j], r[j], r[j + 1] * r[j + 1]) + fmaf(r[j + 2], r[j + 2], r[j + 3] * r[j + 3]);
            }
            warp_sum_multi<W / 2>(q, lane);
            constexpr int kShift = (W == 32) ? 1 : 2;        // lane L holds value L >> kShift = 2 * quad + {0: sum, 1: sumsq}
            const int vi = lane >> kShift;
            if ((lane & ((1 << kShift) - 1)) == 0 && col0 + 4 * (vi >> 1) < p.n_valid)
                p.st_quads[((grow_in_z >> 5) * (long long)(p.n_valid >> 2)) * 2 + (col0 >> 1) + vi] = q[0];
        }
    }

    if (p.edm_out) {
        // D = c_skip * x + c_out * F, written NCHW (reference: networks_edm.py:488-495)
        const int HW = p.rows_per_sample;
        const long long n = grow_in_z / HW;
        const long long hw = grow_in_z % HW;
        if (p.edm_out == 2) {
#pragma unroll
            for (int j = 0; j < W; ++j) {
                const int c = col0 + j;
                if (c < p.edm_C) p.edm_D[(n * p.edm_C + c) * HW + hw] = r[j];
            }
            return;
        }
        const float cskip = __ldg(p.edm_coef + n * p.edm_coef_stride + 0);
        const float cout = __ldg(p.edm_coef + n * p.edm_coef_stride + 1);
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = col0 + j;
            if (c < p.edm_C) {
                const long long idx = (n * p.edm_C + c) * HW + hw;
                p.edm_D[idx] = cskip * __ldg(p.edm_x + idx) + cout * r[j];
            }
        }
        return;
    }

    const long long obase = (long long)zb * p.o_zb + (long long)zh * p.o_zh + grow_in_z * p.ldo + col0;
    // Each thread owns one output row, so a plain 16-byte store per thread writes HALF of 32 different 32-byte sectors per warp
    // instruction (2x the payload over the crossbar).  Lanes 2i / 2i+1 swap halves of an 8-float group instead: both then write the two halves of ONE sector of row 2i,
    // and of row 2i+1 with the second store -- full sectors only.
    const int odd = threadIdx.x & 1;
    if (p.out_f32) {
        float* o = p.out_f32 + obase;
        if (full && warp_rows_ok) {
            float* oe = o - odd * p.ldo + odd * 4;           // the even lane's row, this lane's half of the group
#pragma unroll
            for (int j = 0; j < W; j += 8) {
                float x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) x[k] = __shfl_xor_sync(0xffffffffu, odd ? r[j + k] : r[j + 4 + k], 1);
                const float4 s1 = odd ? make_float4(x[0], x[1], x[2], x[3]) : make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]);
                const float4 s2 = odd ? make_float4(r[j + 4], r[j + 5], r[j + 6], r[j + 7]) : make_float4(x[0], x[1], x[2], x[3]);
                *reinterpret_cast<float4*>(oe + j) = s1;
                *reinterpret_cast<float4*>(oe + p.ldo + j) = s2;
            }
        } else if (full) {
#pragma unroll
            for (int j = 0; j < W; j += 4) *reinterpret_cast<float4*>(o + j) = make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (col0 + j < p.n_valid) o[j] = r[j];
        }
    }
    if (p.out_h16) {
        __half* oh = p.out_h16 + obase;
        if (full) {
            __align__(16) __half hi[W];
            __align__(16) __half lo[W];
#pragma unroll
            for (int j = 0; j < W; ++j) {
                hi[j] = __float2half_rn(r[j]);
                lo[j] = __float2half_rn(r[j] - __half2float(hi[j]));
            }
            if (warp_rows_ok && W % 16 == 0) {
                // the same sector pairing for the fp16 planes: groups of 16 halves (32 bytes), lanes 2i / 2i+1 swap 16-byte halves
                __half* he = oh - odd * p.ldo + odd * 8;
#pragma unroll
                for (int pl = 0; pl < 2; ++pl) {
                    if (pl == 1 && !p.o_plane) break;
                    const __half* src = pl ? lo : hi;
                    __half* dst = he + (pl ? p.o_plane : 0);
#pragma unroll
                    for (int j = 0; j < W; j += 16) {
                        const uint4 a = *reinterpret_cast<const uint4*>(src + j), b = *reinterpret_cast<const uint4*>(src + j + 8);
                        const uint4 snd = odd ? a : b;
                        uint4 x;
                        x.x = __shfl_xor_sync(0xffffffffu, snd.x, 1); x.y = __shfl_xor_sync(0xffffffffu, snd.y, 1);
                        x.z = __shfl_xor_sync(0xffffffffu, snd.z, 1); x.w = __shfl_xor_sync(0xffffffffu, snd.w, 1);
                        *reinterpret_cast<uint4*>(dst + j) = odd ? x : a;
                        *reinterpret_cast<uint4*>(dst + p.ldo + j) = odd ? b : x;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < W; j += 8) *reinterpret_cast<uint4*>(oh + j) = *reinterpret_cast<const uint4*>(hi + j);
                if (p.o_plane) {
#pragma unroll
                    for (int j = 0; j < W; j += 8)
                        *reinterpret_cast<uint4*>(oh + p.o_plane + j) = *reinterpret_cast<const uint4*>(lo + j);
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (col0 + j < p.n_valid) {
                    const __half h = __float2half_rn(r[j]);
                    oh[j] = h;
                    if (p.o_plane) oh[p.o_plane + j] = __float2half_rn(r[j] - __half2float(h));
                }
        }
    }
}

struct RingPos {
    int stage;
    uint32_t phase;
};

struct TileCoord {
    int mt, nt, zb, zh;
};

__device__ __forceinline__ TileCoord tile_coord(const GemmKernelParams& p, int tile) {
    const int tiles_per_z = p.m_tiles * p.n_tiles;
    const int z = tile / tiles_per_z;
    const int t2 = tile - z * tiles_per_z;
    TileCoord c;
    c.mt = t2 / p.n_tiles;
    c.nt = t2 - c.mt * p.n_tiles;
    c.zb = z / p.nh;
    c.zh = z - c.zb * p.nh;
    return c;
}

// ------------------------------------------------------------------------------------------ TMA producer: the K loop of one tile
// Walks (pass, tap, channel block) with running coordinates: no division, one parameter load per tap.  The whole warp runs the loop;
// one elected lane issues the copies.
__device__ __forceinline__ void producer_tile(const GemmKernelParams& p, uint8_t* smem, SmemCtl* ctl, RingPos& r, const int block_bytes,
                                              const int aw0, const int ah0, const int an0, const int a_c_off, const int b_k_off,
                                              const int b_row, const int b_z) {
    const uint32_t tx_bytes = (uint32_t)block_bytes;
    auto load = [&](const CUtensorMap* ma, int ac, int aw, int ah, int an, const CUtensorMap* mb, int bk, int bz) {
        mbar_wait_warp(&ctl->empty[r.stage], r.phase ^ 1);
        uint8_t* sa = smem + r.stage * block_bytes;
        uint64_t* full = &ctl->full[r.stage];
        if (elect_one()) {
            mbar_arrive_expect_tx(full, tx_bytes);
            tma_load_4d(ma, full, sa, ac, aw, ah, an);
            tma_load_3d(mb, full, sa + kATileBytes, bk, b_row, bz);
        }
        __syncwarp();
        if (++r.stage == p.num_stages) { r.stage = 0; r.phase ^= 1; }
    };
    if (p.f8) {
        // e4m3 blocks (128 channels = one 128-byte swizzle row): A_lo8 x W_hi8 over all of K, then A_hi8 x W_lo8
        for (int pass8 = 0; pass8 < 2; ++pass8) {
            const int an8 = an0 + pass8 * p.a8_plane_n;
            int bk = 0;
            for (int tap = 0; tap < p.taps; ++tap) {
                const int aw = aw0 + p.tap_dw[tap], ah = ah0 + p.tap_dh[tap];
                for (int cb = 0; cb < p.cpb8; ++cb, bk += 128) load(&p.tmA8, cb * 128, aw, ah, an8, &p.tmB8, bk, pass8);
            }
            for (int j = 0; j < p.nkb8_aux; ++j, bk += 128) load(&p.tmA2_8, j * 128, aw0, ah0, an8, &p.tmB8, bk, pass8);
        }
    }
    // fp16 passes: (lo x hi, hi x lo,) then hi x hi.  Every wgmma adds an error proportional to the accumulator's current
    // magnitude (on H100 the fp32 accumulation error grows linearly with K), so the two small correction products go first, while
    // the sum is still ~2^-11 of its final size, as the e4m3 corrections do in f8 mode; only the main product then accumulates at
    // full magnitude.
    const int npass16 = p.f8 ? 1 : p.npass;
    for (int pi = 0; pi < npass16; ++pi) {
        const int pass = npass16 == 3 ? (pi + 1) % 3 : pi;
        const int an = an0 + (pass == 1 ? p.a_plane_n : 0);
        const int an2 = an0 + (pass == 1 ? p.a2_plane_n : 0);
        const int bz = b_z + (pass == 2 ? p.b_plane_batch : 0);
        int bk = b_k_off;
        for (int tap = 0; tap < p.taps; ++tap) {
            const int aw = aw0 + p.tap_dw[tap], ah = ah0 + p.tap_dh[tap];
            const int ac0 = p.tap_cb[tap] + a_c_off;
            for (int cb = 0; cb < p.cpb; ++cb, bk += 64) load(&p.tmA, ac0 + cb * 64, aw, ah, an, &p.tmB, bk, bz);
        }
        for (int j = 0; j < p.nkb_aux; ++j, bk += 64) load(&p.tmA2, j * 64, aw0, ah0, an2, &p.tmB, bk, bz);
    }
}

// ------------------------------------------------------------------------------------------ consumer: the K loop of one tile
// One consumer warpgroup, 64 rows.  Walks the ring in the producer's order; every stage is one wgmma group, issued and committed in
// one straight block (fence, its MMAs, commit).  ptxas then marks only the group's last MMA as the commit point, so the wait for
// "one group in flight" really leaves this stage's MMAs running and retires the previous stage, which is released at once.  Keep
// the commit in that block: after a branch merge ptxas carries it on an empty MMA of its own, the wait drains every real MMA, and
// the consumers hold one retired stage the producer could already refill (tests/test_gemm_sass.py).
template <int BN>
__device__ __forceinline__ void mma_tile(const GemmKernelParams& p, uint8_t* smem, SmemCtl* ctl, RingPos& r, const int block_bytes,
                                         const int wg, float (&acc)[BN / 2]) {
    const bool leader = (threadIdx.x & 127) == 0;
    int prev = -1;
    uint32_t scale0 = 0u;                      // only the tile's first MMA overwrites the accumulators
    auto stage = [&](auto f8, auto steps) {
        constexpr bool F8 = decltype(f8)::value;
        constexpr int NS = decltype(steps)::value;
        mbar_wait(&ctl->full[r.stage], r.phase);
        const uint32_t s0 = smem_u32(smem + r.stage * block_bytes);
        const uint64_t da = wgmma_desc_sw128(s0 + wg * 64 * 128);
        const uint64_t db = wgmma_desc_sw128(s0 + kATileBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < NS; ++k)           // 32 e4m3 = 32 bytes per MMA: the same +2 descriptor step (16-byte units) as 16 fp16
            wgmma_ss<BN, F8>(acc, da + 2 * k, db + 2 * k, k > 0 ? 1u : scale0);
        wgmma_commit();
        wgmma_fence_regs(acc);
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&ctl->empty[prev]);
        prev = r.stage;
        if (++r.stage == p.num_stages) { r.stage = 0; r.phase ^= 1; }
        scale0 = 1u;
    };
    using f8_t = std::true_type;
    using f16_t = std::false_type;
    using full_t = std::integral_constant<int, 4>;
    using half_t = std::integral_constant<int, 2>;
    if (p.f8) {
        // e4m3 blocks of a pass: per tap cpb8 channel blocks (the last one half empty when f8_last_steps == 2), then the aux blocks
        const int full8 = p.f8_last_steps == 2 ? p.cpb8 - 1 : p.cpb8;
        for (int pass8 = 0; pass8 < 2; ++pass8) {
            for (int tap = 0; tap < p.taps; ++tap) {
                for (int cb = 0; cb < full8; ++cb) stage(f8_t{}, full_t{});
                if (full8 < p.cpb8) stage(f8_t{}, half_t{});
            }
            for (int j = 0; j < p.nkb8_aux; ++j) stage(f8_t{}, full_t{});
        }
    }
    const int n16 = (p.f8 ? 1 : p.npass) * (p.nkb_main + p.nkb_aux);
    for (int i = 0; i < n16; ++i) stage(f16_t{}, full_t{});
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && leader) mbar_arrive(&ctl->empty[prev]);
}

// ------------------------------------------------------------------------------------------ consumer: the epilogue of one tile
// Accumulator fragment (m64nBN): register g of lane L in warp w holds row 16 w + L / 4 + 8 ((g >> 1) & 1), column 8 (g / 4) + 2 (L % 4)
// + (g & 1).  Per 64-column chunk the warpgroup stages its 64 x 64 block in shared memory; then warp w takes rows 32 (w & 1) + lane
// (one row per lane: the layout epilogue_chunk expects, 32-row slabs for the GroupNorm partials) and columns 32 (w >> 1) .. + 32.
//
// Staging rows are 64 floats (256 bytes) with no padding; the 16-byte chunk c of row r is stored at chunk c ^ f(r & 7),
// f = {0,2,4,6,1,3,5,7}.  Fragment stores (float2): each half warp writes 4 rows x 2 adjacent chunks {2i, 2i+1}; f(r) >> 1 differs
// across those rows, so the 8 chunks land in 8 different bank groups.  Row reads (float4): each quarter warp reads one chunk of 8
// consecutive rows; f is a permutation of 0..7, so again 8 different bank groups.  An address is a per-row key (row base + f) with
// the in-row offset XORed on: rows are 256-byte aligned and no in-row offset carries into bit 8.  Without the padding the ring
// gets one more stage at BN = 256 (4) and at BN = 128 (6).
__device__ __forceinline__ uint32_t stg_swz(uint32_t r) { return (((r & 3) << 1) | ((r >> 2) & 1)) << 4; }

// The lane id, re-read wherever it is used: the staging keys derived from it are then rebuilt per chunk instead of being held in
// registers across the whole epilogue (at BN = 256 the accumulators leave no room for them).
__device__ __forceinline__ uint32_t lane_id_here() {
    uint32_t l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}
__device__ __forceinline__ void sts_f2(uint32_t a, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}

template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmKernelParams& p, float* stg, const int wg, const TileCoord& tc, const float (&acc)[BN / 2]) {
    const int lane = threadIdx.x & 31;
    const int w = (threadIdx.x >> 5) & 3;
    const int row = 32 * (w & 1) + lane;
    const long long grow = (long long)tc.mt * 128 + wg * 64 + row;
    const bool row_ok = grow < p.m_valid;
    const int ch = 32 * (w >> 1);
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += 64) {
        uint32_t ln = lane_id_here();
        // fragment row 16 w + ln / 4 (+ 8), columns 8 i + 2 (ln % 4): (row & 7) == ln / 4
        const uint32_t wkey = smem_u32(stg) + (16 * w + (ln >> 2)) * 256 + ((8 * (ln & 3)) ^ stg_swz(ln >> 2));
#pragma unroll
        for (int g = 0; g < 32; g += 2) {
            const int gi = c0 / 2 + g;
            if (gi < BN / 2) sts_f2((wkey + 2048 * ((g >> 1) & 1)) ^ (32 * (g >> 2)), acc[gi], acc[gi + 1]);
        }
        warpgroup_sync(1 + wg);
        const int width = min(32, BN - c0 - ch);
        const int col0 = tc.nt * BN + c0 + ch;
        ln = lane_id_here();
        const uint32_t rkey = smem_u32(stg) + (32 * (w & 1) + ln) * 256 + 4 * ch + stg_swz(ln);      // (row & 7) == ln % 8
        if (width >= 32) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(v + j) = lds_f4(rkey ^ (4 * j));
            if (col0 < p.n_valid) epilogue_chunk<32>(p, v, grow, col0, row_ok, tc.zb, tc.zh);
        } else if (width >= 16) {
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(v + j) = lds_f4(rkey ^ (4 * j));
            if (col0 < p.n_valid) epilogue_chunk<16>(p, v, grow, col0, row_ok, tc.zb, tc.zh);
        }
        warpgroup_sync(1 + wg);
    }
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmKernelParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // 1024-byte alignment is required by the 128B swizzle; the runtime only guarantees 16.
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int block_bytes = kATileBytes + BN * 128;
    float* stg = reinterpret_cast<float*>(smem + p.num_stages * block_bytes);
    SmemCtl* ctl = reinterpret_cast<SmemCtl*>(smem + p.num_stages * block_bytes + kStgBytes);

    const int warp = threadIdx.x >> 5;
    const int wg = threadIdx.x >> 7;
    const int total_tiles = p.num_z * p.m_tiles * p.n_tiles;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        if (p.nkb_aux) tma_prefetch_desc(&p.tmA2);
        if (p.f8) {
            tma_prefetch_desc(&p.tmA8);
            tma_prefetch_desc(&p.tmB8);
            if (p.nkb8_aux) tma_prefetch_desc(&p.tmA2_8);
        }
        for (int s = 0; s < p.num_stages; ++s) {
            mbar_init(&ctl->full[s], 1);
            mbar_init(&ctl->empty[s], 2);                                 // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer (warp 0, converged; the copies elected)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0) {
            RingPos ring{0, 0u};
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(p, tile);
                int aw0, ah0, an0;
                if (p.a_mode == 0) {
                    // 128 consecutive NHWC pixels: whole image rows (W <= 128) or a 128-pixel segment of one row (W a multiple of 128)
                    const int HW = p.conv_H * p.conv_W;
                    const int p0 = tc.mt * 128;
                    an0 = p0 / HW;
                    const int rem = p0 - an0 * HW;
                    ah0 = rem / p.conv_W;
                    aw0 = rem - ah0 * p.conv_W;
                } else {
                    aw0 = tc.mt * 128;
                    ah0 = 0;
                    an0 = tc.zb * p.a_n_per_zb + tc.zh * p.a_n_per_zh;
                }
                const int a_c_off = tc.zh * p.a_c_per_zh;
                const int b_k_off = p.b_k0 + tc.zh * p.b_k_per_zh;
                const int b_row = tc.nt * BN + tc.zh * p.b_row_per_zh;
                const int b_z = tc.zb * p.b_z_per_zb + tc.zh * p.b_z_per_zh;
                producer_tile(p, smem, ctl, ring, block_bytes, aw0, ah0, an0, a_c_off, b_k_off, b_row, b_z);
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers (warpgroups 1, 2: rows 0..63 / 64..127)
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = wg - 1;
        float* my_stg = stg + cw * 64 * kStgPitch;
        RingPos ring{0, 0u};
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const TileCoord tc = tile_coord(p, tile);
            float acc[BN / 2];
            mma_tile<BN>(p, smem, ctl, ring, block_bytes, cw, acc);
            epilogue_tile<BN>(p, my_stg, cw, tc, acc);
        }
    }
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

static int encode_map_typed(CUtensorMap* m, const void* ptr, int rank, const int64_t* dims, const int64_t* strides_bytes,
                            const int32_t* box, bool bytes8) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return -1;
    cuuint64_t gd[5];
    cuuint64_t gs[4];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) { gd[i] = (cuuint64_t)dims[i]; bx[i] = (cuuint32_t)box[i]; es[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gs[i] = (cuuint64_t)strides_bytes[i];
    CUresult r = fn(m, bytes8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[dsb] cuTensorMapEncodeTiled failed: %d (rank %d dims %lld %lld %lld %lld box %d %d %d %d)\n", (int)r, rank,
                (long long)dims[0], (long long)dims[1], (long long)dims[2], rank > 3 ? (long long)dims[3] : 0LL, box[0], box[1], box[2],
                rank > 3 ? box[3] : 0);
        return -2;
    }
    return 0;
}

// fp16 tensors (also used by attention.cu)
int encode_map(CUtensorMap* m, const void* ptr, int rank, const int64_t* dims, const int64_t* strides_bytes, const int32_t* box) {
    return encode_map_typed(m, ptr, rank, dims, strides_bytes, box, false);
}

OpCheck gemm_check(const ds_gemm_desc& d) {
    if (d.BN < 16 || d.BN > 256 || (d.BN % 16) != 0) return {-10, "gemm: BN"};
    // A conv box of whole image rows (a_box[1] == conv_W <= 128) holds 128 pixels only when conv_W divides 128
    if (d.a_box[0] != 64 || d.a_box[1] * d.a_box[2] * d.a_box[3] != 128) return {-11, "gemm: a_box"};
    if (d.npass != 1 && d.npass != 3) return {-12, "gemm: npass"};
    // cuTensorMapEncodeTiled limits of the A map (what its failed encode returns): extents <= 2^32, strides multiples of 16 below 2^40
    for (int i = 0; i < 4; ++i) if (d.a_dims[i] > (int64_t(1) << 32)) return {-1, "gemm: A tensor map"};
    for (int i = 0; i < 3; ++i) if (d.a_strides[i] % 16 || d.a_strides[i] >= (int64_t(1) << 40)) return {-1, "gemm: A tensor map"};
    if (d.st_unit != 0 && d.st_unit != 2 && d.st_unit != 4) return {-14, "gemm: st_unit"};
    if (d.f8 & 1) {
        // e4m3 correction passes: conv mode, one z slice, three passes, a lo plane; the byte planes have no phase channel bases
        if (d.a_mode != 0 || d.num_z != 1 || d.npass != 3 || d.a_plane_n <= 0) return {-16, "gemm: f8"};
        for (int t = 0; t < 9; ++t) if (d.tap_cb[t]) return {-16, "gemm: f8 with tap_cb"};
        // the e4m3 planes are read in 128-channel boxes whose zero fill the packed weight does not mirror
        if (d.a_dims[0] % 64 || d.a2_c % 64) return {-16, "gemm: f8 channel remainder"};
    }
    if (d.taps != 1 && d.taps != 9) return {-15, "gemm: taps"};
    // image rows wider than one M tile: the tile is a 128-pixel segment of one row
    if (d.a_mode == 0 && d.conv_W > 128 && (d.conv_W % 128 != 0 || d.a_box[1] != 128)) return {-13, "gemm: row segment"};
    // fused statistics: whole 32-row slabs (row validity is then warp-uniform), whole channel quads, one z slice, fp32 output
    if (d.st_quads && (d.num_z != 1 || d.m_valid % 32 != 0 || d.n_valid % (d.st_unit == 2 ? 2 : 4) != 0 || d.edm_out != 0))
        return {-14, "gemm: st_quads"};
    return {0, nullptr};
}

int gemm_build(const ds_gemm_desc* d, GemmKernelParams* kp) {
    memset(kp, 0, sizeof(*kp));
    if (const int rc = gemm_check(*d).rc) return rc;
    if (encode_map(&kp->tmA, d->a_ptr, 4, d->a_dims, d->a_strides, d->a_box)) return -1;
    if (d->a2_c > 0) {
        int64_t dims2[4] = {d->a2_c, d->a_dims[1], d->a_dims[2], d->a_dims[3]};
        // aux tensor shares (w,h,n) extents with A; strides follow its own channel count
        int64_t st2[3] = {d->a2_c * 2, d->a2_c * 2 * d->a_dims[1], d->a2_c * 2 * d->a_dims[1] * d->a_dims[2]};
        if (encode_map(&kp->tmA2, d->a2_ptr, 4, dims2, st2, d->a_box)) return -2;
    }
    int32_t bbox[3] = {64, d->BN, 1};
    if (encode_map(&kp->tmB, d->b_ptr, 3, d->b_dims, d->b_strides, bbox)) return -3;

    kp->BN = d->BN; kp->m_tiles = d->m_tiles; kp->n_tiles = d->n_tiles; kp->num_z = d->num_z; kp->nh = d->nh > 0 ? d->nh : 1;
    kp->taps = d->taps; kp->cpb = d->cpb; kp->nkb_main = d->taps * d->cpb; kp->nkb_aux = d->a2_c > 0 ? (int)((d->a2_c + 63) / 64) : 0;
    kp->npass = d->npass; kp->a_mode = d->a_mode; kp->conv_H = d->conv_H; kp->conv_W = d->conv_W;
    kp->a_plane_n = d->a_plane_n; kp->a2_plane_n = d->a2_plane_n; kp->b_plane_batch = d->b_plane_batch;
    kp->a_c_per_zh = d->a_c_per_zh; kp->a_n_per_zb = d->a_n_per_zb; kp->a_n_per_zh = d->a_n_per_zh;
    kp->b_k0 = d->b_k0; kp->b_k_per_zh = d->b_k_per_zh; kp->b_row_per_zh = d->b_row_per_zh;
    kp->b_z_per_zb = d->b_z_per_zb; kp->b_z_per_zh = d->b_z_per_zh;
    kp->m_valid = d->m_valid; kp->n_valid = d->n_valid;
    kp->out_f32 = d->out_f32; kp->out_h16 = reinterpret_cast<__half*>(d->out_h16);
    kp->o_zb = d->o_zb; kp->o_zh = d->o_zh; kp->ldo = d->ldo; kp->o_plane = d->o_plane;
    kp->bias_n = d->bias_n; kp->bias_m = d->bias_m; kp->rowvec = d->rowvec; kp->rowvec_stride = d->rowvec_stride;
    kp->rows_per_sample = d->rows_per_sample > 0 ? d->rows_per_sample : 1;
    kp->residual = d->residual; kp->ldr = d->ldr; kp->scale = d->scale;
    kp->edm_out = d->edm_out; kp->edm_x = d->edm_x; kp->edm_coef = d->edm_coef; kp->edm_coef_stride = d->edm_coef_stride;
    kp->edm_C = d->edm_C; kp->edm_D = d->edm_D;
    kp->st_quads = d->st_quads;
    kp->st_unit = d->st_unit == 2 ? 2 : 4;
    kp->acc_scale = d->acc_scale == 0.f ? 1.f : d->acc_scale;
    kp->relu = d->relu != 0;
    if (d->f8 & 1) {
        // e4m3 correction passes: byte planes behind the fp16 plane of each operand (layout: csrc/ops.h)
        const int64_t C = d->a_dims[0], Wd = d->a_dims[1], Hd = d->a_dims[2], Bn = d->a_plane_n;
        const int32_t box8[4] = {128, d->a_box[1], d->a_box[2], d->a_box[3]};
        const int64_t dims8[4] = {C, Wd, Hd, 2 * Bn};
        const int64_t st8[3] = {C, Wd * C, Hd * Wd * C};
        const char* a8 = static_cast<const char*>(d->a_ptr) + Bn * Hd * Wd * C * 2;
        if (encode_map_typed(&kp->tmA8, a8, 4, dims8, st8, box8, true)) return -17;
        kp->f8 = 1;
        kp->f8_last_steps = (d->cpb & 1) ? 2 : 4;
        kp->a8_plane_n = (int)Bn;
        kp->cpb8 = (d->cpb + 1) / 2;
        kp->nkb8_main = d->taps * kp->cpb8;
        kp->nkb8_aux = 0;
        if (d->a2_c > 0) {
            const int64_t C2 = d->a2_c;
            const int64_t dims28[4] = {C2, Wd, Hd, 2 * Bn};
            const int64_t st28[3] = {C2, Wd * C2, Hd * Wd * C2};
            const char* a28 = static_cast<const char*>(d->a2_ptr) + Bn * Hd * Wd * C2 * 2;
            if (encode_map_typed(&kp->tmA2_8, a28, 4, dims28, st28, box8, true)) return -18;
            kp->nkb8_aux = (int)((C2 + 127) / 128);
        }
        const int64_t ktot8 = (int64_t)(kp->nkb8_main + kp->nkb8_aux) * 128;
        const int64_t rows = d->b_dims[1];
        const int64_t bd8[3] = {ktot8, rows, 2};
        const int64_t bs8[2] = {ktot8, rows * ktot8};
        const int32_t bbox8[3] = {128, d->BN, 1};
        const char* b8 = static_cast<const char*>(d->b_ptr) + rows * d->b_dims[0] * 2;
        if (encode_map_typed(&kp->tmB8, b8, 3, bd8, bs8, bbox8, true)) return -19;
    }
    for (int t = 0; t < 9; ++t) { kp->tap_dh[t] = d->tap_dh[t]; kp->tap_dw[t] = d->tap_dw[t]; kp->tap_cb[t] = d->tap_cb[t]; }
    const int stage_bytes = kATileBytes + d->BN * 128;
    int ns = (kSmemLimit - 1024 - kStgBytes - (int)sizeof(SmemCtl)) / stage_bytes;
    if (ns > kMaxStages) ns = kMaxStages;
    kp->num_stages = ns;
    return 0;
}

size_t gemm_params_size() { return sizeof(GemmKernelParams); }
void gemm_patch_edm(GemmKernelParams* kp, const float* x, float* D) { kp->edm_x = x; kp->edm_D = D; }

// cudaFuncSetAttribute is per device: one process may drive several GPUs (tests, notebooks), so the opt-in shared-memory size is set once per
// (device, N tile) and the SM count is kept per device.
static int g_num_sms[64] = {};
static bool g_attr_set[64][17] = {};

template <int BN>
static int gemm_launch(const GemmKernelParams* kp, cudaStream_t stream, int slot) {
    if (!g_attr_set[slot][BN / 16]) {
        if (cudaFuncSetAttribute(gemm_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) != cudaSuccess) return -20;
        g_attr_set[slot][BN / 16] = true;
    }
    const size_t smem = (size_t)kp->num_stages * (kATileBytes + BN * 128) + kStgBytes + sizeof(SmemCtl) + 1024;
    const int tiles = kp->num_z * kp->m_tiles * kp->n_tiles;
    const int grid = tiles < g_num_sms[slot] ? tiles : g_num_sms[slot];
    if (grid <= 0) return 0;
    gemm_tc_kernel<BN><<<grid, kThreads, smem, stream>>>(*kp);
    return cudaGetLastError() == cudaSuccess ? 0 : -21;
}

int gemm_run(const GemmKernelParams* kp, cudaStream_t stream) {
    int dev = 0;
    cudaGetDevice(&dev);
    const int slot = (dev < 0 || dev >= 64) ? 0 : dev;
    if (!g_num_sms[slot]) cudaDeviceGetAttribute(&g_num_sms[slot], cudaDevAttrMultiProcessorCount, slot);
    switch (kp->BN / 16) {
        case 1: return gemm_launch<16>(kp, stream, slot);
        case 2: return gemm_launch<32>(kp, stream, slot);
        case 3: return gemm_launch<48>(kp, stream, slot);
        case 4: return gemm_launch<64>(kp, stream, slot);
        case 5: return gemm_launch<80>(kp, stream, slot);
        case 6: return gemm_launch<96>(kp, stream, slot);
        case 7: return gemm_launch<112>(kp, stream, slot);
        case 8: return gemm_launch<128>(kp, stream, slot);
        case 9: return gemm_launch<144>(kp, stream, slot);
        case 10: return gemm_launch<160>(kp, stream, slot);
        case 11: return gemm_launch<176>(kp, stream, slot);
        case 12: return gemm_launch<192>(kp, stream, slot);
        case 13: return gemm_launch<208>(kp, stream, slot);
        case 14: return gemm_launch<224>(kp, stream, slot);
        case 15: return gemm_launch<240>(kp, stream, slot);
        case 16: return gemm_launch<256>(kp, stream, slot);
        default: return -10;
    }
}

}  // namespace dsb

extern "C" int ds_gemm_launch(const ds_gemm_desc* d, cudaStream_t stream) {
    dsb::GemmKernelParams kp;
    int rc = dsb::gemm_build(d, &kp);
    if (rc) return rc;
    return dsb::gemm_run(&kp, stream);
}

extern "C" int ds_gemm_config(const void* desc, int* info) {
    dsb::GemmKernelParams kp;
    int rc = dsb::gemm_build(static_cast<const ds_gemm_desc*>(desc), &kp);
    if (rc) return rc;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -20;
    const int tiles = kp.num_z * kp.m_tiles * kp.n_tiles;
    info[0] = kp.num_stages;
    info[1] = tiles < sms ? tiles : sms;
    return 0;
}

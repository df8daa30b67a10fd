// Internal op descriptors shared by the kernels (csrc/*.cu) and the plan executor (engine.cu).
// Plain C structs: the Python plan compiler mirrors them with ctypes (diff-sampler_b200/_cstructs.py).
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#ifdef __cplusplus
extern "C" {
#endif

// ---------------------------------------------------------------------------------------------
// Tensor-core GEMM / implicit-GEMM convolution (wgmma, fp16 operands, fp32 accumulate in registers).
//   D[m][n] = sum_k A[m][k] * B[n][k]     (both operands K-major)
// A is described as a 4-D tensor (c, w, h, n) of fp16 so that one 128-row M tile is a TMA box
// (64 c, bw, bh, bn) with bw*bh*bn == 128:
//   a_mode 0 (conv):  rows are NHWC pixels; a 3x3 tap is a shifted box, halo zero-filled by TMA.
//   a_mode 1 (rows):  plain row-major matrices, optionally batched over z = (zb, zh).
// B is a 3-D tensor (k, row, batch).  Split precision: npass == 3 accumulates
//   A_lo*B_hi + A_hi*B_lo + A_hi*B_hi (the small corrections first), with the 'lo' planes found at a_plane_n / b_plane_batch.
//
// f8 == 1 ("fp16f8", conv mode only): the two correction products run as e4m3 MMAs (kind::f8f6f4, twice the fp16 rate, 128
// channels per K block).  Operand layout (all scales are powers of two, so the fp16 roundings are those of the unscaled values):
//   A buffer  = [fp16 (v * 2^DS_F8_SH_A16)] [e4m3 ((v - hi) * 2^DS_F8_SH_LO8)] [e4m3 (hi * 2^DS_F8_SH_HI8)]   (2 + 1 + 1 bytes/elem,
//               each plane [Bn][H][W][C]; written by ds_gn_apply with fmt == 1), same for the aux (skip) operand;
//   B buffer  = [fp16 (w * 2^b)][cout_pad][ktot] then [2][cout_pad][ktot8] e4m3: (w_hi * 2^b1), (w_lo * 2^b2), K padded per tap to a
//               multiple of 128, with b + A16 == b1 + LO8 == b2 + HI8 == S  (gemm_desc.pack_conv_weight_f8);
//   the accumulator then holds 2^S * result and the epilogue multiplies by acc_scale = 2^-S before bias / residual.
// The e4m3 blocks are issued first so that they accumulate among themselves before the large fp16 term arrives.
enum { DS_F8_SH_A16 = 6, DS_F8_SH_LO8 = 13, DS_F8_SH_HI8 = 2 };
typedef struct ds_gemm_desc {
    // A operand
    const void* a_ptr;
    int64_t a_dims[4];      // elements: (c, w, h, n)   (n already includes the lo plane if present)
    int64_t a_strides[3];   // bytes: stride of w, h, n
    int32_t a_box[4];       // (64, bw, bh, bn)
    int32_t a_plane_n;      // n-offset of the lo plane
    // optional aux A operand (1x1 skip input appended along K); same (w,h,n) geometry, own channel count
    const void* a2_ptr;
    int64_t a2_c;           // channels of the aux tensor (multiple of 64); 0 = none
    int32_t a2_plane_n;
    int32_t nkb_aux;        // a2_c / 64
    // B operand
    const void* b_ptr;
    int64_t b_dims[3];      // elements: (k, row, batch)
    int64_t b_strides[2];   // bytes: stride of row, batch
    int32_t b_plane_batch;  // batch-offset of the lo plane
    // tiling
    int32_t BN;             // N tile, multiple of 16, <= 256
    int32_t m_tiles, n_tiles, num_z, nh;   // z = zb * nh + zh
    int32_t taps;           // 1 or 9
    int32_t cpb;            // 64-channel blocks per tap
    int32_t npass;          // 1 or 3
    int32_t a_mode;         // 0 conv, 1 rows
    int32_t conv_H, conv_W;
    // z -> operand coordinates
    int32_t a_c_per_zh, a_n_per_zb, a_n_per_zh;
    int32_t b_k0, b_k_per_zh, b_row_per_zh, b_z_per_zb, b_z_per_zh;
    // output
    int32_t m_valid;        // valid rows per z
    int32_t n_valid;        // valid columns
    float* out_f32;         // may be NULL
    void* out_h16;          // may be NULL (fp16 hi plane; lo plane at +o_plane elements if o_plane != 0)
    int64_t o_zb, o_zh;     // element offsets per zb / zh
    int64_t ldo;            // row pitch (elements)
    int64_t o_plane;
    // epilogue:  v = (acc + bias_n[col] + bias_m[row] + rowvec[sample][col] + residual[row][col]) * scale
    const float* bias_n;
    const float* bias_m;
    const float* rowvec;
    int64_t rowvec_stride;  // elements between samples (0 = broadcast)
    int32_t rows_per_sample;
    int32_t f8;             // 1: fp8 correction passes (see above); requires a_mode == 0, num_z == 1, npass == 3, tap_cb == 0
    const float* residual;
    int64_t ldr;
    float scale;
    // EDM output fold (final conv): D[n][c][hw] = cskip[n]*x[n][c][hw] + cout[n]*v   (NCHW fp32)
    int32_t edm_out;        // 1: EDM combine below; 2: plain NCHW fp32 write of the epilogue value (LDM eps output)
    const float* edm_x;
    const float* edm_coef;  // [nsig][4] = (c_skip, c_out, c_in, c_noise)
    int32_t edm_coef_stride;// 0 (one sigma) or 4 (per-sample)
    int32_t edm_C;
    float* edm_D;
    // fused GroupNorm statistics of the fp32 output (conv mode, m_valid % 32 == 0, n_valid % 4 == 0): the epilogue stores, per
    // 32-row slab and per channel QUAD (4 consecutive channels), the partial {sum, sumsq}:
    //   st_quads[((row/32) * (n_valid/4) + channel/4) * 2 + {0,1}]
    // Plain coalesced stores, no atomics, independent of how consumers group the channels (every GroupNorm here has groups that
    // are unions of quads); ds_gn_finalize adds the slabs of a sample and the quads of a group into the fp64 sums gn_apply reads.
    float* st_quads;
    // conv taps: K block `tap` reads the pixel box shifted by (tap_dh, tap_dw) from channel base tap_cb.  A 3x3 stride-1 conv uses
    // (kh-1, kw-1, 0); a 3x3 stride-2 conv over a space-to-depth input [B][H/2][W/2][4C] uses shifts in {-1,0} and the phase's
    // channel base (LDM Downsample, openaimodel.py:134-160).
    int32_t tap_dh[9];
    int32_t tap_dw[9];
    int32_t tap_cb[9];
    float acc_scale;        // accumulator pre-scale (0 is read as 1); 2^-S in f8 mode
    int32_t st_unit;        // channels per statistics partial of st_quads: 4 (default; 0 is read as 4) or 2 (channel PAIRS, for consumers whose
                            // GroupNorm groups are even but not multiples of 4 channels: the 6-, 18-, 30-channel groups of the ADM net);
                            // layout st_quads[((row/32) * (n_valid/unit) + channel/unit) * 2 + {0,1}]
    int32_t relu;           // 1: v = max(v, 0) after bias / residual / scale, before the statistics and every store (Inception's BasicConv2d)
} ds_gemm_desc;

int ds_gemm_launch(const ds_gemm_desc* d, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// GroupNorm statistics over NHWC fp32 (optionally the virtual concat [src0 | src1] along C).
// Accumulates per-(sample, group) double sums {sum, sumsq}; the buffer must be zeroed beforehand.
// Reference: networks_edm.py:96-98 (torch.nn.functional.group_norm).
typedef struct ds_gn_stats_desc {
    const float* src0;
    const float* src1;      // NULL if C1 == 0
    int32_t C0, C1;
    int32_t HW;             // pixels per sample
    int32_t B;
    int32_t groups;
    int32_t pad0;
    double* sums;           // [B][groups][2]
} ds_gn_stats_desc;

// GroupNorm apply (+ adaptive scale/shift) (+ SiLU) (+ 2x resample) -> fp16 hi/lo planes, NHWC.
// Also optionally emits the raw (un-normalised) input, resampled the same way, as fp16 planes
// (operand of the fused 1x1 skip projection) and/or as fp32 (weight-less skip of ADM up/down blocks).
// Reference: networks_edm.py:160 silu(norm0(x)), :165 addcmul(shift, norm1(x), scale+1), :167, :74-77 resample.
typedef struct ds_gn_apply_desc {
    const float* src0;
    const float* src1;
    int32_t C0, C1;
    int32_t H, W;           // input resolution
    int32_t B;
    int32_t groups;
    const double* sums;     // NULL -> no normalisation (raw pass-through only)
    const float* gamma;
    const float* beta;
    float eps;
    int32_t silu;
    const float* ada;       // adaptive [nE][2*C]: scale = ada[c], shift = ada[C + c]; NULL if unused
    int64_t ada_stride;     // elements between samples (0 = broadcast)
    int32_t resample;       // 0 none, 1 down (2x2 mean), 2 up (nearest x2), 3 space-to-depth (out [B][H/2][W/2][4C], phase-major)
    int32_t nplanes;        // 1 or 2 (hi / hi+lo)
    void* out_act;          // fp16 [nplanes][B][Ho][Wo][C]; may be NULL
    void* out_raw;          // fp16 planes of the raw input; may be NULL
    float* out_raw_f32;     // fp32 raw input at output resolution; may be NULL
    int32_t fmt;            // 0: fp16 hi/lo planes.  1: operand layout of an f8 GEMM (ds_gemm_desc.f8), for out_act and out_raw
    int32_t pad0;           // resample 3: channel pitch of each phase (0 = C); channels C .. pad0 of a phase are written as zeros
    // Precomputed per-(sample, channel) coefficients [B][C][2] = {a, b} with y = x * a + b  (a = rstd * gamma * (1 + ada_scale),
    // b = beta * (1 + ada_scale) + ada_shift - mean * a), written by ds_gn_finalize.  When set (resample == 0 only) the kernel reads
    // them instead of deriving them from `sums` in an fp64 prologue per thread, and runs the persistent, evenly split variant.
    const float* coef;
} ds_gn_apply_desc;

// GroupNorm statistics from the quad partials written by the producing GEMM epilogues (ds_gemm_desc.st_quads) of the one or two
// (virtually concatenated) source tensors: sums[n][g] = {sum, sumsq} (fp64) over the sample's slabs and the group's quads.
// Replaces the ds_gn_stats pass over the tensor itself (reads B*HW*C/64 floats instead of B*HW*C).
typedef struct ds_gn_finalize_desc {
    const float* quads0;    // [B * slabs_per_sample][C0/4][2]
    const float* quads1;    // [B * slabs_per_sample][C1/4][2]; NULL when C1 == 0
    int32_t C0, C1;
    int32_t slabs_per_sample;   // H*W / 32
    int32_t B;
    int32_t groups;         // (C0 + C1) / groups must be a multiple of the partial units (when quads0 != NULL)
    int32_t unit0;          // channels per partial of quads0: 4 (0 is read as 4) or 2 (ds_gemm_desc.st_unit of its producer)
    double* sums;           // [B][groups][2]: overwritten from the quads; with quads0 == NULL it is the INPUT (written by ds_gn_stats)
    // optional second product (coef != NULL): the per-(sample, channel) coefficients ds_gn_apply_desc.coef describes
    const float* gamma;
    const float* beta;
    const float* ada;       // adaptive [nE][2*C] (scale | shift), NULL if unused
    int64_t ada_stride;
    float eps;
    int32_t HW;             // pixels per sample (statistics count = HW * C / groups)
    float* coef;            // [B][C0 + C1][2]
    int32_t unit1;          // channels per partial of quads1 (as unit0)
    int32_t pad1;
} ds_gn_finalize_desc;

// Fused softmax attention (attention.cu): out[b][l][h*hd + c] = sum_k softmax_k(scale * q_l . k_k) v_k[c], hd = the head width (pad0).
// All operands are fp16 hi/lo planes, plane p of a [B]-batched tensor at batch index p*B + b.
// Reference: networks_edm.py:105-118, :174-178; ldm/modules/attention.py:152-196.
typedef struct ds_attn_desc {
    const void* q;          // [2][B][L][q_pitch]; head h reads channels q_c0 + h*hd ..
    const void* k;          // [2][B][Lk][k_pitch]; head h reads channels k_c0 + h*hd ..
    const void* vt;         // [2][B][nh*hd][vt_pitch]: V transposed, keys contiguous (Lk <= vt_pitch valid)
    void* out;              // [2][B][L][o_pitch]
    int32_t B, nh, L, Lk;
    int32_t q_pitch, q_c0, k_pitch, k_c0, vt_pitch, o_pitch;
    int32_t nplanes;        // must be 2
    float scale;            // > 0
    int32_t causal;         // 1: query l attends to keys <= l only (CLIP text encoder; L == Lk)
    int32_t pad0;           // head width hd: 0 or 64; 32 (heads in pairs: nh even; q/k/out channels and V^T rows at nh*32); or 72 .. 128, a
                            // multiple of 8 (attn_wide_kernel: unpadded heads, no causal mask)
} ds_attn_desc;

// Row softmax: P = softmax(S) over the last dim, fp32 in, fp16 hi/lo planes out. Reference: networks_edm.py:108.
typedef struct ds_softmax_desc {
    const float* S;
    void* P;
    int64_t rows;
    int32_t L;              // valid row length
    int32_t nplanes;
    int32_t pitch_in;       // elements between rows of S (0 -> L)
    int32_t pitch_out;      // elements between rows of P (0 -> L)
} ds_softmax_desc;

// sigma -> EDM coefficients + positional embedding. Reference: networks_edm.py:488-491, :192-198, :315.
typedef struct ds_posemb_desc {
    const float* sigma;     // device, nsig values
    int32_t nsig;
    int32_t num_channels;   // embedding width
    int32_t endpoint;       // PositionalEmbedding(endpoint=...)
    int32_t swap_sincos;    // SongUNet swaps to [sin, cos]
    float sigma_data;
    int32_t mode;           // 0: EDM (sigma -> coefficients + embedding of c_noise).  1: LDM timestep_embedding (util.py:151-171):
                            //    `sigma` holds the timesteps, emb = [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / half); coef untouched
    float* coef;            // [nsig][4] = (c_skip, c_out, c_in, c_noise)
    float* emb;             // [nsig][num_channels]
    float noise_scale;      // mode 0: the embedding argument is noise_scale * c_noise (Consistency Models: 1000); 0 means 1
    int32_t pad0;
} ds_posemb_desc;

// Small dense layer on CUDA cores (embedding MLP and all per-block affines in one launch):
//   out[n][o] = act( sum_i in_scale * in[n][i] * W[o][i] + b[o] + add[n][o] )
typedef struct ds_linear_desc {
    const float* in;
    int64_t in_stride;      // elements between rows of `in` (0 = single row broadcast to all n)
    const float* W;         // [out_f][in_f]
    const float* b;         // may be NULL
    const float* add;       // may be NULL
    int64_t add_stride;
    float* out;             // [n_rows][out_f]
    int32_t n_rows, in_f, out_f;
    int32_t act;            // 0 none, 1 silu
    float in_scale;
    int32_t pad0;
} ds_linear_desc;

// Network input: x (NCHW fp32) * c_in[n] -> fp16 planes NHWC with channels zero-padded to 64.
// Reference: networks_edm.py:493 (c_in * x).
// With `codebook` set (first stage of a VQ autoencoder, VQModelInterface.decode -> VectorQuantizer2, autoencoder.py:274-282), each
// pixel's C-vector v = c_in * x is first replaced by its nearest codebook row: argmin_j sum_c (v_c - e_jc)^2 in fp32, ties to the lowest
// j as torch.argmin.  C <= 8 then.
typedef struct ds_prep_input_desc {
    const float* x;
    const float* coef;      // from ds_posemb_desc
    int32_t coef_stride;    // 0 or 4
    int32_t B, C, HW;
    int32_t nplanes;
    int32_t x_batch;        // 0 or B: batch of x; sample n reads x[n % x_batch] (classifier-free guidance evaluates [x, x])
    void* out;              // fp16 [nplanes][B][HW][64]
    const float* codebook;  // [n_embed][C] fp32, or NULL (no quantization)
    int32_t* idx;           // [B][HW] chosen codebook rows (debug read-out), or NULL
    int32_t n_embed;
    int32_t pad0;
} ds_prep_input_desc;

// LayerNorm over the last dim of fp32 [rows][C] -> fp16 hi/lo planes (LDM BasicTransformerBlock.norm1/2/3, attention.py:203-215).
typedef struct ds_layernorm_desc {
    const float* src;
    const float* gamma;
    const float* beta;
    void* out;              // fp16 [nplanes][rows][C]
    int64_t rows;
    int32_t C;
    int32_t nplanes;
    float eps;
    int32_t fmt;            // 0: fp16 hi/lo planes.  1: operand image of an f8 GEMM (ds_gemm_desc.f8).  2: fp32 [rows][C] (final LayerNorm of
                            // the CLIP text encoder: the output IS the conditioning tensor)
} ds_layernorm_desc;

// GEGLU gate: out = x[:, :I] * gelu(x[:, I:]) on fp32 [rows][2I] -> fp16 hi/lo planes [rows][I]  (attention.py:42-44, exact erf GELU).
typedef struct ds_geglu_desc {
    const float* src;
    void* out;
    int64_t rows;
    int32_t I;
    int32_t nplanes;
    int32_t fmt;            // as ds_layernorm_desc.fmt (0 or 1)
    int32_t mode;           // 0: GEGLU (above).  1: quick-GELU, out = x * sigmoid(1.702 x) on fp32 [rows][I] (CLIP MLP, modeling_clip.py quick_gelu).
                            // 2: exact erf GELU, out = gelu(x) on fp32 [rows][I] (open_clip ViT-g-14 MLP, nn.GELU()).  Modes 1 and 2 take fmt 0 only.
} ds_geglu_desc;

// Token + position embedding (CLIPTextEmbeddings.forward): out[row][c] = tok[ids[row]][c] + pos[row % T][c], fp32.
typedef struct ds_embed_desc {
    const int32_t* ids;     // [rows] token ids
    const float* tok;       // [vocab][C]
    const float* pos;       // [T][C]
    float* out;             // [rows][C]
    int64_t rows;
    int32_t T, C;
    int32_t vocab;
    int32_t pad0;
} ds_embed_desc;

// Channel mean of an NHWC fp32 tensor (AMED bottleneck read-out, solvers_amed.py:24,27).
typedef struct ds_chanmean_desc {
    const float* src;
    float* out;             // [rows]
    int64_t rows;
    int32_t C;
    int32_t pad0;
} ds_chanmean_desc;

// Fused solver update.  One pass over the state:
//   m0   = D | clamp(D,-s,s)/s | (xs - D)/t | xs/t | (none)          (the "model output" entry the solver stores)
//   out  = cx*xb + c0*m0 + c1*h1 + c2*h2 + c3*h3 + c4*h4
// Covers Euler/Heun/DPM-2/iPNDM(_v)/DEIS/DPM-Solver++/UniPC/AMED updates (reference: solvers.py:80-81,
// :163-168, :252-258, :346-352, :451-477, :576-585; solver_utils.py:102-163, :250-285), see SURVEY.md App. B.
enum { DS_M_X0 = 0, DS_M_EPS = 1, DS_M_DIV = 2, DS_M_NONE = 3 };
typedef struct ds_update_desc {
    float* out_x;
    float* out_m;           // may be NULL
    const float* xb;
    const float* xs;        // NULL -> xb
    const float* D;         // NULL for DS_M_DIV / DS_M_NONE
    const float* h[4];
    const float* thr;       // [B] per-sample threshold s for DS_M_X0 (dynamic thresholding); NULL = none
    const float* coef_dev;  // optional per-sample coefficients, layout [6][B] (cx, c0, c1..c4)
    const float* t_dev;     // optional per-sample divisor [B]
    float coef[6];
    float t;
    int32_t mode;
    int32_t nhist;          // number of history buffers used (0..4)
    int32_t B;
    int64_t n_per_sample;
    // optional fused image epilogue of the LAST step (sample.py:311): out_u8[n][hw][c] = uint8(clip(out * 127.5 + 128, 0, 255)),
    // NCHW fp32 -> NHWC uint8 in the same pass (n_per_sample == u8_C * u8_HW, u8_HW % 4 == 0)
    unsigned char* out_u8;
    int32_t u8_C, u8_HW;
} ds_update_desc;

// Per-sample dynamic threshold s = max(quantile(|x0|, 0.995), 1)  (solver_utils.py:77-86), exact radix select.
typedef struct ds_threshold_desc {
    const float* x0;
    float* thr;             // [B]
    int32_t B;
    int32_t row_len;
    float q;                // 0.995
    float floor_val;        // 1.0
} ds_threshold_desc;

// GITS cost-matrix reductions (gits-main/gits_utils.py:115-132): for every teacher pair i < j and sample b, with
//   x_ij = traj[i] + (t[j] - t[i]) * eps[i]      (a single Euler jump i -> j)
// accumulate  out[i][j][b] = { sum|x_ij - traj[j]|, sum (x_ij - traj[j])^2, sum (c - x_ij)^2, sum (c - x_ij)(c - b0) }
// where b0 = traj[0], c = traj[N-1] (the chord used by cal_deviation, :237-255).  fp64 accumulators.
typedef struct ds_gits_cost_desc {
    const float* traj;      // [N][B][n]
    const float* eps;       // [N-1][B][n]
    const float* t;         // [N] device
    double* out;            // [N][N][B][4]
    int32_t N, B;
    int64_t n;
} ds_gits_cost_desc;

int ds_gits_cost_launch(const ds_gits_cost_desc* d, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Optimal (empirical-Bayes) denoiser over a dataset y_0..y_{N-1} of D = C*H*W values each (optimal.cu; numerics in DESIGN.md 4.9):
//   D*(x; sigma) = sum_i softmax_i(u_i / sigma^2) y_i,   u_i = x.y_i - 0.5 ||y_i||^2.
// The two contractions run on the GEMM kernel (rows mode); these ops prepare and finish them.
//
// x [B][D] fp32 -> fp16 hi/lo planes [2][B][pitch] (columns D..pitch-1 zero) and ||x||^2 in fp64.
typedef struct ds_opt_prep_desc {
    const float* x;
    void* planes;
    double* xn2;            // [B]
    int32_t B, D;
    int32_t pitch, pad0;
} ds_opt_prep_desc;

// Row softmax of the logits GEMM.  part[s][b][i] (s < nslice, row pitch ldp) are the fp32 partials of x_b.y_i over channel slice s;
// they are added in order s = 0, 1, ... in fp64, 0.5 ||y_i||^2 is subtracted, and u_i is kept in fp32 in slice 0.  Rows whose logit
// error bound E_row exceeds DS_OPT_TAU and whose band (keys within 2 E_row + DS_OPT_BAND_NATS of the row maximum) holds at most
// DS_OPT_CAP keys are rescored from exact fp32 distances; every other key then has weight 0.
// P = 2^DS_OPT_P_SHIFT * softmax, as fp16 hi/lo planes [2][B][ldP] (columns N..ldP-1 zero).
// status[b]: DS_OPT_PLAIN, DS_OPT_RESCORED, or DS_OPT_UNREFINED (E_row > tau but the band exceeded the cap).
enum { DS_OPT_CAP = 1024, DS_OPT_P_SHIFT = 15, DS_OPT_BAND_NATS = 40 };
#define DS_OPT_TAU 0.01f
#define DS_OPT_EPS 7.62939453125e-06    /* 2^-17: relative error of u_i per ||x|| ||y_i|| (DESIGN.md 4.9) */
enum { DS_OPT_PLAIN = 0, DS_OPT_RESCORED = 1, DS_OPT_UNREFINED = 2 };
typedef struct ds_opt_softmax_desc {
    float* part;
    const double* hy2;      // [N] 0.5 ||y_i||^2 (fp64)
    const double* xn2;      // [B] ||x_b||^2 (ds_opt_prep_desc)
    const float* sigma;     // [nsig], nsig in {1, B}
    const float* x;         // [B][D] fp32
    const float* y;         // [N][D] fp32 dataset
    void* P;
    int32_t* status;        // [B], may be NULL
    int64_t ldp, ldP;
    int32_t B, N, D, nslice;
    int32_t nsig;
    float ymax;             // max_i ||y_i||
} ds_opt_softmax_desc;

// out[r][c] = scale * sum_{s < nsplit} part[s][r][c], s in increasing order: the split-K partials of the weighted-sum GEMM, rows of
// pitch ld (a multiple of 4, for the GEMM epilogue's vector stores), into the dense [rows][cols] output (NCHW fp32).
typedef struct ds_opt_reduce_desc {
    const float* part;
    float* out;
    int64_t rows;
    int32_t cols, ld;
    int32_t nsplit;
    float scale;
} ds_opt_reduce_desc;

// k nearest dataset rows of each x_b (k <= DS_KNN_MAX): candidates by u_i from the logits GEMM partials (as ds_opt_softmax_desc),
// widened by the GEMM error bound, then exact distances ||x_b - y_i|| (fp32 differences, fp64 sums), ascending, ties to the lower
// index.  dist [B][k] fp32, idx [B][k] int32.
enum { DS_KNN_MAX = 64, DS_KNN_CAND = 256 };
typedef struct ds_opt_knn_desc {
    float* part;
    const double* hy2;
    const double* xn2;
    const float* x;
    const float* y;
    float* dist;
    int32_t* idx;
    int64_t ldp;
    int32_t B, N, D, nslice;
    int32_t k;
    float ymax;
} ds_opt_knn_desc;

// ---------------------------------------------------------------------------------------------
// Inception-v3 FID feature extractor (inception.cu; the TF graph `inception-2015-12-05` as DESIGN.md 4.10 states it).  Every
// convolution runs on the GEMM kernel (rows mode, relu = 1); these ops feed it and pool between its launches.
//
// Input stage: uint8 images (element (n, c, y, x) at n*sn + c*sc + y*sy + x*sx, so NCHW and the NHWC-permuted view both fit) ->
// TF1 legacy ResizeBilinear to Ho x Wo (source (i H / Ho, j W / Wo), neighbours floor and floor + 1 clamped to H-1 / W-1, no half-pixel
// centres, no antialiasing) -> (v - 128) / 128 as fp32 NHWC [B][Ho][Wo][C].  Coordinates and weights in fp64.
typedef struct ds_img_input_desc {
    const unsigned char* src;
    float* out;
    int64_t sn, sc, sy, sx;     // element strides of src
    int32_t B, C, H, W;
    int32_t Ho, Wo;
} ds_img_input_desc;

// im2col: fp32 NHWC [B][H][W][src_pitch], channels src_c0 .. src_c0 + C -> fp16 planes [nplanes][B*Ho*Wo][K64] (hi, then lo at
// + B*Ho*Wo*K64 elements), row (n, oy, ox), column (i*kw + j)*C + c = src(n, oy*sh - ph + i, ox*sw - pw + j, c), 0 outside the image,
// and columns kh*kw*C .. K64 - 1 zero.  Ho = (H + 2 ph - kh) / sh + 1, Wo likewise.
typedef struct ds_im2col_desc {
    const float* src;
    void* out;
    int32_t B, H, W, C;
    int32_t src_pitch, src_c0;
    int32_t kh, kw, sh, sw, ph, pw;
    int32_t K64;
    int32_t nplanes;        // 1 or 2
} ds_im2col_desc;

// Pooling over fp32 NHWC [B][H][W][src_pitch], channels src_c0 .. src_c0 + C, k x k window, stride, pad:
//   mode 0 max (padding never wins), 1 average over the window's in-image pixels only (count_include_pad=False),
//   2 global mean over H x W (k, stride, pad unused): out_f32 [B][out_pitch] at channel out_c0.
// Modes 0 / 1 write fp32 [B][Ho][Wo][out_pitch] and / or fp16 planes [nplanes][B*Ho*Wo][out_pitch] (lo at + B*Ho*Wo*out_pitch), both
// at channel out_c0; Ho = (H + 2 pad - k) / stride + 1.
enum { DS_POOL_MAX = 0, DS_POOL_AVG = 1, DS_POOL_MEAN = 2 };
typedef struct ds_pool_desc {
    const float* src;
    float* out_f32;         // may be NULL (modes 0 / 1)
    void* out_h16;          // may be NULL; modes 0 / 1 only
    int32_t B, H, W, C;
    int32_t src_pitch, src_c0;
    int32_t out_pitch, out_c0;
    int32_t k, stride, pad;
    int32_t mode;
    int32_t nplanes;        // 1 or 2 (out_h16)
    int32_t pad0;
} ds_pool_desc;

// ---------------------------------------------------------------------------------------------
// CLIP score (clip.cu; open_clip ViT-g-14 as DESIGN.md 4.11 states it).  The towers run on the GEMM, LayerNorm, GELU and attention ops;
// these two ops are the image preprocessing and the pooled heads.
//
// Image input: uint8 images (element (n, c, y, x) at n*sn + c*sc + y*sy + x*sx) -> Pillow's antialiased bicubic resize, horizontal pass
// then vertical, each pass accumulating uint8 samples times 22-bit fixed-point weights in int32 from 2^21 and clamping (v >> 22) to
// uint8 -> the S x S centre crop -> (v / 255 - mean[c]) / std[c] in fp32, as fp32 NHWC [B][S][S][3].  The tables are computed on the
// host in double (openclip_plan.bicubic_tables), indexed by OUTPUT (crop) row / column, int32:
//   y0[S] ny[S] x0[S] nx[S] wy[S][ky] wx[S][kx]
// output row i reads source rows y0[i] .. y0[i] + ny[i] - 1 with weights wy[i][0 ..], output column j source columns x0[j] .. with wx[j].
typedef struct ds_clip_input_desc {
    const unsigned char* src;
    const int32_t* tab;
    float* out;
    int64_t sn, sc, sy, sx;     // element strides of src
    int32_t B, H, W, S;
    int32_t ky, kx;             // taps per row of wy / wx
    float mean[3];
    float std[3];
} ds_clip_input_desc;

// Pooled heads, one CTA per sample n:
//   GATHER: out[n * out_stride + c] = src[n * src_stride + r * C + c], c < C, with r = argmax_t ids[n * T + t] (the first maximum, the
//           EOT token of open_clip's text tower) or, ids == NULL, r = row (the class token of the image tower; with src_stride = 0 a
//           weight row broadcast to every sample);
//   L2NORM: out[n][c] = src[n][c] / max(||src[n]||, 1e-12)  (sums of squares in fp64);
//   SCORE:  out[n] = scale * sum_c src[n][c] * src2[n][c]   (fp64 sum).
enum { DS_CLIP_GATHER = 0, DS_CLIP_L2NORM = 1, DS_CLIP_SCORE = 2 };
typedef struct ds_clip_head_desc {
    const float* src;
    const float* src2;
    const int32_t* ids;
    float* out;
    int64_t src_stride, out_stride;
    int32_t B, C, T, row;
    int32_t mode;
    float scale;
} ds_clip_head_desc;

// ---------------------------------------------------------------------------------------------
// Precision, recall, density and coverage (prdc.cu; sfd-main/prdc.py as DESIGN.md 4.12 states it).  Every distance product runs on the
// GEMM kernel (rows mode): part[s][b][i] (s < nslice, row pitch ldp) are the fp32 partials over channel slice s of
// sq st q_b.t_i, the fp16 hi/lo planes of the query and target rows scaled by the powers of two sq and st.  The rows themselves are kept
// in float64 (q [B][D], t [N][D]) with their squared norms qn2 / tn2; d2_bi = qn2_b + tn2_i - 2 (sum_s part) / (sq st) approximates
// ||q_b - t_i||^2 within a per-pair bound (DESIGN.md 4.12).  Pairs the bound cannot decide are recomputed exactly, one warp per pair:
// float64 differences, squares and sums in a fixed order, then sqrt; comparisons are on those float64 distances.  There is no cap on
// the number of recomputed pairs; nres[b] (may be NULL) receives how many pairs row b recomputed.
//
// prdc_kth: rad[b] = the (k+1)-th smallest ||q_b - t_i|| (the target set is the query's own set, so the self distance 0 counts),
// rad2[b] its exact squared distance.  Overwrites part slice 0 with d2 (fp32).  k <= DS_PRDC_KMAX.
enum { DS_PRDC_KMAX = 63, DS_PRDC_LIST = 1024 };
typedef struct ds_prdc_kth_desc {
    float* part;
    const double* q;
    const double* t;
    const double* qn2;      // [B]
    const double* tn2;      // [N]
    double* rad;            // [B]
    double* rad2;           // [B]
    int32_t* nres;          // [B], may be NULL
    int64_t ldp;
    int32_t B, N, D, nslice;
    int32_t k, pad0;
    double sq, st;          // operand scales (powers of two)
} ds_prdc_kth_desc;

// prdc_count: for each query row b against targets with radii tau_i (tau2_i their exact squared distances):
//   cnt_t[b]   = #{i : ||q_b - t_i|| < tau_i};
//   cnt_own[b] = #{i : ||q_b - t_i|| < rho_b}            (rho / rho2 / cnt_own all set, or all NULL);
//   realism[b] = max over {i : tau_i < med} of tau_i / ||q_b - t_i||   (may be NULL; x / 0 = inf, 0 / 0 = nan, nan wins).
typedef struct ds_prdc_count_desc {
    const float* part;
    const double* q;
    const double* t;
    const double* qn2;
    const double* tn2;
    const double* tau;      // [N]
    const double* tau2;     // [N]
    const double* rho;      // [B]
    const double* rho2;     // [B]
    int32_t* cnt_t;         // [B]
    int32_t* cnt_own;       // [B]
    double* realism;        // [B]
    int32_t* nres;          // [B], may be NULL
    int64_t ldp;
    int32_t B, N, D, nslice;
    double sq, st;
    double med;
} ds_prdc_count_desc;

int ds_prdc_kth_launch(const ds_prdc_kth_desc* d, cudaStream_t stream);
int ds_prdc_count_launch(const ds_prdc_count_desc* d, cudaStream_t stream);

int ds_clip_input_launch(const ds_clip_input_desc* d, cudaStream_t stream);
int ds_clip_head_launch(const ds_clip_head_desc* d, cudaStream_t stream);
int ds_img_input_launch(const ds_img_input_desc* d, cudaStream_t stream);
int ds_im2col_launch(const ds_im2col_desc* d, cudaStream_t stream);
int ds_pool_launch(const ds_pool_desc* d, cudaStream_t stream);

int ds_opt_prep_launch(const ds_opt_prep_desc* d, cudaStream_t stream);
int ds_opt_softmax_launch(const ds_opt_softmax_desc* d, cudaStream_t stream);
int ds_opt_reduce_launch(const ds_opt_reduce_desc* d, cudaStream_t stream);
int ds_opt_knn_launch(const ds_opt_knn_desc* d, cudaStream_t stream);
int ds_amed_predict_launch(const float* w, const int* dims6, const float* bott, const float* t_cur, const float* t_next, float scale_dir,
                           float scale_time, float* out, int B, cudaStream_t stream);
int ds_to_uint8_launch(const float* x, unsigned char* out, int B, int Cc, int HW, cudaStream_t stream);
int ds_update_launch(const ds_update_desc* d, cudaStream_t stream);
int ds_threshold_launch(const ds_threshold_desc* d, cudaStream_t stream);
int ds_gn_stats_launch(const ds_gn_stats_desc* d, cudaStream_t stream);
int ds_gn_apply_launch(const ds_gn_apply_desc* d, cudaStream_t stream);
int ds_gn_finalize_launch(const ds_gn_finalize_desc* d, cudaStream_t stream);
int ds_attn_launch(const ds_attn_desc* d, cudaStream_t stream);
int ds_softmax_launch(const ds_softmax_desc* d, cudaStream_t stream);
int ds_posemb_launch(const ds_posemb_desc* d, cudaStream_t stream);
int ds_linear_launch(const ds_linear_desc* d, cudaStream_t stream);
int ds_prep_input_launch(const ds_prep_input_desc* d, cudaStream_t stream);
int ds_chanmean_launch(const ds_chanmean_desc* d, cudaStream_t stream);
int ds_layernorm_launch(const ds_layernorm_desc* d, cudaStream_t stream);
int ds_geglu_launch(const ds_geglu_desc* d, cudaStream_t stream);
int ds_embed_launch(const ds_embed_desc* d, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// Plan records.  The Python plan compiler (diff-sampler_b200/plan.py) lowers one denoiser network at
// one batch size into a flat array of these; the executor (engine.cu) resolves pointer *references*
// and launches them in order.  Pointer fields hold references until resolved:
//   bits 60..63 = space (0 absolute/NULL, 1 arena, 2 weights, 3 io slot), bits 0..59 = byte offset / slot.
enum { DS_OP_GEMM = 1, DS_OP_GN_STATS = 2, DS_OP_GN_APPLY = 3, DS_OP_SOFTMAX = 4, DS_OP_POSEMB = 5, DS_OP_LINEAR = 6,
       DS_OP_PREP_INPUT = 7, DS_OP_CHANMEAN = 8, DS_OP_MEMSET = 9, DS_OP_LAYERNORM = 10, DS_OP_GEGLU = 11,
       DS_OP_GN_FINALIZE = 12, DS_OP_ATTN = 13, DS_OP_EMBED = 14, DS_OP_OPT_PREP = 15, DS_OP_OPT_SOFTMAX = 16,
       DS_OP_OPT_REDUCE = 17, DS_OP_OPT_KNN = 18, DS_OP_IMG_INPUT = 19, DS_OP_IM2COL = 20, DS_OP_POOL = 21,
       DS_OP_CLIP_INPUT = 22, DS_OP_CLIP_HEAD = 23, DS_OP_PRDC_KTH = 24, DS_OP_PRDC_COUNT = 25 };
enum { DS_IO_X = 0, DS_IO_D = 1, DS_IO_SIGMA = 2, DS_IO_LABELS = 3, DS_IO_BOTTLENECK = 4, DS_IO_CTX = 5, DS_IO_COUNT = 6 };

typedef struct ds_memset_desc {
    void* ptr;
    int64_t bytes;
} ds_memset_desc;

typedef struct ds_plan_op {
    int32_t type;
    int32_t tag;            // free-form id for debugging (layer index)
    union {
        ds_gemm_desc gemm;
        ds_gn_stats_desc gn_stats;
        ds_gn_apply_desc gn_apply;
        ds_softmax_desc softmax;
        ds_posemb_desc posemb;
        ds_linear_desc linear;
        ds_prep_input_desc prep_input;
        ds_chanmean_desc chanmean;
        ds_memset_desc memset;
        ds_layernorm_desc layernorm;
        ds_geglu_desc geglu;
        ds_gn_finalize_desc gn_finalize;
        ds_attn_desc attn;
        ds_embed_desc embed;
        ds_opt_prep_desc opt_prep;
        ds_opt_softmax_desc opt_softmax;
        ds_opt_reduce_desc opt_reduce;
        ds_opt_knn_desc opt_knn;
        ds_img_input_desc img_input;
        ds_im2col_desc im2col;
        ds_pool_desc pool;
        ds_clip_input_desc clip_input;
        ds_clip_head_desc clip_head;
        ds_prdc_kth_desc prdc_kth;
        ds_prdc_count_desc prdc_count;
    } u;
} ds_plan_op;

#ifdef __cplusplus
}

namespace dsb {
// The descriptor rules of each launcher, one check per op type next to its launcher, run first by the launcher, by ds_op_check and, on
// every op of a plan, by ds_unet_create.  rc is 0 or the code the launcher returns; rule names the broken rule ("<op>: <rule>").  Pure
// host functions: no CUDA call, and pointers are only tested against NULL, so they hold for plan references as for device addresses.
struct OpCheck {
    int rc;
    const char* rule;
};
OpCheck gemm_check(const ds_gemm_desc& d);
OpCheck attn_check(const ds_attn_desc& d);
OpCheck gn_stats_check(const ds_gn_stats_desc& d);
OpCheck gn_finalize_check(const ds_gn_finalize_desc& d);
OpCheck gn_apply_check(const ds_gn_apply_desc& d);
OpCheck embed_check(const ds_embed_desc& d);
OpCheck layernorm_check(const ds_layernorm_desc& d);
OpCheck geglu_check(const ds_geglu_desc& d);
OpCheck linear_check(const ds_linear_desc& d);
OpCheck prep_input_check(const ds_prep_input_desc& d);
OpCheck opt_prep_check(const ds_opt_prep_desc& d);
OpCheck opt_softmax_check(const ds_opt_softmax_desc& d);
OpCheck opt_reduce_check(const ds_opt_reduce_desc& d);
OpCheck opt_knn_check(const ds_opt_knn_desc& d);
OpCheck img_input_check(const ds_img_input_desc& d);
OpCheck im2col_check(const ds_im2col_desc& d);
OpCheck pool_check(const ds_pool_desc& d);
OpCheck clip_input_check(const ds_clip_input_desc& d);
OpCheck clip_head_check(const ds_clip_head_desc& d);
OpCheck prdc_kth_check(const ds_prdc_kth_desc& d);
OpCheck prdc_count_check(const ds_prdc_count_desc& d);
}  // namespace dsb
#endif

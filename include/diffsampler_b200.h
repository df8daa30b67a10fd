/*
 * diffsampler_b200 — C ABI of the CUDA-native (H100, sm_90a) diffusion ODE sampling hot path.
 *
 * The reference (zju-pi/diff-sampler) is pure Python/PyTorch: its hot path has no FFI today.  The
 * boundary it exposes is the Python call surface
 *     solvers.<name>_sampler(net, latents, ...)          diff-solvers-main/solvers.py:18-821
 *     solver_utils.get_schedule(...)                      diff-solvers-main/solver_utils.py:6-52
 *     get_denoised(net, x, t, ...) -> net(x, sigma, ...)  diff-solvers-main/solvers.py:9-14
 * and the arithmetic underneath it is PyTorch library calls.  This header is the thin C ABI those
 * Python shims (diff-sampler_b200/solvers.py, net.py) bind with ctypes; every entry point names the
 * reference code it replaces.  Plain pointers and sizes only — no torch types, no exceptions; every
 * function returns 0 on success and a negative code on failure (text via ds_last_error()).
 *
 * All device pointers are CUDA device addresses on the current device; `stream` is a cudaStream_t
 * passed as void*.  A handle is bound to one device; calls on one handle must be serialised by the
 * caller (the reference is single-threaded per process, one process per GPU).
 */
#ifndef DIFFSAMPLER_B200_H
#define DIFFSAMPLER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Library version string, e.g. "diffsampler_b200 0.1 (sm_90a)". */
const char* ds_version(void);
/* Text of the last error raised on the calling thread ("" if none). */
const char* ds_last_error(void);

/* ---- denoiser network: replaces net(x, sigma, class_labels) ---------------------------------
 * EDMPrecond.forward + SongUNet/DhariwalUNet.forward, networks_edm.py:482-496, :312-355, :427-453.
 * `weights` is the packed blob produced by diff-sampler_b200/plan.py (fp16 hi/lo K-major conv
 * matrices + fp32 vectors); `plan` is an array of ds_plan_op records (csrc/ops.h) lowered for one
 * batch size.  The library copies the blob to device memory and owns it plus its workspace arena. */
typedef struct ds_weights ds_weights;
typedef struct ds_unet ds_unet;

int ds_weights_create(const void* host_blob, size_t bytes, ds_weights** out);
void ds_weights_destroy(ds_weights* w);

int ds_unet_create(const ds_weights* w, const void* plan_ops, int n_ops, size_t op_size, size_t arena_bytes, ds_unet** out);
void ds_unet_destroy(ds_unet* u);

/* One denoiser evaluation D = net(x, sigma[, labels]).
 *   x            [B, C, H, W] fp32 NCHW (not modified)
 *   sigma        device pointer to 1 or B fp32 values (as lowered in the plan)
 *   labels       [B, label_dim] fp32 or NULL
 *   out_D        [B, C, H, W] fp32 NCHW
 *   out_bottleneck  optional [B, 8*8] channel-mean of the U-Net bottleneck (AMED, solvers_amed.py:7-27) or NULL */
int ds_unet_forward(ds_unet* u, const float* x, const float* sigma, const float* labels, float* out_D,
                    float* out_bottleneck, void* stream);

/* Same with an explicit io table {x, out_D, sigma_or_timesteps, labels_or_coef, out_bottleneck, context}: used by the latent-diffusion
 * (CFGPrecond + UNetModel, networks_edm.py:670-696, openaimodel.py:710-741) plans, whose inputs are the timesteps c_noise[Bt], a
 * coefficient table [B][4] holding c_in, and the text context [Bt, 77, context_dim]; out_D receives eps in NCHW. */
int ds_unet_forward_io(ds_unet* u, const void* const* io, int n_io, void* stream);

/* CUDA-graph replay of the op list (SURVEY.md section 7 step 5: the per-NFE launch list as one graph).  io_bytes[k] = size of io slot k
 * {x, out_D, sigma, labels, out_bottleneck, context} for this plan (0 = slot unused).  After this call ds_unet_forward[_io] stages the
 * inputs into fixed device buffers (device-to-device copies on the caller's stream), replays ONE instantiated graph of all kernels
 * (captured on the second call, after a plain warm-up run) and copies the outputs back: 257 (EDM) / 520 (SD) launches become one. */
int ds_unet_enable_graph(ds_unet* u, const size_t* io_bytes, int n_io);

/* Debug/test access to the workspace arena (device -> host copy, synchronises the stream). */
int ds_unet_debug_read(ds_unet* u, size_t arena_offset, void* host_dst, size_t bytes, void* stream);
/* Number of kernels launched by the last ds_unet_forward on this handle. */
int ds_unet_last_launch_count(const ds_unet* u);

/* Per-op device timing (bench.py's roofline leg): when enabled, every op of the next forwards is bracketed by CUDA events on
 * the launch stream; ds_unet_get_profile synchronises and returns the last elapsed ms of each op (returns the op count). */
int ds_unet_set_profiling(ds_unet* u, int enable);
int ds_unet_get_profile(ds_unet* u, float* ms_per_op, int n);
int ds_unet_op_type(const ds_unet* u, int i);

/* ---- solver update: replaces the 4-12 elementwise ATen launches per step ------------------------
 * solvers.py:80-81 (Euler), :163-168 (Heun), :252-258 (DPM-2), :346-352 (iPNDM), :451-477 (iPNDM_v),
 * :576-585 (DEIS); solver_utils.py:102-163 (DPM-Solver++), :250-285 (UniPC); amed solver_utils.py:90-160.
 *   m0  = D | clamp(D,-s,s)/s | (xs - D)/t | xs/t | none        (mode 0..3; s = thr[b])
 *   out = coef[0]*xb + coef[1]*m0 + sum_k coef[2+k]*hist[k]
 * Coefficients are scalars (coef) or per-sample device vectors coef_dev[6][B] (AMED).  */
int ds_solver_update(float* out_x, float* out_m, const float* xb, const float* xs, const float* D,
                     const float* const* hist, int nhist, const float* thr, int mode, float t, const float* t_dev,
                     const float* coef6, const float* coef_dev, int64_t n_per_sample, int B, void* stream);

/* Same update with the image epilogue of sample.py:311 fused in (the LAST step of a sampling run):
 *   out_u8[n][hw][c] = uint8(clip(out * 127.5 + 128, 0, 255))   NCHW fp32 -> NHWC uint8, in the same pass over the state.
 * C * HW == n_per_sample, HW % 4 == 0; out_x may be NULL when only the byte image is wanted. */
int ds_solver_update_u8(float* out_x, float* out_m, unsigned char* out_u8, int C, int HW, const float* xb, const float* xs, const float* D,
                        const float* const* hist, int nhist, const float* thr, int mode, float t, const float* t_dev,
                        const float* coef6, const float* coef_dev, int64_t n_per_sample, int B, void* stream);

/* ---- dynamic thresholding: replaces torch.quantile(|x0|, 0.995) per sample ---------------------
 * solver_utils.py:77-86.  thr[b] = max(quantile_linear(|x0[b]|, q), floor_val).  Exact selection. */
int ds_dyn_threshold(const float* x0, float* thr, int B, int row_len, float q, float floor_val, void* stream);

/* ---- GITS cost matrix: replaces the O(N_tea^2) loop of tiny reductions --------------------------------
 * gits-main/gits_utils.py:115-132 (+ cal_deviation :237-255).  For every teacher pair i < j and sample b:
 *   x_ij = traj[i] + (t[j]-t[i])*eps[i];  out[i][j][b] = { sum|x_ij-traj[j]|, sum(x_ij-traj[j])^2, sum(c-x_ij)^2, sum(c-x_ij)(c-b0) }
 * with b0 = traj[0], c = traj[N-1].  traj [N][B][n], eps [N-1][B][n] fp32; out [N][N][B][4] fp64 (entries i >= j untouched). */
int ds_gits_cost(const float* traj, const float* eps, const float* t_steps, double* out, int N, int B, int64_t n_per_sample, void* stream);

/* ---- AMED predictor: replaces AMED_predictor.forward + the t_mid formula ------------------------------------------
 * amed-solver-main/training/networks.py:121-155, solvers_amed.py:22-55,:119.  One launch per sampling step:
 *   out4[0][b] = r, out4[1][b] = scale_dir, out4[2][b] = scale_time, out4[3][b] = t_mid = t_next^r * t_cur^(1-r)
 * weights: packed fp32 buffer (diff-sampler_b200/amed_predictor.py:pack); dims6 = {bottleneck_dim, hidden, z, noise_channels, has_dir,
 * has_time}; bottleneck [B][bottleneck_dim] or NULL (analytical first step: zeros, solvers_amed.py:24); t_cur / t_next: device scalars. */
int ds_amed_predict(const float* weights, const int* dims6, const float* bottleneck, const float* t_cur, const float* t_next,
                    float scale_dir, float scale_time, float* out4, int B, void* stream);

/* ---- image epilogue: replaces (images * 127.5 + 128).clip(0, 255).to(uint8).permute(0, 2, 3, 1) -------------
 * sample.py:311.  images [B, C, H*W] fp32 NCHW -> out [B, H*W, C] uint8 NHWC (what is written to PNG / gathered for FID). */
int ds_images_to_uint8(const float* images, unsigned char* out, int B, int C, int HW, void* stream);

/* ---- kernel-level entry points (used by the parity tests and micro-benchmarks) ------------------
 * `desc` points to the matching struct of csrc/ops.h with absolute device pointers. */
int ds_op_launch(int op_type, const void* desc, size_t desc_size, void* stream);
/* The descriptor check ds_op_launch's launcher runs first, without launching: 0, or the code the launcher would return with
 * "<op>: <rule>" in ds_last_error().  Needs no GPU; pointers are only tested against NULL.  ds_unet_create checks every op of a plan
 * this way before it allocates anything. */
int ds_op_check(int op_type, const void* desc, size_t desc_size);
/* sizeof() of the descriptor structs as compiled (0 = ds_plan_op, else DS_OP_* code); lets bindings verify their mirrors. */
size_t ds_sizeof(int which);
/* How the GEMM kernel would run `desc` (a ds_gemm_desc) on the current device: info[0] shared-memory ring stages, info[1] CTAs in
 * the persistent grid. */
int ds_gemm_config(const void* desc, int* info);

#ifdef __cplusplus
}
#endif
#endif

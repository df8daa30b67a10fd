// Plan executor + C ABI (include/diffsampler_b200.h).
// A ds_unet is: packed weights (device), a workspace arena (device), and a list of resolved ops whose
// tensor maps were encoded once at creation.  Forward = patch the io pointers, launch the ops in order
// on the caller's stream.  No host synchronisation, no allocation on the forward path.
#include "../../include/diffsampler_b200.h"
#include "ops.h"
#include "ptx.cuh"
#include <cuda_fp16.h>
#include <nvtx3/nvToolsExt.h>      // header-only NVTX3: ranges cost nothing unless a profiler (nsys / ncu --nvtx) is attached
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

namespace dsb {
struct GemmKernelParams;
int gemm_build(const ds_gemm_desc* d, GemmKernelParams* kp);
int gemm_run(const GemmKernelParams* kp, cudaStream_t stream);
size_t gemm_params_size();
void gemm_patch_edm(GemmKernelParams* kp, const float* x, float* D);
struct AttnKernelParams;
int attn_build(const ds_attn_desc* d, AttnKernelParams* kp);
int attn_run(const AttnKernelParams* kp, cudaStream_t stream);
size_t attn_params_size();
}  // namespace dsb

static thread_local std::string g_err;

// NVTX range per denoiser evaluation (= one NFE) and per solver update: `ncu --nvtx --nvtx-include "ds_unet_forward/"` or an nsys
// timeline then groups the launch list by NFE (SURVEY.md section 5).
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
static int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

struct ds_weights {
    void* dev = nullptr;
    size_t bytes = 0;
};

struct IoFix {
    int op;
    size_t field_off;   // byte offset of the pointer field inside ds_plan_op
    int slot;
};

struct ds_unet {
    const ds_weights* w = nullptr;
    void* arena = nullptr;
    size_t arena_bytes = 0;
    std::vector<ds_plan_op> ops;
    std::vector<std::vector<unsigned char>> gemm_params;   // prebuilt kernel params (tensor maps) per GEMM / attention op, else empty
    std::vector<IoFix> fixes;
    int last_launches = 0;
    // optional per-op timing (bench/profiling only): one event pair per op, read back on demand
    bool profiling = false;
    std::vector<cudaEvent_t> ev0, ev1;
    std::vector<char> ev_used;
    // optional CUDA-graph replay of the op list (ds_unet_enable_graph): the io slots are staged through fixed device buffers so that one
    // instantiated graph serves every call; [0] = without, [1] = with the bottleneck read-out
    bool graph_on = false;
    void* stage[DS_IO_COUNT] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    size_t stage_bytes[DS_IO_COUNT] = {0, 0, 0, 0, 0, 0};
    cudaGraphExec_t gexec[2] = {nullptr, nullptr};
    int gnodes[2] = {0, 0};
    int warm_runs = 0;
    cudaStream_t cap_stream = nullptr;
};

template <class F>
static void visit_ptrs(ds_plan_op& op, F f) {
#define P(field) f((void**)(void*)(&(field)))
    switch (op.type) {
        case DS_OP_GEMM: {
            ds_gemm_desc& g = op.u.gemm;
            P(g.a_ptr); P(g.a2_ptr); P(g.b_ptr); P(g.out_f32); P(g.out_h16); P(g.bias_n); P(g.bias_m); P(g.rowvec);
            P(g.residual); P(g.edm_x); P(g.edm_coef); P(g.edm_D); P(g.st_quads);
            break;
        }
        case DS_OP_GN_STATS: { auto& d = op.u.gn_stats; P(d.src0); P(d.src1); P(d.sums); break; }
        case DS_OP_GN_APPLY: {
            auto& d = op.u.gn_apply;
            P(d.src0); P(d.src1); P(d.sums); P(d.gamma); P(d.beta); P(d.ada); P(d.out_act); P(d.out_raw); P(d.out_raw_f32); P(d.coef);
            break;
        }
        case DS_OP_SOFTMAX: { auto& d = op.u.softmax; P(d.S); P(d.P); break; }
        case DS_OP_POSEMB: { auto& d = op.u.posemb; P(d.sigma); P(d.coef); P(d.emb); break; }
        case DS_OP_LINEAR: { auto& d = op.u.linear; P(d.in); P(d.W); P(d.b); P(d.add); P(d.out); break; }
        case DS_OP_PREP_INPUT: { auto& d = op.u.prep_input; P(d.x); P(d.coef); P(d.out); P(d.codebook); P(d.idx); break; }
        case DS_OP_CHANMEAN: { auto& d = op.u.chanmean; P(d.src); P(d.out); break; }
        case DS_OP_MEMSET: { auto& d = op.u.memset; P(d.ptr); break; }
        case DS_OP_LAYERNORM: { auto& d = op.u.layernorm; P(d.src); P(d.gamma); P(d.beta); P(d.out); break; }
        case DS_OP_GEGLU: { auto& d = op.u.geglu; P(d.src); P(d.out); break; }
        case DS_OP_GN_FINALIZE: { auto& d = op.u.gn_finalize; P(d.quads0); P(d.quads1); P(d.sums); P(d.gamma); P(d.beta); P(d.ada); P(d.coef); break; }
        case DS_OP_ATTN: { auto& d = op.u.attn; P(d.q); P(d.k); P(d.vt); P(d.out); break; }
        case DS_OP_EMBED: { auto& d = op.u.embed; P(d.ids); P(d.tok); P(d.pos); P(d.out); break; }
        case DS_OP_OPT_PREP: { auto& d = op.u.opt_prep; P(d.x); P(d.planes); P(d.xn2); break; }
        case DS_OP_OPT_SOFTMAX: { auto& d = op.u.opt_softmax; P(d.part); P(d.hy2); P(d.xn2); P(d.sigma); P(d.x); P(d.y); P(d.P); P(d.status); break; }
        case DS_OP_OPT_REDUCE: { auto& d = op.u.opt_reduce; P(d.part); P(d.out); break; }
        case DS_OP_OPT_KNN: { auto& d = op.u.opt_knn; P(d.part); P(d.hy2); P(d.xn2); P(d.x); P(d.y); P(d.dist); P(d.idx); break; }
        case DS_OP_IMG_INPUT: { auto& d = op.u.img_input; P(d.src); P(d.out); break; }
        case DS_OP_IM2COL: { auto& d = op.u.im2col; P(d.src); P(d.out); break; }
        case DS_OP_POOL: { auto& d = op.u.pool; P(d.src); P(d.out_f32); P(d.out_h16); break; }
        case DS_OP_CLIP_INPUT: { auto& d = op.u.clip_input; P(d.src); P(d.tab); P(d.out); break; }
        case DS_OP_CLIP_HEAD: { auto& d = op.u.clip_head; P(d.src); P(d.src2); P(d.ids); P(d.out); break; }
        case DS_OP_PRDC_KTH: {
            auto& d = op.u.prdc_kth;
            P(d.part); P(d.q); P(d.t); P(d.qn2); P(d.tn2); P(d.rad); P(d.rad2); P(d.nres);
            break;
        }
        case DS_OP_PRDC_COUNT: {
            auto& d = op.u.prdc_count;
            P(d.part); P(d.q); P(d.t); P(d.qn2); P(d.tn2); P(d.tau); P(d.tau2); P(d.rho); P(d.rho2); P(d.cnt_t); P(d.cnt_own);
            P(d.realism); P(d.nres);
            break;
        }
        default: break;
    }
#undef P
}

// The launcher's descriptor check of the op (ops.h).  Posemb, softmax, chanmean and memset accept every descriptor.
static dsb::OpCheck check_op(const ds_plan_op& op) {
    switch (op.type) {
        case DS_OP_GEMM: return dsb::gemm_check(op.u.gemm);
        case DS_OP_GN_STATS: return dsb::gn_stats_check(op.u.gn_stats);
        case DS_OP_GN_APPLY: return dsb::gn_apply_check(op.u.gn_apply);
        case DS_OP_LINEAR: return dsb::linear_check(op.u.linear);
        case DS_OP_PREP_INPUT: return dsb::prep_input_check(op.u.prep_input);
        case DS_OP_LAYERNORM: return dsb::layernorm_check(op.u.layernorm);
        case DS_OP_GEGLU: return dsb::geglu_check(op.u.geglu);
        case DS_OP_GN_FINALIZE: return dsb::gn_finalize_check(op.u.gn_finalize);
        case DS_OP_ATTN: return dsb::attn_check(op.u.attn);
        case DS_OP_EMBED: return dsb::embed_check(op.u.embed);
        case DS_OP_OPT_PREP: return dsb::opt_prep_check(op.u.opt_prep);
        case DS_OP_OPT_SOFTMAX: return dsb::opt_softmax_check(op.u.opt_softmax);
        case DS_OP_OPT_REDUCE: return dsb::opt_reduce_check(op.u.opt_reduce);
        case DS_OP_OPT_KNN: return dsb::opt_knn_check(op.u.opt_knn);
        case DS_OP_IMG_INPUT: return dsb::img_input_check(op.u.img_input);
        case DS_OP_IM2COL: return dsb::im2col_check(op.u.im2col);
        case DS_OP_POOL: return dsb::pool_check(op.u.pool);
        case DS_OP_CLIP_INPUT: return dsb::clip_input_check(op.u.clip_input);
        case DS_OP_CLIP_HEAD: return dsb::clip_head_check(op.u.clip_head);
        case DS_OP_PRDC_KTH: return dsb::prdc_kth_check(op.u.prdc_kth);
        case DS_OP_PRDC_COUNT: return dsb::prdc_count_check(op.u.prdc_count);
        case DS_OP_SOFTMAX: case DS_OP_POSEMB: case DS_OP_CHANMEAN: case DS_OP_MEMSET: return {0, nullptr};
        default: return {-100, "unknown op type"};
    }
}

static int launch_op(const ds_plan_op& op, const unsigned char* gemm_kp, cudaStream_t s) {
    switch (op.type) {
        case DS_OP_GEMM:
            if (gemm_kp) return dsb::gemm_run(reinterpret_cast<const dsb::GemmKernelParams*>(gemm_kp), s);
            return ds_gemm_launch(&op.u.gemm, s);
        case DS_OP_GN_STATS: return ds_gn_stats_launch(&op.u.gn_stats, s);
        case DS_OP_GN_APPLY: return ds_gn_apply_launch(&op.u.gn_apply, s);
        case DS_OP_SOFTMAX: return ds_softmax_launch(&op.u.softmax, s);
        case DS_OP_POSEMB: return ds_posemb_launch(&op.u.posemb, s);
        case DS_OP_LINEAR: return ds_linear_launch(&op.u.linear, s);
        case DS_OP_PREP_INPUT: return ds_prep_input_launch(&op.u.prep_input, s);
        case DS_OP_CHANMEAN: return ds_chanmean_launch(&op.u.chanmean, s);
        case DS_OP_LAYERNORM: return ds_layernorm_launch(&op.u.layernorm, s);
        case DS_OP_GEGLU: return ds_geglu_launch(&op.u.geglu, s);
        case DS_OP_GN_FINALIZE: return ds_gn_finalize_launch(&op.u.gn_finalize, s);
        case DS_OP_EMBED: return ds_embed_launch(&op.u.embed, s);
        case DS_OP_OPT_PREP: return ds_opt_prep_launch(&op.u.opt_prep, s);
        case DS_OP_OPT_SOFTMAX: return ds_opt_softmax_launch(&op.u.opt_softmax, s);
        case DS_OP_OPT_REDUCE: return ds_opt_reduce_launch(&op.u.opt_reduce, s);
        case DS_OP_OPT_KNN: return ds_opt_knn_launch(&op.u.opt_knn, s);
        case DS_OP_IMG_INPUT: return ds_img_input_launch(&op.u.img_input, s);
        case DS_OP_IM2COL: return ds_im2col_launch(&op.u.im2col, s);
        case DS_OP_POOL: return ds_pool_launch(&op.u.pool, s);
        case DS_OP_CLIP_INPUT: return ds_clip_input_launch(&op.u.clip_input, s);
        case DS_OP_CLIP_HEAD: return ds_clip_head_launch(&op.u.clip_head, s);
        case DS_OP_PRDC_KTH: return ds_prdc_kth_launch(&op.u.prdc_kth, s);
        case DS_OP_PRDC_COUNT: return ds_prdc_count_launch(&op.u.prdc_count, s);
        case DS_OP_ATTN:
            if (gemm_kp) return dsb::attn_run(reinterpret_cast<const dsb::AttnKernelParams*>(gemm_kp), s);
            return ds_attn_launch(&op.u.attn, s);
        case DS_OP_MEMSET:
            return cudaMemsetAsync(op.u.memset.ptr, 0, (size_t)op.u.memset.bytes, s) == cudaSuccess ? 0 : -1;
        default: return -100;
    }
}

extern "C" {

const char* ds_version(void) { return "diffsampler_b200 0.1 (sm_90a, wgmma/TMA)"; }
const char* ds_last_error(void) { return g_err.c_str(); }

int ds_weights_create(const void* host_blob, size_t bytes, ds_weights** out) {
    if (!host_blob || !out) return fail(-1, "ds_weights_create: null argument");
    ds_weights* w = new ds_weights();
    if (cudaMalloc(&w->dev, bytes ? bytes : 16) != cudaSuccess) {
        delete w;
        return fail(-2, std::string("ds_weights_create: cudaMalloc failed: ") + cudaGetErrorString(cudaGetLastError()));
    }
    if (cudaMemcpy(w->dev, host_blob, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(w->dev);
        delete w;
        return fail(-3, "ds_weights_create: cudaMemcpy failed");
    }
    w->bytes = bytes;
    *out = w;
    return 0;
}

void ds_weights_destroy(ds_weights* w) {
    if (!w) return;
    cudaFree(w->dev);
    delete w;
}

int ds_unet_create(const ds_weights* w, const void* plan_ops, int n_ops, size_t op_size, size_t arena_bytes, ds_unet** out) {
    if (!w || !plan_ops || !out) return fail(-1, "ds_unet_create: null argument");
    if (op_size != sizeof(ds_plan_op)) {
        char buf[128];
        snprintf(buf, sizeof buf, "ds_unet_create: ds_plan_op size mismatch (caller %zu, library %zu)", op_size, sizeof(ds_plan_op));
        return fail(-4, buf);
    }
    // refuse a plan with an op its launcher would refuse before anything is allocated (the checks hold on pointer references)
    for (int i = 0; i < n_ops; ++i) {
        const ds_plan_op& op = reinterpret_cast<const ds_plan_op*>(plan_ops)[i];
        const dsb::OpCheck c = check_op(op);
        if (c.rc) {
            char buf[160];
            snprintf(buf, sizeof buf, "ds_unet_create: op %d (type %d tag %d) refused (rc %d): %s", i, op.type, op.tag, c.rc, c.rule);
            return fail(-6, buf);
        }
    }
    ds_unet* u = new ds_unet();
    u->w = w;
    u->arena_bytes = arena_bytes;
    if (cudaMalloc(&u->arena, arena_bytes ? arena_bytes : 16) != cudaSuccess) {
        delete u;
        return fail(-2, std::string("ds_unet_create: cudaMalloc(arena) failed: ") + cudaGetErrorString(cudaGetLastError()));
    }
    cudaMemset(u->arena, 0, arena_bytes);
    u->ops.assign(reinterpret_cast<const ds_plan_op*>(plan_ops), reinterpret_cast<const ds_plan_op*>(plan_ops) + n_ops);
    u->gemm_params.resize(n_ops);
    int bad = 0;
    for (int i = 0; i < n_ops; ++i) {
        ds_plan_op& op = u->ops[i];
        visit_ptrs(op, [&](void** field) {
            const uint64_t ref = reinterpret_cast<uint64_t>(*field);
            const uint64_t space = ref >> 60;
            const uint64_t off = ref & ((1ull << 60) - 1);
            if (space == 0) return;
            if (space == 1) {
                if (off >= arena_bytes) bad = i + 1;
                *field = static_cast<char*>(u->arena) + off;
            } else if (space == 2) {
                if (off >= w->bytes) bad = i + 1;
                *field = static_cast<char*>(w->dev) + off;
            } else if (space == 3) {
                IoFix fx;
                fx.op = i;
                fx.field_off = reinterpret_cast<char*>(field) - reinterpret_cast<char*>(&op);
                fx.slot = (int)off;
                u->fixes.push_back(fx);
                *field = nullptr;
            } else {
                bad = i + 1;
            }
        });
    }
    if (bad) {
        char buf[96];
        snprintf(buf, sizeof buf, "ds_unet_create: bad pointer reference in op %d", bad - 1);
        ds_unet_destroy(u);
        return fail(-5, buf);
    }
    for (int i = 0; i < n_ops; ++i) {
        const int type = u->ops[i].type;
        if (type != DS_OP_GEMM && type != DS_OP_ATTN) continue;
        u->gemm_params[i].resize((type == DS_OP_GEMM ? dsb::gemm_params_size() : dsb::attn_params_size()) + 64);
        // keep 64-byte alignment for the embedded CUtensorMaps
        unsigned char* p = u->gemm_params[i].data();
        unsigned char* al = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 63) & ~uintptr_t(63));
        int rc = type == DS_OP_GEMM ? dsb::gemm_build(&u->ops[i].u.gemm, reinterpret_cast<dsb::GemmKernelParams*>(al))
                                    : dsb::attn_build(&u->ops[i].u.attn, reinterpret_cast<dsb::AttnKernelParams*>(al));
        if (rc) {
            char buf[96];
            snprintf(buf, sizeof buf, "ds_unet_create: %s failed (rc %d) for op %d tag %d", type == DS_OP_GEMM ? "gemm_build" : "attn_build", rc, i,
                     u->ops[i].tag);
            ds_unet_destroy(u);
            return fail(-6, buf);
        }
    }
    *out = u;
    return 0;
}

void ds_unet_destroy(ds_unet* u) {
    if (!u) return;
    for (auto e : u->ev0) cudaEventDestroy(e);
    for (auto e : u->ev1) cudaEventDestroy(e);
    for (int v = 0; v < 2; ++v) if (u->gexec[v]) cudaGraphExecDestroy(u->gexec[v]);
    for (int k = 0; k < DS_IO_COUNT; ++k) if (u->stage[k]) cudaFree(u->stage[k]);
    if (u->cap_stream) cudaStreamDestroy(u->cap_stream);
    cudaFree(u->arena);
    delete u;
}

int ds_unet_forward_io(ds_unet* u, const void* const* io_in, int n_io, void* stream);

int ds_unet_forward(ds_unet* u, const float* x, const float* sigma, const float* labels, float* out_D, float* out_bottleneck,
                    void* stream) {
    const void* io[DS_IO_COUNT] = {x, out_D, sigma, labels, out_bottleneck, nullptr};
    return ds_unet_forward_io(u, io, DS_IO_COUNT, stream);
}

// Launch the op list on `s` with the io slots bound to `io`.  Returns the number of launches, or a negative code.
static int run_ops(ds_unet* u, const void* const* io, cudaStream_t s, bool profiling) {
    for (const IoFix& fx : u->fixes) {
        if (fx.slot < 0 || fx.slot >= DS_IO_COUNT) return fail(-7, "ds_unet_forward: bad io slot");
        void** field = reinterpret_cast<void**>(reinterpret_cast<char*>(&u->ops[fx.op]) + fx.field_off);
        *field = const_cast<void*>(io[fx.slot]);
    }
    int launches = 0;
    for (size_t i = 0; i < u->ops.size(); ++i) {
        ds_plan_op& op = u->ops[i];
        const unsigned char* kp = nullptr;
        if (op.type == DS_OP_GEMM || op.type == DS_OP_ATTN) {
            unsigned char* p = u->gemm_params[i].data();
            unsigned char* al = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 63) & ~uintptr_t(63));
            if (op.type == DS_OP_GEMM && op.u.gemm.edm_out)
                dsb::gemm_patch_edm(reinterpret_cast<dsb::GemmKernelParams*>(al), op.u.gemm.edm_x, op.u.gemm.edm_D);
            kp = al;
        }
        if (op.type == DS_OP_CHANMEAN && op.u.chanmean.out == nullptr) continue;   // bottleneck tap not requested
        if (profiling) { cudaEventRecord(u->ev0[i], s); u->ev_used[i] = 1; }
        int rc = launch_op(op, kp, s);
        if (profiling) cudaEventRecord(u->ev1[i], s);
        if (rc) {
            char buf[160];
            snprintf(buf, sizeof buf, "ds_unet_forward: op %zu (type %d tag %d) failed rc=%d cuda=%s", i, op.type, op.tag, rc,
                     cudaGetErrorString(cudaGetLastError()));
            return fail(-8, buf);
        }
        ++launches;
    }
    return launches;
}

// Capture the op list (io slots bound to the staging buffers) into a graph on the private capture stream and instantiate it.
static int build_graph(ds_unet* u, int variant, const void* const* staged_io) {
    if (!u->cap_stream && cudaStreamCreateWithFlags(&u->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
        return fail(-20, "ds_unet_forward: cannot create the capture stream");
    if (cudaStreamBeginCapture(u->cap_stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess)
        return fail(-21, std::string("ds_unet_forward: cudaStreamBeginCapture failed: ") + cudaGetErrorString(cudaGetLastError()));
    const int n = run_ops(u, staged_io, u->cap_stream, false);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(u->cap_stream, &g);
    if (n < 0 || e != cudaSuccess || !g) {
        if (g) cudaGraphDestroy(g);
        if (n < 0) return n;
        return fail(-22, std::string("ds_unet_forward: stream capture failed: ") + cudaGetErrorString(e));
    }
    cudaGraphExec_t ex = nullptr;
    const cudaError_t ei = cudaGraphInstantiate(&ex, g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) return fail(-23, std::string("ds_unet_forward: cudaGraphInstantiate failed: ") + cudaGetErrorString(ei));
    u->gexec[variant] = ex;
    u->gnodes[variant] = n;
    return 0;
}

int ds_unet_forward_io(ds_unet* u, const void* const* io_in, int n_io, void* stream) {
    if (!u) return fail(-1, "ds_unet_forward: null handle");
    NvtxRange nvtx_range("ds_unet_forward");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const void* io[DS_IO_COUNT] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    for (int k = 0; k < n_io && k < DS_IO_COUNT; ++k) io[k] = io_in[k];
    if (!u->graph_on || u->profiling) {
        const int n = run_ops(u, io, s, u->profiling);
        if (n < 0) return n;
        u->last_launches = n;
        return 0;
    }
    // ---- graph replay: inputs -> staging (device-to-device, same stream), one cudaGraphLaunch, staging -> outputs
    static const bool is_input[DS_IO_COUNT] = {true, false, true, true, false, true};       // X, D, SIGMA, LABELS, BOTTLENECK, CTX
    const void* staged[DS_IO_COUNT];
    for (int k = 0; k < DS_IO_COUNT; ++k) {
        staged[k] = (io[k] && u->stage[k]) ? u->stage[k] : nullptr;
        if (io[k] && !u->stage[k]) return fail(-24, "ds_unet_forward: io slot used without a staging buffer (ds_unet_enable_graph sizes)");
        if (io[k] && is_input[k] &&
            cudaMemcpyAsync(u->stage[k], io[k], u->stage_bytes[k], cudaMemcpyDeviceToDevice, s) != cudaSuccess)
            return fail(-25, "ds_unet_forward: staging copy failed");
    }
    const int variant = io[DS_IO_BOTTLENECK] ? 1 : 0;
    int launches = 0;
    if (!u->gexec[variant]) {
        if (u->warm_runs < 1) {
            // first call: plain launches (sets the per-device function attributes outside any capture)
            launches = run_ops(u, staged, s, false);
            if (launches < 0) return launches;
            ++u->warm_runs;
        } else {
            const int rc = build_graph(u, variant, staged);
            if (rc) return rc;
        }
    }
    if (u->gexec[variant]) {
        if (cudaGraphLaunch(u->gexec[variant], s) != cudaSuccess)
            return fail(-26, std::string("ds_unet_forward: cudaGraphLaunch failed: ") + cudaGetErrorString(cudaGetLastError()));
        launches = u->gnodes[variant];
    }
    for (int k = 0; k < DS_IO_COUNT; ++k)
        if (io[k] && !is_input[k] &&
            cudaMemcpyAsync(const_cast<void*>(io[k]), u->stage[k], u->stage_bytes[k], cudaMemcpyDeviceToDevice, s) != cudaSuccess)
            return fail(-25, "ds_unet_forward: staging copy failed");
    u->last_launches = launches;
    return 0;
}

int ds_unet_enable_graph(ds_unet* u, const size_t* io_bytes, int n_io) {
    if (!u || !io_bytes) return fail(-1, "ds_unet_enable_graph: null argument");
    if (u->graph_on) return 0;
    for (int k = 0; k < n_io && k < DS_IO_COUNT; ++k) {
        if (!io_bytes[k]) continue;
        if (cudaMalloc(&u->stage[k], io_bytes[k]) != cudaSuccess)
            return fail(-2, std::string("ds_unet_enable_graph: cudaMalloc failed: ") + cudaGetErrorString(cudaGetLastError()));
        u->stage_bytes[k] = io_bytes[k];
    }
    u->graph_on = true;
    return 0;
}

int ds_unet_debug_read(ds_unet* u, size_t arena_offset, void* host_dst, size_t bytes, void* stream) {
    if (!u || arena_offset + bytes > u->arena_bytes) return fail(-1, "ds_unet_debug_read: out of range");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail(-2, std::string("ds_unet_debug_read: ") + cudaGetErrorString(cudaGetLastError()));
    if (cudaMemcpy(host_dst, static_cast<char*>(u->arena) + arena_offset, bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
        return fail(-3, "ds_unet_debug_read: memcpy failed");
    return 0;
}

int ds_unet_last_launch_count(const ds_unet* u) { return u ? u->last_launches : 0; }

int ds_unet_set_profiling(ds_unet* u, int enable) {
    if (!u) return fail(-1, "ds_unet_set_profiling: null handle");
    if (enable && u->ev0.empty()) {
        u->ev0.resize(u->ops.size());
        u->ev1.resize(u->ops.size());
        u->ev_used.assign(u->ops.size(), 0);
        for (size_t i = 0; i < u->ops.size(); ++i) {
            cudaEventCreate(&u->ev0[i]);
            cudaEventCreate(&u->ev1[i]);
        }
    }
    u->profiling = enable != 0;
    return 0;
}

int ds_unet_get_profile(ds_unet* u, float* ms_per_op, int n) {
    if (!u || u->ev0.empty()) return fail(-1, "ds_unet_get_profile: profiling was not enabled");
    if (cudaDeviceSynchronize() != cudaSuccess) return fail(-2, "ds_unet_get_profile: sync failed");
    for (int i = 0; i < n && i < (int)u->ops.size(); ++i) {
        float ms = 0.f;
        if (u->ev_used[i]) cudaEventElapsedTime(&ms, u->ev0[i], u->ev1[i]);
        ms_per_op[i] = ms;
    }
    return (int)u->ops.size();
}

int ds_unet_op_type(const ds_unet* u, int i) { return (u && i >= 0 && i < (int)u->ops.size()) ? u->ops[i].type : -1; }

static int solver_update_impl(float* out_x, float* out_m, unsigned char* out_u8, int u8_C, int u8_HW, const float* xb, const float* xs,
                              const float* D, const float* const* hist, int nhist, const float* thr, int mode, float t, const float* t_dev,
                              const float* coef6, const float* coef_dev, int64_t n_per_sample, int B, void* stream) {
    if (!xb || nhist < 0 || nhist > 4) return fail(-1, "ds_solver_update: bad argument");
    NvtxRange nvtx_range("ds_solver_update");
    ds_update_desc d;
    memset(&d, 0, sizeof d);
    d.out_x = out_x; d.out_m = out_m; d.xb = xb; d.xs = xs; d.D = D;
    for (int k = 0; k < nhist; ++k) d.h[k] = hist[k];
    d.thr = thr; d.coef_dev = coef_dev; d.t_dev = t_dev;
    if (coef6) for (int k = 0; k < 6; ++k) d.coef[k] = coef6[k];
    d.t = t; d.mode = mode; d.nhist = nhist; d.B = B; d.n_per_sample = n_per_sample;
    d.out_u8 = out_u8; d.u8_C = u8_C; d.u8_HW = u8_HW;
    if ((mode == DS_M_X0 || mode == DS_M_EPS) && !D) return fail(-1, "ds_solver_update: mode needs D");
    int rc = ds_update_launch(&d, static_cast<cudaStream_t>(stream));
    if (rc) return fail(rc, std::string("ds_solver_update: launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int ds_solver_update(float* out_x, float* out_m, const float* xb, const float* xs, const float* D, const float* const* hist, int nhist,
                     const float* thr, int mode, float t, const float* t_dev, const float* coef6, const float* coef_dev,
                     int64_t n_per_sample, int B, void* stream) {
    return solver_update_impl(out_x, out_m, nullptr, 0, 0, xb, xs, D, hist, nhist, thr, mode, t, t_dev, coef6, coef_dev, n_per_sample, B, stream);
}

int ds_solver_update_u8(float* out_x, float* out_m, unsigned char* out_u8, int C, int HW, const float* xb, const float* xs, const float* D,
                        const float* const* hist, int nhist, const float* thr, int mode, float t, const float* t_dev, const float* coef6,
                        const float* coef_dev, int64_t n_per_sample, int B, void* stream) {
    if (!out_u8 || C <= 0 || HW <= 0) return fail(-1, "ds_solver_update_u8: bad image geometry");
    return solver_update_impl(out_x, out_m, out_u8, C, HW, xb, xs, D, hist, nhist, thr, mode, t, t_dev, coef6, coef_dev, n_per_sample, B, stream);
}

int ds_dyn_threshold(const float* x0, float* thr, int B, int row_len, float q, float floor_val, void* stream) {
    ds_threshold_desc d;
    d.x0 = x0; d.thr = thr; d.B = B; d.row_len = row_len; d.q = q; d.floor_val = floor_val;
    int rc = ds_threshold_launch(&d, static_cast<cudaStream_t>(stream));
    if (rc) return fail(rc, std::string("ds_dyn_threshold: launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

size_t ds_sizeof(int which) {
    switch (which) {
        case 0: return sizeof(ds_plan_op);
        case DS_OP_GEMM: return sizeof(ds_gemm_desc);
        case DS_OP_GN_STATS: return sizeof(ds_gn_stats_desc);
        case DS_OP_GN_APPLY: return sizeof(ds_gn_apply_desc);
        case DS_OP_SOFTMAX: return sizeof(ds_softmax_desc);
        case DS_OP_POSEMB: return sizeof(ds_posemb_desc);
        case DS_OP_LINEAR: return sizeof(ds_linear_desc);
        case DS_OP_PREP_INPUT: return sizeof(ds_prep_input_desc);
        case DS_OP_CHANMEAN: return sizeof(ds_chanmean_desc);
        case DS_OP_MEMSET: return sizeof(ds_memset_desc);
        case DS_OP_LAYERNORM: return sizeof(ds_layernorm_desc);
        case DS_OP_GEGLU: return sizeof(ds_geglu_desc);
        case DS_OP_GN_FINALIZE: return sizeof(ds_gn_finalize_desc);
        case DS_OP_ATTN: return sizeof(ds_attn_desc);
        case DS_OP_EMBED: return sizeof(ds_embed_desc);
        case DS_OP_OPT_PREP: return sizeof(ds_opt_prep_desc);
        case DS_OP_OPT_SOFTMAX: return sizeof(ds_opt_softmax_desc);
        case DS_OP_OPT_REDUCE: return sizeof(ds_opt_reduce_desc);
        case DS_OP_OPT_KNN: return sizeof(ds_opt_knn_desc);
        case DS_OP_IMG_INPUT: return sizeof(ds_img_input_desc);
        case DS_OP_IM2COL: return sizeof(ds_im2col_desc);
        case DS_OP_POOL: return sizeof(ds_pool_desc);
        case DS_OP_CLIP_INPUT: return sizeof(ds_clip_input_desc);
        case DS_OP_CLIP_HEAD: return sizeof(ds_clip_head_desc);
        case DS_OP_PRDC_KTH: return sizeof(ds_prdc_kth_desc);
        case DS_OP_PRDC_COUNT: return sizeof(ds_prdc_count_desc);
        default: return 0;
    }
}

int ds_gits_cost(const float* traj, const float* eps, const float* t_steps, double* out, int N, int B, int64_t n_per_sample, void* stream) {
    ds_gits_cost_desc d;
    d.traj = traj; d.eps = eps; d.t = t_steps; d.out = out; d.N = N; d.B = B; d.n = n_per_sample;
    int rc = ds_gits_cost_launch(&d, static_cast<cudaStream_t>(stream));
    if (rc) return fail(rc, std::string("ds_gits_cost: launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int ds_amed_predict(const float* weights, const int* dims6, const float* bottleneck, const float* t_cur, const float* t_next,
                    float scale_dir, float scale_time, float* out4, int B, void* stream) {
    if (!weights || !dims6 || !t_cur || !t_next || !out4) return fail(-1, "ds_amed_predict: null argument");
    NvtxRange nvtx_range("ds_amed_predict");
    int rc = ds_amed_predict_launch(weights, dims6, bottleneck, t_cur, t_next, scale_dir, scale_time, out4, B, static_cast<cudaStream_t>(stream));
    if (rc) return fail(rc, std::string("ds_amed_predict: launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int ds_images_to_uint8(const float* images, unsigned char* out, int B, int C, int HW, void* stream) {
    if (!images || !out) return fail(-1, "ds_images_to_uint8: null argument");
    int rc = ds_to_uint8_launch(images, out, B, C, HW, static_cast<cudaStream_t>(stream));
    if (rc) return fail(rc, std::string("ds_images_to_uint8: launch failed: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int ds_op_launch(int op_type, const void* desc, size_t desc_size, void* stream) {
    ds_plan_op op;
    memset(&op, 0, sizeof op);
    op.type = op_type;
    if (desc_size > sizeof(op.u)) return fail(-1, "ds_op_launch: descriptor too large");
    memcpy(&op.u, desc, desc_size);
    int rc = launch_op(op, nullptr, static_cast<cudaStream_t>(stream));
    if (rc) {
        char buf[128];
        snprintf(buf, sizeof buf, "ds_op_launch: op type %d failed rc=%d cuda=%s", op_type, rc, cudaGetErrorString(cudaGetLastError()));
        return fail(rc, buf);
    }
    return 0;
}

int ds_op_check(int op_type, const void* desc, size_t desc_size) {
    ds_plan_op op;
    memset(&op, 0, sizeof op);
    op.type = op_type;
    if (desc_size > sizeof(op.u)) return fail(-1, "ds_op_check: descriptor too large");
    memcpy(&op.u, desc, desc_size);
    const dsb::OpCheck c = check_op(op);
    return c.rc ? fail(c.rc, c.rule) : 0;
}

}  // extern "C"

"""ctypes mirrors of the descriptor structs in csrc/ops.h (field order and types must match exactly;
`_lib.py` checks every sizeof against the library's ds_sizeof())."""
import ctypes as C

P = C.c_uint64      # pointer fields: absolute device address or a reference (space << 60 | offset)
I32 = C.c_int32
I64 = C.c_int64
F32 = C.c_float
F64 = C.c_double

DS_OP_GEMM, DS_OP_GN_STATS, DS_OP_GN_APPLY, DS_OP_SOFTMAX, DS_OP_POSEMB, DS_OP_LINEAR = 1, 2, 3, 4, 5, 6
DS_OP_PREP_INPUT, DS_OP_CHANMEAN, DS_OP_MEMSET, DS_OP_LAYERNORM, DS_OP_GEGLU, DS_OP_GN_FINALIZE, DS_OP_ATTN, DS_OP_EMBED = 7, 8, 9, 10, 11, 12, 13, 14
DS_OP_OPT_PREP, DS_OP_OPT_SOFTMAX, DS_OP_OPT_REDUCE, DS_OP_OPT_KNN = 15, 16, 17, 18
DS_OP_IMG_INPUT, DS_OP_IM2COL, DS_OP_POOL = 19, 20, 21
DS_OP_CLIP_INPUT, DS_OP_CLIP_HEAD = 22, 23
DS_OP_PRDC_KTH, DS_OP_PRDC_COUNT = 24, 25
DS_PRDC_KMAX, DS_PRDC_LIST = 63, 1024     # csrc/ops.h: largest nearest_k of prdc_kth, length of its rescoring list
DS_CLIP_GATHER, DS_CLIP_L2NORM, DS_CLIP_SCORE = 0, 1, 2
DS_POOL_MAX, DS_POOL_AVG, DS_POOL_MEAN = 0, 1, 2
DS_IO_X, DS_IO_D, DS_IO_SIGMA, DS_IO_LABELS, DS_IO_BOTTLENECK, DS_IO_CTX, DS_IO_COUNT = 0, 1, 2, 3, 4, 5, 6
DS_M_X0, DS_M_EPS, DS_M_DIV, DS_M_NONE = 0, 1, 2, 3
DS_F8_SH_A16, DS_F8_SH_LO8, DS_F8_SH_HI8 = 6, 13, 2      # csrc/ops.h: power-of-two operand scales of the f8 GEMM mode
# csrc/ops.h: optimal-denoiser constants (band cap, P scale, band width in nats, rescoring threshold tau, u error per ||x|| ||y||)
DS_OPT_CAP, DS_OPT_P_SHIFT, DS_OPT_BAND_NATS, DS_OPT_TAU, DS_OPT_EPS = 1024, 15, 40, 0.01, 2.0 ** -17
DS_OPT_PLAIN, DS_OPT_RESCORED, DS_OPT_UNREFINED = 0, 1, 2
DS_KNN_MAX, DS_KNN_CAND = 64, 256

SPACE_ABS, SPACE_ARENA, SPACE_WEIGHTS, SPACE_IO = 0, 1, 2, 3


def ref(space, offset):
    return (space << 60) | int(offset)


class GemmDesc(C.Structure):
    _fields_ = [
        ('a_ptr', P), ('a_dims', I64 * 4), ('a_strides', I64 * 3), ('a_box', I32 * 4), ('a_plane_n', I32),
        ('a2_ptr', P), ('a2_c', I64), ('a2_plane_n', I32), ('nkb_aux', I32),
        ('b_ptr', P), ('b_dims', I64 * 3), ('b_strides', I64 * 2), ('b_plane_batch', I32),
        ('BN', I32), ('m_tiles', I32), ('n_tiles', I32), ('num_z', I32), ('nh', I32),
        ('taps', I32), ('cpb', I32), ('npass', I32), ('a_mode', I32), ('conv_H', I32), ('conv_W', I32),
        ('a_c_per_zh', I32), ('a_n_per_zb', I32), ('a_n_per_zh', I32),
        ('b_k0', I32), ('b_k_per_zh', I32), ('b_row_per_zh', I32), ('b_z_per_zb', I32), ('b_z_per_zh', I32),
        ('m_valid', I32), ('n_valid', I32),
        ('out_f32', P), ('out_h16', P), ('o_zb', I64), ('o_zh', I64), ('ldo', I64), ('o_plane', I64),
        ('bias_n', P), ('bias_m', P), ('rowvec', P), ('rowvec_stride', I64), ('rows_per_sample', I32), ('f8', I32),
        ('residual', P), ('ldr', I64), ('scale', F32),
        ('edm_out', I32), ('edm_x', P), ('edm_coef', P), ('edm_coef_stride', I32), ('edm_C', I32), ('edm_D', P),
        ('st_quads', P),
        ('tap_dh', I32 * 9), ('tap_dw', I32 * 9), ('tap_cb', I32 * 9), ('acc_scale', F32), ('st_unit', I32),
        ('relu', I32),
    ]


class GnStatsDesc(C.Structure):
    _fields_ = [('src0', P), ('src1', P), ('C0', I32), ('C1', I32), ('HW', I32), ('B', I32), ('groups', I32), ('pad0', I32),
                ('sums', P)]


class GnApplyDesc(C.Structure):
    _fields_ = [('src0', P), ('src1', P), ('C0', I32), ('C1', I32), ('H', I32), ('W', I32), ('B', I32), ('groups', I32),
                ('sums', P), ('gamma', P), ('beta', P), ('eps', F32), ('silu', I32), ('ada', P), ('ada_stride', I64),
                ('resample', I32), ('nplanes', I32), ('out_act', P), ('out_raw', P), ('out_raw_f32', P), ('fmt', I32), ('pad0', I32), ('coef', P)]


class SoftmaxDesc(C.Structure):
    _fields_ = [('S', P), ('P', P), ('rows', I64), ('L', I32), ('nplanes', I32), ('pitch_in', I32), ('pitch_out', I32)]


class PosembDesc(C.Structure):
    _fields_ = [('sigma', P), ('nsig', I32), ('num_channels', I32), ('endpoint', I32), ('swap_sincos', I32),
                ('sigma_data', F32), ('mode', I32), ('coef', P), ('emb', P), ('noise_scale', F32), ('pad0', I32)]


class LinearDesc(C.Structure):
    _fields_ = [('in_', P), ('in_stride', I64), ('W', P), ('b', P), ('add', P), ('add_stride', I64), ('out', P),
                ('n_rows', I32), ('in_f', I32), ('out_f', I32), ('act', I32), ('in_scale', F32), ('pad0', I32)]


class PrepInputDesc(C.Structure):
    _fields_ = [('x', P), ('coef', P), ('coef_stride', I32), ('B', I32), ('C', I32), ('HW', I32), ('nplanes', I32),
                ('x_batch', I32), ('out', P), ('codebook', P), ('idx', P), ('n_embed', I32), ('pad0', I32)]


class ChanmeanDesc(C.Structure):
    _fields_ = [('src', P), ('out', P), ('rows', I64), ('C', I32), ('pad0', I32)]


class LayernormDesc(C.Structure):
    _fields_ = [('src', P), ('gamma', P), ('beta', P), ('out', P), ('rows', I64), ('C', I32), ('nplanes', I32), ('eps', F32), ('fmt', I32)]


class GegluDesc(C.Structure):
    _fields_ = [('src', P), ('out', P), ('rows', I64), ('I', I32), ('nplanes', I32), ('fmt', I32), ('mode', I32)]


class GnFinalizeDesc(C.Structure):
    _fields_ = [('quads0', P), ('quads1', P), ('C0', I32), ('C1', I32), ('slabs_per_sample', I32), ('B', I32), ('groups', I32),
                ('unit0', I32), ('sums', P), ('gamma', P), ('beta', P), ('ada', P), ('ada_stride', I64), ('eps', F32), ('HW', I32), ('coef', P),
                ('unit1', I32), ('pad1', I32)]


class AttnDesc(C.Structure):
    _fields_ = [('q', P), ('k', P), ('vt', P), ('out', P), ('B', I32), ('nh', I32), ('L', I32), ('Lk', I32),
                ('q_pitch', I32), ('q_c0', I32), ('k_pitch', I32), ('k_c0', I32), ('vt_pitch', I32), ('o_pitch', I32),
                ('nplanes', I32), ('scale', F32), ('causal', I32), ('pad0', I32)]


class EmbedDesc(C.Structure):
    _fields_ = [('ids', P), ('tok', P), ('pos', P), ('out', P), ('rows', I64), ('T', I32), ('C', I32), ('vocab', I32), ('pad0', I32)]


class OptPrepDesc(C.Structure):
    _fields_ = [('x', P), ('planes', P), ('xn2', P), ('B', I32), ('D', I32), ('pitch', I32), ('pad0', I32)]


class OptSoftmaxDesc(C.Structure):
    _fields_ = [('part', P), ('hy2', P), ('xn2', P), ('sigma', P), ('x', P), ('y', P), ('P', P), ('status', P), ('ldp', I64), ('ldP', I64),
                ('B', I32), ('N', I32), ('D', I32), ('nslice', I32), ('nsig', I32), ('ymax', F32)]


class OptReduceDesc(C.Structure):
    _fields_ = [('part', P), ('out', P), ('rows', I64), ('cols', I32), ('ld', I32), ('nsplit', I32), ('scale', F32)]


class OptKnnDesc(C.Structure):
    _fields_ = [('part', P), ('hy2', P), ('xn2', P), ('x', P), ('y', P), ('dist', P), ('idx', P), ('ldp', I64),
                ('B', I32), ('N', I32), ('D', I32), ('nslice', I32), ('k', I32), ('ymax', F32)]


class ImgInputDesc(C.Structure):
    _fields_ = [('src', P), ('out', P), ('sn', I64), ('sc', I64), ('sy', I64), ('sx', I64), ('B', I32), ('C', I32), ('H', I32), ('W', I32),
                ('Ho', I32), ('Wo', I32)]


class Im2colDesc(C.Structure):
    _fields_ = [('src', P), ('out', P), ('B', I32), ('H', I32), ('W', I32), ('C', I32), ('src_pitch', I32), ('src_c0', I32),
                ('kh', I32), ('kw', I32), ('sh', I32), ('sw', I32), ('ph', I32), ('pw', I32), ('K64', I32), ('nplanes', I32)]


class PoolDesc(C.Structure):
    _fields_ = [('src', P), ('out_f32', P), ('out_h16', P), ('B', I32), ('H', I32), ('W', I32), ('C', I32), ('src_pitch', I32),
                ('src_c0', I32), ('out_pitch', I32), ('out_c0', I32), ('k', I32), ('stride', I32), ('pad', I32), ('mode', I32),
                ('nplanes', I32), ('pad0', I32)]


class ClipInputDesc(C.Structure):
    _fields_ = [('src', P), ('tab', P), ('out', P), ('sn', I64), ('sc', I64), ('sy', I64), ('sx', I64), ('B', I32), ('H', I32), ('W', I32),
                ('S', I32), ('ky', I32), ('kx', I32), ('mean', F32 * 3), ('std', F32 * 3)]


class ClipHeadDesc(C.Structure):
    _fields_ = [('src', P), ('src2', P), ('ids', P), ('out', P), ('src_stride', I64), ('out_stride', I64), ('B', I32), ('C', I32), ('T', I32),
                ('row', I32), ('mode', I32), ('scale', F32)]


class PrdcKthDesc(C.Structure):
    _fields_ = [('part', P), ('q', P), ('t', P), ('qn2', P), ('tn2', P), ('rad', P), ('rad2', P), ('nres', P), ('ldp', I64),
                ('B', I32), ('N', I32), ('D', I32), ('nslice', I32), ('k', I32), ('pad0', I32), ('sq', F64), ('st', F64)]


class PrdcCountDesc(C.Structure):
    _fields_ = [('part', P), ('q', P), ('t', P), ('qn2', P), ('tn2', P), ('tau', P), ('tau2', P), ('rho', P), ('rho2', P), ('cnt_t', P),
                ('cnt_own', P), ('realism', P), ('nres', P), ('ldp', I64), ('B', I32), ('N', I32), ('D', I32), ('nslice', I32),
                ('sq', F64), ('st', F64), ('med', F64)]


class MemsetDesc(C.Structure):
    _fields_ = [('ptr', P), ('bytes', I64)]


class _OpUnion(C.Union):
    _fields_ = [('gemm', GemmDesc), ('gn_stats', GnStatsDesc), ('gn_apply', GnApplyDesc), ('softmax', SoftmaxDesc),
                ('posemb', PosembDesc), ('linear', LinearDesc), ('prep_input', PrepInputDesc), ('chanmean', ChanmeanDesc),
                ('memset', MemsetDesc), ('layernorm', LayernormDesc), ('geglu', GegluDesc), ('gn_finalize', GnFinalizeDesc), ('attn', AttnDesc),
                ('embed', EmbedDesc), ('opt_prep', OptPrepDesc), ('opt_softmax', OptSoftmaxDesc), ('opt_reduce', OptReduceDesc),
                ('opt_knn', OptKnnDesc), ('img_input', ImgInputDesc), ('im2col', Im2colDesc), ('pool', PoolDesc),
                ('clip_input', ClipInputDesc), ('clip_head', ClipHeadDesc), ('prdc_kth', PrdcKthDesc), ('prdc_count', PrdcCountDesc)]


class PlanOp(C.Structure):
    _fields_ = [('type', I32), ('tag', I32), ('u', _OpUnion)]


SIZEOF_CHECKS = {
    0: PlanOp, DS_OP_GEMM: GemmDesc, DS_OP_GN_STATS: GnStatsDesc, DS_OP_GN_APPLY: GnApplyDesc, DS_OP_SOFTMAX: SoftmaxDesc,
    DS_OP_POSEMB: PosembDesc, DS_OP_LINEAR: LinearDesc, DS_OP_PREP_INPUT: PrepInputDesc, DS_OP_CHANMEAN: ChanmeanDesc,
    DS_OP_MEMSET: MemsetDesc, DS_OP_LAYERNORM: LayernormDesc, DS_OP_GEGLU: GegluDesc, DS_OP_GN_FINALIZE: GnFinalizeDesc, DS_OP_ATTN: AttnDesc,
    DS_OP_EMBED: EmbedDesc, DS_OP_OPT_PREP: OptPrepDesc, DS_OP_OPT_SOFTMAX: OptSoftmaxDesc, DS_OP_OPT_REDUCE: OptReduceDesc,
    DS_OP_OPT_KNN: OptKnnDesc, DS_OP_IMG_INPUT: ImgInputDesc, DS_OP_IM2COL: Im2colDesc, DS_OP_POOL: PoolDesc,
    DS_OP_CLIP_INPUT: ClipInputDesc, DS_OP_CLIP_HEAD: ClipHeadDesc, DS_OP_PRDC_KTH: PrdcKthDesc, DS_OP_PRDC_COUNT: PrdcCountDesc,
}

# Union member of each op type of the network plans (plan.py, ldm_plan.py, vae_plan.py, clip_plan.py) ...
UNION_FIELD = {
    DS_OP_GEMM: 'gemm', DS_OP_GN_STATS: 'gn_stats', DS_OP_GN_APPLY: 'gn_apply', DS_OP_SOFTMAX: 'softmax', DS_OP_POSEMB: 'posemb',
    DS_OP_LINEAR: 'linear', DS_OP_PREP_INPUT: 'prep_input', DS_OP_CHANMEAN: 'chanmean', DS_OP_MEMSET: 'memset',
    DS_OP_LAYERNORM: 'layernorm', DS_OP_GEGLU: 'geglu', DS_OP_GN_FINALIZE: 'gn_finalize', DS_OP_ATTN: 'attn', DS_OP_EMBED: 'embed',
}
# ... and of the ops only the optimal-denoiser plans (optimal.py) use around their two GEMMs.
OPT_UNION_FIELD = {DS_OP_OPT_PREP: 'opt_prep', DS_OP_OPT_SOFTMAX: 'opt_softmax', DS_OP_OPT_REDUCE: 'opt_reduce', DS_OP_OPT_KNN: 'opt_knn'}
# ... and of the ops only the Inception-v3 feature extractor (inception_plan.py) uses around its GEMMs.
INCEPTION_UNION_FIELD = {DS_OP_IMG_INPUT: 'img_input', DS_OP_IM2COL: 'im2col', DS_OP_POOL: 'pool'}
# ... and of the ops only the CLIP-score towers (openclip_plan.py) add.
OPENCLIP_UNION_FIELD = {DS_OP_CLIP_INPUT: 'clip_input', DS_OP_CLIP_HEAD: 'clip_head'}
# ... and of the ops only the PRDC plans (prdc.py) add.
PRDC_UNION_FIELD = {DS_OP_PRDC_KTH: 'prdc_kth', DS_OP_PRDC_COUNT: 'prdc_count'}
ALL_UNION_FIELD = {**UNION_FIELD, **OPT_UNION_FIELD, **INCEPTION_UNION_FIELD, **OPENCLIP_UNION_FIELD, **PRDC_UNION_FIELD}
OP_TYPE_OF = {GemmDesc: DS_OP_GEMM, GnStatsDesc: DS_OP_GN_STATS, GnApplyDesc: DS_OP_GN_APPLY, SoftmaxDesc: DS_OP_SOFTMAX,
              PosembDesc: DS_OP_POSEMB, LinearDesc: DS_OP_LINEAR, PrepInputDesc: DS_OP_PREP_INPUT, ChanmeanDesc: DS_OP_CHANMEAN,
              MemsetDesc: DS_OP_MEMSET, LayernormDesc: DS_OP_LAYERNORM, GegluDesc: DS_OP_GEGLU, GnFinalizeDesc: DS_OP_GN_FINALIZE, AttnDesc: DS_OP_ATTN,
              EmbedDesc: DS_OP_EMBED, OptPrepDesc: DS_OP_OPT_PREP, OptSoftmaxDesc: DS_OP_OPT_SOFTMAX, OptReduceDesc: DS_OP_OPT_REDUCE,
              OptKnnDesc: DS_OP_OPT_KNN, ImgInputDesc: DS_OP_IMG_INPUT, Im2colDesc: DS_OP_IM2COL, PoolDesc: DS_OP_POOL,
              ClipInputDesc: DS_OP_CLIP_INPUT, ClipHeadDesc: DS_OP_CLIP_HEAD, PrdcKthDesc: DS_OP_PRDC_KTH, PrdcCountDesc: DS_OP_PRDC_COUNT}

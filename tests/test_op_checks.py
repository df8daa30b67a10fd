"""The launchers' descriptor checks (ds_op_check, csrc/ops.h) without a GPU: every op of the plans the project compiles passes them, and
for every rule the smallest descriptor that breaks it is refused with the launcher's code and the rule's name while its nearest valid
neighbour is accepted.  On the GPU, ds_unet_create refuses a plan with one broken op and names that op.  (The full-size
Consistency-Models plans are checked in tests/test_cm_host.py.)"""
import ctypes

import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import _lib
from diff_sampler_b200 import gemm_desc as G


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    return g._load_build_module().build()


def _refused(pl):
    """(op index, type, tag, rule) of every op of plan `pl` that its launcher would refuse."""
    out = []
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        why = _lib.op_check(getattr(op.u, S.ALL_UNION_FIELD[op.type]))
        if why:
            out.append((i, op.type, op.tag, why))
    return out


def _vq_f4_plans():
    import vq_ref as VQ
    from diff_sampler_b200 import vae_plan
    P, _ = VQ.make_params('vq_f4')
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    yield 'vq_f4 64->256', vae_plan.compile_vae_plan(mods, meta, wb, 1, 64, quantize=True, debug_indices=True)


def _optimal_plans():
    """The optimal-denoiser plans of tests/test_optimal_host.py, and CIFAR-10's 50 000 x 3072 dataset (only the blob layout is needed)."""
    from diff_sampler_b200 import optimal as OPT
    for N, D, B, nsig, knn in ((300, 192, 4, 1, 0), (65, 105, 3, 3, 0), (130, 48, 2, 1, 5), (70, 105, 3, 3, 0), (70, 105, 3, 3, 4),
                               (50000, 3072, 16, 16, 0), (50000, 3072, 16, 1, 5)):
        g = OPT._Geometry(N, D)
        wb, _ = OPT.blob_layout(g)
        yield f'optimal N{N} D{D} B{B} s{nsig} knn{knn}', OPT.compile_plan(g, wb, B, nsig, 1.0, knn=knn)


def _family(name):
    import plan_digest
    if name == 'vq_f4':
        yield from _vq_f4_plans()
    elif name == 'optimal':
        yield from _optimal_plans()
    else:
        for key, pl, _ in getattr(plan_digest, name)():
            yield key, pl


@pytest.mark.parametrize('family', ['_edm_variants', '_small_variants', '_benchmarked', 'vq_f4', 'optimal'])
def test_every_plan_op_passes_its_launcher_check(built, family):
    n = 0
    for key, pl in _family(family):
        assert not _refused(pl), (key, _refused(pl)[:5])
        n += pl.n_ops
    print(f'{family}: {n} ops accepted')
    assert n > 0


# ---------------------------------------------------------------------------------------------------- one rule at a time
def _with(desc, **kw):
    """A copy of desc with fields replaced; a dict value sets array elements by index, a list the whole array."""
    d = type(desc).from_buffer_copy(desc)
    for k, v in kw.items():
        if isinstance(v, dict):
            for i, x in v.items():
                getattr(d, k)[i] = x
        elif isinstance(v, list):
            getattr(d, k)[:] = v
        else:
            setattr(d, k, v)
    return d


def _gemm():
    d, _ = G.conv_gemm(1, 2, 8, 8, 64, 1, 64)                      # 3x3 conv 64 -> 64 over 2 x 8 x 8, box (64, 8, 8, 2)
    return d


def _attn():
    return S.AttnDesc(q=1, k=1, vt=1, out=1, B=2, nh=2, L=64, Lk=64, q_pitch=128, q_c0=0, k_pitch=128, k_c0=0, vt_pitch=64, o_pitch=128,
                      nplanes=2, scale=0.125, causal=0)


def _gn_stats():
    return S.GnStatsDesc(src0=1, src1=0, C0=64, C1=0, HW=64, B=2, groups=32, sums=1)


def _gn_finalize():
    return S.GnFinalizeDesc(quads0=1, quads1=0, C0=64, C1=0, slabs_per_sample=2, B=2, groups=16, unit0=0, sums=1, gamma=1, beta=1, eps=1e-5,
                            HW=64, coef=1, unit1=0)


def _gn_apply():
    return S.GnApplyDesc(src0=1, src1=0, C0=64, C1=0, H=8, W=8, B=2, groups=32, sums=1, coef=0, gamma=1, beta=1, eps=1e-5, silu=1,
                         resample=0, nplanes=2, fmt=0, out_act=1)


def _linear():
    return S.LinearDesc(in_=1, W=1, out=1, n_rows=2, in_f=64, out_f=64, in_scale=1.0)


# (descriptor, the rule, [fields that break it], [nearest fields that do not]); every rule of csrc/ops.h's checks appears.
RULES = [
    (_gemm, -10, 'gemm: BN', [dict(BN=8), dict(BN=264), dict(BN=44)], [dict(BN=16), dict(BN=256), dict(BN=48)]),
    (_gemm, -11, 'gemm: a_box', [dict(a_box=[64, 8, 8, 1]), dict(a_box=[32, 8, 8, 4])], [dict(a_box=[64, 8, 16, 1])]),
    (_gemm, -12, 'gemm: npass', [dict(npass=2)], [dict(npass=1)]),
    (_gemm, -1, 'gemm: A tensor map', [dict(a_dims={3: (1 << 32) + 1}), dict(a_strides={0: 136}), dict(a_strides={2: 1 << 40})],
     [dict(a_dims={3: 1 << 32}), dict(a_strides={0: 144}), dict(a_strides={2: (1 << 40) - 16})]),
    (_gemm, -14, 'gemm: st_unit', [dict(st_unit=3)], [dict(st_unit=2)]),
    (_gemm, -16, 'gemm: f8', [dict(f8=1, a_plane_n=0), dict(f8=1, npass=1), dict(f8=1, a_mode=1), dict(f8=1, num_z=2)], [dict(f8=1)]),
    (_gemm, -16, 'gemm: f8 with tap_cb', [dict(f8=1, tap_cb={8: 64})], [dict(tap_cb={8: 64})]),
    (_gemm, -15, 'gemm: taps', [dict(taps=3)], [dict(taps=1)]),
    (_gemm, -13, 'gemm: row segment', [dict(conv_W=192, a_box=[64, 128, 1, 1]), dict(conv_W=256, a_box=[64, 64, 2, 1])],
     [dict(conv_W=256, a_box=[64, 128, 1, 1])]),
    (_gemm, -14, 'gemm: st_quads', [dict(st_quads=1, m_valid=112), dict(st_quads=1, n_valid=62), dict(st_quads=1, edm_out=2),
                                    dict(st_quads=1, num_z=2), dict(st_quads=1, st_unit=4, n_valid=66)],
     [dict(st_quads=1, m_valid=96), dict(st_quads=1, st_unit=2, n_valid=62)]),
    (_attn, -30, 'attn: args', [dict(nplanes=1), dict(Lk=0), dict(B=0), dict(nh=0), dict(L=0), dict(scale=0.0)], [dict(Lk=8)]),
    (_attn, -31, 'attn: pitch', [dict(o_pitch=132), dict(q_c0=4, q_pitch=256), dict(vt_pitch=68)], [dict(o_pitch=136)]),
    (_attn, -32, 'attn: extent', [dict(Lk=65), dict(q_c0=8), dict(o_pitch=120), dict(k_c0=8)], [dict(Lk=64, q_c0=8, q_pitch=136)]),
    (_attn, -40, 'attn: causal', [dict(causal=1, Lk=32)], [dict(causal=1)]),
    (_gn_stats, -2, 'gn_stats: channels', [dict(groups=24), dict(C0=66), dict(C0=62, C1=2), dict(groups=0), dict(groups=128, C0=256)],
     [dict(groups=16), dict(C0=64, C1=64)]),
    (_gn_stats, -2, 'gn_stats: one-channel groups', [dict(groups=64)], [dict(groups=32)]),
    (_gn_finalize, -2, 'gn_finalize: groups', [dict(groups=24), dict(groups=0), dict(groups=128, C0=256)], [dict(groups=8)]),
    (_gn_finalize, -2, 'gn_finalize: source units', [dict(C1=64), dict(C0=66, C1=62, quads1=1, groups=1)], [dict(C1=64, quads1=1)]),
    (_gn_finalize, -2, 'gn_finalize: group units', [dict(groups=32), dict(C0=46, C1=16, quads1=1, groups=31, unit0=2)],
     [dict(groups=32, unit0=2), dict(C0=46, C1=16, quads1=1, groups=31, unit0=2, unit1=2)]),
    (_gn_finalize, -2, 'gn_finalize: nothing to do', [dict(quads0=0, coef=0)], [dict(quads0=0)]),
    (_gn_finalize, -2, 'gn_finalize: coef inputs', [dict(gamma=0), dict(beta=0), dict(HW=0)], [dict(coef=0, gamma=0, beta=0, HW=0)]),
    (_gn_finalize, -2, 'gn_finalize: shared memory', [dict(C0=6144, groups=64), dict(quads0=0, C0=6144, groups=64)],
     [dict(C0=6140, groups=5), dict(quads0=0, C0=6142, groups=2)]),
    (_gn_apply, -2, 'gn_apply: channels', [dict(C0=60), dict(C0=60, C1=4)], [dict(C0=56), dict(C0=56, C1=8)]),
    (_gn_apply, -2, 'gn_apply: width', [dict(C0=4104), dict(C0=4096, C1=8)], [dict(C0=4096), dict(C0=4088, C1=8)]),
    (_gn_apply, -2, 'gn_apply: fmt', [dict(fmt=1, nplanes=1), dict(fmt=1, resample=3), dict(fmt=2)], [dict(fmt=1), dict(fmt=1, resample=1)]),
    (_gn_apply, -2, 'gn_apply: coef with resample', [dict(coef=1, resample=1), dict(coef=1, resample=2), dict(coef=1, resample=3)],
     [dict(coef=1)]),
    (_gn_apply, -2, 'gn_apply: statistics', [dict(sums=0), dict(sums=0, resample=1)], [dict(sums=0, coef=1), dict(sums=0, out_act=0, out_raw=1)]),
    (_gn_apply, -2, 'gn_apply: resample parity', [dict(resample=1, H=7), dict(resample=1, W=7), dict(resample=3, H=7), dict(resample=3, W=7)],
     [dict(resample=1), dict(resample=3), dict(resample=2, H=7, W=7)]),
    (_gn_apply, -2, 'gn_apply: coef width', [dict(coef=1, sums=0, C0=2056)], [dict(coef=1, sums=0, C0=2048), dict(coef=1, C0=2056)]),
    (_linear, -2, 'linear: in_f', [dict(in_f=2049)], [dict(in_f=2048)]),
    (lambda: S.PrepInputDesc(x=1, coef=1, B=2, C=3, HW=64, nplanes=2, out=1), -2, 'prep_input: C', [dict(C=65)], [dict(C=64)]),
    (lambda: S.PrepInputDesc(x=1, coef=1, B=2, C=3, HW=64, nplanes=2, out=1, codebook=1, n_embed=16), -2, 'prep_input: codebook',
     [dict(C=9), dict(n_embed=0)], [dict(C=8), dict(n_embed=1), dict(C=9, codebook=0)]),
    (lambda: S.LayernormDesc(src=1, gamma=1, beta=1, out=1, rows=4, C=64, nplanes=2, eps=1e-5, fmt=0), -2, 'layernorm: C',
     [dict(C=2052), dict(C=62)], [dict(C=2048), dict(C=60)]),
    (lambda: S.LayernormDesc(src=1, gamma=1, beta=1, out=1, rows=4, C=64, nplanes=2, eps=1e-5, fmt=1), -2, 'layernorm: f8 planes',
     [dict(nplanes=1)], [dict(nplanes=1, fmt=2), dict(nplanes=1, fmt=0)]),
    (lambda: S.GegluDesc(src=1, out=1, rows=4, I=64, nplanes=2, fmt=0, mode=0), -2, 'geglu: I', [dict(I=62)], [dict(I=60)]),
    (lambda: S.GegluDesc(src=1, out=1, rows=4, I=64, nplanes=2, fmt=0, mode=1), -2, 'geglu: quick-GELU fmt', [dict(fmt=1)], [dict(fmt=0)]),
    (lambda: S.GegluDesc(src=1, out=1, rows=4, I=64, nplanes=2, fmt=1, mode=0), -2, 'geglu: f8 planes', [dict(nplanes=1)],
     [dict(nplanes=2), dict(nplanes=1, fmt=0)]),
    (lambda: S.EmbedDesc(ids=1, tok=1, pos=1, out=1, rows=4, T=2, C=8, vocab=10), -2, 'embed: shape',
     [dict(C=6), dict(rows=0), dict(T=0), dict(vocab=0)], [dict(C=4), dict(rows=1), dict(T=1), dict(vocab=1)]),
    (lambda: S.OptPrepDesc(x=1, planes=1, xn2=1, B=2, D=48, pitch=48), -1, 'opt_prep: shape',
     [dict(pitch=52), dict(pitch=40), dict(B=0), dict(D=0)], [dict(pitch=56), dict(D=40, pitch=40)]),
    (lambda: S.OptSoftmaxDesc(part=1, hy2=1, xn2=1, sigma=1, x=1, y=1, P=1, B=2, N=100, D=48, nslice=1, ldp=104, ldP=104, nsig=1), -1,
     'opt_softmax: shape', [dict(ldP=96), dict(ldp=99), dict(nslice=0), dict(B=0), dict(N=0)], [dict(ldP=100, ldp=100)]),
    (lambda: S.OptSoftmaxDesc(part=1, hy2=1, xn2=1, sigma=1, x=1, y=1, P=1, B=2, N=100, D=48, nslice=1, ldp=104, ldP=104, nsig=1), -1,
     'opt_softmax: nsig', [dict(nsig=3), dict(nsig=0)], [dict(nsig=2)]),
    (lambda: S.OptReduceDesc(part=1, out=1, rows=2, cols=48, ld=48, nsplit=2, scale=1.0), -1, 'opt_reduce: shape',
     [dict(ld=44), dict(nsplit=0), dict(rows=0), dict(cols=0)], [dict(ld=52), dict(nsplit=1)]),
    (lambda: S.OptKnnDesc(part=1, hy2=1, xn2=1, x=1, y=1, dist=1, idx=1, ldp=104, B=2, N=100, D=48, nslice=1, k=5), -1, 'opt_knn: shape',
     [dict(ldp=96), dict(B=0), dict(N=0)], [dict(ldp=100)]),
    (lambda: S.OptKnnDesc(part=1, hy2=1, xn2=1, x=1, y=1, dist=1, idx=1, ldp=104, B=2, N=100, D=48, nslice=1, k=5), -1, 'opt_knn: k',
     [dict(k=0), dict(k=S.DS_KNN_MAX + 1), dict(k=40, N=39, ldp=40)], [dict(k=S.DS_KNN_MAX), dict(k=39, N=39, ldp=40)]),
]


def _rc(desc):
    return _lib.load().ds_op_check(S.OP_TYPE_OF[type(desc)], ctypes.byref(desc), ctypes.sizeof(desc))


@pytest.mark.parametrize('make,rc,rule,bad,good', RULES, ids=[r[2] for r in RULES])
def test_each_rule_refuses_what_breaks_it_and_accepts_its_neighbour(built, make, rc, rule, bad, good):
    base = make()
    assert _lib.op_check(base) is None, _lib.op_check(base)
    for kw in bad:
        d = _with(base, **kw)
        assert (_rc(d), _lib.op_check(d)) == (rc, rule), kw
    for kw in good:
        d = _with(base, **kw)
        assert _lib.op_check(d) is None, (kw, _lib.op_check(d))


def test_rule_free_ops_and_unknown_types(built):
    """Posemb, softmax, chanmean and memset have no descriptor rules; an unknown op type is refused as the plan executor refuses it."""
    for desc in (S.PosembDesc(), S.SoftmaxDesc(), S.ChanmeanDesc(), S.MemsetDesc()):
        assert _lib.op_check(desc) is None
    lib = _lib.load()
    d = S.MemsetDesc()
    assert lib.ds_op_check(99, ctypes.byref(d), ctypes.sizeof(d)) == -100
    assert lib.ds_op_check(S.DS_OP_MEMSET, ctypes.byref(d), ctypes.sizeof(S.PlanOp)) == -1          # larger than any descriptor


# ---------------------------------------------------------------------------------------------------- plan creation
@pytest.mark.gpu
def test_unet_create_refuses_a_plan_with_a_broken_op(built):
    """A plan whose one gn_apply has the coefficient table set together with a 2x2 pool is refused by ds_unet_create with that op's
    index, tag and rule, and no handle is made, so no forward can run; the intact plan is accepted."""
    import plan_digest
    key, pl, blob = next(plan_digest._edm_variants())
    plans = _lib.NativePlans(blob, torch.device('cuda', 0))
    plans.get('intact', lambda: pl)
    i = next(i for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_GN_APPLY and pl.ops_array[i].u.gn_apply.resample == 0)
    op = pl.ops_array[i]
    op.u.gn_apply.resample = 1
    op.u.gn_apply.coef = op.u.gn_apply.coef or op.u.gn_apply.sums
    with pytest.raises(_lib.DsError, match=rf'op {i} \(type {S.DS_OP_GN_APPLY} tag {op.tag}\) refused \(rc -2\): gn_apply: coef with resample'):
        plans.get('broken', lambda: pl)
    assert 'broken' not in plans.plans

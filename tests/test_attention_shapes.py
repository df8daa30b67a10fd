"""Inventory of the attentions and row softmaxes the compiled plans launch (no GPU needed).

Every plan tests/plan_digest.py compiles -- the tiny interpreter variants, the compile options (EDM without flash attention among
them), the full-size and the benchmarked nets -- and the tiny SD net with flash_attn=False is reduced to its DS_OP_ATTN and
DS_OP_SOFTMAX descriptors.  Each descriptor is classed as tests/test_gpu_attention.py organises its sweep (attn_class,
softmax_class there), and every class must be one that sweep runs on the GPU.  A plan that launches an attention or a softmax the
sweep never ran fails here, before anyone reaches an H100.  attn_wide_kernel is swept in tests/test_gpu_openclip.py; its classes
come from that module's constants."""
import pytest

import plan_digest
import test_gpu_attention as A
import test_gpu_openclip as W
from diff_sampler_b200 import _cstructs as S


def _tiny_ldm_unfused():
    from diff_sampler_b200 import ldm_plan
    from oracle import ldm_oracle as LO
    P, cfg = LO.make_params('tiny_ldm')
    st = ldm_plan.ldm_structure(P, cfg['num_heads'])
    wb, info = ldm_plan.pack_ldm_weights(st, P)
    yield 'ldm/tiny_ldm/flash_attn=0', ldm_plan.compile_ldm_plan(st, wb, info, 2, 2, 1, cfg['img_resolution'], flash_attn=False), None


def _attn_of(d):
    hd = 64 if d.pad0 == 0 else d.pad0
    kernel = 'pair' if hd == 32 else ('wide' if hd > 64 else 'attn')
    return A.attn_class(kernel, hd, d.q == d.k, d.causal, d.L, d.Lk)


def _wide_classes():
    """The classes test_gpu_openclip.py's wide-kernel sweep runs: plan-layout self-attention at every width and key count, and
    cross-attention from separate buffers."""
    out = {A.attn_class('wide', hd, True, 0, Lk, Lk) for hd in W.WIDE_HDS for Lk in W.WIDE_LKS}
    return out | {A.attn_class('wide', hd, False, 0, L, Lk) for hd in W.WIDE_HDS for L in W.WIDE_LS for Lk in (1, 65, 730)}


@pytest.fixture(scope='module')
def launched():
    """class -> the first (plan, op index) that launches it, for attention and softmax descriptors."""
    attn, smax = {}, {}
    gens = [plan_digest._edm_variants(), plan_digest._edm_options(), plan_digest._cm_variants(), plan_digest._uncond_ldm_variants(),
            plan_digest._vq_variants(), plan_digest._small_variants(), plan_digest._benchmarked(), _tiny_ldm_unfused()]
    for gen in gens:
        for key, pl, _ in gen:
            for i in range(pl.n_ops):
                op = pl.ops_array[i]
                if op.type == S.DS_OP_ATTN:
                    attn.setdefault(_attn_of(op.u.attn), (key, i))
                elif op.type == S.DS_OP_SOFTMAX:
                    d = op.u.softmax
                    smax.setdefault(A.softmax_class(d.L, d.pitch_in, d.pitch_out), (key, i))
    return attn, smax


def test_every_launched_attention_is_swept(launched):
    swept = {A.case_class(c) for c in A.ATTN_CASES} | _wide_classes()
    missing = {cls: where for cls, where in launched[0].items() if cls not in swept}
    print(f'{len(launched[0])} attention classes launched: {sorted(launched[0])}')
    assert launched[0] and not missing, \
        f'attentions no case of tests/test_gpu_attention.py runs ((kernel, head width, self, causal, L % 128, Lk % 64): first plan, op): {missing}'


def test_every_launched_softmax_is_swept(launched):
    swept = {A.softmax_case_class(c) for c in A.SOFTMAX_CASES}
    missing = {cls: where for cls, where in launched[1].items() if cls not in swept}
    print(f'{len(launched[1])} softmax classes launched: {sorted(launched[1])}')
    assert launched[1] and not missing, \
        f'row softmaxes no case of tests/test_gpu_attention.py runs ((kernel, pitch_in - L, pitch_out - L): first plan, op): {missing}'


def test_the_sweep_runs_every_softmax_kernel_and_both_fused_kernels():
    """The sweep reaches each of the launcher's six softmax kernels, and each fused kernel with self- and cross-attention, with and
    without the causal mask, and with whole and partial last query tiles and key blocks."""
    kernels = {A.softmax_case_class(c)[0] for c in A.SOFTMAX_CASES}
    assert kernels == {'reg2', 'reg8', 'cta4', 'cta8', 'warp_f4', 'warp_scalar'}
    classes = {A.case_class(c) for c in A.ATTN_CASES}
    for kernel, hd in (('attn', 64), ('pair', 32)):
        for self_attn in (True, False):
            for causal in (False, True):
                assert any(c[:4] == (kernel, hd, self_attn, causal) for c in classes), (kernel, self_attn, causal)
        for lq in ('whole', 'part'):
            for lk in ('whole', 'part'):
                assert (kernel, hd, False, False, lq, lk) in classes

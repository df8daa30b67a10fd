"""Host logic of the unconditional latent-diffusion eps-net (no GPU): the structure parsed from the LSUN-Bedroom / FFHQ LDM-VQ-f4
state-dict shapes, the legacy qkv reorder, the descriptors of channel remainders and head pairs, the launchers' new check rules, and
the constructor's argument errors."""
import json
import math
import os

import numpy as np
import pytest
import torch

import ldm_uncond_ref as U
from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import _lib
from diff_sampler_b200 import gemm_desc as G
from diff_sampler_b200 import ldm_plan


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    return g._load_build_module().build()


def _shape_params(name):
    """Zero tensors of the state-dict shapes (structure and descriptors only need the shapes)."""
    return {k: torch.zeros(v) for k, v in U.param_shapes(U.CONFIGS[name]).items()}


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_ldm_uncond.npz')


def _golden():
    return np.load(GOLDEN)


def _reference_shapes(name):
    """Names and shapes of the reference UNetModel's state dict (tools/gen_ldm_uncond_golden.py)."""
    return {k: tuple(v) for k, v in json.loads(bytes(_golden()['state_dict_shapes_json']).decode())[name]}


@pytest.mark.parametrize('name', ['tiny_uncond', 'ldm_vq4'])
def test_restated_state_dict_layout_is_the_reference_one(name):
    ref = json.loads(bytes(_golden()['state_dict_shapes_json']).decode())[name]
    ours = list(U.param_shapes(U.CONFIGS[name]).items())
    assert [(k, tuple(v)) for k, v in ref] == [(k, tuple(v)) for k, v in ours]


def test_oracle_against_the_reference_golden():
    """tests/ldm_uncond_ref.py (float64) against the reference UNetModel + CFGPrecond('uncond') run in float32: D at one and at
    per-sample sigma, the middle-block tap, the 'discrete' schedule and a DPM-Solver++(2M) sample."""
    from oracle import solvers_oracle as SO
    G = _golden()
    P, cfg = U.make_params('tiny_uncond')
    on = U.OracleUncondNet(P, cfg)
    assert np.allclose([on.sigma_min, on.sigma_max], G['sigma_range'], rtol=1e-6)
    x = torch.from_numpy(G['x'])
    for sigma in (14.6, 1.0, 0.05):
        on.taps = {}
        D = on(x * sigma, torch.tensor([sigma]))
        tap = on.taps['middle_block'].mean(dim=1)
        ref, rtap = torch.from_numpy(G[f'D/{sigma}']).double(), torch.from_numpy(G[f'tap/{sigma}']).double()
        assert (D - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item()), sigma
        assert (tap - rtap).abs().max().item() < 1e-5 * max(1.0, rtap.abs().max().item()), sigma
    on.taps = None
    sig = torch.tensor([5.0, 0.3])
    ref = torch.from_numpy(G['D/persample']).double()
    assert (on(x * sig[:, None, None, None], sig) - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
    kw = dict(num_steps=5, sigma_min=on.sigma_min, sigma_max=on.sigma_max, schedule_type='discrete', schedule_rho=1)
    assert np.allclose(SO.get_schedule(net=on, **kw).numpy(), G['sched_discrete'], rtol=1e-6)
    out = SO.sample(on, x.double(), 'dpm_pp', max_order=2, predict_x0=False, **kw)
    ref = torch.from_numpy(G['sample_dpmpp']).double()
    assert (out.double() - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


def test_full_size_structure_from_state_dict_shapes():
    """lsun_bedrooms-ldm-vq-4.yaml, from the reference UNetModel's state-dict shapes: attention at 32^2 / 16^2 / 8^2 over
    448 / 672 / 896 channels = 14 / 21 / 28 heads of 32."""
    st = ldm_plan.ldm_structure({k: torch.zeros(v) for k, v in _reference_shapes('ldm_vq4').items()}, 8, 32)
    assert st['model_channels'] == 224 and st['in_channels'] == 3 and st['out_channels'] == 3
    attn = [L for _, ls in st['inp'] + st['mid'] + st['out'] for L in ls if L[0] == 'qkv_attn']
    assert {(L[2], L[3], L[4]) for L in attn} == {(448, 14, 32), (672, 21, 32), (896, 28, 32)}
    assert len(attn) == 2 * 3 + 1 + 3 * 3
    assert not [L for _, ls in st['inp'] + st['mid'] + st['out'] for L in ls if L[0] == 'attn']
    cins = sorted({L[2] for _, ls in st['out'] for L in ls if L[0] == 'res'})
    assert 1568 in cins and 1120 in cins and 672 in cins


@pytest.mark.parametrize('heads', [3, 14, 21])
@pytest.mark.parametrize('pairs', [True, False])
def test_qkv_reorder_matches_legacy_attention(heads, pairs):
    """Attention over the reordered rows (q heads | k heads, v; 32- or 64-row head slots, a zero head to even the pairs) equals
    QKVAttentionLegacy over the reference's [head][q|k|v][d] rows, and the padded proj_out columns see only zeros."""
    torch.manual_seed(heads)
    d, T = 32, 20
    C = heads * d
    w, b = torch.randn(3 * C, C, dtype=torch.float64), torch.randn(3 * C, dtype=torch.float64)
    x = torch.randn(2, C, T, dtype=torch.float64)
    ref = U.legacy_attention(torch.einsum('oc,nct->not', w, x) + b[None, :, None], heads)
    wqk, bqk, wv, bv = (t.double() for t in ldm_plan._legacy_qkv_split(w, b, heads, pairs))
    hs, dp = (heads + heads % 2, 32) if pairs else (heads, 64)
    assert wqk.shape == (2 * hs * dp, C) and wv.shape == (hs * dp, C)
    qk = torch.einsum('oc,nct->nto', wqk, x) + bqk
    v = torch.einsum('oc,nct->nto', wv, x) + bv
    q, k = qk[..., :hs * dp].reshape(2, T, hs, dp), qk[..., hs * dp:].reshape(2, T, hs, dp)
    v = v.reshape(2, T, hs, dp)
    att = torch.softmax(torch.einsum('nthd,nshd->nhts', q, k) / math.sqrt(d), dim=-1)
    o = torch.einsum('nhts,nshd->nthd', att, v)
    if hs > heads:
        assert o[:, :, heads:].abs().max().item() == 0.0
    pw = torch.randn(C, C, dtype=torch.float64)
    cols = ldm_plan._legacy_proj_cols(pw, heads, pairs).double()
    got = torch.einsum('nthd,ohd->not', o, cols.reshape(C, hs, dp))
    want = torch.einsum('nct,oc->not', ref, pw)
    assert (got - want).abs().max().item() < 1e-12 * want.abs().max().item()


def test_conv_descriptor_channel_remainder_and_phase_pitch():
    d, info = G.conv_gemm(1 << 20, 2, 32, 32, 224, 1 << 21, 448, taps=9, a2_ptr=1 << 22, C2=672, out_f32=1 << 23)
    assert d.cpb == 4 and d.a_dims[0] == 224 and d.a_strides[0] == 448 and d.a2_c == 672 and d.nkb_aux == 11
    assert info['ktot'] == 9 * 256 + 704 and d.b_dims[0] == info['ktot']
    d, _ = G.conv_gemm(1 << 20, 2, 16, 16, 224, 1 << 21, 224, taps=9, out_f32=1 << 23, s2d=True)
    assert d.a_dims[0] == 4 * 256 and [d.tap_cb[t] for t in range(9)] == [768, 512, 768, 256, 0, 256, 768, 512, 768]
    assert G.pack_conv_weight(torch.zeros(448, 224, 3, 3), torch.zeros(448, 672, 1, 1)).shape[-1] == 9 * 256 + 704


def _plans(name, pairs, batches=(1, 2, 32)):
    P = _shape_params(name)
    cfg = U.CONFIGS[name]
    st = ldm_plan.ldm_structure(P, 8, cfg['num_head_channels'])
    wb, info = ldm_plan.pack_ldm_weights(st, P, head_pairs=pairs)
    for B in batches:
        yield B, ldm_plan.compile_ldm_plan(st, wb, info, B, B, B if B > 1 else 1, cfg['img_resolution'])


@pytest.mark.parametrize('pairs', [True, False])
def test_every_op_of_the_full_size_plans_passes_the_launch_checks(built, pairs):
    for B, pl in _plans('ldm_vq4', pairs):
        bad = []
        types = set()
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            desc = getattr(op.u, S.ALL_UNION_FIELD[op.type])
            types.add(op.type)
            why = _lib.op_check(desc)
            if why:
                bad.append((i, op.tag, why))
            if op.type == S.DS_OP_ATTN:
                assert desc.pad0 == (32 if pairs else 0) and (desc.nh % 2 == 0 or not pairs)
        assert not bad, (B, bad[:5])
        assert S.DS_OP_ATTN in types


def test_pairs_halve_the_attention_gemm_widths():
    """[q heads | k heads] of 21 heads: 22 x 32 x 2 = 1408 columns with pairs against 21 x 64 x 2 = 2688 padded."""
    widths = {}
    for pairs in (True, False):
        (_, pl), = _plans('ldm_vq4', pairs, batches=(1,))
        widths[pairs] = sorted({int(pl.ops_array[i].u.attn.nh) * (32 if pairs else 64)
                                for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_ATTN})
    assert widths[True] == [448, 704, 896] and widths[False] == [896, 1344, 1792]


def test_uncond_plan_has_no_context_ops():
    (_, pl), = _plans('tiny_uncond', True, batches=(2,))
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        desc = getattr(op.u, S.ALL_UNION_FIELD[op.type])
        for name, _ in desc._fields_:
            v = getattr(desc, name)
            if isinstance(v, int) and v and (v >> 60) == S.SPACE_IO:
                assert (v & ((1 << 60) - 1)) != S.DS_IO_CTX, (i, name)


# --------------------------------------------------------------------------------------------- check rules
def _attn(**kw):
    a = dict(q=1, k=1, vt=1, out=1, B=2, nh=22, L=256, Lk=256, q_pitch=2 * 704, q_c0=0, k_pitch=2 * 704, k_c0=704, vt_pitch=256,
             o_pitch=704, nplanes=2, scale=0.17, causal=0, pad0=32)
    a.update(kw)
    return S.AttnDesc(**a)


def test_attn_pair_rules(built):
    assert _lib.op_check(_attn()) is None
    assert 'attn: head_dim' in _lib.op_check(_attn(pad0=48))
    assert _lib.op_check(_attn(pad0=64, q_pitch=2 * 22 * 64, k_pitch=2 * 22 * 64, k_c0=22 * 64, o_pitch=22 * 64)) is None
    assert 'attn: pair head count' in _lib.op_check(_attn(nh=21, q_pitch=2 * 672, k_pitch=2 * 672, k_c0=672, o_pitch=672))
    assert _lib.op_check(_attn(nh=20)) is None
    assert 'attn: extent' in _lib.op_check(_attn(o_pitch=696))
    assert 'attn: extent' in _lib.op_check(_attn(k_c0=712))
    # a 64-wide head layout at nh x 32 is too narrow for the padded kernel
    assert 'attn: extent' in _lib.op_check(_attn(pad0=0))


def test_gemm_f8_channel_remainder_rule(built):
    base = dict(f8=True, acc_scale=1.0)
    d, _ = G.conv_gemm(1 << 20, 2, 16, 16, 256, 1 << 21, 256, taps=9, out_f32=1 << 23, **base)
    assert _lib.op_check(d) is None
    d, _ = G.conv_gemm(1 << 20, 2, 16, 16, 224, 1 << 21, 256, taps=9, out_f32=1 << 23, **base)
    assert 'gemm: f8 channel remainder' in _lib.op_check(d)
    d, _ = G.conv_gemm(1 << 20, 2, 16, 16, 256, 1 << 21, 256, taps=9, a2_ptr=1 << 22, C2=672, out_f32=1 << 23, **base)
    assert 'gemm: f8 channel remainder' in _lib.op_check(d)
    d, _ = G.conv_gemm(1 << 20, 2, 16, 16, 224, 1 << 21, 256, taps=9, out_f32=1 << 23)
    assert _lib.op_check(d) is None


def _gn(**kw):
    a = dict(src0=1, C0=224, C1=0, H=16, W=16, B=2, groups=32, eps=0.0, silu=0, resample=3, nplanes=2, out_raw=1, pad0=256)
    a.update(kw)
    return S.GnApplyDesc(**a)


def test_gn_apply_phase_pitch_rule(built):
    assert _lib.op_check(_gn()) is None
    assert _lib.op_check(_gn(pad0=224)) is None
    assert _lib.op_check(_gn(pad0=0)) is None
    assert 'gn_apply: phase pitch' in _lib.op_check(_gn(pad0=216))
    assert 'gn_apply: phase pitch' in _lib.op_check(_gn(pad0=252))
    assert 'gn_apply: phase pitch' in _lib.op_check(_gn(resample=2))
    assert 'gn_apply: phase pitch' in _lib.op_check(_gn(out_raw_f32=1))


# --------------------------------------------------------------------------------------------- arguments
def test_constructor_argument_errors():
    from diff_sampler_b200.ldm_net import B200LDMNet
    P = _shape_params('tiny_uncond')
    with pytest.raises(ValueError, match='guidance_type'):
        B200LDMNet(P, img_channels=3, guidance_type='cfg')
    with pytest.raises(ValueError, match='fp16f8'):
        B200LDMNet(P, img_resolution=32, img_channels=3, guidance_type='uncond', num_head_channels=32, precision='fp16f8')


def test_uncond_beta_schedule():
    from diff_sampler_b200 import ldm_net
    from oracle import ldm_oracle as LO
    assert ldm_net.UNCOND_BETAS == U.BETAS
    assert torch.equal(ldm_net.make_alphas_cumprod(*ldm_net.UNCOND_BETAS), LO.make_alphas_cumprod(*U.BETAS))


# --------------------------------------------------------------------------------------------- plans on the float64 interpreter
@pytest.mark.parametrize('pairs', [True, False])
def test_tiny_plan_on_the_interpreter(pairs):
    """The tiny net's plan (channel remainders, phase-pitched space-to-depth, 3- and 9-head levels) op by op in float64 against the
    functional forward: eps and the middle-block read-out."""
    import ldm_uncond_interp as LI
    P, cfg = U.make_params('tiny_uncond')
    st = ldm_plan.ldm_structure(P, 8, cfg['num_head_channels'])
    wb, info = ldm_plan.pack_ldm_weights(st, P, head_pairs=pairs)
    B, R = 2, cfg['img_resolution']
    pl = ldm_plan.compile_ldm_plan(st, wb, info, B, B, B, R)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 3, R, R, generator=g).contiguous()
    t = torch.tensor([417.0, 38.0])
    c_in = torch.tensor([0.37, 0.81])
    eps = torch.zeros(B, 3, R, R)
    bott = torch.zeros(B, 64)
    coef = torch.zeros(B, 4)
    coef[:, 2] = c_in
    LI.run_plan(pl, wb.bytes(), {S.DS_IO_X: x, S.DS_IO_D: eps, S.DS_IO_SIGMA: t, S.DS_IO_LABELS: coef, S.DS_IO_BOTTLENECK: bott})
    Pd = {k: v.double() for k, v in P.items()}
    taps = {}
    with torch.no_grad():
        ref = U.unet_forward(Pd, cfg, x.double() * c_in.double().reshape(-1, 1, 1, 1), t.double(), taps=taps)
    err = (eps.double() - ref).abs().max().item()
    tap = taps['middle_block'].mean(dim=1).reshape(B, 64)
    eb = (bott.double() - tap).abs().max().item()
    print(f'tiny_uncond pairs={pairs}: interpreter vs float64 forward {err:.3e} (max {ref.abs().max().item():.2f}), tap {eb:.3e}')
    assert err < 1e-4 * max(1.0, ref.abs().max().item())
    assert eb < 1e-4 * max(1.0, tap.abs().max().item())


# --------------------------------------------------------------------------------------------- released checkpoint
class _NotATensor:
    """An object a weights_only load refuses (a training checkpoint may carry such callback / config objects)."""


def _ldm_ckpt_state(name='tiny_uncond'):
    """A LatentDiffusion state dict with the released file's key layout: model.diffusion_model.* (the eps-net), first_stage_model.*
    (VQ encoder, quant_conv, codebook, post_quant_conv, decoder) and the schedule buffers."""
    import vq_ref as VQ
    from diff_sampler_b200 import ldm_net
    P, _ = U.make_params(name)
    V, _ = VQ.make_params('tiny_vq')
    sd = {'model.diffusion_model.' + k: v for k, v in P.items()}
    sd.update({'first_stage_model.' + k: v for k, v in V.items()})
    sd['first_stage_model.encoder.conv_in.weight'] = torch.zeros(64, 3, 3, 3)
    sd['first_stage_model.quant_conv.weight'] = torch.zeros(3, 3, 1, 1)
    ac = ldm_net.make_alphas_cumprod(*ldm_net.UNCOND_BETAS)
    sd['alphas_cumprod'] = ac
    sd['betas'] = torch.zeros(1000)
    return sd, P, V, ac


def test_ldm_checkpoint_key_split(tmp_path):
    from diff_sampler_b200 import ldm_net
    sd, P, V, ac = _ldm_ckpt_state()
    path = tmp_path / 'model.ckpt'
    torch.save({'state_dict': sd, 'epoch': 3, 'global_step': 1200}, path)
    unet, first, ac2, sf = ldm_net.load_ldm_checkpoint(str(path))
    assert list(unet) == list(P) and all(torch.equal(unet[k], P[k]) for k in P)
    assert set(first) == set(V) and all(torch.equal(first[k], V[k]) for k in V)
    assert torch.equal(ac2, ac) and sf == 1.0
    st = ldm_plan.ldm_structure(unet, 8, 32)
    assert {L[3] for _, ls in st['inp'] + st['mid'] + st['out'] for L in ls if L[0] == 'qkv_attn'} == {3, 6, 9}


def test_ldm_checkpoint_is_never_unpickled(tmp_path):
    from diff_sampler_b200 import ldm_net
    sd, _, _, _ = _ldm_ckpt_state()
    path = tmp_path / 'model.ckpt'
    torch.save({'state_dict': sd, 'callbacks': _NotATensor()}, path)
    with pytest.raises(ValueError, match='weights_only'):
        ldm_net.load_ldm_checkpoint(str(path))
    torch.save({'model': sd}, path)
    with pytest.raises(ValueError, match='state_dict'):
        ldm_net.load_ldm_checkpoint(str(path))
    torch.save({'state_dict': {k: v for k, v in sd.items() if not k.startswith('first_stage_model.')}}, path)
    with pytest.raises(ValueError, match='first_stage_model'):
        ldm_net.load_ldm_checkpoint(str(path))

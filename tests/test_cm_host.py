"""Consistency-Models LSUN-256 nets (lsun_bedroom, lsun_cat) on the host: the float64 oracle against the real reference
(tests/golden/ref_cm.npz, oracle/gen_cm_golden.py), the importer's structure at the full lsun_setting, the qkv row permutation,
the tiny CM plan on the CPU plan interpreter, the launchers' descriptor checks over the full-size plan, and the other plan kinds
compiling byte for byte as before."""
import json
import os

import numpy as np
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import _lib
from diff_sampler_b200 import cm_net, gemm_desc as G, plan as planner
from oracle import cm_interp as CI
from oracle import cm_oracle as CO

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
TOL = {False: 3e-5, True: 3e-4}          # as tests/test_plan_interp.py


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'ref_cm.npz'))


@pytest.fixture(scope='module')
def tiny():
    sd = cm_net.init_state_dict(cm_net.TINY_SETTING, seed=0)
    return sd, CO.CMOracle(sd, cm_net.TINY_SETTING)


@pytest.fixture(scope='module')
def full():
    """The full lsun_setting net from a random state dict with the released checkpoint's key names and shapes."""
    sd = cm_net.init_state_dict(None, seed=0)
    spec, params = cm_net.convert(sd)
    return sd, spec, params


def test_cm_oracle_matches_reference(ref, tiny):
    _, orc = tiny
    for tag in ('s2', 's80', 's0p002', 'per'):
        x, sig = torch.from_numpy(ref[f'cm/{tag}/x']), torch.from_numpy(ref[f'cm/{tag}/sigma'])
        orc.taps = {}
        D = orc(x, sig)
        want = torch.from_numpy(ref[f'cm/{tag}/D'])
        mid = torch.from_numpy(ref[f'cm/{tag}/middle']).double()
        err = (D - want).abs().max().item()
        err_mid = (orc.taps['middle_block'] - mid).abs().max().item()
        print(f'{tag}: |D - ref| {err:.3e}, |middle_block - ref| {err_mid:.3e}')
        assert err < 1e-5 * max(1.0, want.abs().max().item())
        assert err_mid < 1e-5 * max(1.0, mid.abs().max().item())


def test_qkv_permutation_matches_the_reference_rearrange(ref):
    """QKVFlashAttention reads qkv conv rows as `b (three h d) s -> b s three h d`; the importer must deliver the EDM order
    [head][d][q|k|v] (plan._qkv_split), not the legacy [head][q|k|v][d]."""
    layout = torch.from_numpy(ref['qkv/layout']).long()          # [3, heads, d]: the conv row each slot reads
    heads = int(ref['qkv/heads'])
    rows = torch.arange(layout.numel())
    edm = cm_net.qkv_cm_to_edm(rows, heads).reshape(heads, -1, 3)
    assert torch.equal(edm, layout.permute(1, 2, 0))
    w = torch.randn(layout.numel(), 5, 1, 1)
    wqk, _, wv, _ = planner._qkv_split(cm_net.qkv_cm_to_edm(w, heads), torch.zeros(layout.numel()), heads)
    C = layout.numel() // 3
    assert torch.equal(wqk[:C], w[:C, :, 0, 0]) and torch.equal(wqk[C:], w[C:2 * C, :, 0, 0]) and torch.equal(wv, w[2 * C:, :, 0, 0])


def test_lsun_structure(full):
    sd, spec, params = full
    widths = {256: 256, 128: 256, 64: 512, 32: 512, 16: 1024, 8: 1024}
    assert spec.img_resolution == 256 and spec.stem_cout == 256 and spec.noise_channels == 256 and spec.emb_channels == 1024
    assert spec.noise_scale == 1000.0 and spec.kind == 'cm' and spec.label_dim == 0
    for b in spec.enc + spec.dec:
        assert b.cout == widths[b.res_in if (b.up or b.down) else b.res_out], b      # a resampling block keeps its input width
        assert not b.adaptive_scale and b.skip_scale == 1.0 and b.eps == 1e-5
        assert b.heads == (b.cout // 64 if b.res_out in (32, 16, 8) and not (b.up or b.down) and b.name != 'dec.8x8_in1' else 0), b
        if b.up or b.down:
            assert b.skip == 'resample' and b.cin == b.cout
    assert sum(b.down for b in spec.enc) == 5 and sum(b.up for b in spec.dec) == 5
    # concat widths: the reference's input_block_chans, popped in reverse
    chans = [256]
    for level, m in enumerate((1, 1, 2, 2, 4, 4)):
        chans += [256 * m] * 2 + ([256 * m] if level < 5 else [])
    assert [b.concat for b in spec.dec if b.concat] == chans[::-1]
    assert spec.bottleneck_block == 'dec.8x8_in1' and spec.dec[1].name == 'dec.8x8_in1'
    # the 8x8 middle block: ResBlock + attention folded into in0, ResBlock in1, as middle_block.0 / .1 / .2
    assert torch.equal(params['model.dec.8x8_in1.conv0.weight'], sd['middle_block.2.in_layers.2.weight'])
    assert torch.equal(params['model.dec.8x8_in0.proj.weight'], sd['middle_block.1.proj_out.weight'])
    assert sum(1 for k in sd if not k.startswith(('time_embed', 'out.'))) == sum(1 for k in params if not k.startswith(('model.map_', 'model.out_')))
    assert all(v.dtype == torch.float32 for v in params.values())


def test_fp16_state_dict_is_upcast():
    sd = {k: v.half() if not k.startswith(('time_embed', 'out.')) else v for k, v in cm_net.init_state_dict(cm_net.TINY_SETTING).items()}
    _, params = cm_net.convert(sd, cm_net.TINY_SETTING)
    assert all(v.dtype == torch.float32 for v in params.values())


@pytest.mark.parametrize('field,value', [('use_scale_shift_norm', True), ('class_cond', True), ('learn_sigma', True),
                                         ('num_head_channels', 32), ('resblock_updown', False), ('num_channels', 32)])
def test_unsupported_settings_are_rejected(field, value):
    with pytest.raises(ValueError, match=field):
        cm_net.structure(dict(cm_net.TINY_SETTING, **{field: value}))


def test_state_dict_must_match_the_settings():
    sd = cm_net.init_state_dict(cm_net.TINY_SETTING)
    with pytest.raises(ValueError):
        cm_net.convert(sd, dict(cm_net.TINY_SETTING, num_channels=128))
    with pytest.raises(KeyError):
        cm_net.convert({k: v for k, v in sd.items() if 'middle_block.1.qkv' not in k}, cm_net.TINY_SETTING)


@pytest.mark.parametrize('f8', [False, True])
def test_cm_plan_on_the_cpu_interpreter(ref, tiny, f8):
    sd, orc = tiny
    spec, params = cm_net.convert(sd, cm_net.TINY_SETTING)
    wb, info = planner.pack_weights(spec, params, f8=f8)
    for tag in ('s2', 's80', 'per'):
        x, sig = torch.from_numpy(ref[f'cm/{tag}/x']), torch.from_numpy(ref[f'cm/{tag}/sigma'])
        B = x.shape[0]
        pl = planner.compile_plan(spec, wb, info, B, sig.numel(), 0, npass=3, f8=f8)
        D, bott = torch.zeros_like(x), torch.zeros(B, 64)
        CI.run_plan(pl, wb.bytes(), {S.DS_IO_X: x, S.DS_IO_D: D, S.DS_IO_SIGMA: sig.contiguous(), S.DS_IO_BOTTLENECK: bott})
        orc.taps = {}
        want = orc(x, sig)
        tap = orc.taps['middle_block'].mean(dim=1).reshape(B, 64).float()
        err, err_tap = (D - want).abs().max().item(), (bott - tap).abs().max().item()
        print(f'{tag} f8={f8}: interpreter vs oracle {err:.3e}, middle-block tap {err_tap:.3e}')
        assert err < TOL[f8] * max(1.0, want.abs().max().item())
        assert err_tap < TOL[f8] * max(1.0, tap.abs().max().item())


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    return g._load_build_module().build()


@pytest.mark.parametrize('f8', [False, True])
def test_fullsize_plan_passes_the_launcher_checks(built, full, f8):
    """The shapes new to the EDM plan path -- 256-wide convolutions as 128-pixel row segments, a 3-channel stem at 256x256,
    GroupNorm over 65 536-pixel groups, pooling from a 256-wide input, 1024 + 1024 channel concats -- against the launchers' descriptor
    checks (ds_op_check), at a per-sample-sigma batch of 32 (the affine runs as a GEMM) and at batch 2."""
    _, spec, params = full
    wb, info = planner.pack_weights(spec, params, f8=f8)
    seen = set()
    for B, nsig in ((2, 1), (32, 32)):
        pl = planner.compile_plan(spec, wb, info, B, nsig, 0, npass=3, f8=f8)
        bad = []
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            d = getattr(op.u, S.UNION_FIELD[op.type])
            why = _lib.op_check(d)
            if why:
                bad.append((i, why))
            if op.type == S.DS_OP_GEMM and d.a_mode == 0 and d.conv_W == 256:
                seen.add(('row segment', d.taps, int(d.a_dims[0])))
            if op.type == S.DS_OP_GN_APPLY and d.resample == 1 and d.H == 256:
                seen.add('pool from 256')
            if op.type == S.DS_OP_GN_APPLY and d.C0 == 1024 and d.C1 == 1024:
                seen.add('concat 2048')
            if op.type == S.DS_OP_POSEMB:
                assert d.noise_scale == 1000.0 and d.mode == 0 and not d.endpoint and not d.swap_sincos
        assert not bad, bad[:10]
        print(f'B={B} f8={f8}: {pl.n_ops} ops, {pl.meta["n_gemm"]} GEMMs, arena {pl.arena_bytes / 2 ** 30:.2f} GiB')
    assert ('row segment', 9, 64) in seen and 'pool from 256' in seen and 'concat 2048' in seen
    assert G.conv_box(256, 256) == (128, 1, 1)


def test_other_plans_compile_as_before():
    """EDM / CM / LDM / VAE / VQ / CLIP / optimal-denoiser plan variants and the benchmarked plans: op arrays, arena, meta and weight
    blobs unchanged."""
    import plan_digest
    want = json.load(open(os.path.join(GOLDEN, 'plan_digests.json')))
    got = plan_digest.all_digests()
    assert sorted(got) == sorted(want)
    changed = [k for k in want if got[k] != want[k]]
    assert not changed, changed

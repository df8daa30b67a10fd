"""Host-side logic of the product (CPU): plan lowering, weight packing, coefficient algebra, schedules, GITS dp —
checked against the oracle / golden vectors without touching a GPU."""
import json
import os

import numpy as np
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import edm_nets, gemm_desc as G, gits_utils, plan as planner, solver_utils as U
from oracle import edm_oracle as O
from oracle import solvers_oracle as SO

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'ref_core.npz')


def test_init_matches_reference_digest():
    d = np.load(GOLD)
    meta = json.loads(bytes(d['meta_json']).decode())
    for name in ('tiny_song', 'tiny_adm', 'cifar10'):
        params, cfg = edm_nets.init_params(name, seed=0)
        assert O.params_digest(params) == meta[f'digest/{name}/0']
        edm_nets.dezero_(params, cfg['kind'], seed=0)
        assert O.params_digest(params) == meta[f'digest/{name}/1']


@pytest.mark.parametrize('name,B', [('tiny_song', 3), ('tiny_adm', 5), ('cifar10', 8), ('ffhq', 2)])
def test_plan_lowering_invariants(name, B):
    params, cfg = edm_nets.init_params(name, seed=0)
    spec = edm_nets.spec_from_params(params, cfg['img_resolution'], cfg['img_channels'], cfg.get('label_dim', 0))
    assert spec.aff_total == sum(b.aff_width for b in spec.enc + spec.dec)
    wb, info = planner.pack_weights(spec, params)
    for nsig in (1, B):
        pl = planner.compile_plan(spec, wb, info, B, nsig, B if spec.label_dim else 0, npass=3)
        n_gemm = 0
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            if op.type == S.DS_OP_GEMM:
                g = op.u.gemm
                n_gemm += 1
                assert g.BN % 16 == 0 and 16 <= g.BN <= 256
                assert g.a_box[0] == 64 and g.a_box[1] * g.a_box[2] * g.a_box[3] == 128
                assert g.n_tiles * g.BN >= g.n_valid and g.m_tiles * 128 >= g.m_valid
                assert (g.a_ptr >> 60) in (S.SPACE_ARENA, S.SPACE_WEIGHTS) and (g.b_ptr >> 60) in (S.SPACE_ARENA, S.SPACE_WEIGHTS)
                assert all(s % 16 == 0 for s in g.a_strides) and all(s % 16 == 0 for s in g.b_strides)
        assert n_gemm == pl.meta['n_gemm'] and pl.arena_bytes > 0
    # every conv of the reference is lowered exactly once: stem + 2 per block (+1 head); an attention block adds qk, v, proj and
    # either the fused attention op (64-wide heads) or the QK^T / PV GEMM pair around a softmax
    blocks = spec.enc + spec.dec
    n_attn = sum(1 for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_ATTN)
    n_soft = sum(1 for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_SOFTMAX)
    assert n_attn + n_soft == sum(1 for b in blocks if b.heads)
    assert pl.meta['n_gemm'] == 1 + 2 * len(blocks) + 3 * n_attn + 5 * n_soft + 1


def test_spec_matches_oracle_structure():
    for name in ('tiny_song', 'tiny_adm', 'cifar10', 'imagenet64'):
        P, St = O.make_net(name, seed=0) if name != 'imagenet64' else (None, None)
        if P is None:
            continue
        spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
        for b in spec.enc + spec.dec:
            ob = St['blocks'][b.name]
            assert (b.cin, b.cout, b.up, b.down, b.heads) == (ob['cin'], ob['cout'], ob['up'], ob['down'], ob['heads'])
            assert {None: 'identity', 1: 'conv', 0: 'resample'}[ob['skip_kernel']] == b.skip
            assert abs(b.skip_scale - float(ob['skip_scale'])) < 1e-7 and b.eps == ob['eps']


def test_weight_packing_roundtrip():
    torch.manual_seed(0)
    w = torch.randn(70, 40, 3, 3)
    sk = torch.randn(70, 24, 1, 1)
    p = G.pack_conv_weight(w, sk)
    bn, tiles = G.pick_bn(70)
    assert bn % 16 == 0 and bn * tiles >= 70
    assert p.shape == (2, bn * tiles, 9 * 64 + 64) and p.dtype == torch.float16
    full = p[0].float() + p[1].float()
    ref = torch.zeros(70, 3, 3, 64)
    ref[..., :40] = w.permute(0, 2, 3, 1)
    assert (full[:70, :576] - ref.reshape(70, -1)).abs().max() < 1e-6
    assert (full[:70, 576:600] - sk.reshape(70, 24)).abs().max() < 1e-6 and full[70:].abs().max() == 0
    assert G.pick_bn(256) == (256, 1) and G.pick_bn(384) == (192, 2) and G.pick_bn(3) == (32, 1) and G.pick_bn(576) == (192, 3)
    assert G.pick_bn(320) == (160, 2) and G.pick_bn(1344) == (224, 6)
    # few M tiles: the N tile that minimises (waves over NUM_SMS SMs) x (per-tile cost); many tiles: pick_bn's tiling
    assert G.fill_bn(1280, 8) == (80, 16) and G.fill_bn(1280, 32) == (160, 8) and G.fill_bn(1280, 2048) == (256, 5)
    assert G.fill_bn(256, 256) == (256, 1) and G.fill_bn(256, 64) == (128, 2)
    assert G.conv_box(32, 32) == (32, 4, 1) and G.conv_box(8, 8) == (8, 8, 2) and G.conv_box(64, 64) == (64, 2, 1)
    # qkv de-interleave ([head][c][q|k|v] rows, networks_edm.py:174)
    C_, nh = 8, 2
    wq = torch.arange(3 * C_).float().reshape(3 * C_, 1)
    bq = torch.arange(3 * C_).float()
    wqk, bqk, wv, bv = planner._qkv_split(wq, bq, nh)
    idx = torch.arange(3 * C_).reshape(nh, C_ // nh, 3)
    assert torch.equal(bqk[:C_], idx[:, :, 0].reshape(-1).float()) and torch.equal(bqk[C_:], idx[:, :, 1].reshape(-1).float())
    assert torch.equal(bv, idx[:, :, 2].reshape(-1).float())


def test_f8_operand_packing_and_plan():
    """f8 GEMM mode (csrc/ops.h): operand images are self-consistent (hi + lo reproduces the value to ~2^-15 relative, the three
    scales of each operand pair add up to the same S) and the plan marks exactly the block convolutions."""
    torch.manual_seed(0)
    w = torch.randn(100, 192, 3, 3) / 40
    sk = torch.randn(100, 64, 1, 1) / 8
    blob, shift = G.pack_conv_weight_f8(w, sk)
    bn, tiles = G.pick_bn(100)
    k16, k8 = 9 * 192 + 64, 9 * 256 + 128
    assert blob.dtype == torch.uint8 and blob.numel() == bn * tiles * (2 * k16 + 2 * k8)
    assert shift == S.DS_F8_SH_LO8 + int(np.floor(np.log2(448.0 / max(w.abs().max().item(), sk.abs().max().item()))))
    (m16, s16), (mh8, sh8), (ml8, sl8) = G.decode_conv_weight_f8(blob, shift, 100, 192, 9, 64)
    wk, skk = w.permute(0, 2, 3, 1).reshape(100, 9, 192), sk.reshape(100, 64)
    wmax = max(wk.abs().max().item(), skk.abs().max().item())
    assert (m16 - wk).abs().max() <= 2.0 ** -11 * wmax and (s16 - skk).abs().max() <= 2.0 ** -11 * wmax
    assert (m16 + ml8 - wk).abs().max() <= 2.0 ** -15 * wmax and (s16 + sl8 - skk).abs().max() <= 2.0 ** -15 * wmax
    assert ((mh8 - m16).abs() <= 2.0 ** -4 * m16.abs() + 2.0 ** -10 * wmax).all()
    x = torch.randn(2, 4, 4, 64) * 3
    hi, lo8, hi8 = G.decode_act_planes_f8(G.act_planes_f8(x), x.shape)
    assert (hi - x).abs().max() <= 2.0 ** -11 * 16 and (hi + lo8 - x).abs().max() <= 2.0 ** -15 * 16
    assert ((hi8 - hi).abs() <= 2.0 ** -4 * hi.abs() + 2.0 ** -11).all()
    # saturation instead of inf / nan for out-of-range activations
    big = torch.tensor([[2000.0, -5000.0, 100.0, 1e-9] * 16])
    hi, lo8, hi8 = G.decode_act_planes_f8(G.act_planes_f8(big), big.shape)
    assert torch.isfinite(hi).all() and torch.isfinite(lo8).all() and torch.isfinite(hi8).all() and hi.abs().max() < 1024

    params, cfg = edm_nets.init_params('tiny_song', seed=0)
    spec = edm_nets.spec_from_params(params, cfg['img_resolution'], cfg['img_channels'], cfg.get('label_dim', 0))
    wb, info = planner.pack_weights(spec, params, f8=True)
    pl = planner.compile_plan(spec, wb, info, 3, 1, 0, npass=3, f8=True)
    ref_wb, ref_info = planner.pack_weights(spec, params)
    ref_pl = planner.compile_plan(spec, ref_wb, ref_info, 3, 1, 0, npass=3)
    assert pl.n_ops == ref_pl.n_ops and pl.arena_bytes == ref_pl.arena_bytes and wb.size <= ref_wb.size * 1.35
    n_f8 = n_fmt = 0
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        if op.type == S.DS_OP_GEMM and op.u.gemm.f8:
            g = op.u.gemm
            n_f8 += 1
            assert g.a_mode == 0 and g.num_z == 1 and g.npass == 3 and g.taps == 9 and g.b_dims[2] == 1 and g.a_dims[3] == g.a_plane_n
            assert 0 < g.acc_scale < 1 and np.log2(g.acc_scale) == round(np.log2(g.acc_scale))
        elif op.type == S.DS_OP_GEMM:
            assert op.u.gemm.acc_scale in (0.0, 1.0)
        if op.type == S.DS_OP_GN_APPLY and op.u.gn_apply.fmt == 1:
            n_fmt += 1
    blocks = spec.enc + spec.dec
    assert n_f8 == 2 * len(blocks) + 1 and n_fmt == 2 * len(blocks) + 1          # block convolutions + the head conv
    last_fmt = {}
    for i in range(pl.n_ops):                       # every GEMM reads its operands in the format their last producer wrote
        o = pl.ops_array[i]
        if o.type == S.DS_OP_GN_APPLY:
            for ptr in (o.u.gn_apply.out_act, o.u.gn_apply.out_raw):
                if ptr:
                    last_fmt[ptr] = o.u.gn_apply.fmt
        elif o.type == S.DS_OP_GEMM:
            g = o.u.gemm
            for ptr, used in ((g.a_ptr, True), (g.a2_ptr, bool(g.a2_c)), (g.b_ptr, g.a_mode == 1)):
                if used and ptr in last_fmt:
                    assert last_fmt[ptr] == ((1 if g.f8 & 1 else 0) if ptr != g.b_ptr else 0), (i, o.tag)


@pytest.mark.parametrize('f8,f8_linear', [(False, False), (True, False), (True, True)])
def test_ldm_plan_lowering(f8, f8_linear):
    """The latent-diffusion eps-net lowers on the host (no GPU) in every precision; f8 touches exactly the ResBlock and Upsample convolutions,
    and f8_linear additionally the five single-consumer linears of every transformer block (with their producers' output format)."""
    from diff_sampler_b200 import ldm_plan
    from oracle import ldm_oracle as LO
    P, cfg = LO.make_params('tiny_ldm')
    st = ldm_plan.ldm_structure(P, cfg['num_heads'])
    wb, info = ldm_plan.pack_ldm_weights(st, P, f8=f8, f8_linear=f8_linear)
    pl = ldm_plan.compile_ldm_plan(st, wb, info, 2, 4, 1, cfg['img_resolution'], npass=3, f8=f8, f8_linear=f8_linear)
    layers = [L for _, ls in st['inp'] + st['mid'] + st['out'] for L in ls]
    n_res = sum(1 for L in layers if L[0] == 'res')
    n_att = sum(1 for L in layers if L[0] == 'attn')
    n_up = sum(1 for L in layers if L[0] == 'up')
    ops = [pl.ops_array[i] for i in range(pl.n_ops)]
    n_f8 = sum(1 for o in ops if o.type == S.DS_OP_GEMM and o.u.gemm.f8)
    n_fmt = sum(1 for o in ops if o.type == S.DS_OP_GN_APPLY and o.u.gn_apply.fmt == 1)
    n_ln = sum(1 for o in ops if o.type == S.DS_OP_LAYERNORM and o.u.layernorm.fmt == 1)
    n_gg = sum(1 for o in ops if o.type == S.DS_OP_GEGLU and o.u.geglu.fmt == 1)
    assert pl.n_ops > 50 and pl.arena_bytes > 0 and n_res > 0 and n_att > 0
    lin = 1 if f8_linear else 0
    assert n_up > 0
    assert n_f8 == (2 * n_res + n_up if f8 else 0) + 5 * n_att * lin
    assert n_fmt == (2 * n_res + n_up if f8 else 0) + 2 * n_att * lin    # + norm -> proj_in and the cast before proj_out
    assert (n_ln, n_gg) == (2 * n_att * lin, n_att * lin)                # norm2, norm3; norm1 feeds both an A and a B operand and stays fp16
    assert len(info['f8_shift']) == (2 * n_res + n_up if f8 else 0) + 5 * n_att * lin
    # every f8 GEMM reads an operand some producer wrote in the f8 image: same buffer reference
    f8_inputs = {o.u.gemm.a_ptr for o in ops if o.type == S.DS_OP_GEMM and o.u.gemm.f8} | \
                {o.u.gemm.a2_ptr for o in ops if o.type == S.DS_OP_GEMM and o.u.gemm.f8 and o.u.gemm.a2_c}
    f8_outputs = {o.u.gn_apply.out_act for o in ops if o.type == S.DS_OP_GN_APPLY and o.u.gn_apply.fmt == 1} | \
                 {o.u.gn_apply.out_raw for o in ops if o.type == S.DS_OP_GN_APPLY and o.u.gn_apply.fmt == 1} | \
                 {o.u.layernorm.out for o in ops if o.type == S.DS_OP_LAYERNORM and o.u.layernorm.fmt == 1} | \
                 {o.u.geglu.out for o in ops if o.type == S.DS_OP_GEGLU and o.u.geglu.fmt == 1}
    assert f8_inputs <= f8_outputs
    # order-aware: scratch buffers ('act', 'ln', ...) are reused with different formats, so each GEMM must find its A operand (and the
    # K-appended skip operand) in the format of the LAST producer that wrote that buffer before it
    last_fmt = {}
    for o in ops:
        if o.type == S.DS_OP_GN_APPLY:
            for ptr in (o.u.gn_apply.out_act, o.u.gn_apply.out_raw):
                if ptr:
                    last_fmt[ptr] = o.u.gn_apply.fmt
        elif o.type == S.DS_OP_LAYERNORM:
            last_fmt[o.u.layernorm.out] = o.u.layernorm.fmt
        elif o.type == S.DS_OP_GEGLU:
            last_fmt[o.u.geglu.out] = o.u.geglu.fmt
        elif o.type == S.DS_OP_GEMM:
            g = o.u.gemm
            want = 1 if g.f8 & 1 else 0
            if g.a_ptr in last_fmt:
                assert last_fmt[g.a_ptr] == want, (o.tag, 'A operand format')
            if g.a2_c and g.a2_ptr in last_fmt:
                assert last_fmt[g.a2_ptr] == want, (o.tag, 'skip operand format')
            if g.a_mode == 1 and g.b_ptr in last_fmt:
                assert last_fmt[g.b_ptr] == 0, (o.tag, 'B-side activations are always fp16 hi/lo planes')


@pytest.mark.parametrize('name,R,B', [('tiny_vae', 8, 2), ('wide_vae', 64, 2), ('sd_vae', 64, 1)])
def test_vae_decoder_plan_lowering(name, R, B):
    """First-stage decoder (vae_plan.py): the structure read back from state_dict names equals the oracle's module list (which is pinned
    to the reference Decoder), every module is lowered once, rows wider than one M tile are tiled as 128-pixel row segments."""
    from diff_sampler_b200 import vae_plan
    from oracle import vae_oracle as VO
    P, cfg = VO.make_params(name, seed=0)
    mods, meta = vae_plan.vae_structure(P)
    omods, c_end = VO.structure(cfg)
    assert [tuple(m) for m in mods] == [tuple(m) for m in omods] and meta['c_end'] == c_end
    assert meta['upscale'] == 2 ** (len(cfg['ch_mult']) - 1) and meta['out_ch'] == cfg['out_ch']
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    pl = vae_plan.compile_vae_plan(mods, meta, wb, B, R)
    ops = [pl.ops_array[i] for i in range(pl.n_ops)]
    gemms = [o.u.gemm for o in ops if o.type == S.DS_OP_GEMM]
    n_res = sum(1 for m in mods if m[0] == 'res')
    n_att = sum(1 for m in mods if m[0] == 'attn')
    n_up = sum(1 for m in mods if m[0] == 'up')
    assert len(gemms) == 2 + 2 * n_res + 5 * n_att + n_up + 1            # post_quant + conv_in, 2 per block, qk/v/S/PV/proj, up convs, conv_out
    assert sum(1 for o in ops if o.type == S.DS_OP_GN_STATS) == 2 * n_res + n_att + 1
    assert pl.meta['out_res'] == R * meta['upscale']
    for g in gemms:
        wide = g.a_mode == 0 and g.conv_W > 128
        assert g.f8 & ~1 == 0                                            # bit 0 (e4m3 corrections) is the only flag
        if wide:
            assert g.conv_W % 128 == 0 and tuple(g.a_box) == (64, 128, 1, 1) and g.num_z == 1
        assert g.m_tiles * 128 >= g.m_valid and g.n_tiles * g.BN >= g.n_valid
    last = gemms[-1]
    assert last.edm_out == 2 and last.edm_C == cfg['out_ch'] and last.n_valid == cfg['out_ch']
    assert gemms[0].taps == 1 and gemms[0].ldo == 64 and gemms[0].n_valid == cfg['z_channels'] and gemms[1].a_ptr == gemms[0].out_h16


def test_schedules_and_deis_tables_match_reference_golden():
    d = np.load(GOLD)
    for st in ('polynomial', 'logsnr', 'time_uniform'):
        for n in (4, 6, 7, 11, 18, 61):
            assert np.array_equal(U.get_schedule(n, 0.002, 80, schedule_type=st, schedule_rho=7).float().numpy(), d[f'sched/{st}/{n}'])
    ts = U.get_schedule(61, 0.002, 80)
    assert torch.equal(U.get_schedule(61, 0.002, 80, dp_list=[0, 5, 17, 60]), ts[[0, 5, 17, 60]])          # GITS gather
    for ci, (n, mo, mode) in {7: (7, 4, 'tab'), 8: (6, 4, 'rhoab')}.items():
        C_ = U.get_deis_coeff_list(U.get_schedule(n, 0.002, 80), mo, deis_mode=mode)
        for row, rr in zip(C_, d[f'deis/{ci}']):
            assert np.allclose([float(torch.as_tensor(c).detach()) for c in row], rr[:len(row)], rtol=1e-6, atol=1e-9)
    with pytest.raises(ValueError):
        U.get_schedule(5, 0.002, 80, schedule_type='nope')


def test_update_coefficients_reproduce_reference_formulas():
    torch.manual_seed(0)
    x = torch.randn(2, 3, 4, 4)
    ms = [torch.randn(2, 3, 4, 4) for _ in range(3)]
    ts = [torch.tensor(5.0), torch.tensor(3.0), torch.tensor(2.0)]
    t = torch.tensor(1.2)
    for order in (1, 2, 3):
        for px0 in (True, False):
            ref = SO.dpm_pp_update(x, ms, ts, t, order, predict_x0=px0, scale=0.9)
            c = U.dpm_pp_coefs([float(v) for v in ts], float(t), order, px0, 0.9)
            got = c[0] * x + c[1] * ms[-1] + c[2] * ms[-2] + c[3] * ms[-3]
            assert (ref - got).abs().max() < 5e-6
            for var in ('bh1', 'bh2'):
                class N:
                    def __call__(self, xt, tt, cl):
                        self.xt = xt
                        return self.D
                n = N()
                n.D = torch.randn_like(x) * 0.3
                xr, mr = SO.unipc_update(x, ms, ts, t, order, variant=var, predict_x0=px0, net=n, use_corrector=True)
                pred, corr = U.unipc_coefs([float(v) for v in ts], float(t), order, var, px0, True)
                hist = [ms[-1 - k] for k in range(order)]
                xp = pred[0] * x + sum(pred[1 + k] * hist[k] for k in range(order))
                mt = SO.dynamic_thresholding(n.D) if px0 else (n.xt - n.D) / t
                xc = corr[0] * x + corr[1] * mt + sum(corr[2 + k] * hist[k] for k in range(order))
                assert (xp - n.xt).abs().max() < 1e-5 and (xc - xr).abs().max() < 2e-5
    with pytest.raises(ValueError):
        U.dpm_pp_coefs([1.0], 0.5, 4)


def test_gits_dp_bit_exact_vs_reference():
    d = np.load(GOLD)
    meta = json.loads(bytes(d['meta_json']).decode())
    cm = d['gits/cost']
    for key, ref in meta['gits/dp'].items():
        ns, coeff = key.split('/')
        assert gits_utils.dp(cm, int(ns), cm.shape[0], float(coeff)) == ref
    traj = torch.from_numpy(d['gits/traj'])
    assert np.abs(gits_utils.cal_deviation(traj, 3, 8, bs=3).numpy() - d['gits/dev']).max() <= 1e-5 * np.abs(d['gits/dev']).max()
    with pytest.raises(NotImplementedError):
        gits_utils.get_sampler_fn('nope', 'cpu')


def test_public_surface_matches_reference_signatures():
    """Drop-in check: every function of the reference's solvers / solver_utils / solvers_amed / gits_utils surface exists here with
    the same parameter names, order and defaults (signatures recorded from the real reference into tests/golden/ref_signatures.json;
    the product may only ADD trailing keyword parameters, e.g. `dp_list`, `scale`, `t_steps`)."""
    import inspect
    import importlib
    ref = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'ref_signatures.json')))
    modmap = {'solvers': 'diff_sampler_b200.solvers', 'solver_utils': 'diff_sampler_b200.solver_utils',
              'solvers_amed': 'diff_sampler_b200.solvers_amed', 'gits_utils': 'diff_sampler_b200.gits_utils',
              'amed.solver_utils': 'diff_sampler_b200.solver_utils', 'gits.solver_utils': 'diff_sampler_b200.solver_utils'}
    checked = 0
    for key, params in ref.items():
        modname, fn = key.rsplit('.', 1)
        mod = importlib.import_module(modmap[modname])
        assert hasattr(mod, fn), f'{key} missing'
        mine = list(inspect.signature(getattr(mod, fn)).parameters.items())
        mine_named = [(n, p) for n, p in mine if p.kind not in (inspect.Parameter.VAR_KEYWORD, inspect.Parameter.VAR_POSITIONAL)]
        ref_named = [r for r in params if 'VAR_' not in r[1]]
        ref_has_kwargs = any('VAR_KEYWORD' in r[1] for r in params)
        assert len(mine_named) >= len(ref_named), key
        for (n, p), (rn, _, rd) in zip(mine_named, ref_named):
            assert n == rn, f'{key}: parameter {n} != reference {rn}'
            md = None if p.default is inspect._empty else repr(p.default)
            if rd is not None and md is not None:
                assert md == rd or (rd in ('[]',) and md == rd) or float_eq(md, rd), f'{key}.{n}: default {md} != reference {rd}'
        if ref_has_kwargs:
            assert any(p.kind == inspect.Parameter.VAR_KEYWORD for _, p in mine), f'{key} must swallow **kwargs (sample.py passes the whole CLI dict)'
        checked += 1
    assert checked >= 30


def float_eq(a, b):
    try:
        return float(a) == float(b)
    except ValueError:
        return False


def test_as_native_compiles_only_known_preconditioners_and_tracks_weight_updates(monkeypatch):
    """solvers.as_native (the drop-in entry sample.py's `sampler_fn(net, ...)` goes through): EDMPrecond over SongUNet/DhariwalUNet and
    CFGPrecond over a UNetModel are compiled once and cached with a weight fingerprint; other preconditioners are left alone."""
    import torch.nn as nn
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.ldm_net import B200LDMNet
    from diff_sampler_b200.net import B200Net

    def mk(cls_name, inner_name, path='model'):
        root = type(cls_name, (nn.Module,), {})()
        m = root
        parts = path.split('.')
        for i, part in enumerate(parts):
            child = type(inner_name if i == len(parts) - 1 else 'Node', (nn.Module,), {})()
            m.add_module(part, child)
            m = child
        m.register_parameter('w', nn.Parameter(torch.ones(3), requires_grad=False))
        return root
    made = []
    monkeypatch.setattr(B200Net, 'from_reference', classmethod(lambda cls, net, **kw: made.append(('edm', kw)) or object.__new__(B200Net)))
    monkeypatch.setattr(B200LDMNet, 'from_reference', classmethod(lambda cls, net, **kw: made.append(('ldm', kw)) or object.__new__(B200LDMNet)))
    edm = mk('EDMPrecond', 'SongUNet')
    a = solvers.as_native(edm)
    assert isinstance(a, B200Net) and solvers.as_native(edm) is a and len(made) == 1
    with torch.no_grad():
        edm.model.w.add_(1.0)                                   # in-place update (optimizer / EMA / load_state_dict): version counter moves
    b = solvers.as_native(edm)
    assert b is not a and len(made) == 2
    solvers.invalidate_native(edm)
    assert solvers.as_native(edm) is not b and len(made) == 3
    for other in ('VPPrecond', 'VEPrecond', 'iDDPMPrecond'):    # different c_skip / c_out / c_noise: never evaluated as EDM
        m = mk(other, 'SongUNet')
        assert solvers.as_native(m) is m
    assert len(made) == 3
    cfg = mk('CFGPrecond', 'UNetModel', 'model.model.diffusion_model')
    cfg.guidance_type = 'classifier-free'
    c = solvers.as_native(cfg)
    assert isinstance(c, B200LDMNet) and made[-1][0] == 'ldm' and solvers.as_native(cfg) is c
    fn = lambda x, s: x
    assert solvers.as_native(fn) is fn


def test_solver_update_rejects_missing_history_and_miscounted_coefficients():
    from diff_sampler_b200 import solver_utils as U
    x = torch.zeros(2, 4)
    with pytest.raises(ValueError, match='None'):
        U.solver_update(x, x, [1.0, 0.0, 0.5], hist=[None])
    with pytest.raises(ValueError, match='coefficients'):
        U.solver_update(x, x, [1.0, 0.0, 0.5, 0.5], hist=[x])


def test_benchmark_plans_cover_the_gemm_tile_configurations():
    """tests/test_gpu_gemm_tiles.py replays every GEMM configuration of the benchmarked plans against float64.  The EDM plans at the
    benchmark's batch and precision must keep offering it the cases that matter: N tiles 32 to 256, f8 blocks whose last 128-channel
    e4m3 block is half empty, both statistics granularities, the EDM output fold and rows mode."""
    from diff_sampler_b200 import gemm_replay
    cfgs = set()
    for name, B, fmin in (('cifar10', 512, 0), ('ffhq', 256, 256), ('imagenet64', 256, 0)):
        cfgs |= set(gemm_replay.plan_configs(gemm_replay.edm_plan(name, B, fmin)))
    assert {c.BN for c in cfgs} >= {32, 64, 128, 192, 256}
    assert any(c.f8 and ((c.C // 64) % 2 or (c.C2 // 64) % 2) for c in cfgs)
    assert {c.st_unit for c in cfgs} >= {2, 4}
    assert any(c.edm == 1 for c in cfgs)
    assert any(c.mode == 'rows' for c in cfgs)
    assert any(c.f8 and c.BN in (192, 256) for c in cfgs)


def _tiny_plans():
    """(name, plan, weight bytes, io) of every plan kind, at the sizes tests/test_plan_interp.py runs them."""
    from diff_sampler_b200 import clip_plan, ldm_plan, vae_plan
    from oracle import clip_oracle as CO, ldm_oracle as LO, vae_oracle as VO
    for name, f8 in (('tiny_song', False), ('tiny_adm', False), ('tiny_song', True), ('tiny_adm', True)):
        P, St = O.make_net(name, seed=0, dezero=True)
        spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
        spec.sigma_data = 0.5
        wb, info = planner.pack_weights(spec, P, f8=f8)
        B, R = 3, St['img_resolution']
        pl = planner.compile_plan(spec, wb, info, B, 1, B if spec.label_dim else 0, npass=3, f8=f8)
        lab = torch.eye(spec.label_dim)[torch.arange(B) % spec.label_dim].contiguous() if spec.label_dim else None
        yield (f'{name} f8={f8}', pl, wb.bytes(), {S.DS_IO_X: O.stacked_randn(range(B), (3, R, R)) * 2.0, S.DS_IO_D: torch.zeros(B, 3, R, R),
                                                  S.DS_IO_SIGMA: torch.tensor([2.0]), S.DS_IO_LABELS: lab, S.DS_IO_BOTTLENECK: torch.zeros(B, 64)})
    P, cfg = LO.make_params('tiny_ldm')
    st = ldm_plan.ldm_structure(P, cfg['num_heads'])
    for mode in ('fp16x3', 'f8', 'f8_linear'):
        f8, f8l = mode != 'fp16x3', mode == 'f8_linear'
        wb, info = ldm_plan.pack_ldm_weights(st, P, f8=f8, f8_linear=f8l)
        B, Bt, R, C = 2, 4, cfg['img_resolution'], cfg['in_channels']
        pl = ldm_plan.compile_ldm_plan(st, wb, info, B, Bt, 1, R, npass=3, f8=f8, f8_linear=f8l)
        g = torch.Generator().manual_seed(5)
        yield (f'tiny_ldm {mode}', pl, wb.bytes(), {S.DS_IO_X: torch.randn(B, C, R, R, generator=g), S.DS_IO_D: torch.zeros(Bt, C, R, R),
                                                    S.DS_IO_SIGMA: torch.tensor([417.0]), S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 0.37, 0.0]]),
                                                    S.DS_IO_BOTTLENECK: torch.zeros(Bt, 64),
                                                    S.DS_IO_CTX: torch.randn(Bt, 77, cfg['context_dim'], generator=g)})
    P, cfg = VO.make_params('tiny_vae', seed=0)
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    pl = vae_plan.compile_vae_plan(mods, meta, wb, 2, 8)
    z = torch.randn(2, cfg['z_channels'], 8, 8, generator=torch.Generator().manual_seed(3)) * cfg['scale_factor'] * 1.3
    yield ('tiny_vae', pl, wb.bytes(), {S.DS_IO_X: z, S.DS_IO_D: torch.zeros(2, meta['out_ch'], 8 * meta['upscale'], 8 * meta['upscale']),
                                        S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0 / cfg['scale_factor'], 0.0]])})
    P, cfg = CO.make_params('tiny_clip', seed=0)
    ccfg = clip_plan.clip_config(P)
    wb = clip_plan.pack_clip_weights(P, ccfg)
    ids = torch.randint(0, cfg['vocab_size'], (2, 77), generator=torch.Generator().manual_seed(4)).to(torch.int32)
    pl = clip_plan.compile_clip_plan(ccfg, wb, 2, 77)
    yield ('tiny_clip', pl, wb.bytes(), {S.DS_IO_X: ids, S.DS_IO_D: torch.zeros(2, 77, cfg['hidden_size'])})


def test_plan_op_write_spans_cover_every_store_of_the_interpreter():
    """tests/plan_spans.writes() is the span table the GPU op replay (tests/test_gpu_plan_ops.py) fills with NaN and outside of which
    it demands the arena unchanged byte for byte.  Here every op of every plan kind runs on the CPU interpreter, and every byte it
    changes -- arena and io slots -- must lie inside the op's spans; every pointer field must resolve."""
    from oracle import plan_interp as PI
    from plan_spans import resolve, writes
    seen = set()
    for name, pl, wb, io in _tiny_plans():
        io = {k: (v.contiguous() if v is not None else None) for k, v in io.items()}
        mem = PI.Memory(pl.arena_bytes, wb, io)
        regions = {S.SPACE_ARENA: mem.arena}
        regions.update({(S.SPACE_IO, k): v.reshape(-1).view(torch.uint8) for k, v in io.items() if v is not None})
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            seen.add(op.type)
            resolve(op, mem.arena, mem.weights, io)
            before = {k: r.clone() for k, r in regions.items()}
            PI.run_op(mem, op)
            inside = {k: torch.zeros(r.numel(), dtype=torch.bool) for k, r in regions.items()}
            for s in writes(op):
                space, off = s.ref >> 60, s.ref & PI.MASK60
                key = space if space == S.SPACE_ARENA else (space, off)
                if key not in inside:
                    continue
                o = off if space == S.SPACE_ARENA else 0
                assert o + s.nbytes <= inside[key].numel(), (name, i, s)
                inside[key][o:o + s.nbytes] = True
            for k, r in regions.items():
                stray = (r != before[k]) & ~inside[k]
                assert not stray.any(), (name, i, S.UNION_FIELD[op.type], op.tag, k, stray.nonzero()[:4].reshape(-1).tolist())
    assert seen == set(S.UNION_FIELD), sorted(S.UNION_FIELD[t] for t in set(S.UNION_FIELD) - seen)


def test_plan_op_spans_and_resolve_handle_the_benchmarked_plans():
    """Every op type of the five benchmarked plans (host-compiled, as tests/test_gpu_gemm_tiles.bench_plan builds them) has a span
    table entry and resolves."""
    from plan_spans import resolve, writes
    from test_gpu_gemm_tiles import WORKLOADS, bench_plan
    class Buf:                                   # stands in for a device buffer: resolve() only needs a base address and a size
        def __init__(self, base, n):
            self.base, self.n = base, n

        def data_ptr(self):
            return self.base

        def numel(self):
            return self.n
    for name in WORKLOADS:
        pl = bench_plan(name)
        types = set()
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            types.add(S.UNION_FIELD[op.type])
            resolve(op, Buf(1 << 40, pl.arena_bytes), Buf(1 << 44, 1 << 40), {k: Buf((k + 1) << 32, 1) for k in range(6)})
            spans = writes(op)
            assert spans or op.type == S.DS_OP_CHANMEAN, (name, i)
            assert all(s.nbytes > 0 and s.ref >> 60 in (S.SPACE_ARENA, S.SPACE_IO) for s in spans), (name, i, spans)
            for s in spans:
                if s.ref >> 60 == S.SPACE_ARENA:
                    assert (s.ref & ((1 << 60) - 1)) + s.nbytes <= pl.arena_bytes, (name, i, s)
        print(name, pl.n_ops, sorted(types))
        assert {'gemm', 'gn_apply', 'memset'} <= types

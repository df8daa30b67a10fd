"""Plans as data, checked without a GPU: the CPU plan interpreter (oracle/plan_interp.py) executes what the plan compilers emit --
arena offsets, operand planes and formats, packed weights and their scales, tap tables, epilogue options -- and the result must agree
with the network oracles (which are pinned to the real reference).  The EDM cases double as the interpreter's own validation: those
plans are the ones the GPU runs green in tests/test_gpu_parity.py."""
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import edm_nets, ldm_plan, plan as planner, vae_plan
from oracle import edm_oracle as O
from oracle import ldm_oracle as LO
from oracle import plan_interp as PI
from oracle import vae_oracle as VO

TOL = {False: 3e-5, True: 3e-4}          # fp16 hi/lo planes carry ~2^-22; the f8 mode adds ~3 % of the single-pass fp16 error


@pytest.mark.parametrize('name,f8', [('tiny_song', False), ('tiny_adm', False), ('tiny_song4', False), ('tiny_song', True), ('tiny_adm', True)])
def test_edm_plan_on_the_cpu_interpreter(name, f8):
    P, St = O.make_net(name, seed=0, dezero=True)
    spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
    spec.sigma_data = 0.5
    wb, info = planner.pack_weights(spec, P, f8=f8)
    B = 2
    pl = planner.compile_plan(spec, wb, info, B, 1, B if spec.label_dim else 0, npass=3, f8=f8)
    x = (O.stacked_randn(range(B), (3, St['img_resolution'], St['img_resolution'])) * 2.0).contiguous()
    sig = torch.tensor([2.0])
    lab = torch.eye(spec.label_dim)[torch.arange(B) % spec.label_dim].contiguous() if spec.label_dim else None
    D = torch.zeros_like(x)
    bott = torch.zeros(B, 64)
    PI.run_plan(pl, wb.bytes(), {S.DS_IO_X: x, S.DS_IO_D: D, S.DS_IO_SIGMA: sig, S.DS_IO_LABELS: lab, S.DS_IO_BOTTLENECK: bott})
    ref = O.OracleNet(P, St)(x, sig[0], class_labels=lab)
    err = (D - ref).abs().max().item()
    print(f'{name} f8={f8}: interpreter vs oracle {err:.3e}')
    assert err < TOL[f8] * max(1.0, ref.abs().max().item())


def test_edm_plan_mixed_precision_by_channel_count():
    """fp16f8 with f8_min_channels: narrow blocks stay fp16x3, wide ones run in the f8 mode; each GEMM finds its operands in its own format."""
    P, St = O.make_net('tiny_song', seed=0, dezero=True)
    spec = edm_nets.spec_from_params(P, 16, 3, 0)
    spec.sigma_data = 0.5
    x = (O.stacked_randn(range(2), (3, 16, 16)) * 2.0).contiguous()
    sig = torch.tensor([2.0])
    ref = O.OracleNet(P, St)(x, sig[0])
    counts, errs = [], []
    for thr in (0, 128, 1000):
        wb, info = planner.pack_weights(spec, P, f8=True, f8_min_channels=thr)
        pl = planner.compile_plan(spec, wb, info, 2, 1, 0, npass=3, f8=True)
        counts.append(sum(1 for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_GEMM and pl.ops_array[i].u.gemm.f8))
        D = torch.zeros_like(x)
        PI.run_plan(pl, wb.bytes(), {S.DS_IO_X: x, S.DS_IO_D: D, S.DS_IO_SIGMA: sig, S.DS_IO_BOTTLENECK: torch.zeros(2, 64)})
        errs.append((D - ref).abs().max().item())
    assert counts[0] > counts[1] > counts[2] == 0
    assert errs[0] < TOL[True] and errs[1] < errs[0] and errs[2] < TOL[False]


def test_edm_plan_variants_per_sample_sigma_and_broadcast_label():
    """The (batch, #sigma, #labels) plan variants: per-sample sigma (AMED evaluates the net at scale_time * t_mid per sample) and one
    class label broadcast to the batch (networks_edm.py:485)."""
    P, St = O.make_net('tiny_adm', seed=0, dezero=True)
    spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
    spec.sigma_data = 0.5
    wb, info = planner.pack_weights(spec, P)
    B = 3
    x0 = O.stacked_randn(range(B), (3, St['img_resolution'], St['img_resolution']))
    on = O.OracleNet(P, St)
    for nsig, nlab in ((B, B), (1, 1), (B, 1)):
        pl = planner.compile_plan(spec, wb, info, B, nsig, nlab, npass=3)
        sig = torch.tensor([3.0, 0.4, 11.0])[:nsig].contiguous()
        x = (x0 * (sig[:, None, None, None] if nsig > 1 else sig[0])).contiguous()
        lab = torch.eye(spec.label_dim)[torch.tensor([1, 4, 7])[:nlab]].contiguous()
        D = torch.zeros_like(x)
        PI.run_plan(pl, wb.bytes(), {S.DS_IO_X: x, S.DS_IO_D: D, S.DS_IO_SIGMA: sig, S.DS_IO_LABELS: lab, S.DS_IO_BOTTLENECK: torch.zeros(B, 64)})
        ref = on(x, sig if nsig > 1 else sig[0], class_labels=lab if nlab > 1 else lab.expand(B, -1))
        err = (D - ref).abs().max().item()
        print(f'tiny_adm nsig={nsig} nlab={nlab}: {err:.3e}')
        assert err < TOL[False] * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('mode', ['fp16x3', 'f8', 'f8_linear'])
def test_ldm_plan_on_the_cpu_interpreter(mode):
    f8, f8l = mode != 'fp16x3', mode == 'f8_linear'
    P, cfg = LO.make_params('tiny_ldm')
    st = ldm_plan.ldm_structure(P, cfg['num_heads'])
    wb, info = ldm_plan.pack_ldm_weights(st, P, f8=f8, f8_linear=f8l)
    B = Bt = 2
    R = cfg['img_resolution']
    pl = ldm_plan.compile_ldm_plan(st, wb, info, B, Bt, 1, R, npass=3, f8=f8, f8_linear=f8l)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, cfg['in_channels'], R, R, generator=g).contiguous()
    ctx = torch.randn(Bt, 77, cfg['context_dim'], generator=g).contiguous()
    t = torch.tensor([417.0])
    c_in = 0.37
    eps = torch.zeros(Bt, cfg['in_channels'], R, R)
    io = {S.DS_IO_X: x, S.DS_IO_D: eps, S.DS_IO_SIGMA: t, S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, c_in, 0.0]]), S.DS_IO_BOTTLENECK: torch.zeros(Bt, 64),
          S.DS_IO_CTX: ctx}
    PI.run_plan(pl, wb.bytes(), io)
    with torch.no_grad():
        ref = LO.unet_forward(P, cfg, x * c_in, t.expand(Bt), ctx)
    err = (eps - ref).abs().max().item()
    print(f'tiny_ldm {mode}: interpreter vs oracle {err:.3e}')
    assert err < TOL[f8] * max(1.0, ref.abs().max().item())


def test_vae_decoder_plan_on_the_cpu_interpreter():
    """The first-stage decoder lowering (vae_plan.py) has not run on hardware yet; as data it reproduces the oracle module by module."""
    P, cfg = VO.make_params('tiny_vae', seed=0)
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    B, R = 2, 8
    pl = vae_plan.compile_vae_plan(mods, meta, wb, B, R)
    g = torch.Generator().manual_seed(3)
    z = (torch.randn(B, cfg['z_channels'], R, R, generator=g) * cfg['scale_factor'] * 1.3).contiguous()
    out = torch.zeros(B, meta['out_ch'], R * meta['upscale'], R * meta['upscale'])
    io = {S.DS_IO_X: z, S.DS_IO_D: out, S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0 / cfg['scale_factor'], 0.0]])}
    mem = PI.run_plan(pl, wb.bytes(), io)
    taps = {}
    with torch.no_grad():
        ref = VO.decode(P, cfg, z, taps=taps)
    for mname, t in taps.items():
        n, c, h, w = t.shape
        mine = PI.read_buffer(mem, pl, 'h:' + mname, (n, h, w, c)).permute(0, 3, 1, 2)
        assert (mine - t).abs().max().item() < 3e-5 * max(1.0, t.abs().max().item()), mname
    assert (out - ref).abs().max().item() < 3e-5


def test_clip_text_encoder_plan_on_the_cpu_interpreter():
    """The text-encoder plan (embedding gather, pre-LN layers with the causal fused attention, quick-GELU MLP, fp32 final LayerNorm)
    against transformers' CLIPTextModel output (tests/golden/ref_clip.npz) and the oracle."""
    import os
    import numpy as np
    from diff_sampler_b200 import clip_plan
    from oracle import clip_oracle as CO
    d = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_clip.npz'))
    P, cfg = CO.make_params('tiny_clip', seed=0)
    got_cfg = clip_plan.clip_config(P)
    assert all(got_cfg[k] == cfg[k] for k in got_cfg)
    wb = clip_plan.pack_clip_weights(P, got_cfg)
    ids = torch.from_numpy(d['tiny_clip/ids'])
    B, T = ids.shape
    pl = clip_plan.compile_clip_plan(got_cfg, wb, B, T)
    assert pl.meta['n_gemm'] == 5 * cfg['num_hidden_layers']
    out = torch.zeros(B, T, cfg['hidden_size'])
    PI.run_plan(pl, wb.bytes(), {S.DS_IO_X: ids.to(torch.int32).contiguous(), S.DS_IO_D: out})
    err = (out - torch.from_numpy(d['tiny_clip/out'])).abs().max().item()
    print(f'clip plan on the interpreter vs transformers: {err:.3e}')
    assert err < 3e-5
    # a shorter sequence is its own plan (position rows 0..T-1; causal => equal to the prefix of the long run)
    T2 = 20
    pl2 = clip_plan.compile_clip_plan(got_cfg, wb, B, T2)
    out2 = torch.zeros(B, T2, cfg['hidden_size'])
    PI.run_plan(pl2, wb.bytes(), {S.DS_IO_X: ids[:, :T2].to(torch.int32).contiguous(), S.DS_IO_D: out2})
    assert (out2 - out[:, :T2]).abs().max().item() < 3e-5
    with pytest.raises(ValueError):
        clip_plan.compile_clip_plan(got_cfg, wb, B, 78)

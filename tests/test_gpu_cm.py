"""Consistency-Models LSUN-256 nets on the H100: the posemb kernel's noise scale, the native denoiser against the float64 oracle
(oracle/cm_oracle.py, pinned to the reference by tests/golden/ref_cm.npz) at the tiny and the full lsun_setting size, every op of the
full-size plan against the plan interpreter, the samplers end to end, and the two entry points (B200Net.from_cm, from_cm_checkpoint)."""
import io
import math

import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import cm_net

pytestmark = pytest.mark.gpu

TOL = 1e-3                               # fp16x3 and fp16f8 (tests/test_gpu_parity.py); single-pass fp16 has its own, looser bound
TOL_FP16 = 2e-2


def _dev():
    return torch.device('cuda:0')


def _tiny():
    from oracle import cm_oracle as CO
    sd = cm_net.init_state_dict(cm_net.TINY_SETTING, seed=0)
    return sd, CO.CMOracle(sd, cm_net.TINY_SETTING)


def _native(sd, setting, precision=None):
    from diff_sampler_b200.net import B200Net
    spec, params = cm_net.convert(sd, setting)
    return B200Net(params, spec.img_resolution, spec.img_channels, 0, precision=precision, device=_dev(), spec=spec)


def _latents(B, R, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, R, R, generator=g)


def test_posemb_noise_scale():
    """Mode 0 with noise_scale = 1000 embeds 1000 ln(sigma) / 4 ([cos | sin], endpoint=False) and leaves the coefficients alone."""
    from diff_sampler_b200 import _lib
    sig = torch.tensor([0.002, 1.0, 80.0, 0.37, 13.0], device=_dev())
    B, nc = sig.numel(), 256
    coef = torch.zeros(B, 4, device=_dev())
    emb = torch.zeros(B, nc, device=_dev())
    _lib.op_launch(S.PosembDesc(sigma=sig.data_ptr(), nsig=B, num_channels=nc, endpoint=0, swap_sincos=0, sigma_data=0.5,
                                coef=coef.data_ptr(), emb=emb.data_ptr(), noise_scale=1000.0))
    torch.cuda.synchronize()
    s = sig.double()
    t = 1000 * s.log() / 4
    a = t[:, None] * torch.exp(-math.log(10000.0) * torch.arange(nc // 2, device=_dev(), dtype=torch.float64) / (nc // 2))[None]
    ref = torch.cat([a.cos(), a.sin()], dim=1)
    # |argument| reaches 1000 ln(80) / 4 = 1095: one fp32 ulp of it (1.2e-4) is the floor of any fp32 evaluation
    err = (emb.double() - ref).abs().max().item()
    s2 = s ** 2 + 0.25
    refc = torch.stack([0.25 / s2, s * 0.5 / s2.sqrt(), 1 / s2.sqrt(), s.log() / 4], dim=1)
    errc = ((coef.double() - refc).abs() / refc.abs().clamp_min(1e-3)).max().item()
    print(f'posemb noise_scale=1000: emb err {err:.3e}, coef rel err {errc:.3e}')
    assert err < 5e-4 and errc < 1e-6


@pytest.mark.parametrize('precision,tol', [('fp16x3', TOL), ('fp16', TOL_FP16), ('fp16f8', TOL)])
def test_tiny_denoiser_parity(precision, tol):
    sd, orc = _tiny()
    nat = _native(sd, cm_net.TINY_SETTING, precision)
    x0 = _latents(3, 32)
    for sigma in (80.0, 2.5, 0.05, 0.002):
        x = x0 * sigma
        ref = orc(x, torch.tensor(sigma))
        got = nat(x.to(_dev()), torch.tensor(sigma, device=_dev())).cpu()
        err = (got - ref).abs().max().item()
        print(f'tiny CM {precision} sigma={sigma}: max-abs err {err:.3e} (max|D| {ref.abs().max().item():.2f})')
        assert err < tol
    sig = torch.tensor([3.0, 0.4, 11.0])
    x = x0 * sig[:, None, None, None]
    ref = orc(x, sig)
    got = nat(x.to(_dev()), sig.to(_dev())).cpu()
    err = (got - ref).abs().max().item()
    print(f'tiny CM {precision} per-sample sigma: {err:.3e}')
    assert err < tol


@pytest.fixture(scope='module')
def full():
    from oracle import cm_oracle as CO
    sd = cm_net.init_state_dict(None, seed=0)
    return sd, CO.CMOracle(sd, cm_net.lsun_setting(), device=_dev())


@pytest.mark.parametrize('precision,tol', [('fp16x3', TOL), ('fp16', TOL_FP16), ('fp16f8', TOL)])
def test_fullsize_denoiser_parity(full, precision, tol):
    """lsun_setting at batch 2 with random de-zeroed weights (zero_module layers given O(1) weights)."""
    sd, orc = full
    nat = _native(sd, None, precision)
    x0 = _latents(2, 256)
    for sigma in (40.0, 1.0, 0.02):
        x = x0 * sigma
        ref = orc(x, torch.tensor(sigma))
        got = nat(x.to(_dev()), torch.tensor(sigma, device=_dev())).cpu()
        err = (got - ref).abs().max().item()
        print(f'lsun CM {precision} sigma={sigma}: max-abs err {err:.3e} (max|D| {ref.abs().max().item():.2f})')
        assert err < tol
    del nat
    torch.cuda.empty_cache()


def test_fullsize_plan_ops_against_the_interpreter(full, monkeypatch):
    """Every op of the full-size fp16f8 plan at batch 2, replayed alone on 0xFF-filled outputs against the float64 interpreter, as
    tests/test_gpu_plan_ops.py does for the benchmarked plans."""
    import test_gpu_plan_ops as TPO
    from diff_sampler_b200 import _lib, plan as planner
    sd, _ = full
    spec, params = cm_net.convert(sd)
    wb, info = planner.pack_weights(spec, params, f8=True)
    B = 2
    pl = planner.compile_plan(spec, wb, info, B, 1, 0, npass=3, f8=True)
    g = torch.Generator().manual_seed(11)
    io_host = {S.DS_IO_X: torch.randn(B, 3, 256, 256, generator=g) * 2.5, S.DS_IO_D: torch.zeros(B, 3, 256, 256),
               S.DS_IO_SIGMA: torch.tensor([2.5]), S.DS_IO_BOTTLENECK: torch.zeros(B, 64)}
    monkeypatch.setattr(TPO, 'workload', lambda name: (pl, wb.bytes(), io_host))
    from oracle import cm_interp as CI
    monkeypatch.setitem(TPO.PI._DISPATCH, S.DS_OP_POSEMB, CI.DISPATCH_ENTRY)     # the interpreter's posemb with the noise scale
    res = TPO.replay(_lib, 'cm_lsun')
    # the embedding argument is 1000 ln(sigma) / 4 = 229 here: its fp32 rounding alone is ~1.4e-5, so the posemb bound of the
    # benchmarked plans (2e-6 absolute, for |ln(sigma) / 4| < 1.1) scales with |argument|
    t_emb = max(1.0, 1000.0 * abs(math.log(2.5)) / 4)
    bad = [r for r in res['rows'] if r['ratio'] > (t_emb if r['type'] == 'posemb' else 1.0) or r['problems']]
    worst = {}
    for r in res['rows']:
        worst[r['type']] = max(worst.get(r['type'], 0.0), r['ratio'])
    print(f"cm_lsun: {res['n_ops']} ops, {res['seconds']:.1f} s, peak {res['peak'] / 2 ** 30:.2f} GiB; worst ratio per type "
          + ', '.join(f'{k} {v:.3f}' for k, v in sorted(worst.items())))
    assert len(res['rows']) == res['n_ops'] and {r['type'] for r in res['rows']} == res['types']
    assert all(res['rows'][i]['type'] == 'gn_stats' for i in res['skips'])
    assert not bad, '\n'.join(TPO._fmt('cm_lsun', r) for r in bad[:20])


SAMPLERS = [('heun', dict(num_steps=5)), ('dpm_pp', dict(num_steps=6, max_order=2, predict_x0=True)),
            ('ipndm', dict(num_steps=6, max_order=4))]


@pytest.mark.parametrize('solver,kw', SAMPLERS, ids=[s for s, _ in SAMPLERS])
def test_tiny_sampler_parity(solver, kw):
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    sd, orc = _tiny()
    nat = _native(sd, cm_net.TINY_SETTING)
    lat = _latents(4, 32, seed=1)
    ref = SO.sample(orc, lat, solver, **kw)
    got = getattr(solvers, solver + '_sampler')(nat, lat.to(_dev()), **kw).cpu()
    err = (got - ref).abs().max().item()
    print(f'tiny CM {solver} {kw}: final max-abs err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
    assert err < TOL


def test_tiny_gits_schedule_parity():
    """DPM-Solver++(2M) on a GITS schedule: 5 steps picked from an 11-point polynomial teacher grid."""
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    sd, orc = _tiny()
    nat = _native(sd, cm_net.TINY_SETTING)
    dp_list = [0, 2, 4, 7, 10]
    t_ref = SO.get_schedule(11, 0.002, 80, dp_list=dp_list)
    lat = _latents(4, 32, seed=2)
    kw = dict(num_steps=5, max_order=2, predict_x0=True)
    ref = SO.sample(orc, lat, 'dpm_pp', t_steps=t_ref, **kw)
    got = solvers.dpm_pp_sampler(nat, lat.to(_dev()), t_steps=t_ref.to(_dev()), **kw).cpu()
    err = (got - ref).abs().max().item()
    print(f'tiny CM dpm_pp on GITS schedule {dp_list}: {err:.3e}')
    assert err < TOL


def test_tiny_amed_dpmpp_with_the_middle_block_tap():
    """AMED-DPM++ plug-in: the predictor reads mean(middle_block output, dim=1), [B, 8, 8] (solvers_amed.py:11-14)."""
    import os
    import numpy as np
    from oracle import amed_oracle as AO
    from diff_sampler_b200 import solvers_amed
    from diff_sampler_b200.amed_predictor import AMEDPredictor
    sd, orc = _tiny()
    nat = _native(sd, cm_net.TINY_SETTING)
    B = 3
    x = _latents(B, 32, seed=3) * 5.0
    bott = torch.zeros(B, 64, device=_dev())
    nat(x.to(_dev()), torch.tensor(5.0, device=_dev()), bottleneck=bott)
    orc.taps = {}
    orc(x, torch.tensor(5.0))
    tap = orc.taps['middle_block'].mean(dim=1).reshape(B, 64).float()
    err_tap = (bott.cpu() - tap).abs().max().item()
    print(f'middle-block tap: {err_tap:.3e}')
    assert err_tap < TOL
    d = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_amed.npz'))
    ci = 5                                                   # dpm_pp, max_order 3, predict_x0, scale_dir 0.05 (test_gpu_parity.AMED_CASES)
    W = {k[len(f'amed/{ci}/pred/'):]: torch.from_numpy(d[k]) for k in d.files if k.startswith(f'amed/{ci}/pred/')}
    cfg = dict(scale_dir=0.05, scale_time=0.0)
    kw = dict(num_steps=5, max_order=3, predict_x0=True)
    lat = _latents(B, 32, seed=4)
    ref = AO.sample_amed(orc, lat, 'dpm_pp', W, cfg, bottleneck_block='middle_block', **kw)
    got = solvers_amed.dpm_pp_sampler(nat, lat.to(_dev()), AMED_predictor=AMEDPredictor(W, **cfg).to(_dev()), **kw).cpu()
    err = (got - ref).abs().max().item()
    print(f'AMED-DPM++ on the tiny CM net: {err:.3e}')
    assert err < TOL


class _CMPrecondStandIn(torch.nn.Module):
    """The attributes and state_dict layout of the reference's CMPrecond (networks_edm.py:504-531) around a UNetModel."""

    def __init__(self, sd, img_resolution, sigma_min=0.002, sigma_max=80.0, sigma_data=0.5):
        super().__init__()
        self.model = torch.nn.Module()
        for k, v in sd.items():
            mod = self.model
            *path, leaf = k.split('.')
            for p in path:
                if not hasattr(mod, p):
                    mod.add_module(p, torch.nn.Module())
                mod = getattr(mod, p)
            mod.register_parameter(leaf, torch.nn.Parameter(v.clone(), requires_grad=False))
        self.img_resolution, self.img_channels, self.label_dim = img_resolution, 3, 0
        self.sigma_min, self.sigma_max, self.sigma_data = sigma_min, sigma_max, sigma_data


def test_from_cm_and_from_cm_checkpoint():
    from diff_sampler_b200.net import B200Net
    sd, orc = _tiny()
    mod = _CMPrecondStandIn({k: v.half() for k, v in sd.items()}, 32, sigma_max=60.0)
    a = B200Net.from_cm(mod, setting=cm_net.TINY_SETTING, device=_dev())
    assert (a.img_resolution, a.sigma_min, a.sigma_max, a.sigma_data, a.label_dim) == (32, 0.002, 60.0, 0.5, 0)
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    b = B200Net.from_cm_checkpoint(buf, setting=cm_net.TINY_SETTING, device=_dev())
    assert (b.sigma_min, b.sigma_max, b.sigma_data) == (0.002, 80.0, 0.5) and b.spec.noise_scale == 1000.0
    x = _latents(2, 32, seed=5) * 3.0
    ref = orc(x, torch.tensor(3.0))
    gb = b(x.to(_dev()), torch.tensor(3.0, device=_dev())).cpu()
    ga = a(x.to(_dev()), torch.tensor(3.0, device=_dev())).cpu()
    from oracle import cm_oracle as CO
    ref16 = CO.CMOracle({k: v.half().float() for k, v in sd.items()}, cm_net.TINY_SETTING)(x, torch.tensor(3.0))
    ea, eb = (ga - ref16).abs().max().item(), (gb - ref).abs().max().item()
    print(f'from_cm (fp16 torso) {ea:.3e}, from_cm_checkpoint {eb:.3e}')
    assert ea < TOL and eb < TOL
    with pytest.raises((KeyError, ValueError)):
        B200Net.from_cm(mod, device=_dev())                      # the default lsun_setting does not describe this state dict

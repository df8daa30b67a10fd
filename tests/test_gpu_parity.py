"""Parity proper (GPU): the native denoiser and every sampler, called through the reference-facing API
(B200Net(x, sigma, class_labels) / solvers.<name>_sampler(net, latents, ...)), against the CPU oracle
(oracle/ — pinned to the real reference by tests/golden) on the same seeded latents and weights.

Tolerance (BASELINE.json north_star): max-abs <= 1e-3 per pixel on identical latents/weights.  The weight set is the
'de-zeroed' random init (|F_x| = O(1)); the reference-init nets (init_zero layers ~1e-5) are a vacuous gate and are
checked too.  precision='fp16x3' (split-precision wgmma, 3 MMAs per product) is the mode that must hold 1e-3;
precision='fp16' (single pass) is reported with its own, looser bound.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


TOL = 1e-3


def _dev():
    return torch.device('cuda:0')


def _oracle(name, dezero=True, seed=0):
    from oracle import edm_oracle as O
    P, S = O.make_net(name, seed=seed, dezero=dezero)
    return O.OracleNet(P, S), P, S


def _native(P, S, precision=None):
    from diff_sampler_b200.net import B200Net
    return B200Net(P, S['img_resolution'], S['img_channels'], S['label_dim'], precision=precision, device=_dev())


def _labels(S, B, seed=0):
    if not S['label_dim']:
        return None
    g = torch.Generator().manual_seed(seed)
    return torch.eye(S['label_dim'])[torch.randint(S['label_dim'], (B,), generator=g)]


@pytest.mark.parametrize('name,precision', [('tiny_song', 'fp16x3'), ('tiny_adm', 'fp16x3'),
                                            ('tiny_song', 'fp16f8'), ('tiny_adm', 'fp16f8')])
def test_block_outputs_localise(name, precision):
    """Per-block activations of the native plan vs the oracle's (diagnostic: names the first block that drifts)."""
    from oracle import edm_oracle as O
    on, P, S = _oracle(name)
    nat = _native(P, S, precision)
    B = 3
    x = O.stacked_randn(range(B), (S['img_channels'], S['img_resolution'], S['img_resolution'])) * 3.0
    lab = _labels(S, B)
    sig = torch.tensor(1.7)
    on.taps = {}
    ref = on(x, sig, class_labels=lab)
    got = nat(x.to(_dev()), sig.to(_dev()), class_labels=None if lab is None else lab.to(_dev()))
    torch.cuda.synchronize()
    nlab = B if lab is not None else 0
    worst = 0.0
    for bname, t in on.taps.items():
        n, c, h, w = t.shape
        mine = nat.debug_read(B, 1, nlab, 'x:' + bname, n * c * h * w).reshape(n, h, w, c).permute(0, 3, 1, 2)
        err = (mine - t).abs().max().item()
        worst = max(worst, err / max(1.0, t.abs().max().item()))
        print(f'{bname:28s} max|ref| {t.abs().max().item():9.4f}  err {err:.3e}')
    err = (got.cpu() - ref).abs().max().item()
    print(f'{name}: D err {err:.3e}')
    assert worst < (1e-4 if precision == 'fp16x3' else 5e-4) and err < TOL


@pytest.mark.parametrize('name,precision,tol', [('tiny_song', 'fp16x3', TOL), ('tiny_adm', 'fp16x3', TOL), ('tiny_song', 'fp16', 2e-2),
                                                ('tiny_adm', 'fp16', 2e-2)])
def test_denoiser_parity(name, precision, tol):
    from oracle import edm_oracle as O
    on, P, S = _oracle(name)
    nat = _native(P, S, precision)
    B = 5
    x0 = O.stacked_randn(range(B), (S['img_channels'], S['img_resolution'], S['img_resolution']))
    lab = _labels(S, B)
    labd = None if lab is None else lab.to(_dev())
    for sigma in (80.0, 2.5, 0.05):
        x = x0 * sigma
        ref = on(x, torch.tensor(sigma), class_labels=lab)
        got = nat(x.to(_dev()), torch.tensor(sigma, device=_dev()), class_labels=labd).cpu()
        err = (got - ref).abs().max().item()
        print(f'{name} {precision} sigma={sigma}: max-abs err {err:.3e} (max|D| {ref.abs().max().item():.2f})')
        assert err < tol
    # per-sample sigma (AMED evaluates the net at scale_time * t_mid per sample)
    sig = torch.tensor([3.0, 0.4, 11.0, 0.9, 50.0])
    x = x0 * sig[:, None, None, None]
    ref = on(x, sig, class_labels=lab)
    got = nat(x.to(_dev()), sig.to(_dev()), class_labels=labd).cpu()
    err = (got - ref).abs().max().item()
    print(f'{name} {precision} per-sample sigma: {err:.3e}')
    assert err < tol


@pytest.mark.parametrize('name', ['tiny_song', 'tiny_adm', 'cifar10'])
def test_denoiser_parity_f8_mode(name):
    """precision='fp16f8': block convolutions as fp16 hi x hi + two e4m3 correction products (2 MMA units per product instead of 3).
    Expected error ~1e-4 on the de-zeroed nets (tests/study_fp8_corrections.py), inside the 1e-3 contract."""
    from oracle import edm_oracle as O
    on, P, S = _oracle(name)
    nat = _native(P, S, 'fp16f8')
    ref_nat = _native(P, S, 'fp16x3')
    B = 3
    x0 = O.stacked_randn(range(B), (S['img_channels'], S['img_resolution'], S['img_resolution']))
    lab = _labels(S, B)
    labd = None if lab is None else lab.to(_dev())
    for sigma in (80.0, 2.5, 0.05):
        x = x0 * sigma
        ref = on(x, torch.tensor(sigma), class_labels=lab)
        got = nat(x.to(_dev()), torch.tensor(sigma, device=_dev()), class_labels=labd).cpu()
        got3 = ref_nat(x.to(_dev()), torch.tensor(sigma, device=_dev()), class_labels=labd).cpu()
        err, err3 = (got - ref).abs().max().item(), (got3 - ref).abs().max().item()
        print(f'{name} fp16f8 sigma={sigma}: max-abs err {err:.3e} (fp16x3 {err3:.3e}, max|D| {ref.abs().max().item():.2f})')
        assert err < TOL / 2


def test_sampler_parity_f8_mode():
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    on, P, S = _oracle('tiny_song')
    nat = _native(P, S, 'fp16f8')
    lat = O.stacked_randn(range(4), (3, 16, 16))
    for solver, kw in (('heun', dict(num_steps=6)), ('dpm_pp', dict(num_steps=7, max_order=3, predict_x0=True))):
        ref = SO.sample(on, lat, solver, **kw)
        got = getattr(solvers, solver + '_sampler')(nat, lat.to(_dev()), **kw).cpu()
        err = (got - ref).abs().max().item()
        print(f'tiny_song fp16f8 {solver}: final-image max-abs err {err:.3e}')
        assert err < TOL


@pytest.mark.parametrize('name,solver,kw', [('cifar10', 'heun', dict(num_steps=10)),
                                            ('imagenet64', 'dpm_pp', dict(num_steps=11, max_order=2, predict_x0=True))])
def test_fullsize_sampler_parity_f8_mode(name, solver, kw):
    """The configurations bench.py runs in fp16f8 by default (PRECISION_FOR): BASELINE config 2 (CIFAR-10, Heun NFE=18) and config 4's
    net and solver (ImageNet-64, DPM-Solver++(2M) NFE=10), full-size nets, final images against the CPU oracle within the 1e-3 contract."""
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    on, P, S = _oracle(name)
    nat = _native(P, S, 'fp16f8')
    B = 2
    lat = O.stacked_randn(range(B), (3, S['img_resolution'], S['img_resolution']))
    lab = _labels(S, B)
    ref = SO.sample(on, lat, solver, class_labels=lab, **kw)
    got = getattr(solvers, solver + '_sampler')(nat, lat.to(_dev()), class_labels=None if lab is None else lab.to(_dev()), **kw).cpu()
    err = (got - ref).abs().max().item()
    print(f'{name} fp16f8 {solver} {kw}: final-image max-abs err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
    assert err < TOL


@pytest.mark.parametrize('fuse', [True, False])
def test_fused_groupnorm_stats_plan_matches(fuse):
    """The plan with GroupNorm statistics taken from the GEMM epilogues (default) and the one with the separate gn_stats pass give the
    same denoiser output."""
    from oracle import edm_oracle as O
    from diff_sampler_b200.net import B200Net
    on, P, S = _oracle('tiny_adm')
    nat = B200Net(P, S['img_resolution'], S['img_channels'], S['label_dim'], device=_dev(), fuse_stats=fuse)
    x = O.stacked_randn(range(3), (3, 16, 16)) * 2.0
    lab = _labels(S, 3)
    ref = on(x, torch.tensor(2.0), class_labels=lab)
    got = nat(x.to(_dev()), torch.tensor(2.0, device=_dev()), class_labels=lab.to(_dev())).cpu()
    assert (got - ref).abs().max().item() < TOL


def test_reference_init_weights_are_a_vacuous_gate():
    """With the reference's own init (init_zero layers ~1e-5) |F_x| ~ 3e-5 and even single-pass fp16 is ~1e-7 off."""
    from oracle import edm_oracle as O
    on, P, S = _oracle('tiny_song', dezero=False)
    nat = _native(P, S, 'fp16')
    x = O.stacked_randn(range(4), (3, 16, 16)) * 2.0
    ref = on(x, torch.tensor(2.0))
    got = nat(x.to(_dev()), torch.tensor(2.0, device=_dev())).cpu()
    err = (got - ref).abs().max().item()
    print(f'reference-init tiny_song fp16: {err:.3e}')
    assert err < 1e-5


@pytest.mark.parametrize('name', ['cifar10', 'ffhq', 'imagenet64'])
def test_fullsize_denoiser_parity(name):
    """BASELINE config net (55.7 M parameters), batch 2, one evaluation at three noise levels."""
    from oracle import edm_oracle as O
    on, P, S = _oracle(name)
    nat = _native(P, S)
    x0 = O.stacked_randn(range(2), (3, S['img_resolution'], S['img_resolution']))
    lab = _labels(S, 2)
    labd = None if lab is None else lab.to(_dev())
    for sigma in (40.0, 1.0):
        x = x0 * sigma
        ref = on(x, torch.tensor(sigma), class_labels=lab)
        got = nat(x.to(_dev()), torch.tensor(sigma, device=_dev()), class_labels=labd).cpu()
        err = (got - ref).abs().max().item()
        print(f'{name} sigma={sigma}: max-abs err {err:.3e} (max|D| {ref.abs().max().item():.2f})')
        assert err < TOL


SAMPLER_CASES = [
    ('euler', dict(num_steps=6)),
    ('euler', dict(num_steps=5, afs=True, denoise_to_zero=True)),
    ('heun', dict(num_steps=5)),
    ('dpm_2', dict(num_steps=5, r=0.4)),
    ('ipndm', dict(num_steps=7, max_order=4)),
    ('ipndm', dict(num_steps=6, max_order=3, afs=True)),
    ('ipndm_v', dict(num_steps=7, max_order=4)),
    ('deis', dict(num_steps=7, max_order=4, deis_mode='tab')),
    ('deis', dict(num_steps=6, max_order=4, deis_mode='rhoab')),
    ('dpm_pp', dict(num_steps=7, max_order=3, predict_x0=True)),
    ('dpm_pp', dict(num_steps=6, max_order=2, predict_x0=False)),
    ('dpm_pp', dict(num_steps=6, max_order=3, predict_x0=True, afs=True, lower_order_final=False)),
    ('unipc', dict(num_steps=7, max_order=3, predict_x0=True, variant='bh2')),
    ('unipc', dict(num_steps=6, max_order=2, predict_x0=False, variant='bh1')),
    ('unipc', dict(num_steps=6, max_order=3, predict_x0=True, afs=True)),
]


@pytest.mark.parametrize('solver,kw', SAMPLER_CASES, ids=[f'{s}-{i}' for i, (s, _) in enumerate(SAMPLER_CASES)])
@pytest.mark.parametrize('name', ['tiny_song', 'tiny_adm'])
def test_sampler_parity(name, solver, kw):
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers, solver_utils
    on, P, S = _oracle(name)
    nat = _native(P, S)
    B = 4
    lat = O.stacked_randn(range(B), (S['img_channels'], S['img_resolution'], S['img_resolution']))
    lab = _labels(S, B)
    kw = dict(kw)
    mode = kw.pop('deis_mode', None)
    common = dict(sigma_min=0.002, sigma_max=80, schedule_type='polynomial', schedule_rho=7)
    okw, nkw = dict(kw), dict(kw)
    if solver == 'deis':
        ts = SO.get_schedule(kw['num_steps'], 0.002, 80)
        okw['coeff_list'] = SO.get_deis_coeff_list(ts, kw['max_order'], deis_mode=mode)
        nkw['coeff_list'] = solver_utils.get_deis_coeff_list(ts, kw['max_order'], deis_mode=mode)
    ref = SO.sample(on, lat, solver, class_labels=lab, **common, **okw)
    fn = getattr(solvers, solver + '_sampler')
    got = fn(nat, lat.to(_dev()), class_labels=None if lab is None else lab.to(_dev()), **common, **nkw).cpu()
    err = (got - ref).abs().max().item()
    print(f'{name} {solver} {kw}: final max-abs err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
    assert err < TOL


def test_trajectory_and_eps_outputs():
    """return_inters / return_eps stacking (solvers.py:82-95) — what GITS consumes."""
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    on, P, S = _oracle('tiny_song')
    nat = _native(P, S)
    lat = O.stacked_randn(range(3), (3, 16, 16))
    for solver in ('euler', 'ipndm', 'dpm_pp'):
        rt, re = SO.sample(on, lat, solver, num_steps=6, return_inters=True, return_eps=True, denoise_to_zero=(solver == 'euler'))
        gt, ge = getattr(solvers, solver + '_sampler')(nat, lat.to(_dev()), num_steps=6, return_inters=True, return_eps=True,
                                                       denoise_to_zero=(solver == 'euler'))
        assert tuple(gt.shape) == tuple(rt.shape) and tuple(ge.shape) == tuple(re.shape)
        e1, e2 = (gt.cpu() - rt).abs().max().item(), (ge.cpu() - re).abs().max().item()
        print(f'{solver}: traj err {e1:.3e} eps err {e2:.3e}')
        assert e1 < TOL and e2 < TOL


# --------------------------------------------------------------------------------------------- AMED / GITS
AMED_CASES = [
    ('amed', 'amed_sampler', dict(num_steps=4), dict(scale_dir=0.01, scale_time=0.2)),
    ('euler', 'euler_sampler', dict(num_steps=4, afs=True), dict(scale_dir=0.01, scale_time=0.2)),
    ('ipndm', 'ipndm_sampler', dict(num_steps=5, max_order=3), dict(scale_dir=0.01, scale_time=0.2)),
    ('dpm_2', 'dpm_2_sampler', dict(num_steps=4), dict(scale_dir=0.0, scale_time=0.2)),
    ('dpm_pp', 'dpm_pp_sampler', dict(num_steps=4, max_order=2, predict_x0=False, afs=True), dict(scale_dir=0.01, scale_time=0.2)),
    ('dpm_pp', 'dpm_pp_sampler', dict(num_steps=5, max_order=3, predict_x0=True), dict(scale_dir=0.05, scale_time=0.0)),
]


@pytest.mark.parametrize('ci', range(len(AMED_CASES)))
def test_amed_sampler_parity(ci):
    """AMED plug-in samplers (per-sample r / scale_dir / scale_time, second evaluation at per-sample sigma) vs the oracle and
    vs the REAL reference's recorded output (tests/golden/ref_amed.npz)."""
    import os
    import numpy as np
    from oracle import amed_oracle as AO
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers_amed
    from diff_sampler_b200.amed_predictor import AMEDPredictor
    osolver, fn, kw, cfg = AMED_CASES[ci]
    d = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_amed.npz'))
    W = {k[len(f'amed/{ci}/pred/'):]: torch.from_numpy(d[k]) for k in d.files if k.startswith(f'amed/{ci}/pred/')}
    on, P, S = _oracle('tiny_song4')
    nat = _native(P, S)
    lat = O.stacked_randn(range(3), (3, 16, 16))
    ref = AO.sample_amed(on, lat, osolver, W, cfg, **kw)
    pred = AMEDPredictor(W, **cfg).to(_dev())
    got = getattr(solvers_amed, fn)(nat, lat.to(_dev()), AMED_predictor=pred, **kw).cpu()
    e_or = (got - ref).abs().max().item()
    e_ref = (got - torch.from_numpy(d[f'amed/{ci}/out'])).abs().max().item()
    print(f'AMED {fn} {kw}: vs oracle {e_or:.3e}, vs recorded reference {e_ref:.3e}')
    assert e_or < TOL and e_ref < TOL


@pytest.mark.parametrize('metric', ['l1', 'l2', 'dev'])
def test_gits_cost_matrix_and_dp(metric):
    """One-kernel cost matrix (ds_gits_cost) vs the oracle's pairwise loop; the DP on it returns the same index list."""
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import gits_utils
    on, P, S = _oracle('tiny_song')
    lat = O.stacked_randn(range(4), (3, 16, 16))
    N = 13
    ts = SO.get_schedule(N, 0.002, 80)
    traj, eps = SO.sample(on, lat, 'euler', t_steps=ts, num_steps=N, return_inters=True, return_eps=True)
    ref = SO.gits_cost_matrix(traj, eps, ts, metric, 3, 16)
    got = gits_utils.cost_matrix(traj.to(_dev()), eps.to(_dev()), ts.to(_dev()), metric, 3, 16).cpu()
    err = (got - ref).abs().max().item()
    print(f'gits cost {metric}: max err {err:.3e} (max {ref.abs().max().item():.3f})')
    assert err <= 2e-4 * ref.abs().max().item()
    for ns, coeff in ((5, 1.0), (7, 1.15)):
        assert gits_utils.dp(got.numpy(), ns, N, coeff) == SO.dp(ref.numpy(), ns, N, coeff)


def test_gits_get_dp_list_end_to_end():
    from diff_sampler_b200 import gits_utils, solver_utils, solvers
    _, P, S = _oracle('tiny_song')
    nat = _native(P, S)
    kw = dict(dataset_name='cifar10', num_warmup=8, max_batch_size=8, sigma_min=0.002, sigma_max=80, num_steps=5, num_steps_tea=11,
              schedule_type='polynomial', schedule_rho=7, afs=False, metric='dev', coeff=1.15, model_source='edm', solver='dpmpp',
              solver_tea='euler', max_order=2, deis_mode='tab', prompt=None, guidance_rate=1.0)
    torch.manual_seed(0)
    dp_list = gits_utils.get_dp_list(nat, _dev(), **kw)
    print('dp_list', dp_list)
    assert dp_list[0] == 0 and dp_list[-1] == 10 and len(dp_list) == 5 and dp_list == sorted(set(dp_list))
    t_steps = solver_utils.get_schedule(11, 0.002, 80, device=_dev(), dp_list=dp_list)
    out = solvers.dpm_pp_sampler(nat, torch.randn(4, 3, 16, 16, device=_dev()), num_steps=5, max_order=2, t_steps=t_steps)
    assert torch.isfinite(out).all()


# --------------------------------------------------------------------------------------------- BASELINE-size properties
def test_fullsize_batch_independence_and_properties():
    """At the BASELINE size (CIFAR-10 net, batch 512) the oracle is too slow; check size-independent properties instead:
    a sample's output does not depend on the batch it rides in, the update kernel is linear, thresholding is idempotent."""
    from diff_sampler_b200 import solver_utils as U
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200.net import B200Net
    net = B200Net.from_config('cifar10', seed=0, dezero=True, device=_dev())
    g = torch.Generator(device=_dev()).manual_seed(7)
    x = torch.randn(512, 3, 32, 32, generator=g, device=_dev()) * 5.0
    sig = torch.tensor(5.0, device=_dev())
    big = net(x, sig).clone()
    small = net(x[100:104].contiguous(), sig)
    e = (big[100:104] - small).abs().max().item()
    print(f'batch-512 vs batch-4 rows: {e:.3e}')
    assert e < 2e-5
    assert torch.isfinite(big).all()
    # update kernel linearity in (x, D, history) at full size
    a, b_, h = (torch.randn(512, 3, 32, 32, generator=g, device=_dev()) for _ in range(3))
    f = lambda X, D, H: U.solver_update(torch.empty_like(X), X, [0.7, -1.3, 0.4], mode=S.DS_M_EPS, D=D, t=3.0, hist=[H])
    lhs = f(a + 2 * b_, b_ - a, h + a)
    rhs = f(a, b_, h) + 2 * f(b_, -0.5 * a, 0.5 * a)
    assert (lhs - rhs).abs().max().item() < 1e-4
    # dynamic thresholding: s >= 1, |out| <= 1, idempotent, ~0.5% of the entries clipped when s > 1
    x0 = b_ * 3.0
    s = U.dyn_threshold(x0)
    y = U.dynamic_thresholding_fn(x0)
    assert (s >= 1).all() and y.abs().max().item() <= 1.0 + 1e-6
    frac = ((x0.abs() > s[:, None, None, None]).float().mean().item())
    assert abs(frac - 0.005) < 0.001
    y2 = U.dynamic_thresholding_fn(y)
    assert (y2 - y).abs().max().item() == 0.0


@pytest.mark.parametrize('name', ['tiny_song', 'tiny_adm'])
def test_unfused_attention_plan_matches(name):
    """flash_attn=False keeps the QK^T GEMM -> softmax -> PV GEMM lowering (used for heads wider than 64); both lowerings hold the
    oracle tolerance on the nets whose heads are 64 wide (where the default is the fused kernel)."""
    from oracle import edm_oracle as O
    from diff_sampler_b200.net import B200Net
    on, P, S = _oracle(name)
    x = O.stacked_randn(range(3), (3, 16, 16)) * 2.0
    lab = _labels(S, 3)
    ref = on(x, torch.tensor(2.0), class_labels=lab)
    for flash in (True, False):
        nat = B200Net(P, S['img_resolution'], S['img_channels'], S['label_dim'], device=_dev(), flash_attn=flash)
        got = nat(x.to(_dev()), torch.tensor(2.0, device=_dev()), class_labels=None if lab is None else lab.to(_dev())).cpu()
        err = (got - ref).abs().max().item()
        print(f'{name} flash_attn={flash}: {err:.3e}')
        assert err < TOL


def test_batched_embedding_gemm_path():
    """>= 32 embedding rows (per-sample labels and sigmas) lower the affine layer to the wgmma GEMM instead of the warp-per-feature
    linear kernel; same tolerance against the oracle."""
    from oracle import edm_oracle as O
    from diff_sampler_b200.net import B200Net
    from diff_sampler_b200 import _cstructs as CS
    on, P, S = _oracle('tiny_adm')
    B = 40
    nat = B200Net(P, S['img_resolution'], S['img_channels'], S['label_dim'], device=_dev())
    x = O.stacked_randn(range(B), (3, 16, 16))
    sig = torch.linspace(0.05, 40.0, B)
    lab = _labels(S, B)
    ref = on(x * sig[:, None, None, None], sig, class_labels=lab)
    got = nat((x * sig[:, None, None, None]).to(_dev()), sig.to(_dev()), class_labels=lab.to(_dev())).cpu()
    _, pl = nat._plan(B, B, B)
    n_lin = sum(1 for i in range(pl.n_ops) if pl.ops_array[i].type == CS.DS_OP_LINEAR)
    assert n_lin == 3                                    # map_layer0, map_layer1, map_label; the affine layer is a GEMM here
    err = (got - ref).abs().max().item()
    print(f'tiny_adm B={B} per-sample labels/sigma (embedding GEMM): {err:.3e}')
    assert err < TOL


def test_ldm_unfused_attention_matches():
    from oracle import edm_oracle as O
    on, nat, cfg = _ldm_pair(flash_attn=False)
    B, R = 2, cfg['img_resolution']
    x0 = O.stacked_randn(range(B), (4, R, R))
    g = torch.Generator().manual_seed(6)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    ref = on(x0 * 2.0, torch.tensor([2.0]), condition=c, unconditional_condition=uc)
    got = nat((x0 * 2.0).to(_dev()), torch.tensor([2.0], device=_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev())).cpu()
    assert (got - ref).abs().max().item() < TOL * max(1.0, ref.abs().max().item())


# --------------------------------------------------------------------------------------------- latent diffusion (config 5)
def _ldm_pair(name='tiny_ldm', guidance=7.5, precision=None, flash_attn=True):
    from oracle import ldm_oracle as LO
    from diff_sampler_b200.ldm_net import B200LDMNet
    P, cfg = LO.make_params(name)
    on = LO.OracleCFGNet(P, cfg, guidance_rate=guidance)
    nat = B200LDMNet(P, img_resolution=cfg['img_resolution'], img_channels=cfg['in_channels'], num_heads=cfg['num_heads'],
                     guidance_rate=guidance, precision=precision, device=_dev(), flash_attn=flash_attn)
    return on, nat, cfg


def test_ldm_eps_net_blocks_localise():
    """Per-module activations of the native latent-diffusion eps-net vs the oracle (names the first module that drifts)."""
    from oracle import edm_oracle as O
    on, nat, cfg = _ldm_pair()
    B, R = 2, cfg['img_resolution']
    x = O.stacked_randn(range(B), (4, R, R)) * 2.0
    g = torch.Generator().manual_seed(5)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    on.taps = {}
    ref = on(x, torch.tensor([2.0]), condition=c, unconditional_condition=uc)
    got = nat(x.to(_dev()), torch.tensor([2.0], device=_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev()))
    torch.cuda.synchronize()
    h, pl = nat._plan(B, 2 * B, 1)
    worst = 0.0
    for name, t in on.taps.items():
        key = 'h:' + name
        if key not in pl.arena_offsets:
            continue
        n, cch, hh, ww = t.shape
        buf = torch.empty(n * cch * hh * ww)
        import ctypes as C
        from diff_sampler_b200 import _lib
        _lib.check(nat.lib.ds_unet_debug_read(h, pl.arena_offsets[key], buf.data_ptr(), buf.numel() * 4, None), 'debug_read')
        mine = buf.reshape(n, hh, ww, cch).permute(0, 3, 1, 2)
        err = (mine - t).abs().max().item()
        worst = max(worst, err / max(1.0, t.abs().max().item()))
        print(f'{name:40s} max|ref| {t.abs().max().item():9.3f} err {err:.3e}')
    e = (got.cpu() - ref).abs().max().item()
    print(f'tiny_ldm D (cfg 7.5): err {e:.3e} (max|D| {ref.abs().max().item():.2f})')
    assert worst < 1e-4 and e < TOL * max(1.0, ref.abs().max().item())


def test_ldm_cfg_denoiser_parity_f8_mode():
    """precision='fp16f8' on the latent-diffusion eps-net: ResBlock convolutions in the f8 GEMM mode, transformer GEMMs in fp16x3."""
    from oracle import edm_oracle as O
    on, nat, cfg = _ldm_pair(precision='fp16f8')
    _, nat3, _ = _ldm_pair(precision='fp16x3')
    B, R = 3, cfg['img_resolution']
    x0 = O.stacked_randn(range(B), (4, R, R))
    g = torch.Generator().manual_seed(6)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    for sigma in (10.0, 0.5):
        ref = on(x0 * sigma, torch.tensor([sigma]), condition=c, unconditional_condition=uc)
        args = ((x0 * sigma).to(_dev()), torch.tensor([sigma], device=_dev()))
        got = nat(*args, condition=c.to(_dev()), unconditional_condition=uc.to(_dev())).cpu()
        got3 = nat3(*args, condition=c.to(_dev()), unconditional_condition=uc.to(_dev())).cpu()
        err, err3 = (got - ref).abs().max().item(), (got3 - ref).abs().max().item()
        print(f'ldm fp16f8 sigma={sigma}: err {err:.3e} (fp16x3 {err3:.3e}, max|D| {ref.abs().max().item():.1f})')
        assert err < TOL * max(1.0, ref.abs().max().item())


def test_ldm_cfg_denoiser_parity_f8_linear():
    """fp16f8 with f8_linear=True: ResBlock convolutions and the single-consumer transformer linears in the f8 GEMM mode."""
    from oracle import edm_oracle as O
    from oracle import ldm_oracle as LO
    from diff_sampler_b200.ldm_net import B200LDMNet
    P, cfg = LO.make_params('tiny_ldm')
    on = LO.OracleCFGNet(P, cfg, guidance_rate=7.5)
    nat = B200LDMNet(P, img_resolution=cfg['img_resolution'], img_channels=cfg['in_channels'], num_heads=cfg['num_heads'], guidance_rate=7.5,
                     precision='fp16f8', device=_dev(), f8_linear=True)
    assert nat.f8_linear
    B, R = 3, cfg['img_resolution']
    x0 = O.stacked_randn(range(B), (4, R, R))
    g = torch.Generator().manual_seed(6)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    for sigma in (10.0, 0.5):
        ref = on(x0 * sigma, torch.tensor([sigma]), condition=c, unconditional_condition=uc)
        got = nat((x0 * sigma).to(_dev()), torch.tensor([sigma], device=_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev())).cpu()
        err = (got - ref).abs().max().item()
        print(f'ldm fp16f8 + f8_linear sigma={sigma}: err {err:.3e} (max|D| {ref.abs().max().item():.1f})')
        assert err < TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('guidance', [7.5, 1.0])
def test_ldm_cfg_denoiser_parity(guidance):
    from oracle import edm_oracle as O
    on, nat, cfg = _ldm_pair(guidance=guidance)
    B, R = 3, cfg['img_resolution']
    x0 = O.stacked_randn(range(B), (4, R, R))
    g = torch.Generator().manual_seed(6)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    cd, ucd = c.to(_dev()), uc.to(_dev())
    for sigma in (10.0, 0.5):
        ref = on(x0 * sigma, torch.tensor([sigma]), condition=c, unconditional_condition=uc)
        got = nat((x0 * sigma).to(_dev()), torch.tensor([sigma], device=_dev()), condition=cd, unconditional_condition=ucd).cpu()
        err = (got - ref).abs().max().item()
        print(f'ldm g={guidance} sigma={sigma}: err {err:.3e} (max|D| {ref.abs().max().item():.1f})')
        assert err < TOL * max(1.0, ref.abs().max().item())
    sig = torch.tensor([3.0, 0.4, 9.0])
    ref = on(x0 * sig[:, None, None, None], sig, condition=c, unconditional_condition=uc)
    got = nat((x0 * sig[:, None, None, None]).to(_dev()), sig.to(_dev()), condition=cd, unconditional_condition=ucd).cpu()
    err = (got - ref).abs().max().item()
    print(f'ldm g={guidance} per-sample sigma: err {err:.3e}')
    assert err < TOL * max(1.0, ref.abs().max().item())
    # sigma <-> t mapping and the 'discrete' schedule (solver_utils.py:42-48)
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solver_utils
    assert abs(nat.sigma_min - on.sigma_min) < 1e-6 and abs(nat.sigma_max - on.sigma_max) < 1e-4
    ts_ref = SO.get_schedule(6, on.sigma_min, on.sigma_max, schedule_type='discrete', schedule_rho=1, net=on)
    ts = solver_utils.get_schedule(6, nat.sigma_min, nat.sigma_max, device=_dev(), schedule_type='discrete', schedule_rho=1, net=nat)
    assert (ts.cpu() - ts_ref).abs().max().item() <= 2e-5 * ts_ref.abs().max().item()


def test_ldm_sampler_parity():
    """BASELINE config-5 shape: DPM-Solver++(2M) eps-mode on the 'discrete' schedule with classifier-free guidance."""
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    on, nat, cfg = _ldm_pair()
    B, R = 2, cfg['img_resolution']
    lat = O.stacked_randn(range(B), (4, R, R))
    g = torch.Generator().manual_seed(7)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g)
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g)
    kw = dict(num_steps=5, sigma_min=on.sigma_min, sigma_max=on.sigma_max, schedule_type='discrete', schedule_rho=1, max_order=2, predict_x0=False)
    ref = SO.sample(on, lat, 'dpm_pp', condition=c, unconditional_condition=uc, **kw)
    got = solvers.dpm_pp_sampler(nat, lat.to(_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev()), **kw).cpu()
    err = (got - ref).abs().max().item()
    print(f'ldm dpm_pp(2M) NFE=4 cfg: err {err:.3e} (max|x| {ref.abs().max().item():.1f})')
    assert err < TOL * max(1.0, ref.abs().max().item())


def test_sd15_fullsize_parity():
    """Full Stable-Diffusion-v1.5-sized eps-net (859.5 M parameters, 4x64x64 latents, 77x768 context) under classifier-free
    guidance, batch 1: native vs the CPU oracle.  Weights come from the seeded recipe of oracle/ldm_oracle.make_params."""
    import time
    from oracle import edm_oracle as O
    torch.set_num_threads(min(16, torch.get_num_threads()))
    t0 = time.time()
    on, nat, cfg = _ldm_pair('sd15')
    x = O.stacked_randn(range(1), (4, 64, 64)) * 3.0
    g = torch.Generator().manual_seed(8)
    c = torch.randn(1, 77, 768, generator=g)
    uc = torch.randn(1, 77, 768, generator=g)
    got = nat(x.to(_dev()), torch.tensor([3.0], device=_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev())).cpu()
    t1 = time.time()
    ref = on(x, torch.tensor([3.0]), condition=c, unconditional_condition=uc)
    err = (got - ref).abs().max().item()
    print(f'sd15 cfg 7.5 batch 1: err {err:.3e} (max|D| {ref.abs().max().item():.2f}); build+native {t1 - t0:.0f}s, oracle {time.time() - t1:.0f}s')
    assert err < TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('name', ['tiny_song', 'tiny_adm'])
def test_cuda_graph_replay_matches_plain_launches(name):
    """ds_unet_enable_graph: every denoiser evaluation after the first two is ONE cudaGraphLaunch of the captured op list over staged io
    buffers.  Same bits as the plain launch loop for changing inputs / sigmas / labels, with and without the AMED bottleneck read-out,
    and through a sampler run."""
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.net import B200Net
    on, P, S = _oracle(name)
    mk = lambda g: B200Net(P, S['img_resolution'], S['img_channels'], S['label_dim'], device=_dev(), cuda_graph=g)
    plain, graph = mk(False), mk(True)
    B = 4
    lab = _labels(S, B)
    labd = None if lab is None else lab.to(_dev())
    for k, sigma in enumerate((80.0, 7.0, 1.3, 0.4, 0.02)):
        x = (O.stacked_randn(range(k, k + B), (3, 16, 16)) * sigma).to(_dev())
        sig = torch.tensor(sigma, device=_dev())
        bott_p, bott_g = torch.zeros(B, 64, device=_dev()), torch.zeros(B, 64, device=_dev())
        want_b = k >= 2
        a = plain(x, sig, class_labels=labd, bottleneck=bott_p if want_b else None)
        b = graph(x, sig, class_labels=labd, bottleneck=bott_g if want_b else None)
        assert torch.equal(a, b), (k, (a - b).abs().max().item())
        if want_b:
            assert torch.equal(bott_p, bott_g) and bott_g.abs().sum().item() > 0
    assert graph.launches_last_forward == plain.launches_last_forward
    lat = O.stacked_randn(range(B), (3, 16, 16)).to(_dev())
    a = solvers.heun_sampler(plain, lat, class_labels=labd, num_steps=5)
    b = solvers.heun_sampler(graph, lat, class_labels=labd, num_steps=5)
    assert torch.equal(a, b)
    # per-sample sigma uses another plan (and its own graph)
    sigs = torch.tensor([3.0, 0.4, 11.0, 0.9], device=_dev())
    x = lat * sigs[:, None, None, None]
    for _ in range(3):
        assert torch.equal(plain(x, sigs, class_labels=labd), graph(x, sigs, class_labels=labd))


def test_cuda_graph_replay_ldm():
    from oracle import edm_oracle as O
    from oracle import ldm_oracle as LO
    from diff_sampler_b200.ldm_net import B200LDMNet
    P, cfg = LO.make_params('tiny_ldm')
    mk = lambda g: B200LDMNet(P, img_resolution=cfg['img_resolution'], img_channels=cfg['in_channels'], num_heads=cfg['num_heads'],
                              guidance_rate=7.5, device=_dev(), cuda_graph=g)
    plain, graph = mk(False), mk(True)
    B, R = 2, cfg['img_resolution']
    g = torch.Generator().manual_seed(6)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g).to(_dev())
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g).to(_dev())
    for k, sigma in enumerate((10.0, 2.0, 0.5, 0.1)):
        x = (O.stacked_randn(range(k, k + B), (4, R, R)) * sigma).to(_dev())
        sig = torch.tensor([sigma], device=_dev())
        bp, bg = torch.zeros(B, 64, device=_dev()), torch.zeros(B, 64, device=_dev())
        a = plain(x, sig, condition=c, unconditional_condition=uc, bottleneck=bp if k % 2 else None)
        b = graph(x, sig, condition=c, unconditional_condition=uc, bottleneck=bg if k % 2 else None)
        assert torch.equal(a, b) and torch.equal(bp, bg)


def test_fused_uint8_image_epilogue_in_the_last_update():
    """f1: `images_uint8=` makes the LAST update kernel of a sampling run also write (x * 127.5 + 128).clip(0, 255).uint8 in NHWC
    (sample.py:311) -- bit-exact against the torch expression on the fp32 images the same call returns; samplers without a fused
    final update (denoise_to_zero, UniPC) fall back to the one-pass conversion kernel with the same result."""
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers
    on, P, S = _oracle('tiny_song')
    nat = _native(P, S)
    B = 5
    lat = O.stacked_randn(range(B), (3, 16, 16)).to(_dev())
    for fn, kw in (('heun_sampler', dict(num_steps=4)), ('euler_sampler', dict(num_steps=4)), ('ipndm_sampler', dict(num_steps=5, max_order=3)),
                   ('dpm_pp_sampler', dict(num_steps=5, max_order=2)), ('dpm_2_sampler', dict(num_steps=3)),
                   ('euler_sampler', dict(num_steps=4, denoise_to_zero=True)), ('unipc_sampler', dict(num_steps=5))):
        u8 = torch.full((B, 16, 16, 3), 7, dtype=torch.uint8, device=_dev())
        l0 = __import__('diff_sampler_b200.solver_utils', fromlist=['LAUNCHES']).LAUNCHES[0]
        img = getattr(solvers, fn)(nat, lat, images_uint8=u8, **kw)
        n_launch = __import__('diff_sampler_b200.solver_utils', fromlist=['LAUNCHES']).LAUNCHES[0] - l0
        plain = getattr(solvers, fn)(nat, lat, **kw)
        assert torch.equal(img, plain)                                           # the fp32 result is unchanged
        want = (img * 127.5 + 128).clip(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
        assert torch.equal(u8, want), (fn, kw, (u8.int() - want.int()).abs().max().item())
        print(f'{fn} {kw}: uint8 image epilogue bit-exact ({n_launch} solver-kernel launches)')


# --------------------------------------------------------------------------------------------- BASELINE configs as configured
def test_config3_ffhq_ipndm_fullsize_sampler_parity():
    """BASELINE config 3: EDM FFHQ-64 net (full size), iPNDM num_steps=7 (NFE=6), max_order=4 (4-term multistep history), final
    images against the CPU oracle.  Checked for the library default (fp16x3) and for the mode bench.py runs this config in."""
    import bench
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.net import B200Net
    on, P, S = _oracle('ffhq')
    B = 2
    lat = O.stacked_randn(range(B), (3, 64, 64))
    kw = dict(num_steps=7, max_order=4, sigma_min=0.002, sigma_max=80, schedule_type='polynomial', schedule_rho=7)
    ref = SO.sample(on, lat, 'ipndm', **kw)
    modes = [('fp16x3', 0)]
    bm = (bench.PRECISION_FOR['ffhq'], bench.F8_MIN_CHANNELS_FOR.get('ffhq', 0))
    if bm not in modes:
        modes.append(bm)
    for prec, fmin in modes:
        nat = B200Net(P, 64, 3, 0, precision=prec, f8_min_channels=fmin, device=_dev())
        got = solvers.ipndm_sampler(nat, lat.to(_dev()), **kw).cpu()
        err = (got - ref).abs().max().item()
        print(f'ffhq ipndm NFE=6 {prec} f8_min_channels={fmin}: final-image max-abs err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
        assert err < TOL
        del nat


def test_config4_imagenet64_dpmpp_on_gits_schedule_parity():
    """BASELINE config 4: ImageNet-64 class-conditional ADM net (full size), DPM-Solver++(2M) NFE=10 on a GITS schedule: t_steps are
    picked from the 61-point polynomial teacher grid by the DP over the native teacher trajectories (gits_utils.get_dp_list, coeff 1.15),
    so the grid is non-uniform; final images against the CPU oracle on the same t_steps, in the precision bench.py runs this config in."""
    import bench
    from oracle import edm_oracle as O
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import gits_utils, solver_utils, solvers
    on, P, S = _oracle('imagenet64')
    nat = _native(P, S, bench.PRECISION_FOR['imagenet64'])
    kw = dict(dataset_name='imagenet64', num_warmup=4, max_batch_size=4, sigma_min=0.002, sigma_max=80, num_steps=11, num_steps_tea=61,
              schedule_type='polynomial', schedule_rho=7, afs=False, metric='dev', coeff=1.15, model_source='edm', solver='dpmpp',
              solver_tea='dpmpp', max_order=2, deis_mode='tab', prompt=None, guidance_rate=1.0, predict_x0=True, lower_order_final=True)
    torch.manual_seed(0)
    dp_list = gits_utils.get_dp_list(nat, _dev(), **kw)
    print('GITS dp_list', dp_list)
    assert len(dp_list) == 11 and dp_list[0] == 0 and dp_list[-1] == 60 and dp_list == sorted(set(dp_list))
    t_steps = solver_utils.get_schedule(61, 0.002, 80, device=_dev(), schedule_type='polynomial', schedule_rho=7, dp_list=dp_list)
    poly = solver_utils.get_schedule(11, 0.002, 80, device=_dev())
    assert (t_steps - poly).abs().max().item() > 1e-3                      # not the plain 11-point polynomial grid
    t_ref = SO.get_schedule(61, 0.002, 80, dp_list=dp_list)
    assert torch.equal(t_steps.cpu(), t_ref)                               # integer gather: bit-exact
    B = 2
    lat = O.stacked_randn(range(B), (3, 64, 64))
    lab = _labels(S, B)
    skw = dict(num_steps=11, max_order=2, predict_x0=True, lower_order_final=True)
    ref = SO.sample(on, lat, 'dpm_pp', class_labels=lab, t_steps=t_ref, **skw)
    got = solvers.dpm_pp_sampler(nat, lat.to(_dev()), class_labels=lab.to(_dev()), t_steps=t_steps, **skw).cpu()
    err = (got - ref).abs().max().item()
    print(f'imagenet64 dpm_pp(2M) NFE=10 on GITS t_steps ({nat.precision}): final-image max-abs err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
    assert err < TOL


AMED_ADM_CASES = [
    ('amed', 'amed_sampler', dict(num_steps=4), dict(scale_dir=0.01, scale_time=0.2)),
    ('dpm_pp', 'dpm_pp_sampler', dict(num_steps=4, max_order=2, predict_x0=True, afs=True), dict(scale_dir=0.01, scale_time=0.2)),
    ('ipndm', 'ipndm_sampler', dict(num_steps=4, max_order=4, afs=True), dict(scale_dir=0.01, scale_time=0.0)),
]
AMED_LDM_CASES = [
    (7.5, dict(num_steps=4, afs=True, max_order=2, predict_x0=False, lower_order_final=True), dict(scale_dir=0.0, scale_time=0.2)),
    (7.5, dict(num_steps=3, afs=False, max_order=3, predict_x0=False, lower_order_final=True), dict(scale_dir=0.01, scale_time=0.2)),
]


def _amed_tap_case(group, ci):
    import numpy as np
    d = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_amed_taps.npz'))
    pre = f'{group}/{ci}/pred/'
    W = {k[len(pre):]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre)}
    return d, W, torch.from_numpy(d[f'{group}/{ci}/out'])


@pytest.mark.parametrize('ci', range(len(AMED_ADM_CASES)))
def test_amed_class_conditional_tap_parity(ci):
    """AMED samplers on a class-conditional EDM net: the predictor reads enc['8x8_block2'] (solvers_amed.py:16).  Native vs the oracle and
    vs the REAL reference's recorded output (tests/golden/ref_amed_taps.npz)."""
    from oracle import amed_oracle as AO
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers_amed
    from diff_sampler_b200.amed_predictor import AMEDPredictor
    osolver, fn, kw, cfg = AMED_ADM_CASES[ci]
    d, W, rec = _amed_tap_case('adm', ci)
    on, P, S = _oracle('tiny_adm3')
    nat = _native(P, S)
    assert nat.spec.bottleneck_block.endswith('8x8_block2')
    lat = O.stacked_randn(range(3), (3, 16, 16))
    lab = torch.from_numpy(d['adm/labels'])
    ref = AO.sample_amed(on, lat, osolver, W, cfg, class_labels=lab, **kw)
    pred = AMEDPredictor(W, **cfg).to(_dev())
    got = getattr(solvers_amed, fn)(nat, lat.to(_dev()), class_labels=lab.to(_dev()), AMED_predictor=pred, **kw).cpu()
    e_or, e_ref = (got - ref).abs().max().item(), (got - rec).abs().max().item()
    print(f'AMED {fn} on tiny_adm3 (8x8_block2 tap) {kw}: vs oracle {e_or:.3e}, vs recorded reference {e_ref:.3e}')
    assert e_or < TOL and e_ref < TOL


@pytest.mark.parametrize('ci', range(len(AMED_LDM_CASES)))
def test_config5_amed_dpmpp_ldm_cfg_tap_parity(ci):
    """BASELINE config 5's sampler/net pair: solvers_amed.dpm_pp_sampler (AMED plug-in on DPM-Solver++, afs, eps-prediction, 'discrete'
    schedule rho=1; launch.sh:57-61) on a latent-diffusion net under classifier-free guidance 7.5: the predictor reads the channel mean
    of middle_block's output, conditional half of the doubled batch (solvers_amed.py:11-12, :24-26).  Native vs oracle vs the REAL
    reference's recorded output."""
    from oracle import amed_oracle as AO
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers_amed
    from diff_sampler_b200.amed_predictor import AMEDPredictor
    guidance, kw, cfg = AMED_LDM_CASES[ci]
    d, W, rec = _amed_tap_case('ldm', ci)
    on, nat, lcfg = _ldm_pair(guidance=guidance)
    lat = O.stacked_randn(range(2), (4, 16, 16))
    c, uc = torch.from_numpy(d['ldm/c']), torch.from_numpy(d['ldm/uc'])
    common = dict(schedule_type='discrete', schedule_rho=1)
    ref = AO.sample_amed(on, lat, 'dpm_pp', W, cfg, condition=c, unconditional_condition=uc, sigma_min=on.sigma_min, sigma_max=on.sigma_max,
                         **common, **kw)
    pred = AMEDPredictor(W, **cfg).to(_dev())
    got = solvers_amed.dpm_pp_sampler(nat, lat.to(_dev()), condition=c.to(_dev()), unconditional_condition=uc.to(_dev()), AMED_predictor=pred,
                                      sigma_min=nat.sigma_min, sigma_max=nat.sigma_max, **common, **kw).cpu()
    scale = max(1.0, ref.abs().max().item())
    e_or, e_ref = (got - ref).abs().max().item(), (got - rec).abs().max().item()
    print(f'AMED dpm_pp on tiny_ldm cfg {guidance} {kw}: vs oracle {e_or:.3e}, vs recorded reference {e_ref:.3e} (max|x| {scale:.1f})')
    assert e_or < TOL * scale and e_ref < TOL * scale


# --------------------------------------------------------------------------------------------- the drop-in entry points
def _module_from_params(P, cls_name, sub=None):
    """An nn.Module stand-in carrying a flat parameter dict under the reference's state_dict names (class NAME as the reference's, which
    is what as_native inspects).  `sub` = {dotted child path: class name} renames inner modules (e.g. {'model': 'SongUNet'})."""
    import torch.nn as nn
    sub = sub or {}
    root = type(cls_name, (nn.Module,), {})()
    for k, v in P.items():
        parts = k.split('.')
        m, path = root, ''
        for part in parts[:-1]:
            path = part if not path else path + '.' + part
            if part not in m._modules:
                m.add_module(part, type(sub.get(path, 'Node'), (nn.Module,), {})())
            m = m._modules[part]
        m.register_parameter(parts[-1], nn.Parameter(v.clone(), requires_grad=False))
    return root


@pytest.mark.parametrize('name', ['tiny_song', 'tiny_adm'])
def test_dropin_as_native_and_from_reference(name):
    """sample.py hands the samplers a torch EDMPrecond module (sample.py:301): `solvers.<x>_sampler(net, ...)` must compile it once
    (as_native -> B200Net.from_reference), cache it, notice weight updates, and give the same images as B200Net(P, ...)."""
    from oracle import edm_oracle as O
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.net import B200Net
    on, P, S = _oracle(name)
    mod = _module_from_params(P, 'EDMPrecond', {'model': 'SongUNet' if S['kind'] == 'song' else 'DhariwalUNet'}).to(_dev())
    mod.img_resolution, mod.img_channels, mod.label_dim = S['img_resolution'], S['img_channels'], S['label_dim']
    mod.sigma_min, mod.sigma_max, mod.sigma_data, mod.use_fp16 = 0.002, 80.0, 0.5, False
    direct = _native(P, S)
    nat = solvers.as_native(mod)
    assert isinstance(nat, B200Net) and solvers.as_native(mod) is nat                       # compiled once, cached on the module
    viaref = B200Net.from_reference(mod, device=_dev())
    B = 3
    lat = O.stacked_randn(range(B), (3, 16, 16)).to(_dev())
    lab = _labels(S, B)
    labd = None if lab is None else lab.to(_dev())
    a = solvers.heun_sampler(direct, lat, class_labels=labd, num_steps=4)
    b = solvers.heun_sampler(mod, lat, class_labels=labd, num_steps=4)                      # the torch module itself, as sample.py passes it
    c = solvers.heun_sampler(viaref, lat, class_labels=labd, num_steps=4)
    assert torch.equal(a, b) and torch.equal(a, c)
    ref = __import__('oracle.solvers_oracle', fromlist=['sample']).sample(on, lat.cpu(), 'heun', class_labels=lab, num_steps=4)
    assert (b.cpu() - ref).abs().max().item() < TOL
    # a weight update invalidates the cached snapshot (fingerprint = storage address + version counter of every tensor)
    with torch.no_grad():
        next(iter(mod.parameters())).mul_(1.0)
    assert solvers.as_native(mod) is not nat
    # other preconditioners are not compiled as EDM (their c_skip / c_out / c_noise differ): the object is returned unchanged
    vp = _module_from_params(P, 'VPPrecond', {'model': 'SongUNet'})
    assert solvers.as_native(vp) is vp


def test_dropin_from_pickle():
    """`B200Net.from_pickle(network-snapshot.pkl)` (what sample.py:81-82 unpickles) on the GPU: same denoiser output as B200Net built
    from the snapshot's state_dict, and equal to the oracle on those weights.  The fixture (64-channel DDPM++ net, the narrowest the
    native kernels run) was written by the real reference classes through torch_utils/persistence.py (oracle/gen_edm_pickle.py)."""
    import json
    from oracle import edm_oracle as O
    from diff_sampler_b200 import checkpoint as CK
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.net import B200Net
    gold = os.path.join(os.path.dirname(__file__), 'golden')
    meta = json.load(open(os.path.join(gold, 'edm_snapshot.json')))['song64']
    path = os.path.join(gold, meta['file'])
    net = B200Net.from_pickle(path, device=_dev())
    params, m = CK.load_edm_pickle(path)
    net2 = B200Net(params, m['img_resolution'], m['img_channels'], m['label_dim'], device=_dev())
    R = m['img_resolution']
    x = O.stacked_randn(range(4), (3, R, R)) * 2.0
    sig = torch.tensor(2.0)
    a = net(x.to(_dev()), sig.to(_dev())).cpu()
    b = net2(x.to(_dev()), sig.to(_dev())).cpu()
    assert torch.equal(a, b)
    _, S = O.make_songunet(img_resolution=R, in_channels=3, out_channels=3, augment_dim=9, model_channels=64, channel_mult=(1,), num_blocks=1,
                           attn_resolutions=(8,))
    S['sigma_data'], S['sigma_min'], S['sigma_max'] = 0.5, 0.002, 80.0
    on = O.OracleNet(params, S)
    err = (a - on(x, sig)).abs().max().item()
    print(f'from_pickle song64: D err vs oracle {err:.3e}')
    assert err < TOL
    lat = O.stacked_randn(range(4), (3, R, R))
    from oracle import solvers_oracle as SO
    got = solvers.euler_sampler(net, lat.to(_dev()), num_steps=5).cpu()
    assert (got - SO.sample(on, lat, 'euler', num_steps=5)).abs().max().item() < TOL
    assert (net.sigma_min, net.sigma_max) == (0.002, 80.0) and net.checkpoint_meta['class_name'] == 'EDMPrecond'


def test_dropin_ldm_from_reference_and_as_native():
    """A torch CFGPrecond module (net.model.model.diffusion_model = UNetModel, net.model.alphas_cumprod) handed to the samplers is
    compiled by as_native -> B200LDMNet.from_reference and gives the images of B200LDMNet(P, ...)."""
    from oracle import edm_oracle as O
    from oracle import ldm_oracle as LO
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.ldm_net import B200LDMNet
    on, direct, cfg = _ldm_pair()
    P, _ = LO.make_params('tiny_ldm')
    mod = _module_from_params({'model.model.diffusion_model.' + k: v for k, v in P.items()}, 'CFGPrecond',
                              {'model.model.diffusion_model': 'UNetModel'}).to(_dev())
    mod.model.model.diffusion_model.num_heads = cfg['num_heads']
    mod.model.alphas_cumprod = LO.make_alphas_cumprod()
    mod.img_resolution, mod.img_channels, mod.label_dim = cfg['img_resolution'], cfg['in_channels'], True
    mod.guidance_type, mod.guidance_rate = 'classifier-free', 7.5
    nat = solvers.as_native(mod)
    assert isinstance(nat, B200LDMNet) and solvers.as_native(mod) is nat
    mod.sigma_min, mod.sigma_max = nat.sigma_min, nat.sigma_max
    mod.sigma, mod.sigma_inv = nat.sigma, nat.sigma_inv                      # CFGPrecond methods the 'discrete' schedule calls (solver_utils.py:42-48)
    B, R = 2, cfg['img_resolution']
    lat = O.stacked_randn(range(B), (4, R, R)).to(_dev())
    g = torch.Generator().manual_seed(7)
    c = torch.randn(B, 77, cfg['context_dim'], generator=g).to(_dev())
    uc = torch.randn(B, 77, cfg['context_dim'], generator=g).to(_dev())
    kw = dict(condition=c, unconditional_condition=uc, num_steps=4, sigma_min=nat.sigma_min, sigma_max=nat.sigma_max, schedule_type='discrete',
              schedule_rho=1, max_order=2, predict_x0=False)
    a = solvers.dpm_pp_sampler(direct, lat, **kw)
    b = solvers.dpm_pp_sampler(mod, lat, **kw)
    assert torch.equal(a, b)


# --------------------------------------------------------------------------------------------- first-stage decoder
@pytest.mark.parametrize('name,R', [('tiny_vae', 8), ('wide_vae', 64)])
def test_vae_decoder_parity(name, R):
    """decode_first_stage through B200VAEDecoder vs the CPU oracle (pinned to the reference Decoder): per-module activations and the
    final image; 'wide_vae' at R = 64 reaches 256-pixel rows (pair-kernel row segments)."""
    from oracle import vae_oracle as VO
    from diff_sampler_b200.vae_net import B200VAEDecoder
    P, cfg = VO.make_params(name, seed=0)
    vae = B200VAEDecoder(P, scale_factor=cfg['scale_factor'], device=_dev())
    g = torch.Generator().manual_seed(3)
    B = 2
    z = torch.randn(B, cfg['z_channels'], R, R, generator=g) * cfg['scale_factor'] * 1.3
    taps = {}
    with torch.no_grad():
        ref = VO.decode(P, cfg, z, taps=taps)
    got = vae.decode(z.to(_dev())).cpu()
    torch.cuda.synchronize()
    for mname, t in taps.items():
        n, c, h, w = t.shape
        mine = vae.debug_read(B, R, 'h:' + mname, n * c * h * w).reshape(n, h, w, c).permute(0, 3, 1, 2)
        print(f'{mname:32s} max|ref| {t.abs().max().item():9.4f}  err {(mine - t).abs().max().item():.3e}')
    err = (got - ref).abs().max().item()
    print(f'{name}: image err {err:.3e} (max|x| {ref.abs().max().item():.2f})')
    assert got.shape == ref.shape and err < TOL



# --------------------------------------------------------------------------------------------- text encoder
@pytest.mark.parametrize('name,B', [('tiny_clip', 3), ('clip_l', 2)])
def test_clip_text_encoder_parity(name, B):
    """get_learned_conditioning's encoder through B200CLIPTextEncoder vs the CPU oracle (pinned to transformers' CLIPTextModel) and, for
    tiny_clip, the committed transformers output itself; clip_l has the dimensions Stable Diffusion v1.x conditions on (12 layers,
    12 x 64 heads, 768 wide, 49408 tokens), seeded weights."""
    import os
    import numpy as np
    from oracle import clip_oracle as CO
    from diff_sampler_b200.clip_net import B200CLIPTextEncoder
    P, cfg = CO.make_params(name, seed=0)
    enc = B200CLIPTextEncoder(P, num_heads=cfg['num_attention_heads'], device=_dev())
    if name == 'tiny_clip':
        d = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_clip.npz'))
        ids = torch.from_numpy(d['tiny_clip/ids'])[:B]
    else:
        g = torch.Generator().manual_seed(5)
        ids = torch.randint(0, cfg['vocab_size'], (B, 77), generator=g)
        ids[:, 0] = 49406
        ids[0, 9:] = 49407
    taps = {}
    with torch.no_grad():
        ref = CO.text_forward(P, cfg, ids, taps=taps)
    got = enc(ids.to(_dev())).cpu()
    torch.cuda.synchronize()
    err = (got - ref).abs().max().item()
    print(f'{name}: last_hidden_state err {err:.3e} (max|x| {ref.abs().max().item():.2f}); launches {enc.total_launches}')
    assert got.shape == ref.shape == (B, 77, cfg['hidden_size']) and err < TOL
    if name == 'tiny_clip':
        assert (got - torch.from_numpy(d['tiny_clip/out'])[:B]).abs().max().item() < TOL
    with pytest.raises(Exception):
        enc(ids)                                           # host tensor: no CPU fallback

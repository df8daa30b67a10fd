"""Optimal denoiser on the GPU (csrc/optimal.cu + the GEMM kernel) against the float64 oracle (tests/opt_ref.py).

  * D at every sigma of the 18-step rho = 7 schedule and at {0.002 .. 80}, scalar and per-sample sigma, batches 1 / 3 / 64 / 512 and
    one larger than the 512-row chunk, on a CIFAR-shaped set of 50 000 structured uint8 images: within the per-row bound of DESIGN.md
    4.9 and never above 1e-3;
  * near-duplicate sets (pairs one level apart in 1..16 values, exact duplicates) at sigma <= 0.05: every row rescored, <= 1e-6;
  * odd shapes: N in {1, 2, 63, 65, 4097} x D in {105, 3072, 12288};
  * no row ever needs rescoring without getting it (last_unrefined_rows == 0), and two calls are bit-identical;
  * optimal_sampler (afs, denoise_to_zero, t_steps) and the native euler / heun / dpm_pp samplers with the denoiser as `net`;
  * nearest(): indices and distances against the float64 argsort.

Every output D is written into the body of a NaN-filled buffer whose head and tail guards must come back untouched."""
import gc
import math

import pytest
import torch

import opt_ref as O
from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import optimal as OPT
from diff_sampler_b200 import solvers

pytestmark = pytest.mark.gpu

GUARD = 64
FLOOR = 5e-5            # weighted-sum GEMM accumulation (2048 keys per fp32 accumulator, three passes) + P rounding (DESIGN.md 4.9)
SCHEDULE = [float(v) for v in O.polynomial_schedule(18).to(torch.float32)]
EXTRA = [0.002, 0.01, 0.05, 0.2, 1.0, 3.0, 5.0, 10.0, 30.0, 80.0]


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda', 0)


@pytest.fixture(scope='module')
def cifar(dev):
    y = O.uint8_images(50000, 3, 32, 32, seed=1234)
    den = OPT.B200OptimalDenoiser(y, device=dev)
    return y.to(dev), den


def guarded_call(den, x, sigma):
    n = x.numel()
    buf = torch.full((n + 2 * GUARD,), float('nan'), device=x.device)
    out = buf[GUARD:GUARD + n].view(x.shape)
    r = den(x, sigma, out=out)
    assert r.data_ptr() == out.data_ptr()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), 'guard overwritten'
    assert torch.isfinite(out).all(), 'unwritten or non-finite output'
    return out


def row_bound(den, x, sigma, D, y):
    """Per-row bound on |D - D*|_inf: 2 E_row max_i |y_i - D|_inf for rows on GEMM logits, plus FLOOR."""
    B = x.shape[0]
    s = torch.as_tensor(sigma, dtype=torch.float64, device=x.device).reshape(-1).expand(B)
    xn = x.double().reshape(B, -1).norm(dim=1)
    D_ = x[0].numel()
    E = (xn + den.ymax) * (S.DS_OPT_EPS * den.ymax + math.sqrt(D_) * 2.0 ** -25) / (s * s)
    spread = y.abs().max().double() + D.double().reshape(B, -1).abs().amax(dim=1)
    plain = den.last_row_status == S.DS_OPT_PLAIN
    return torch.where(plain, 2 * E * spread, torch.zeros_like(E)) + FLOOR


def check(den, y, x, sigma, tol=1e-3):
    got = guarded_call(den, x, sigma)
    ref = O.denoise_opt(x, sigma, y)
    err = (got.double() - ref).reshape(x.shape[0], -1).abs().amax(dim=1)
    assert den.last_unrefined_rows == 0, den.last_row_status.tolist()
    bound = row_bound(den, x, sigma, got, y)
    assert (err <= bound).all(), (err.max().item(), bound.min().item())
    assert err.max().item() <= tol, (err.max().item(), den.last_row_status.tolist())
    return got


def noisy(y, B, sigma, seed):
    g = torch.Generator(device=y.device).manual_seed(seed)
    idx = torch.randint(0, y.shape[0], (B,), generator=g, device=y.device)
    s = torch.as_tensor(sigma, dtype=torch.float32, device=y.device).reshape(-1, *([1] * (y.dim() - 1)))
    return (y[idx] + s * torch.randn((B,) + tuple(y.shape[1:]), generator=g, device=y.device)).contiguous()


@pytest.mark.parametrize('sigma', sorted(set(SCHEDULE + EXTRA)))
def test_cifar_every_sigma(cifar, sigma):
    y, den = cifar
    check(den, y, noisy(y, 64, sigma, seed=int(sigma * 1000) % 9973), sigma)


def test_cifar_per_sample_sigma_mixing_extremes(cifar):
    y, den = cifar
    sig = torch.tensor([80.0, 0.002, 1.0, 0.05, 5.0, 0.2, 30.0, 0.01] * 8, device=y.device)
    x = noisy(y, 64, sig, seed=5)
    check(den, y, x, sig)
    st = den.last_row_status.cpu()
    assert (st[1::8] == S.DS_OPT_RESCORED).all() and (st[0::8] == S.DS_OPT_PLAIN).all()


@pytest.mark.parametrize('B', [1, 3, 512, 1100])
def test_cifar_batches(cifar, B):
    y, den = cifar
    assert den.chunk == 512
    for sigma in (80.0, 1.0, 0.002):
        check(den, y, noisy(y, B, sigma, seed=B), sigma)


def test_bit_identical_repeats(cifar):
    y, den = cifar
    for sigma in (40.0, 0.5, 0.002):
        x = noisy(y, 64, sigma, seed=3)
        a = den(x, sigma).clone()
        b = den(x, sigma)
        assert torch.equal(a, b)


@pytest.mark.parametrize('sigma', [0.002, 0.01, 0.05])
def test_near_duplicates_rescored(dev, sigma):
    y = O.near_duplicates(4000, 3, 32, 32, seed=77).to(dev)
    den = OPT.B200OptimalDenoiser(y, device=dev)
    x = noisy(y, 256, sigma, seed=17)
    got = check(den, y, x, sigma, tol=1e-6)
    assert (den.last_row_status == S.DS_OPT_RESCORED).all()
    # rows exactly on a duplicate pair: the two keys share the weight
    dup = y[0:2000:34]                        # pair index k = 0, 17, 34 ... are exact duplicates (rows 2k, 2k + 1)
    check(den, y, dup.contiguous(), sigma, tol=1e-6)
    del den, got
    gc.collect()


@pytest.mark.parametrize('N', [1, 2, 63, 65, 4097])
@pytest.mark.parametrize('shape', [(3, 5, 7), (3, 32, 32), (3, 64, 64)])
def test_odd_shapes(dev, N, shape):
    y = O.uint8_images(N, *shape, seed=N).to(dev)
    den = OPT.B200OptimalDenoiser(y, device=dev)
    for sigma in (80.0, 1.0, 0.01):
        check(den, y, noisy(y, 3, sigma, seed=N + 1), sigma)
    del den
    gc.collect()


def _sampler_case(y, den, lat, **kw):
    got = OPT.optimal_sampler(None, lat, y, **kw)
    okw = {k: v for k, v in kw.items() if k not in ('return_denoised', 'return_eps')}
    ref = O.optimal_sampler(lat, y, denoiser=lambda x, s: O.denoise_opt(x.float(), s, y), **okw)
    return got, ref


def test_optimal_sampler_variants(cifar, monkeypatch):
    y, den = cifar
    monkeypatch.setattr(OPT, '_CACHE', {OPT._dataset_key(y) + (str(y.device),): den})
    lat = torch.randn(64, 3, 32, 32, generator=torch.Generator(device=y.device).manual_seed(9), device=y.device)
    got, ref = _sampler_case(y, den, lat, num_steps=18, afs=True)
    assert (got.double() - ref).abs().max().item() <= 1e-3
    t_given = torch.tensor([80.0, 20.0, 5.0, 1.5, 0.6, 0.2, 0.05, 0.01, 0.002], device=y.device)
    for kw in (dict(num_steps=18, denoise_to_zero=True), dict(t_steps=t_given)):
        got, ref = _sampler_case(y, den, lat, return_inters=True, return_denoised=True, return_eps=True, **kw)
        xt, dn, ep = got
        rxt, rdn, rep = ref
        assert xt.shape == rxt.shape and dn.shape == rdn.shape and ep.shape == rep.shape
        scale = rxt.abs().amax(dim=(1, 2, 3, 4)).clamp_min(1.0)
        assert ((xt.double() - rxt).abs().amax(dim=(1, 2, 3, 4)) / scale).max().item() <= 1e-3
        assert (dn.double() - rdn).abs().max().item() <= 1e-3
        tt = list(t_given.tolist()) if 't_steps' in kw else SCHEDULE
        tt = tt + [tt[-1]] * (ep.shape[0] - len(tt) + 1)
        for i in range(ep.shape[0]):                       # eps * t = x - D: compare in the units of x
            t = tt[i + 1] if (kw.get('denoise_to_zero') and i == ep.shape[0] - 1) else tt[i]
            assert (ep[i].double() - rep[i]).abs().max().item() * t <= 1e-3, i
        assert (xt[-1].double() - rxt[-1]).abs().max().item() <= 1e-3


@pytest.mark.parametrize('name', ['euler', 'heun', 'dpm_pp'])
def test_native_samplers_take_the_denoiser_as_net(cifar, name):
    from oracle import solvers_oracle as SO
    y, den = cifar
    lat = torch.randn(64, 3, 32, 32, generator=torch.Generator(device=y.device).manual_seed(21), device=y.device)
    got = getattr(solvers, f'{name}_sampler')(den, lat, num_steps=18)
    ref = SO.sample(lambda x, t, class_labels=None: O.denoise_opt(x.float(), t, y), lat.double(), name, num_steps=18)
    assert (got.double() - ref).abs().max().item() <= 1e-3


@pytest.mark.parametrize('k', [1, 10, 64])
def test_nearest(cifar, k):
    y, den = cifar
    for sigma in (0.05, 1.0):
        x = noisy(y, 64, sigma, seed=k)
        dist, idx = den.nearest(x, k)
        assert dist.shape == (64, k) and idx.shape == (64, k)
        assert torch.isfinite(dist).all() and (idx >= 0).all() and (idx < y.shape[0]).all()
        rd, ri, sd = O.knn(x, y, k)
        tol = 4e-7 * (1 + sd[:, :k + 1].sqrt())                   # fp32 rounding of the distances
        assert ((dist.double() - rd).abs() <= tol[:, :k]).all()
        gaps = sd[:, 1:k + 1].sqrt() - sd[:, :k].sqrt()
        for b in range(64):
            if (gaps[b] > 2 * tol[b, :k]).all():
                assert torch.equal(idx[b], ri[b]), b
            elif k < sd.shape[1] and gaps[b, k - 1] > 2 * tol[b, k - 1]:
                assert set(idx[b].tolist()) == set(ri[b].tolist()), b


def test_nearest_exact_duplicates_tie_to_lower_index(dev):
    y = O.near_duplicates(200, 3, 8, 8, seed=3).to(dev)
    den = OPT.B200OptimalDenoiser(y, device=dev)
    x = y[[0, 34, 68]].contiguous()               # pairs 0, 17, 34: exact duplicates of rows 1, 35, 69
    dist, idx = den.nearest(x, 2)
    assert idx.tolist() == [[0, 1], [34, 35], [68, 69]]
    assert (dist == 0).all()

"""PRDC on the GPU: bit-identical to the reference on its exact golden cases, equal to the float64 restatement on continuous features,
exact where many pairs sit within the GEMM's error bound of a radius, and deterministic across calls, chunkings and CUDA-graph replay;
one 50 000 x 50 000 x 2048 run within the workspace bound."""
import os

import numpy as np
import pytest
import torch

import prdc_ref as O
from diff_sampler_b200 import prdc as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda'


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_prdc.npz')))


def _same(a, b):
    assert list(a) == list(b)
    for key in a:
        if key == 'realism':
            assert np.array_equal(a[key], b[key], equal_nan=True), key
        else:
            assert type(a[key]) is np.float64 and a[key] == b[key], (key, a[key], b[key])


def _inception_like(n, D, seed, device='cpu'):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(n, D, generator=g, device=device).abs()


@pytest.mark.parametrize('name', [c[0] for c in O.golden_cases()])
def test_golden_cases_are_bit_identical_to_the_reference(golden, name):
    r, f, k = golden[f'{name}/real'] / 16.0, golden[f'{name}/fake'] / 16.0, int(golden[f'{name}/k'])
    m = P.B200PRDC(r, k)
    got = m.score(f, realism=True)
    want = {key: golden[f'{name}/{key}'][()] for key in list(O.KEYS) + ['realism']}
    _same(got, want)
    assert np.array_equal(m.radii, golden[f'{name}/radii']) and np.array_equal(m.fake_radii, golden[f'{name}/fake_radii'])
    _same(P.compute_prdc(torch.from_numpy(r).to(DEV), torch.from_numpy(f).float(), k, realism=True), want)   # fp32 codes / 16 are exact


@pytest.mark.parametrize('n_r,n_f,dtype,on_gpu', [(4000, 3500, np.float32, False), (2500, 3000, np.float64, True)])
def test_continuous_features_match_the_restatement(n_r, n_f, dtype, on_gpu):
    real = _inception_like(n_r, 2048, 1).numpy().astype(dtype)
    fake = (_inception_like(n_f, 2048, 2) * 1.05).numpy().astype(dtype)
    args = (torch.from_numpy(real).to(DEV), torch.from_numpy(fake).to(DEV)) if on_gpu else (real, fake)
    m = P.B200PRDC(args[0], 5)
    got = m.score(args[1], realism=True)
    want, rad, frad = O.prdc(torch.from_numpy(real).double().to(DEV), torch.from_numpy(fake).double().to(DEV), 5, realism=True)
    for key in O.KEYS:
        assert got[key] == want[key], key
    for a, b in ((m.radii, rad), (m.fake_radii, frad), (got['realism'], want['realism'])):
        assert np.all(np.abs(a - b) <= 1e-12 * np.abs(b))
    print(f'rescored pairs: {m.last_rescored_pairs}')


def test_pairs_at_the_radii_are_counted_exactly():
    """Fake rows that copy real rows put pairs exactly at real radii (the copy of real row i's (k+1)-th neighbour), inside the GEMM's
    bound of the threshold; features on a 1/16 grid keep every sum exact, so each count is decided by the exact distances alone."""
    g = torch.Generator().manual_seed(5)
    real = torch.randint(0, 64, (3000, 256), generator=g).double() / 16
    fake = torch.randint(0, 64, (2000, 256), generator=g).double() / 16
    fake[:1500] = real[torch.randperm(3000, generator=g)[:1500]]
    m = P.B200PRDC(real, 5)
    got = m.score(fake, realism=True)
    want, rad, frad = O.prdc(real.to(DEV), fake.to(DEV), 5, realism=True)
    _same(got, want)
    assert np.array_equal(m.radii, rad) and np.array_equal(m.fake_radii, frad)
    assert m.last_rescored_pairs > 1500
    print(f'rescored pairs: {m.last_rescored_pairs}')


def test_chunks_calls_and_graph_replay_are_bit_identical(monkeypatch):
    real, fake = _inception_like(2000, 2048, 3), _inception_like(1700, 2048, 4)
    ref = P.B200PRDC(real, 5, cuda_graph=False)
    a = ref.score(fake, realism=True)
    _same(ref.score(fake, realism=True), a)
    g = P.B200PRDC(real, 5, cuda_graph=True)
    for _ in range(3):                                               # eager warm-up, capture, replay
        _same(g.score(fake, realism=True), a)
    assert np.array_equal(g.radii, ref.radii)
    monkeypatch.setattr(P, 'WORKSPACE_BYTES', 8 * 256 * 2048 * 4)      # 256-row chunks
    small = P.B200PRDC(real, 5)
    _same(small.score(fake, realism=True), a)
    assert np.array_equal(small.radii, ref.radii) and np.array_equal(small.fake_radii, ref.fake_radii)


def test_empty_realism_mask_is_refused():
    x = torch.zeros(10, 4, dtype=torch.float64)
    m = P.B200PRDC(x, 3)                                             # every radius 0: none below the median
    with pytest.raises(ValueError, match='realism'):
        m.score(x, realism=True)
    assert m.score(x)['precision'] == 0.0


def test_fid_sized_sets_run_within_the_workspace_bound():
    n, D = 50000, 2048
    real, fake = _inception_like(n, D, 7, DEV), _inception_like(n, D, 8, DEV) * 1.02
    m = P.B200PRDC(real, 5)
    got = m.score(fake)
    assert P.chunk_rows(n, n, D) * P.slices(D)[1] * P._pad(n) * 4 <= P.WORKSPACE_BYTES
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:64]
    for x, rad in ((real, m.radii), (fake, m.fake_radii)):
        d2 = O.exact_d2(x[rows.to(DEV)].double(), x.double()).kthvalue(6, dim=1).values
        want = O.sqrt(d2).cpu().numpy()
        assert np.all(np.abs(rad[rows.numpy()] - want) <= 1e-12 * want)
    assert all(0.0 <= got[k] <= 1.0 for k in ('precision', 'recall', 'coverage'))
    print(got, f'rescored pairs: {m.last_rescored_pairs}')

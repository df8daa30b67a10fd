"""PRDC, host side (no GPU): the float64 restatement against the reference's own compute_prdc (tests/golden/ref_prdc.npz), the
radii and score plans on the float64 plan interpreter against the restatement, the launcher rules of the two new ops, and the
argument errors, which match the reference's failure conditions."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import prdc_ref as O
from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import prdc as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = [c[0] for c in O.golden_cases()]


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_prdc.npz')))


@pytest.fixture(scope='module')
def built():
    from diff_sampler_b200 import _lib
    try:
        _lib.load()
    except _lib.DsError as e:
        pytest.skip(str(e))
    return _lib


def test_golden_inputs_are_the_seeded_ones(golden):
    for name, r, f, k in O.golden_cases():
        assert np.array_equal(golden[f'{name}/real'], r.numpy()) and np.array_equal(golden[f'{name}/fake'], f.numpy())
        assert int(golden[f'{name}/k']) == k


@pytest.mark.parametrize('name', NAMES)
def test_restatement_equals_the_reference_bit_for_bit(golden, name):
    r, f, k = golden[f'{name}/real'], golden[f'{name}/fake'], int(golden[f'{name}/k'])
    got, rad, frad = O.prdc(O.features(torch.from_numpy(r)), O.features(torch.from_numpy(f)), k, realism=True)
    assert list(got) == list(O.KEYS) + ['realism']
    for key in O.KEYS:
        assert type(got[key]) is np.float64 and got[key] == golden[f'{name}/{key}'], key
    assert np.array_equal(got['realism'], golden[f'{name}/realism'], equal_nan=True)
    assert np.array_equal(rad, golden[f'{name}/radii']) and np.array_equal(frad, golden[f'{name}/fake_radii'])


def test_golden_covers_the_edge_cases(golden):
    """Duplicates across the sets (zero distances and inf realism), zero radii with a zero distance (nan realism)."""
    assert np.isinf(golden['d2048/realism']).any()
    assert np.isnan(golden['zero/realism']).any() and (golden['zero/radii'] == 0).any()
    assert {int(golden[f'{n}/k']) for n in NAMES} >= {1, 5, 8}


def _near_threshold_sets(seed=3, n=300, m=260, D=64):
    """Continuous features with fake rows placed exactly at (and a hair inside / outside) real radii, so that many pairs sit within
    the GEMM's error bound of a threshold."""
    g = torch.Generator().manual_seed(seed)
    real = torch.rand(n, D, generator=g, dtype=torch.float64) * 4
    fake = torch.rand(m, D, generator=g, dtype=torch.float64) * 4
    r = O.radii(real, 5)[0]
    for j in range(0, 120, 3):
        i = j // 3
        u = torch.randn(D, generator=g, dtype=torch.float64)
        for t, s in enumerate((1.0, 1 - 1e-12, 1 + 1e-12)):
            fake[j + t] = real[i] + u / u.norm() * r[i] * s
    return real, fake


def _scores(out, k):
    cnt_f = out['cnt_f'].astype(np.int64)
    return dict(precision=(cnt_f > 0).mean(), recall=(out['cnt_r'] > 0).mean(), density=(1. / float(k)) * cnt_f.mean(),
                coverage=(out['own_r'] > 0).mean())


@pytest.mark.parametrize('case', ['zero', 'near', 'near_chunked'])
def test_plans_on_the_interpreter_reproduce_the_restatement(built, golden, monkeypatch, case):
    if case == 'zero':
        real, fake, k = O.features(torch.from_numpy(golden['zero/real'])), O.features(torch.from_numpy(golden['zero/fake'])), 5
    else:
        (real, fake), k = _near_threshold_sets(), 5
    if case == 'near_chunked':
        monkeypatch.setattr(P, 'WORKSPACE_BYTES', 128 * 4 * 320)       # 128-row chunks: three GEMM launches per pass
    hs = O.HostSets(real, fake, k)
    out = hs.run(realism=True)
    want, rad, frad = O.prdc(real, fake, k, realism=True)
    assert np.array_equal(out['radii'], rad) and np.array_equal(out['fake_radii'], frad)
    got = _scores(out, k)
    for key in O.KEYS:
        assert got[key] == want[key], key
    assert np.array_equal(out['realism'], want['realism'], equal_nan=True)
    n_gemm = [pl.meta['n_gemm'] for pl in out['plans']]
    assert n_gemm == ([3, 9] if case == 'near_chunked' else [1, 3])
    for pl in out['plans']:
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            assert built.op_check(getattr(op.u, S.ALL_UNION_FIELD[op.type])) is None


def test_chunks_cover_every_query_row_within_the_workspace():
    for nq, nt, D in ((50000, 50000, 2048), (10000, 10000, 2048), (7, 9, 3), (300, 260, 64)):
        c = P.chunk_rows(nq, nt, D)
        _, ns = P.slices(D)
        assert 1 <= c <= nq and ns * c * P._pad(nt) * 4 <= P.WORKSPACE_BYTES
        assert c == nq or c % 128 == 0
    assert P.chunk_rows(50000, 50000, 2048) == 1280


def test_operand_scale_keeps_the_hi_plane_in_range():
    for m in (1e-30, 3e-3, 1.0, 17.5, 2.0 ** 14, 6e4, 1e30):
        x = torch.tensor([[m, -m / 3]], dtype=torch.float64)
        s = P.operand_scale(x)
        assert 2.0 ** 13 <= m * s < 2.0 ** 14 and s == 2.0 ** round(np.log2(s))
        assert torch.isfinite(P.split_rows(x, s, 64).float()).all()
    assert P.operand_scale(torch.zeros(2, 3, dtype=torch.float64)) == 1.0


# ---------------------------------------------------------------------------------------------------- launcher rules
def _with(desc, **kw):
    d = type(desc).from_buffer_copy(desc)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _kth():
    return S.PrdcKthDesc(part=1, q=1, t=1, qn2=1, tn2=1, rad=1, rad2=1, nres=1, ldp=320, B=128, N=300, D=64, nslice=1, k=5, sq=1.0,
                         st=2.0)


def _count():
    return S.PrdcCountDesc(part=1, q=1, t=1, qn2=1, tn2=1, tau=1, tau2=1, rho=1, rho2=1, cnt_t=1, cnt_own=1, realism=1, nres=1, ldp=320,
                           B=128, N=300, D=64, nslice=1, sq=1.0, st=2.0, med=0.5)


RULES = [   # (make, rule, a breaking change, its nearest valid neighbour)
    (_kth, 'prdc_kth: shape', dict(ldp=299), dict(ldp=300)),
    (_kth, 'prdc_kth: shape', dict(nslice=0), dict(nslice=2)),
    (_kth, 'prdc_kth: k', dict(k=0), dict(k=1)),
    (_kth, 'prdc_kth: k', dict(k=S.DS_PRDC_KMAX + 1), dict(k=S.DS_PRDC_KMAX)),
    (_kth, 'prdc_kth: k', dict(N=5, ldp=5), dict(N=6, ldp=6)),
    (_kth, 'prdc_kth: scale', dict(sq=0.0), dict(sq=2.0 ** -20)),
    (_kth, 'prdc_kth: operands', dict(rad2=0), dict(nres=0)),
    (_count, 'prdc_count: shape', dict(D=0), dict(D=1)),
    (_count, 'prdc_count: scale', dict(st=float('nan')), dict(st=2.0 ** 40)),
    (_count, 'prdc_count: operands', dict(tau2=0), dict(realism=0)),
    (_count, 'prdc_count: own', dict(cnt_own=0), dict(cnt_own=0, rho=0, rho2=0)),
    (_count, 'prdc_count: own', dict(rho2=0), dict(rho2=0, rho=0, cnt_own=0)),
]


@pytest.mark.parametrize('make,rule,bad,good', RULES, ids=[f'{r[1]}-{i}' for i, r in enumerate(RULES)])
def test_each_rule_refuses_what_breaks_it_and_accepts_its_neighbour(built, make, rule, bad, good):
    assert built.op_check(make()) is None
    assert built.op_check(_with(make(), **bad)) == rule
    assert built.op_check(_with(make(), **good)) is None


def test_descriptor_sizes_and_plan_op_size(built):
    lib = built.load()
    for t in (S.DS_OP_PRDC_KTH, S.DS_OP_PRDC_COUNT):
        assert lib.ds_sizeof(t) == C.sizeof(S.SIZEOF_CHECKS[t])
    assert C.sizeof(S.PlanOp) == 528 == lib.ds_sizeof(0)          # every existing plan keeps its bytes
    assert (S.DS_OP_PRDC_KTH, S.DS_OP_PRDC_COUNT) == (24, 25)


def test_existing_plan_digests_are_unchanged():
    import plan_digest
    want = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'plan_digests.json')))
    got = plan_digest.all_digests(benchmarked=False)
    assert got and all(got[k] == want[k] for k in got)


# ---------------------------------------------------------------------------------------------------- arguments
def _f(n, d=8, dtype=np.float64):
    return np.random.default_rng(n).random((n, d)).astype(dtype)


@pytest.mark.parametrize('real,fake,k,match', [
    (_f(20), _f(20, 9), 5, 'features per row'),
    (_f(6), _f(20), 5, 'real_features has 6 rows'),            # argpartition needs k + 1 <= N - 1 in the reference
    (_f(20), _f(6), 5, 'fake_features has 6 rows'),
    (_f(20), _f(20), 0, 'nearest_k must be an integer >= 1'),
    (_f(200), _f(200), 64, 'at most 63'),
    (np.where(np.arange(160).reshape(20, 8) == 7, np.nan, _f(20)), _f(20), 5, 'non-finite'),
    (_f(20), np.where(np.arange(160).reshape(20, 8) == 7, np.inf, _f(20)), 5, 'non-finite'),
    (_f(20).astype(np.float16), _f(20), 5, 'float32 or float64'),
    (_f(20)[0], _f(20), 5, r'\[N, D\]'),
])
def test_arguments_are_refused_where_the_reference_fails(real, fake, k, match):
    with pytest.raises(ValueError, match=match):
        P.compute_prdc(real, fake, k)


def test_smallest_sets_the_reference_accepts_pass_validation():
    r, f = P._rows(_f(7), 'r'), P._rows(torch.from_numpy(_f(7, dtype=np.float32)), 'f')
    P._check_rows(r, 5, 'r')
    P._check_rows(f, 5, 'f')
    assert r.dtype == f.dtype == torch.float64

"""Optimal denoiser, host side (no GPU): the float64 oracle against the reference's own outputs (tests/golden/ref_opt.npz), the
optimal plan on the float64 plan interpreter against the oracle, descriptor sizes, argument errors, the dataset cache and the
reference quirks optimal_sampler keeps or rejects, and the kernels' register use."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import opt_ref as O
from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import _lib
from diff_sampler_b200 import optimal as OPT
from oracle import plan_interp as PI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_opt.npz')))


def test_golden_inputs_are_the_seeded_ones(golden):
    assert torch.equal(torch.from_numpy(golden['dataset']), O.golden_dataset())
    assert torch.equal(torch.from_numpy(golden['latents']), O.golden_latents())


@pytest.mark.parametrize('j', range(len(O.GOLDEN_SIGMAS)))
def test_oracle_denoiser_matches_reference(golden, j):
    ds = torch.from_numpy(golden['dataset'])
    x = torch.from_numpy(golden[f'opt_x_{j}'])
    got = O.denoise_opt(x, O.GOLDEN_SIGMAS[j], ds)
    ref = torch.from_numpy(golden[f'opt_d_{j}']).double()
    assert (got - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize('name', sorted(O.GOLDEN_SAMPLER_RUNS))
def test_oracle_sampler_matches_reference(golden, name):
    ds = torch.from_numpy(golden['dataset'])
    lat = torch.from_numpy(golden['latents'])
    kw = dict(O.GOLDEN_SAMPLER_RUNS[name])
    kw.pop('return_denoised', None)
    kw.pop('return_eps', None)
    r = O.optimal_sampler(lat, ds, **kw)
    if isinstance(r, tuple):
        for k, v in zip(('xt', 'den', 'eps'), r):
            ref = torch.from_numpy(golden[f'{name}_{k}']).double()
            assert v.shape == ref.shape, (k, v.shape, ref.shape)
            assert (v - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item()), k
    else:
        ref = torch.from_numpy(golden[f'{name}_x']).double()
        assert (r - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


def _interp(y, x, sigma):
    """The optimal plan for x [B, ...] run on the float64 plan interpreter: (D, per-row status)."""
    N, B = y.shape[0], x.shape[0]
    g = OPT._Geometry(N, int(np.prod(y.shape[1:])))
    blob, wb, ymax = OPT.pack_dataset(y.reshape(N, -1).float(), g)
    sig = torch.as_tensor(sigma, dtype=torch.float32).reshape(-1)
    pl = OPT.compile_plan(g, wb, B, sig.numel(), ymax)
    out = torch.full_like(x, float('nan'))
    status = torch.full((B,), -1, dtype=torch.int32)
    PI.run_plan(pl, blob.numpy().tobytes(), {S.DS_IO_X: x.contiguous(), S.DS_IO_D: out, S.DS_IO_SIGMA: sig,
                                             S.DS_IO_BOTTLENECK: status})
    return out, status


@pytest.mark.parametrize('sigma', [80.0, 5.0, 1.0, 0.2, 0.05, 0.002])
def test_plan_on_interpreter_matches_oracle(golden, sigma):
    ds = torch.from_numpy(golden['dataset'])
    lat = torch.from_numpy(golden['latents'])
    x = (ds[[3, 50, 100, 299]] + sigma * lat).float()
    got, status = _interp(ds, x, sigma)
    ref = O.denoise_opt(x, sigma, ds)
    assert torch.isfinite(got).all()
    assert (got.double() - ref).abs().max().item() < 1e-5
    assert (status != S.DS_OPT_UNREFINED).all()
    if sigma <= 0.05:
        assert (status == S.DS_OPT_RESCORED).all()


def test_plan_on_interpreter_odd_shape_and_per_sample_sigma():
    y = O.uint8_images(65, 3, 5, 7, seed=3)
    sig = torch.tensor([80.0, 0.002, 0.5])
    x = (y[[0, 1, 64]] + sig.reshape(-1, 1, 1, 1) * torch.randn(3, 3, 5, 7, generator=torch.Generator().manual_seed(1))).float()
    got, status = _interp(y, x, sig)
    ref = O.denoise_opt(x, sig, y)
    assert (got.double() - ref).abs().max().item() < 1e-5
    assert status[1].item() == S.DS_OPT_RESCORED and status[0].item() == S.DS_OPT_PLAIN


def test_knn_plan_on_interpreter():
    y = O.uint8_images(130, 3, 4, 4, seed=5)
    x = (y[[7, 9]] + 0.3 * torch.randn(2, 3, 4, 4, generator=torch.Generator().manual_seed(2))).float()
    g = OPT._Geometry(130, 48)
    blob, wb, ymax = OPT.pack_dataset(y.reshape(130, -1), g)
    pl = OPT.compile_plan(g, wb, 2, 1, ymax, knn=5)
    dist = torch.zeros(2, 5)
    idx = torch.zeros(2, 5, dtype=torch.int32)
    PI.run_plan(pl, blob.numpy().tobytes(), {S.DS_IO_X: x, S.DS_IO_D: dist, S.DS_IO_BOTTLENECK: idx})
    rd, ri, _ = O.knn(x, y, 5)
    assert torch.equal(idx.long(), ri)
    assert (dist.double() - rd).abs().max().item() < 1e-5


@pytest.mark.parametrize('knn', [0, 4])
def test_plan_stores_stay_inside_their_spans(knn):
    """Every byte an op of the optimal plans changes on the interpreter -- arena and io slots -- lies inside the op's store spans
    (opt_ref.writes), and every op type of the family occurs."""
    y = O.uint8_images(70, 3, 5, 7, seed=9)
    g = OPT._Geometry(70, 105)
    blob, wb, ymax = OPT.pack_dataset(y.reshape(70, -1), g)
    B = 3
    pl = OPT.compile_plan(g, wb, B, B, ymax, knn=knn)
    x = (y[:B] + 0.1).contiguous()
    io = {S.DS_IO_X: x, S.DS_IO_SIGMA: torch.tensor([80.0, 0.5, 0.002]), S.DS_IO_D: torch.zeros(B, knn or 105),
          S.DS_IO_BOTTLENECK: torch.zeros(B * (knn or 1), dtype=torch.int32)}
    mem = PI.Memory(pl.arena_bytes, blob.numpy().tobytes(), io)
    regions = {S.SPACE_ARENA: mem.arena}
    regions.update({(S.SPACE_IO, k): v.reshape(-1).view(torch.uint8) for k, v in io.items()})
    seen = set()
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        seen.add(op.type)
        before = {k: r.clone() for k, r in regions.items()}
        PI.run_op(mem, op)
        inside = {k: torch.zeros(r.numel(), dtype=torch.bool) for k, r in regions.items()}
        for sp in O.writes(op):
            space, off = sp.ref >> 60, sp.ref & PI.MASK60
            key = space if space == S.SPACE_ARENA else (space, off)
            o = off if space == S.SPACE_ARENA else 0
            assert o + sp.nbytes <= inside[key].numel(), (i, sp)
            inside[key][o:o + sp.nbytes] = True
        for k, r in regions.items():
            assert not ((r != before[k]) & ~inside[k]).any(), (i, op.type, k)
    want = {S.DS_OP_GEMM, S.DS_OP_OPT_PREP} | ({S.DS_OP_OPT_KNN} if knn else {S.DS_OP_OPT_SOFTMAX, S.DS_OP_OPT_REDUCE})
    assert seen == want


def test_geometry_and_workspace_bound():
    g = OPT._Geometry(50000, 3072)
    assert (g.Dp, g.Np, g.nslice, g.slice_c) == (3072, 50048, 12, 256)
    assert g.ksplit % 64 == 0 and g.nsplit * g.ksplit >= 50000 and g.ksplit <= OPT.KEYS_PER_SPLIT
    c = g.chunk()
    assert c == 512 and c * g.row_bytes() <= OPT.WORKSPACE_BYTES
    big = OPT._Geometry(50000, 12288)
    assert big.chunk() * big.row_bytes() <= OPT.WORKSPACE_BYTES and big.chunk() % 128 == 0


def test_descriptor_sizes_keep_the_plan_record():
    assert ctypes.sizeof(S.PlanOp) == 528                   # every existing plan keeps its bytes (tests/golden/plan_digests.json)
    for cls in (S.OptPrepDesc, S.OptSoftmaxDesc, S.OptReduceDesc, S.OptKnnDesc):
        assert ctypes.sizeof(cls) < ctypes.sizeof(S.GemmDesc)
    assert min(S.DS_OP_OPT_PREP, S.DS_OP_OPT_SOFTMAX, S.DS_OP_OPT_REDUCE, S.DS_OP_OPT_KNN) > S.DS_OP_EMBED


def test_constants_mirror_the_header():
    src = open(os.path.join(ROOT, 'diff-sampler_b200', 'csrc', 'ops.h')).read()
    for name in ('DS_OPT_CAP', 'DS_OPT_P_SHIFT', 'DS_OPT_BAND_NATS', 'DS_KNN_MAX', 'DS_KNN_CAND'):
        assert int(re.search(name + r' = (\d+)', src).group(1)) == getattr(S, name), name
    assert float(re.search(r'#define DS_OPT_TAU ([0-9.e+-]+)f', src).group(1)) == S.DS_OPT_TAU
    assert float(re.search(r'#define DS_OPT_EPS ([0-9.e+-]+)', src).group(1)) == S.DS_OPT_EPS


def test_constructor_rejects_bad_datasets():
    with pytest.raises(ValueError):
        OPT.B200OptimalDenoiser(torch.zeros(4, 3, 8))
    with pytest.raises(ValueError):
        OPT.B200OptimalDenoiser(torch.zeros(4, 3, 8, 8, dtype=torch.int32))
    with pytest.raises(ValueError):
        OPT.B200OptimalDenoiser(torch.zeros(0, 3, 8, 8))
    with pytest.raises(_lib.DsError):
        OPT.B200OptimalDenoiser(torch.zeros(4, 3, 8, 8), device='cpu')


def test_input_checks():
    den = object.__new__(OPT.B200OptimalDenoiser)
    den.shape, den.device = (3, 8, 8), torch.device('cuda', 0)
    with pytest.raises(_lib.DsError):
        den(torch.zeros(2, 3, 8, 8), 1.0)
    with pytest.raises(_lib.DsError):
        den.nearest(torch.zeros(2, 3, 8, 8), 3)


def test_sampler_rejects_reference_failures():
    lat = torch.zeros(2, 3, 8, 8)
    ds = torch.zeros(5, 3, 8, 8)
    with pytest.raises(ValueError, match='afs'):
        OPT.optimal_sampler(None, lat, ds, num_steps=4, afs=True, return_denoised=True)
    for kw in (dict(), dict(return_denoised=True), dict(return_eps=True)):
        with pytest.raises(ValueError, match='return_inters'):
            OPT.optimal_sampler(None, lat, ds, num_steps=4, return_inters=True, **kw)


def test_dataset_cache_keyed_by_storage_shape_and_version(monkeypatch):
    made = []

    class Fake:
        def __init__(self, dataset, device=None):
            made.append(dataset)

    monkeypatch.setattr(OPT, 'B200OptimalDenoiser', Fake)
    monkeypatch.setattr(OPT, '_CACHE', {})
    ds = torch.zeros(5, 3, 4, 4)
    a = OPT.denoiser_for(ds)
    assert OPT.denoiser_for(ds) is a and len(made) == 1
    ds.add_(1.0)                                            # in-place write: version bump -> re-pack
    b = OPT.denoiser_for(ds)
    assert b is not a and len(made) == 2
    other = torch.zeros(5, 3, 4, 4)
    OPT.denoiser_for(other)
    assert len(made) == 3 and len(OPT._CACHE) == 1          # at most one dataset kept
    OPT.denoiser_for(ds)
    assert len(made) == 4


def test_solvers_reexport_the_drop_ins():
    from diff_sampler_b200 import solvers
    assert solvers.get_denoised_opt is OPT.get_denoised_opt
    assert solvers.optimal_sampler is OPT.optimal_sampler
    import inspect
    sig = inspect.signature(OPT.optimal_sampler)
    assert list(sig.parameters)[:3] == ['net', 'latents', 'cifar10_dataset']
    assert {k: v.default for k, v in sig.parameters.items() if v.default is not inspect._empty} == dict(
        class_labels=None, num_steps=None, sigma_min=0.002, sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False,
        denoise_to_zero=False, return_inters=False, return_denoised=False, return_eps=False, t_steps=None)
    assert list(inspect.signature(OPT.get_denoised_opt).parameters) == ['x', 't', 'cifar10_dataset']


def test_kernels_compile_without_spills(tmp_path):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not available')
    src = os.path.join(ROOT, 'diff-sampler_b200', 'csrc', 'optimal.cu')
    r = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c', src, '-o',
                        str(tmp_path / 'o.o')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    assert len(kernels) == 4, kernels
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', r.stderr)
    assert len(spills) == 4 and all(s == ('0', '0') for s in spills), r.stderr

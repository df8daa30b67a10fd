"""The FID feature extractor on the GPU: the three new kernels against float64 at every shape the plans launch, the GEMM's ReLU
epilogue, op-by-op replay of two plans against the float64 plan interpreter, the features against the float64 oracle in both
precisions, chunked batches, CUDA-graph replay, and sample -> uint8 -> features -> FID end to end.

Weights: torchvision's random init with BatchNorm statistics calibrated on random images (oracle/inception_oracle.make_state_dict)."""
import numpy as np
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import inception_plan as IP
from oracle import inception_oracle as O
from oracle import plan_interp as PI
from plan_spans import resolve, writes

import inception_interp as II

pytestmark = pytest.mark.gpu

SIZES = (32, 64, 256, 512)


def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


@pytest.fixture(scope='module')
def sd():
    return O.make_state_dict(0)


@pytest.fixture(scope='module')
def wb(sd):
    return IP.pack_inception_weights(sd)


@pytest.fixture(scope='module')
def oracle_sd(sd):
    return {k: v.to(dev()) for k, v in sd.items()}


def _images(B, H, W, seed=0):
    return torch.randint(0, 256, (B, 3, H, W), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _key(desc):
    val = lambda v: tuple(v) if hasattr(v, '__len__') else v            # ctypes arrays (the GEMM's dims, strides, taps)
    return tuple((k, val(getattr(desc, k))) for k, t in type(desc)._fields_ if t is not S.P)


def _unique_ops(plans, types):
    """(plan, op) for the first op of each distinct descriptor (pointer fields aside) of the given types."""
    seen, out = set(), []
    for pl in plans:
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            if op.type not in types:
                continue
            k = (op.type, _key(getattr(op.u, S.ALL_UNION_FIELD[op.type])))
            if k not in seen:
                seen.add(k)
                out.append((pl, op))
    return out


def _locate(arena, io, span):
    space, off = span.ref >> 60, span.ref & PI.MASK60
    if space == S.SPACE_ARENA:
        return arena[off:off + span.nbytes]
    return io[off].reshape(-1).view(torch.uint8)[:span.nbytes]


def _run_both(lib, pl, op, wdev, io, seed):
    """The op on a seeded random fp32 arena: (spans, kernel bytes, interpreter bytes).  Needs II.install."""
    g = torch.Generator(device=dev()).manual_seed(seed)
    arena = (torch.rand(pl.arena_bytes // 4, generator=g, device=dev()) * 2.5 - 0.5).view(torch.uint8)
    snap, snap_io = arena.clone(), {k: v.clone() for k, v in io.items()}
    PI.run_op(PI.Memory(0, None, snap_io, device=dev(), arena=snap, weights=wdev), op)
    lib.op_launch(resolve(op, arena, wdev, io))
    torch.cuda.synchronize()
    spans = writes(op)
    return spans, [_locate(arena, io, s) for s in spans], [_locate(snap, snap_io, s) for s in spans]


def test_new_kernels_match_float64_at_every_plan_shape(lib, wb, monkeypatch):
    """ds_img_input (both input layouts, every input size), ds_im2col and ds_pool at every descriptor the plans launch: im2col and
    max pooling exact, the averages and the resize within 1e-6 of max |value|."""
    II.install(monkeypatch)
    wdev = torch.frombuffer(bytearray(wb.bytes()), dtype=torch.uint8).to(dev())
    B = 3
    plans = []
    for size in SIZES:
        x = _images(B, size, size, seed=size)
        for layout in ('nchw', 'nhwc'):
            xs = x if layout == 'nchw' else x.permute(0, 2, 3, 1).contiguous()
            strides = None if layout == 'nchw' else tuple(xs.permute(0, 3, 1, 2).stride())
            pl = IP.compile_inception_plan(wb, B, size, size, 3, strides)
            plans.append(pl)
            io = {S.DS_IO_X: xs.to(dev()), S.DS_IO_D: torch.zeros(B, IP.FEATURES, device=dev())}
            (pl0, op), = _unique_ops([pl], {S.DS_OP_IMG_INPUT})
            spans, got, want = _run_both(lib, pl0, op, wdev, io, 0)
            g, w = got[0].view(torch.float32).double(), want[0].view(torch.float32).double()
            assert (g - w).abs().max().item() <= 1e-6 * max(1.0, w.abs().max().item()), (size, layout)
    plans.append(IP.compile_inception_plan(wb, B, 64, 64, 1))          # the fp16 plans write one plane
    io = {S.DS_IO_X: _images(B, 64, 64).to(dev()), S.DS_IO_D: torch.zeros(B, IP.FEATURES, device=dev())}
    checked = {S.DS_OP_IM2COL: 0, S.DS_OP_POOL: 0}
    for n, (pl, op) in enumerate(_unique_ops(plans, {S.DS_OP_IM2COL, S.DS_OP_POOL})):
        spans, got, want = _run_both(lib, pl, op, wdev, io, n + 1)
        checked[op.type] += 1
        exact = op.type == S.DS_OP_IM2COL or op.u.pool.mode == S.DS_POOL_MAX
        for s, g, w in zip(spans, got, want):
            if exact:
                assert torch.equal(g, w), (n, s.fmt)
                continue
            if s.fmt == 'f32':
                gv, wv = g.view(torch.float32).double(), w.view(torch.float32).double()
            else:
                h = lambda b: b.view(torch.float16).double()
                gv, wv = h(g), h(w)
                if s.nplanes == 2:
                    k = gv.numel() - s.plane
                    gv, wv = gv[:k] + gv[s.plane:], wv[:k] + wv[s.plane:]
            # the gaps between the written channel windows hold the random arena bytes (identical on both sides, NaN as fp16 at times)
            diff = (gv - wv).nan_to_num(0.0, posinf=0.0, neginf=0.0)
            # a lone fp16 plane: an fp32 mean one ulp off a rounding boundary may round to the neighbouring fp16 value (2^-10 relative)
            rel = 2.0 ** -10 if s.fmt == 'f16' and s.nplanes == 1 else 1e-6
            assert diff.abs().max().item() <= rel * wv.nan_to_num(0.0, posinf=0.0, neginf=0.0).abs().max().item(), (n, s.fmt)
    print(f'checked {checked[S.DS_OP_IM2COL]} im2col and {checked[S.DS_OP_POOL]} pool descriptors')
    assert checked[S.DS_OP_IM2COL] > 20 and checked[S.DS_OP_POOL] >= 6


def test_gemm_relu_is_max_of_the_plain_epilogue(lib, wb):
    """Every distinct GEMM of a plan, relu = 1 against relu = 0 on the same operands: bitwise max(v, 0) of the fp32 output."""
    pl = IP.compile_inception_plan(wb, 2, 64, 64, 3)
    wdev = torch.frombuffer(bytearray(wb.bytes()), dtype=torch.uint8).to(dev())
    g = torch.Generator(device=dev()).manual_seed(5)
    arena = (torch.rand(pl.arena_bytes // 2, generator=g, device=dev()) * 2 - 1).half().view(torch.uint8)
    io = {S.DS_IO_D: torch.zeros(2, IP.FEATURES, device=dev())}
    n = 0
    for _, op in _unique_ops([pl], {S.DS_OP_GEMM}):
        d = resolve(op, arena, wdev, io)
        d.out_h16, d.o_plane = 0, 0
        m, nv, ldo = int(d.m_valid), int(d.n_valid), int(d.ldo)
        out = lambda: torch.as_strided(arena[int(d.out_f32) - arena.data_ptr():].view(torch.float32), (m, nv), (ldo, 1)).clone()
        d.relu = 0
        lib.op_launch(d)
        plain = out()
        d.relu = 1
        lib.op_launch(d)
        got = out()
        assert torch.equal(got, plain.clamp_min(0.0)) and (plain < 0).any(), (n, m, nv)
        n += 1
    assert n > 40


def test_plan_ops_against_the_interpreter(lib, wb, monkeypatch):
    """Op-by-op replay of the 32^2 and 256^2 plans (batch 2) against the float64 plan interpreter, as tests/test_gpu_plan_ops.py does
    for the benchmarked plans: stores only inside each op's spans, every element the reference writes written and within tolerance."""
    import test_gpu_plan_ops as TPO
    II.install(monkeypatch)

    def workload(name):
        size = int(name.split('_')[1])
        return (IP.compile_inception_plan(wb, 2, size, size, 3), wb.bytes(),
                {S.DS_IO_X: _images(2, size, size, seed=size), S.DS_IO_D: torch.zeros(2, IP.FEATURES)})
    monkeypatch.setattr(TPO, 'workload', workload)
    for name in ('inception_32', 'inception_256'):
        res = TPO.replay(lib, name)
        bad = [r for r in res['rows'] if r['ratio'] > 1.0 or r['problems']]
        worst = {}
        for r in res['rows']:
            worst[r['type']] = max(worst.get(r['type'], 0.0), r['ratio'])
        print(f"{name}: {res['n_ops']} ops, worst error / bound per type {worst}")
        assert not res['skips'] and len(res['rows']) == res['n_ops']
        assert not bad, '\n'.join(TPO._fmt(name, r) for r in bad[:20])


@pytest.mark.parametrize('precision', ['fp16x3', 'fp16'])
def test_features_against_the_oracle(lib, sd, oracle_sd, precision):
    from diff_sampler_b200.inception_net import B200InceptionV3
    det = B200InceptionV3(sd, precision=precision)
    worst = 0.0
    for size in SIZES:
        x = _images(3, size, size, seed=size).to(dev())
        got = det(x).double()
        want = O.features(x, oracle_sd)
        fmax = want.abs().max().item()
        err = (got - want).abs().max().item()
        print(f'{precision} {size}x{size}: max |f| {fmax:.3f}, max |diff| {err:.3e} = {err / fmax:.2e} of max |f|')
        worst = max(worst, err / max(1.0, fmax) if precision == 'fp16x3' else err / fmax)
        nhwc = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)          # the samplers' NHWC images, viewed as NCHW
        assert torch.equal(det(nhwc), got.float())
    # fp16x3: the project's gate.  fp16 (one fp16 pass per product, 94 layers deep): measured on an H100 80GB HBM3, 2.1e-2 of max |f|
    # at 32 x 32 on these weights; the bound leaves room for the other sizes and seeds
    assert worst <= (1e-3 if precision == 'fp16x3' else 5e-2), worst
    with pytest.raises(NotImplementedError):
        det(x, return_features=False)


def test_chunked_batch_equals_single_images(lib, sd):
    from diff_sampler_b200.inception_net import B200InceptionV3
    det = B200InceptionV3(sd, max_batch=64)
    x = _images(250, 64, 64, seed=9).to(dev())
    got = det(x)
    one = torch.cat([det(x[i:i + 1]) for i in range(250)])
    err = (got - one).abs().max().item()
    print(f'batch 250 in chunks of 64 vs one image at a time: max |diff| {err:.3e}, max |f| {one.abs().max().item():.3f}')
    assert err <= 1e-6 * one.abs().max().item()


def test_cuda_graph_replay_is_bitwise_eager(lib, sd):
    from diff_sampler_b200.inception_net import B200InceptionV3
    eager = B200InceptionV3(sd, cuda_graph=False)
    graph = B200InceptionV3(sd, cuda_graph=True)
    for k in range(3):                                         # plain warm-up, capture, replay
        x = _images(5, 48, 48, seed=k).to(dev())
        assert torch.equal(eager(x), graph(x)), k


def test_sample_to_fid_end_to_end(lib, sd, oracle_sd):
    """euler_sampler(images_uint8=...) on a tiny EDM net -> FeatureStats.append_images(u8, det) -> frechet_distance, against the FID
    of the oracle's features of the same uint8 images."""
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.fid_stats import FeatureStats, frechet_distance
    from diff_sampler_b200.inception_net import B200InceptionV3
    from diff_sampler_b200.net import B200Net
    from oracle import edm_oracle as EO
    P, Sp = EO.make_net('tiny_song', seed=0, dezero=True)
    net = B200Net(P, Sp['img_resolution'], Sp['img_channels'], Sp['label_dim'], device=dev())
    det = B200InceptionV3(sd)
    ours, ref = FeatureStats(), FeatureStats()
    images = []
    for b in range(3):
        lat = EO.stacked_randn(range(16 * b, 16 * b + 16), (3, 16, 16)).to(dev())
        u8 = torch.empty(16, 16, 16, 3, dtype=torch.uint8, device=dev())
        solvers.euler_sampler(net, lat, num_steps=4, images_uint8=u8)
        ours.append_images(u8, det)
        ref.append(O.features(u8.permute(0, 3, 1, 2), oracle_sd))
        images.append(u8)
    mu, sig = ours.finalize()
    mu_r, sig_r = ref.finalize()
    g = torch.Generator().manual_seed(1)
    mu0, sig0 = mu_r + torch.randn(mu_r.shape, generator=g, dtype=torch.float64).numpy() * 0.1, np.eye(mu_r.shape[0])  # 48 images: sig_r is singular
    fid, fid_ref = frechet_distance(mu, sig, mu0, sig0), frechet_distance(mu_r, sig_r, mu0, sig0)
    print(f'FID {fid:.6f} against the oracle features {fid_ref:.6f}')
    assert abs(fid - fid_ref) <= 1e-4 * abs(fid_ref)

"""The FID feature extractor on the CPU: the float64 oracle (oracle/inception_oracle.py) pinned to torchvision's Inception3 and to the
TF graph's pools, the input resize pinned to NVIDIA's affine_grid / grid_sample formulation, the BatchNorm fold, the plan on the
float64 plan interpreter against the oracle, and the launcher checks of the three new ops."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import inception_plan as IP
from oracle import inception_oracle as O

import inception_interp as II

SIZES = (32, 64, 256, 512)


@pytest.fixture(scope='module')
def sd():
    return O.make_state_dict(0)


@pytest.fixture(scope='module')
def wb(sd):
    return IP.pack_inception_weights(sd)


@pytest.fixture(scope='module')
def built():
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    from diff_sampler_b200 import _lib
    return _lib


def _tv_model(sd):
    import torchvision
    m = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=False, transform_input=False)
    m.load_state_dict(sd, strict=False)
    return m.double().eval()


def _images(B, H, W, seed=0):
    return torch.randint(0, 256, (B, 3, H, W), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def test_oracle_without_quirks_is_torchvision(sd):
    m = _tv_model(sd)
    cap = {}
    m.avgpool.register_forward_hook(lambda mod, i, o: cap.__setitem__('f', o.flatten(1)))
    x = O.input_stage(_images(2, 64, 64))
    with torch.no_grad():
        m(x)
    got = O.body(x, sd, tf_quirks=False).mean(dim=(2, 3))
    assert (got - cap['f']).abs().max().item() <= 1e-10 * cap['f'].abs().max().item()


@pytest.mark.parametrize('name,cin,hw', [('Mixed_5b', 192, 35), ('Mixed_5c', 256, 35), ('Mixed_5d', 288, 35), ('Mixed_6b', 768, 17),
                                         ('Mixed_6c', 768, 17), ('Mixed_6d', 768, 17), ('Mixed_6e', 768, 17), ('Mixed_7b', 1280, 8),
                                         ('Mixed_7c', 2048, 8)])
def test_quirk_blocks_are_torchvision_blocks_with_the_tf_pools(sd, name, cin, hw, monkeypatch):
    """Each patched block equals torchvision's with its pool branch replaced: an average without the padding in the count, and for
    Mixed_7c a 3 x 3 stride-1 max pool."""
    m = _tv_model(sd)
    x = torch.rand(2, cin, hw, hw, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    avg = F.avg_pool2d
    if name == 'Mixed_7c':
        monkeypatch.setattr(F, 'avg_pool2d', lambda t, kernel_size, stride, padding: F.max_pool2d(t, kernel_size, stride, padding))
    else:
        monkeypatch.setattr(F, 'avg_pool2d', lambda t, kernel_size, stride, padding: avg(t, kernel_size, stride, padding, count_include_pad=False))
    with torch.no_grad():
        want = getattr(m, name)(x)
    monkeypatch.undo()
    kind = {'5': 'a', '6': 'c', '7': 'e'}[name[6]]
    args = (True, True) if name == 'Mixed_7c' else (True,)
    got = getattr(O, 'block_' + kind)(x, sd, name, *args)
    assert (got - want).abs().max().item() <= 1e-10 * want.abs().max().item()
    # and the quirk changes the result (the test would not notice a pool left as torchvision's)
    plain = getattr(O, 'block_' + kind)(x, sd, name, False)
    assert (plain - want).abs().max().item() > 1e-6 * want.abs().max().item()


def _nvidia_resize(x):
    """NVIDIA's port of the TF resize: affine_grid with the theta shift, grid_sample(bilinear, border, align_corners=False)."""
    B, C, H, W = x.shape
    theta = torch.eye(2, 3, dtype=torch.float64)
    theta[0, 2] += theta[0, 0] / W - theta[0, 0] / 299
    theta[1, 2] += theta[1, 1] / H - theta[1, 1] / 299
    grid = F.affine_grid(theta.unsqueeze(0).repeat(B, 1, 1), [B, C, 299, 299], align_corners=False)
    return F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=False)


@pytest.mark.parametrize('size', [32, 64, 256, 512, 299])
def test_resize_is_nvidia_grid_sample_and_the_closed_form(size):
    x = _images(2, size, size, seed=size).double()
    got = O.resize_tf_legacy(x)
    assert (got - _nvidia_resize(x)).abs().max().item() < 1e-9
    g = torch.Generator().manual_seed(3)
    for _ in range(64):                                        # the closed form, pixel by pixel
        i, j = (int(v) for v in torch.randint(0, 299, (2,), generator=g))
        fy, fx = i * size / 299, j * size / 299
        y0, x0 = int(fy), int(fx)
        y1, x1 = min(y0 + 1, size - 1), min(x0 + 1, size - 1)
        dy, dx = fy - y0, fx - x0
        p = x[1, 2]
        top = p[y0, x0] + (p[y0, x1] - p[y0, x0]) * dx
        bot = p[y1, x0] + (p[y1, x1] - p[y1, x0]) * dx
        assert abs(float(top + (bot - top) * dy) - float(got[1, 2, i, j])) < 1e-9
    if size == 299:
        assert torch.equal(got, x)


def test_bn_fold_reproduces_conv_bn(sd):
    x = torch.randn(2, 288, 17, 17, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    for name, (cin, cout, (kh, kw), s, (ph, pw)) in IP.layers().items():
        if cin != 288:
            continue
        w, b = IP.fold_bn(sd, name)
        w4 = w.reshape(cout, kh, kw, cin).permute(0, 3, 1, 2)
        got = F.relu(F.conv2d(x, w4, b, stride=s, padding=(ph, pw)))
        want = O.basic_conv(x, sd, name, stride=s, padding=(ph, pw))
        assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item(), name


@pytest.mark.parametrize('size,layout', [(32, 'nchw'), (64, 'nchw'), (32, 'nhwc')])
def test_plan_on_the_interpreter_equals_the_oracle(sd, wb, size, layout):
    B = 2
    x = _images(B, size, size, seed=size)
    if layout == 'nhwc':
        xs = x.permute(0, 2, 3, 1).contiguous()               # the memory of the samplers' NHWC uint8 images
        strides = tuple(xs.permute(0, 3, 1, 2).stride())
    else:
        xs, strides = x, None
    pl = IP.compile_inception_plan(wb, B, size, size, 3, strides)
    D = torch.zeros(B, IP.FEATURES)
    II.run_plan(pl, wb.bytes(), {S.DS_IO_X: xs, S.DS_IO_D: D})
    want = O.features(x, sd)
    err = (D.double() - want).abs().max().item()
    # the plan's operands are fp16 hi/lo pairs (~2^-22 relative) and its folded weights fp32: measured 2e-5 of max |f| after 94 layers
    assert err <= 1e-4 * want.abs().max().item(), (err, want.abs().max().item())


def test_every_op_of_the_plans_passes_its_launcher_check(built, wb):
    for B in (1, 64):
        for size in SIZES:
            pl = IP.compile_inception_plan(wb, B, size, size, 3)
            for i in range(pl.n_ops):
                op = pl.ops_array[i]
                why = built.op_check(getattr(op.u, S.ALL_UNION_FIELD[op.type]))
                assert why is None, (B, size, i, op.tag, why)


def _with(desc, **kw):
    d = type(desc).from_buffer_copy(desc)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _img_input():
    return S.ImgInputDesc(src=1, out=1, sn=3 * 64 * 64, sc=64 * 64, sy=64, sx=1, B=2, C=3, H=64, W=64, Ho=299, Wo=299)


def _im2col():
    return S.Im2colDesc(src=1, out=1, B=2, H=35, W=35, C=48, src_pitch=48, src_c0=0, kh=5, kw=5, sh=1, sw=1, ph=2, pw=2, K64=1216, nplanes=2)


def _pool():
    return S.PoolDesc(src=1, out_f32=1, out_h16=1, B=2, H=35, W=35, C=288, src_pitch=288, src_c0=0, out_pitch=768, out_c0=480, k=3, stride=2,
                      pad=0, mode=S.DS_POOL_MAX, nplanes=2)


RULES = [   # (make, rule, a breaking change, its nearest valid neighbour)
    (_img_input, 'img_input: shape', dict(Ho=0), dict(Ho=1)),
    (_im2col, 'im2col: shape', dict(ph=-1), dict(ph=0)),
    (_im2col, 'im2col: K64', dict(K64=1200), dict(K64=1280)),
    (_im2col, 'im2col: channels', dict(src_c0=8), dict(src_c0=8, src_pitch=56)),
    (_im2col, 'im2col: nplanes', dict(nplanes=3), dict(nplanes=1)),
    (_pool, 'pool: mode', dict(mode=3), dict(mode=S.DS_POOL_AVG)),
    (_pool, 'pool: shape', dict(C=0), dict(C=4)),
    (_pool, 'pool: window', dict(pad=3), dict(pad=2)),
    (_pool, 'pool: channels', dict(out_c0=484), dict(out_c0=480, out_pitch=768)),
    (_pool, 'pool: alignment', dict(out_c0=482, out_pitch=772), dict(out_c0=484, out_pitch=772)),
    (_pool, 'pool: outputs', dict(out_f32=0, out_h16=0), dict(out_f32=0)),
    (_pool, 'pool: outputs', dict(mode=S.DS_POOL_MEAN), dict(mode=S.DS_POOL_MEAN, out_h16=0)),
    (_pool, 'pool: nplanes', dict(nplanes=0), dict(nplanes=1)),
]


@pytest.mark.parametrize('make,rule,bad,good', RULES, ids=[f'{r[1]}-{i}' for i, r in enumerate(RULES)])
def test_each_rule_refuses_what_breaks_it_and_accepts_its_neighbour(built, make, rule, bad, good):
    assert built.op_check(make()) is None
    assert built.op_check(_with(make(), **bad)) == rule
    assert built.op_check(_with(make(), **good)) is None


def test_gemm_descriptor_keeps_its_size(built):
    lib = built.load()
    assert C.sizeof(S.GemmDesc) == 520 == lib.ds_sizeof(S.DS_OP_GEMM)
    assert S.GemmDesc.st_unit.offset == 512 and S.GemmDesc.relu.offset == 516
    assert C.sizeof(S.PlanOp) == 528 == lib.ds_sizeof(0)
    for t in (S.DS_OP_IMG_INPUT, S.DS_OP_IM2COL, S.DS_OP_POOL):
        assert lib.ds_sizeof(t) == C.sizeof(S.SIZEOF_CHECKS[t])

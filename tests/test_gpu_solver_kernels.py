"""Solver-side kernels (csrc/solver.cu) against exact references, at the sizes the samplers run them (GPU).

Each kernel is called through the C ABI as solver_utils.py, gits_utils.py and dist_utils.py call it, and compared with a float64 or
exact-integer reference of the same operation:

  * the uint8 image conversion (ds_images_to_uint8, and the epilogue of ds_solver_update_u8) for every fp32 bit pattern;
  * the fused update, all 20 update_kernel<NH, MODE> instantiations, at the samplers' shapes (grids of up to three sweeps);
  * the dynamic-thresholding quantile on its three launch paths and at the rank edge cases of its radix select;
  * the GITS cost reductions at the benchmark's teacher sizes, each sum against its own roundoff bound.

Every output buffer sits between a head and a tail guard (NaN for floats; 0xFF or 0x00 for bytes) that must come back untouched, and
its body is pre-filled the same way, so an element the kernel never writes shows up as a NaN or as a wrong byte.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
GUARD = 64              # guard elements before and after every output; 64 keeps the body 16-byte aligned for the float4 paths
X0, EPS, DIV, NONE = 0, 1, 2, 3     # DS_M_* (csrc/ops.h)


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


def dev():
    return torch.device('cuda:0')


def stream():
    return C.c_void_p(torch.cuda.current_stream(dev()).cuda_stream)


def ptr(t):
    return None if t is None else t.data_ptr()


def bits(t):
    """Integer view of a tensor's storage, for bitwise comparisons."""
    return t.view({torch.float32: torch.int32, torch.float64: torch.int64}.get(t.dtype, t.dtype))


class Guarded:
    """GUARD + n + GUARD elements filled with `fill`; the kernel writes `body`, the n elements in the middle."""

    def __init__(self, n, dtype, fill):
        self.n = n
        self.full = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=dev())
        self.body = self.full[GUARD:GUARD + n]
        self.fill = bits(self.full[:1].clone())

    def guards_intact(self):
        ends = torch.cat([self.full[:GUARD], self.full[GUARD + self.n:]])
        return bool((bits(ends) == self.fill).all())


def u8_expr(x):
    """sample.py:311's (x * 127.5 + 128).clip(0, 255).to(uint8), in place on one fp32 temporary.  Every torch op is its own kernel,
    so the product and the sum are rounded separately in fp32, as on the CPU."""
    r = x.mul(127.5)
    r.add_(128)
    r.clamp_(0, 255)
    return r.to(torch.uint8)


# --------------------------------------------------------------------------------------------- uint8 conversion, every fp32 input
CHUNK = 1 << 26         # 2^32 bit patterns in 64 chunks: ~1 GiB of device memory at the peak


def _patterns(k, total):
    """fp32 tensor of `total` values: chunk k of all 2^32 bit patterns (int32 order), then the chunk's head again as padding."""
    b = torch.arange(total, dtype=torch.int32, device=dev())
    b[CHUNK:] -= CHUNK
    b += -2 ** 31 + k * CHUNK
    return b.view(torch.float32)


def _u8_mismatches(x, got, out):
    """Compares the bytes `got` (in x's order) with u8_expr(x).  Returns the mismatching input patterns of the chunk proper as rows
    (bits, reference, kernel), and the mismatch count over the padded tensor."""
    assert out.guards_intact(), 'a byte outside the image was written'
    nan = torch.isnan(x)
    assert (got[nan] == 0).all(), 'NaN must convert to 0 (fmaxf(NaN, 0) = 0)'
    want = u8_expr(x)
    diff = (got != want) & ~nan              # torch's NaN -> uint8 cast is undefined: NaN is checked above instead
    idx = diff[:CHUNK].nonzero().flatten()
    rows = torch.stack([bits(x)[idx].long() & 0xFFFFFFFF, want[idx].long(), got[idx].long()], 1).cpu()
    return rows, int(diff.sum())


def u8_sweep(lib):
    """Converts all 2^32 fp32 bit patterns through both entry points.  Returns {entry point: (rows of mismatching unique inputs,
    total mismatches including the padding)}.

    ds_images_to_uint8 runs with C = 1, 3, 4 in turn and an odd pixel count, so the NHWC scatter is checked as well; the bytes are
    permuted back to the input's NCHW order.  ds_solver_update_u8 runs with mode NONE and coefficients (1, 0): out_x = 1 * xb + 0 * 0
    equals xb exactly (NaN stays NaN), so its epilogue sees the same values; C = 3, HW = 4096, B > 1.  Guards and bodies are filled
    with 0xFF in even chunks and 0x00 in odd chunks."""
    l = lib.load()
    found = {'ds_images_to_uint8': [], 'ds_solver_update_u8': []}
    count = dict.fromkeys(found, 0)
    hist = (C.c_void_p * 4)()
    coef = (C.c_float * 6)(1.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    for k in range((1 << 32) // CHUNK):
        fill = 0xFF if k % 2 == 0 else 0x00
        Cc, HW = (1, 3, 4)[k % 3], 4095
        B = -(-CHUNK // (Cc * HW))
        x = _patterns(k, B * Cc * HW)
        out = Guarded(x.numel(), torch.uint8, fill)
        lib.check(l.ds_images_to_uint8(x.data_ptr(), out.body.data_ptr(), B, Cc, HW, stream()), 'ds_images_to_uint8')
        rows, n = _u8_mismatches(x, out.body.view(B, HW, Cc).permute(0, 2, 1).reshape(-1), out)
        found['ds_images_to_uint8'].append(rows)
        count['ds_images_to_uint8'] += n
        del x, out

        Cc, HW = 3, 4096
        B = -(-CHUNK // (Cc * HW))
        x = _patterns(k, B * Cc * HW)
        ox = Guarded(x.numel(), torch.float32, float('nan'))
        out = Guarded(x.numel(), torch.uint8, fill)
        lib.check(l.ds_solver_update_u8(ox.body.data_ptr(), None, out.body.data_ptr(), Cc, HW, x.data_ptr(), None, None, hist, 0, None,
                                        NONE, 1.0, None, coef, None, Cc * HW, B, stream()), 'ds_solver_update_u8')
        assert ox.guards_intact()
        assert bool(((ox.body == x) | (torch.isnan(ox.body) & torch.isnan(x))).all()), 'out_x = 1 * xb + 0 * 0 must equal xb'
        del ox
        rows, n = _u8_mismatches(x, out.body.view(B, HW, Cc).permute(0, 2, 1).reshape(-1), out)
        found['ds_solver_update_u8'].append(rows)
        count['ds_solver_update_u8'] += n
        del x, out
    return {name: (torch.cat(found[name]), count[name]) for name in found}


def test_uint8_conversion_every_fp32_input(lib):
    """Both uint8 entry points against the torch expression, byte for byte, for every fp32 input but NaN (which must give 0).

    sample.py:311 rounds x * 127.5 and then the sum with 128; a single FMA rounds once, and the truncation then gives one less for
    inputs within an ulp of a boundary (N - 128) / 127.5 (e.g. 0x3C008040 = 0.0078430772: 129, not 128)."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    res = u8_sweep(lib)
    torch.cuda.synchronize()
    print(f'uint8 sweep of 2^32 inputs x 2 entry points: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')
    msg = []
    for name, (rows, n) in res.items():
        print(f'  {name}: {rows.shape[0]} mismatching inputs')
        if rows.shape[0] or n:
            ex = ', '.join(f'0x{b:08X} ({float(np.uint32(b).view(np.float32))!r}): want {w} got {g}'
                           for b, w, g in rows[:6].tolist())
            msg.append(f'{name}: {rows.shape[0]} inputs convert differently from (x * 127.5 + 128).clip(0, 255).to(uint8), e.g. {ex}')
    assert not msg, '; '.join(msg)
    # and through the Python front end the samplers' fallback uses (dist_utils.to_uint8_nhwc), on image-like values and the examples
    from diff_sampler_b200 import dist_utils
    g = torch.Generator().manual_seed(15)
    x = (torch.randn(9, 3, 32, 32, generator=g) * 0.8).to(dev())
    x[0, 0, 0, :3] = torch.from_numpy(np.array([0xBF7CFCFD, 0xBC0080A1, 0x3C008040], np.uint32).view(np.float32)).to(dev())
    x[0, 0, 1, :4] = torch.tensor([-1.0, 1.0, 0.99999, -5.0], device=dev())
    assert torch.equal(dist_utils.to_uint8_nhwc(x), u8_expr(x).permute(0, 2, 3, 1))


# --------------------------------------------------------------------------------------------- fused update
SHAPES = {                                    # (B, C, HW): n_per_sample = C * HW
    'cifar10_512x3x32x32': (512, 3, 32 * 32),
    'imagenet64_256x3x64x64': (256, 3, 64 * 64),
    'sd_latent_8x4x64x64': (8, 4, 64 * 64),
    'cfg_16x4x64x64': (16, 4, 64 * 64),
    'cm_lsun256_32x3x256x256': (32, 3, 256 * 256),
    'n4_x1000': (1000, 1, 4),                 # sample boundaries inside a warp: 1 float4 per sample
    'n12_x333': (333, 3, 4),                  # 3 float4 per sample
}

# per-sample inputs each mode reads: every combination of them, alone and together
_VARIANTS = {X0: [(), ('thr',), ('coef_dev',), ('thr', 'coef_dev')],
             EPS: [(), ('t_dev',), ('coef_dev',), ('t_dev', 'coef_dev')],
             DIV: [(), ('t_dev',), ('coef_dev',), ('t_dev', 'coef_dev')],
             NONE: [(), ('coef_dev',)]}


def _update_cases():
    cases = []
    for nh in range(5):
        for mode in (X0, EPS, DIV, NONE):
            var = _VARIANTS[mode]
            cases.append(dict(name=f'nhist{nh}_{("x0", "eps", "div", "none")[mode]}', nh=nh, mode=mode, per_sample=var[nh % len(var)],
                              xs=mode in (EPS, DIV) and nh % 2 == 1, out_m=nh != 2, u8=nh == 3))
    # the aliasing and NULL outputs of the samplers' own calls
    cases += [
        # last step of a multistep run that records no trajectory: x is updated in place and the byte image written (solvers.py:261)
        dict(name='inplace_eps_u8', nh=3, mode=EPS, out_x='xb', out_m=True, u8=True),
        # DPM++ with dynamic thresholding, in place (solvers.py:374)
        dict(name='inplace_x0_thr', nh=2, mode=X0, per_sample=('thr',), out_x='xb', out_m=True),
        # AMED second leg: per-sample divisor and coefficients, xs set, in place (solvers_amed.py:165, 280)
        dict(name='inplace_amed', nh=1, mode=EPS, xs=True, per_sample=('t_dev', 'coef_dev'), out_x='xb', out_m=False),
        # dynamic_thresholding_fn: xb and D are the same tensor, no out_x (solver_utils.py:132)
        dict(name='dynamic_thresholding_fn', nh=0, mode=X0, per_sample=('thr',), out_x=None, out_m=True, D_is_xb=True),
        # d_cur only, no out_x (solvers.py:373, :414)
        dict(name='eps_out_m_only', nh=0, mode=EPS, out_x=None, out_m=True),
        # classifier-free guidance combine over the two halves of one [2B] eps buffer (ldm_net.py:154, :161)
        dict(name='cfg_halves', nh=2, mode=NONE, per_sample=('coef_dev',), hist_halves=True, out_m=False),
        dict(name='cfg_halves_scalar', nh=2, mode=NONE, hist_halves=True, out_m=False),
    ]
    for c in cases:
        c.setdefault('per_sample', ())
        c.setdefault('xs', False)
        c.setdefault('out_x', 'new')
        c.setdefault('u8', False)
        c.setdefault('D_is_xb', False)
        c.setdefault('hist_halves', False)
    return cases


def _per_sample(B, mult, period, g):
    """fp32 [B] > 0 whose binary exponents ((b * mult) % period - period // 2) jump by at least min(mult, period - mult) between
    neighbouring samples: a value read for the wrong sample b is off by a large factor."""
    e = (torch.arange(B) * mult) % period - period // 2
    return ((torch.rand(B, generator=g) + 0.5) * 2.0 ** e).float()


def _grid_sweeps(B, n):
    """Grid-stride sweeps of update_kernel: ds_update_launch caps the grid at 16 CTAs of 256 threads per SM, one float4 per thread."""
    n4 = B * n // 4
    sms = torch.cuda.get_device_properties(dev()).multi_processor_count
    grid = min(-(-n4 // 256), 16 * sms)
    return -(-n4 // (grid * 256))


def _update_case(lib, case, B, Cc, HW, inp, g):
    """Runs one case; returns a list of failure messages."""
    n = Cc * HW
    nh, mode = case['nh'], case['mode']
    ps = case['per_sample']
    fails = []
    # coefficients: scalars of either sign, or per-sample vectors [6][B]
    coef = [float(np.float32(s * m)) for s, m in zip(np.where(torch.rand(6, generator=g).numpy() < 0.5, -1.0, 1.0),
                                                      0.25 + 3.75 * torch.rand(6, generator=g).numpy())]
    coef = coef[:2 + nh] + [0.0] * (4 - nh)
    coef_dev = None
    if 'coef_dev' in ps:
        coef_dev = torch.stack([_per_sample(B, 7, 13, g) * (1 if k % 2 else -1) for k in range(6)]).to(dev()).contiguous()
        coef_dev[2 + nh:] = 0
    t = float(np.float32(0.5 + 79.5 * torch.rand(1, generator=g).item()))
    t_dev = (_per_sample(B, 5, 11, g) * 4).to(dev()) if 't_dev' in ps else None
    thr = (_per_sample(B, 4, 9, g) * 2).to(dev()) if 'thr' in ps else None
    # inputs
    xb_buf = Guarded(B * n, torch.float32, float('nan'))
    xb = xb_buf.body.view(B, n)
    xb.copy_(inp['xb'])
    xb0 = xb.clone()
    xs = inp['xs'] if case['xs'] else None
    D = xb if case['D_is_xb'] else (inp['D'] if mode in (X0, EPS) else None)
    hist = [inp['F'][:B], inp['F'][B:]][:nh] if case['hist_halves'] else inp['h'][:nh]
    # outputs
    ox = Guarded(B * n, torch.float32, float('nan')) if case['out_x'] == 'new' else None
    out_x = ox.body.view(B, n) if ox is not None else (xb if case['out_x'] == 'xb' else None)
    om = Guarded(B * n, torch.float32, float('nan')) if case['out_m'] else None
    u8 = Guarded(B * n, torch.uint8, 0xFF) if case['u8'] else None

    l = lib.load()
    hp = (C.c_void_p * 4)(*[h.data_ptr() for h in hist], *([None] * (4 - nh)))
    cf = (C.c_float * 6)(*coef)
    args = (ptr(xb), ptr(xs), ptr(D), hp, nh, ptr(thr), mode, t, ptr(t_dev), cf, ptr(coef_dev), n, B, stream())
    out_m = om.body if om is not None else None
    if u8 is not None:
        lib.check(l.ds_solver_update_u8(ptr(out_x), ptr(out_m), u8.body.data_ptr(), Cc, HW, *args), 'ds_solver_update_u8')
    else:
        lib.check(l.ds_solver_update(ptr(out_x), ptr(out_m), *args), 'ds_solver_update')

    # m0 in fp32 on the CPU (IEEE division; the library is built without fast math)
    xb_np = xb0.cpu().numpy()
    xs_np = xs.cpu().numpy() if xs is not None else xb_np
    tt = t_dev.cpu().numpy()[:, None] if t_dev is not None else np.float32(t)
    if mode == X0:
        m = xb_np if case['D_is_xb'] else D.cpu().numpy()
        if thr is not None:
            s = thr.cpu().numpy()[:, None]
            m = np.minimum(np.maximum(m, -s), s) / s
    elif mode == EPS:
        m = (xs_np - D.cpu().numpy()) / tt
    elif mode == DIV:
        m = xs_np / tt
    else:
        m = np.zeros_like(xb_np)
    m = torch.from_numpy(np.ascontiguousarray(m, dtype=np.float32)).to(dev())
    if out_m is not None:
        if not om.guards_intact():
            fails.append('out_m guard overwritten')
        if not torch.equal(bits(out_m.view(B, n)), bits(m)):
            bad = (bits(out_m.view(B, n)) != bits(m)).nonzero()[:3].tolist()
            fails.append(f'out_m differs from fp32 m0 at [sample, element] {bad}')
    # out_x against the float64 combination of the same fp32 operands
    cd = coef_dev.double() if coef_dev is not None else torch.tensor(coef, dtype=torch.float64, device=dev())[:, None].expand(6, B)
    terms = [xb0, m] + list(hist)
    ref = torch.zeros(B, n, dtype=torch.float64, device=dev())
    mag = torch.zeros_like(ref)
    for k, v in enumerate(terms):
        tk = cd[k][:, None] * v.double()
        ref += tk
        mag += tk.abs()
    if out_x is not None:
        if ox is not None and not ox.guards_intact():
            fails.append('out_x guard overwritten')
        if not xb_buf.guards_intact():
            fails.append('xb guard overwritten')
        if not torch.isfinite(out_x).all():
            fails.append('out_x has elements that were not written')
        err = (out_x.double() - ref).abs()
        bound = (nh + 2) * U * (1 + 2 ** -20) * mag
        if not bool((err <= bound).all()):
            w = ((err - bound) / mag.clamp_min(1e-300)).argmax().item()
            fails.append(f'out_x exceeds the roundoff bound at sample {w // n} element {w % n}: err {err.view(-1)[w].item():.3e} '
                         f'bound {bound.view(-1)[w].item():.3e}')
        case['ratio'] = (err / bound.clamp_min(1e-300)).max().item()
        if mode == NONE and nh == 0 and not torch.equal(out_x, cd[0].float()[:, None] * xb0):
            fails.append('mode NONE without history: out_x must be the fp32 product cx * xb itself (c0 * 0 adds nothing)')
    if u8 is not None:
        if not u8.guards_intact():
            fails.append('out_u8 guard overwritten')
        want = u8_expr(out_x).view(B, Cc, HW).permute(0, 2, 1).reshape(-1)
        if not torch.equal(u8.body, want):
            fails.append(f'out_u8 differs from the torch expression at {(u8.body != want).sum().item()} bytes')
        if out_x is not None and case['out_x'] == 'new':
            # header: out_x may be NULL when only the byte image is wanted; the bytes must not depend on it
            u8b = Guarded(B * n, torch.uint8, 0x00)
            lib.check(l.ds_solver_update_u8(None, None, u8b.body.data_ptr(), Cc, HW, *args), 'ds_solver_update_u8')
            if not (u8b.guards_intact() and torch.equal(u8b.body, u8.body)):
                fails.append('out_u8 without out_x differs from out_u8 with it')
    return [f'{case["name"]}: {f}' for f in fails]


def test_fused_update_at_sampler_shapes(lib):
    """At every shape of SHAPES, one after the other (failures are collected per shape and case):
    all 20 update_kernel<NH, MODE> instantiations (nhist 0..4 x mode X0 / EPS / DIV / NONE) with every per-sample input their mode
    reads (thr, t_dev, coef_dev: alone and together), xs NULL and set, out_m NULL and set, the uint8 epilogue, and the aliasing the
    samplers use (out_x is xb; xb is D with out_x NULL; history in the two halves of one buffer).  Per-sample coefficients, divisors
    and thresholds of neighbouring samples differ by a factor of 5 or more, so a wrong sample index b in any sweep shows up.

    out_m (m0 = D | clamp(D, -s, s) / s | (xs - D) / t | xs / t | 0) is one fp32 subtraction and one IEEE division per element: it
    must equal fp32 numpy bit for bit.
    out_x = cx*xb + c0*m0 + sum_k c_k*h_k is nhist + 2 roundings in fp32 (a product, then nhist + 1 additions or FMAs).  Each rounding
    adds at most u = 2^-24 of a partial sum bounded by sum |c_k * term_k|, so |out_x - exact| <= (nhist + 2) * u * sum |c_k * term_k|
    (to first order; the factor 1 + 2^-20 covers the rest), with `exact` the float64 combination of the same fp32 operands.
    out_u8 must equal the torch expression of sample.py:311 on the out_x the kernel wrote, byte for byte."""
    fails = []
    for shape in SHAPES:
        fails += _update_shape(lib, shape)
    assert not fails, '\n'.join(fails)


def _update_shape(lib, shape):
    """Every case of _update_cases() at one sampler shape; returns the failure messages."""
    B, Cc, HW = SHAPES[shape]
    n = Cc * HW
    torch.cuda.reset_peak_memory_stats()
    sweeps = _grid_sweeps(B, n)
    if shape.startswith('cm_lsun256'):
        assert sweeps >= 3, f'the largest case must run at least three grid-stride sweeps, got {sweeps}'
    g = torch.Generator().manual_seed(list(SHAPES).index(shape))
    inp = dict(xb=(torch.randn(B, n, generator=g) * 20).to(dev()), xs=(torch.randn(B, n, generator=g) * 20 + 0.5).to(dev()),
               D=(torch.randn(B, n, generator=g) * 3).to(dev()), h=[torch.randn(B, n, generator=g).to(dev()) for _ in range(4)],
               F=torch.randn(2 * B, n, generator=g).to(dev()))
    fails, worst = [], 0.0
    cases = _update_cases()
    t0 = time.time()
    for case in cases:
        fails += _update_case(lib, case, B, Cc, HW, inp, g)
        worst = max(worst, case.get('ratio', 0.0))
    torch.cuda.synchronize()
    print(f'update {shape}: {len(cases)} cases, {sweeps} grid sweep(s), worst |err| / bound {worst:.3f}, {time.time() - t0:.1f} s, '
          f'peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')
    return [f'{shape} {f}' for f in fails]


# --------------------------------------------------------------------------------------------- dynamic threshold
Q = 0.995
# 10240 / 10241: static / opt-in shared memory; 51200 / 51201: opt-in shared / global memory (ds_threshold_launch); 201: fp32(q) * 200
# is the integer 199; the rest are the samplers' rows (CIFAR-10, ImageNet-64 / FFHQ, SD latents, 256x256 pixel models)
LENGTHS = [(1, 2), (2, 2), (201, 2), (1000, 2), (3072, 2), (10240, 2), (10241, 2), (12288, 2), (16384, 2), (51200, 2), (51201, 2),
           (196608, 2), (12288, 32)]
KINDS = ['normal', 'ties_span', 'ties_end_at_k', 'all_equal', 'zeros', 'subnormal', 'shared_top_bytes', 'huge']


def _rank(n, q=Q):
    """torch.quantile's rank arithmetic for an fp32 input: rank = fp32(q) * (n - 1) in fp32; below / above = floor / ceil; weight =
    rank - below in fp32."""
    rank = np.float32(np.float32(q) * np.float32(n - 1))
    below = int(np.floor(rank))
    return below, int(np.ceil(rank)), np.float32(rank - np.float32(below))


def _q_exact(n, j):
    """An fp32 q with fp32(q * (n - 1)) == j: the quantile at q is then the j-th order statistic itself (weight 0)."""
    if n == 1:
        return np.float32(Q)
    q = np.float32(j / (n - 1))
    for _ in range(64):
        r = np.float32(q * np.float32(n - 1))
        if r == j:
            return q
        q = np.nextafter(q, np.float32(np.inf) if r < j else np.float32(-np.inf))
    raise AssertionError(f'no fp32 q gives rank {j} of {n}')


def _threshold_rows(n, reps, seed):
    """reps rows of each kind, as fp32 [rows, n] (random signs, so zeros include -0.0; shuffled).  The kinds put these keys at the
    selected rank k = floor(fp32(q) * (n - 1)):
      normal           |N(0, 1)| times a per-row scale in [1e-3, 1e3]
      ties_span        equal keys over ranks k-2 .. k+3: ranks k and k+1 tie (the `s_less + eq > k + 1` branch)
      ties_end_at_k    equal keys over ranks k-3 .. k, a larger key at k+1 (the `s_min_above` branch)
      all_equal        one value everywhere
      zeros            +-0 up to rank k, a positive key at k+1
      subnormal        only subnormal keys
      shared_top_bytes keys 0x3F80xxxx: the first two radix passes see one bin, the last two decide
      huge             magnitudes log-uniform in [1e-30, 1e30]"""
    g = np.random.default_rng(seed)
    k = _rank(n)[0]
    kinds = KINDS if n >= 8 else ['normal', 'all_equal', 'zeros', 'huge']
    rows = []
    for _ in range(reps):
        for kind in kinds:
            a = np.sort(np.abs(g.standard_normal(n)).astype(np.float32) * np.float32(10.0 ** g.uniform(-3, 3)))
            if kind == 'ties_span':
                a[k - 2:k + 4] = a[k - 2]
                assert a[k] == a[k + 1]
            elif kind == 'ties_end_at_k':
                a[k - 3:k + 1] = a[k - 3]
                assert a[k - 1] == a[k] < a[k + 1]
            elif kind == 'all_equal':
                a[:] = np.float32(0.37)
            elif kind == 'zeros':
                a[:k + 1] = 0
            elif kind == 'subnormal':
                a = np.sort(g.integers(1, 1 << 23, n).astype(np.uint32)).view(np.float32)
            elif kind == 'shared_top_bytes':
                a = np.sort(g.integers(0x3F800000, 0x3F810000, n).astype(np.uint32)).view(np.float32)
            elif kind == 'huge':
                a = np.sort((10.0 ** g.uniform(-30, 30, n)).astype(np.float32))
            sign = np.where(g.random(n) < 0.5, np.float32(-1), np.float32(1))
            rows.append((a * sign)[g.permutation(n)])
    return np.stack(rows)


def _threshold(lib, x, q, floor):
    B, n = x.shape
    out = Guarded(B, torch.float32, float('nan'))
    lib.check(lib.load().ds_dyn_threshold(x.data_ptr(), out.body.data_ptr(), B, n, float(q), float(floor), stream()), 'ds_dyn_threshold')
    torch.cuda.synchronize()
    assert out.guards_intact(), 'thr written outside [0, B)'
    got = out.body.cpu().numpy()
    assert np.isfinite(got).all(), 'a thr entry was not written'
    return got


@pytest.mark.parametrize('n,reps', LENGTHS, ids=[f'n{n}-B{r * (len(KINDS) if n >= 8 else 4)}' for n, r in LENGTHS])
def test_dyn_threshold_launch_paths_and_rank_edges(lib, n, reps):
    """ds_dyn_threshold (exact radix select + torch's lerp) on all three launch paths, with rows built to hit each branch.

    Reference: |x| sorted in fp32; lo, hi = the order statistics at torch.quantile's fp32 floor / ceil of the rank, w its fp32 weight.
      * with floor 0 (the raw quantile): within 1 fp32 ulp of the float64 lerp lo + w (hi - lo), and exactly lo when w = 0 or lo = hi.
        In these rows hi - lo is exact (Sterbenz: hi <= 2 lo, or lo = 0), and the kernel's lerp rounds once (FMA), i.e. <= 1/2 ulp.
      * each order statistic exactly: with an fp32 q' whose rank fp32(q' (n - 1)) is exactly k (then k + 1), the output is the k-th
        (k+1-th) smallest |x| itself, bit for bit.
      * within 1 ulp of torch.quantile(|x|, q) on the GPU;
      * with floor 1: exactly max(raw quantile, 1)."""
    rows = _threshold_rows(n, reps, seed=n)
    x = torch.from_numpy(rows).to(dev())
    k, above, w = _rank(n)
    srt = np.sort(np.abs(rows), axis=1)
    lo, hi = srt[:, k], srt[:, above]
    got = _threshold(lib, x, Q, 0.0)
    lerp = lo.astype(np.float64) + float(w) * (hi.astype(np.float64) - lo.astype(np.float64))
    ulp = np.spacing(np.abs(lerp).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - lerp)
    print(f'dyn threshold n={n} B={rows.shape[0]} k={k} w={w}: max |err| / ulp {np.max(err / ulp):.3f}')
    assert (err <= ulp).all(), f'rows {np.nonzero(err > ulp)[0].tolist()}: got {got[err > ulp]} want {lerp[err > ulp]}'
    exact = (w == 0) | (lo == hi)
    assert np.array_equal(got[exact].view(np.uint32), lo[exact].view(np.uint32))
    for j in (k, k + 1):
        if j < n:
            gj = _threshold(lib, x, _q_exact(n, j), 0.0)
            assert np.array_equal(gj.view(np.uint32), srt[:, j].view(np.uint32)), \
                f'order statistic {j}: rows {np.nonzero(gj != srt[:, j])[0].tolist()}'
    tq = torch.quantile(x.abs(), Q, dim=1).cpu().numpy()
    tol = np.spacing(np.maximum(np.abs(tq), np.abs(got)))
    assert (np.abs(got - tq) <= tol).all(), f'vs torch.quantile: rows {np.nonzero(np.abs(got - tq) > tol)[0].tolist()}'
    got1 = _threshold(lib, x, Q, 1.0)
    assert np.array_equal(got1, np.maximum(got, np.float32(1.0)))


# --------------------------------------------------------------------------------------------- GITS cost matrix
GITS = [(61, 16, 12288), (21, 4, 3072), (2, 3, 1332), (5, 2, 20)]     # bench.py's ImageNet-64 / CIFAR-10 teachers; N = 2; n % 1024 != 0


def _teacher(N, B, n, g):
    """An Euler-like teacher trajectory on the EDM schedule (80 -> 0.002, rho 7): traj[i+1] = traj[i] + (t[i+1] - t[i]) eps[i] plus
    a small perturbation, so the near-diagonal jump errors are small as in a real run."""
    idx = torch.arange(N, dtype=torch.float64)
    t = ((80 ** (1 / 7) + idx / max(N - 1, 1) * (0.002 ** (1 / 7) - 80 ** (1 / 7))) ** 7).float()
    base = torch.randn(B, n, generator=g)
    eps = torch.stack([base + 0.1 * torch.randn(B, n, generator=g) for _ in range(N - 1)])
    traj = [torch.randn(B, n, generator=g) * 80]
    for i in range(N - 1):
        traj.append(traj[-1] + (t[i + 1] - t[i]) * eps[i] + 1e-3 * torch.randn(B, n, generator=g))
    return torch.stack(traj).to(dev()), eps.to(dev()), t.to(dev())


@pytest.mark.parametrize('N,B,n', GITS)
def test_gits_cost_sums_within_their_roundoff_bounds(lib, N, B, n):
    """ds_gits_cost: every (i < j, b) entry, each of its four sums against a bound derived from the kernel's arithmetic; entries
    i >= j stay NaN.

    Per element, with exact (float64) X = traj[i] + h eps[i] (h = fp32(t[j] - t[i])), H = |h eps[i]|, R = traj[j], c = traj[N-1],
    b0 = traj[0], E = X - R, Ec = c - X, Cb = c - b0, T = |X| + H + |E|, Tc = |X| + H + |Ec|, and u = 2^-24:
      xs = fp32(X) costs <= u (|X| + H) (one FMA, or a product and a sum); e = fp32(xs - R) then differs from E by <= u T, and
      ca = fp32(c - xs) from Ec by <= u Tc; cb = fp32(c - b0) from Cb by <= u |Cb|.  Each thread adds 4 elements in fp32 (<= 4
      roundings of partial sums bounded by the sum of |terms|) and accumulates those partials in fp64 (~2^-53: negligible).  So
        |S1 - sum |E||        <= u sum (|X| + H + 4 |E|)
        |S2 - sum E^2|        <= u sum (6 |E| + u T) T            (2 |E| u T + (u T)^2 + 4 u E^2)
        |S3 - sum Ec^2|       <= u sum (6 |Ec| + u Tc) Tc
        |S4 - sum Ec Cb|      <= u sum (5 |Ec| + Tc) |Cb|         (|Ec| u |Cb| + |Cb| u Tc + 4 u |Ec Cb|)
    to first order; the test allows twice that.  The bound of an entry scales with its own terms: the small near-diagonal entries,
    which the DP compares, are held to their own size, not to the largest entry of the matrix."""
    g = torch.Generator().manual_seed(N * 1000 + n)
    traj, eps, t = _teacher(N, B, n, g)
    torch.cuda.reset_peak_memory_stats()
    out = Guarded(N * N * B * 4, torch.float64, float('nan'))
    lib.check(lib.load().ds_gits_cost(traj.data_ptr(), eps.data_ptr(), t.data_ptr(), out.body.data_ptr(), N, B, n, stream()), 'ds_gits_cost')
    torch.cuda.synchronize()
    assert out.guards_intact()
    got = out.body.view(N, N, B, 4)
    upper = torch.ones(N, N, dtype=torch.bool, device=dev()).triu(1)
    assert torch.isnan(got[~upper]).all(), 'an entry with i >= j was written'
    assert torch.isfinite(got[upper]).all(), 'an entry with i < j was not written'
    c, b0 = traj[N - 1].double(), traj[0].double()
    Cb = c - b0
    worst = [0.0] * 4
    fails = []
    for i in range(N - 1):
        for j0 in range(i + 1, N, 16):
            j1 = min(j0 + 16, N)
            h = (t[j0:j1] - t[i]).double()[:, None, None]                 # fp32 subtraction, as the kernel
            HE = h * eps[i].double()                                        # exact: a product of two fp32 values
            X = traj[i].double() + HE
            E = X - traj[j0:j1].double()
            Ec = c - X
            T = X.abs() + HE.abs() + E.abs()
            Tc = X.abs() + HE.abs() + Ec.abs()
            ref = [E.abs().sum(-1), (E * E).sum(-1), (Ec * Ec).sum(-1), (Ec * Cb).sum(-1)]
            bound = [2 * U * (X.abs() + HE.abs() + 4 * E.abs()).sum(-1), 2 * U * ((6 * E.abs() + U * T) * T).sum(-1),
                     2 * U * ((6 * Ec.abs() + U * Tc) * Tc).sum(-1), 2 * U * ((5 * Ec.abs() + Tc) * Cb.abs()).sum(-1)]
            for s in range(4):
                err = (got[i, j0:j1, :, s] - ref[s]).abs()
                worst[s] = max(worst[s], (err / bound[s]).max().item())
                if not bool((err <= bound[s]).all()):
                    jj, bb = divmod((err - bound[s]).argmax().item(), B)
                    fails.append(f'sum {s + 1} at (i={i}, j={j0 + jj}, b={bb}): got {got[i, j0 + jj, bb, s].item():.9e} '
                                 f'want {ref[s][jj, bb].item():.9e}, bound {bound[s][jj, bb].item():.3e}')
    print(f'gits cost N={N} B={B} n={n}: worst |err| / bound per sum {", ".join(f"{w:.3f}" for w in worst)}; '
          f'peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')
    assert not fails, '\n'.join(fails[:20])

"""GroupNorm end to end (GPU): every statistics source and apply kernel against float64 GroupNorm, at every GroupNorm shape the
compiled plans launch and at the branch edges of the kernels.

The shapes are harvested on the host from the ops of the plans of tests/plan_digest.py (the tiny interpreter variants and the five
benchmarked plans), the full-size Consistency-Models LSUN-256 plan and the VQ-f4 decode plan, and keyed on what selects a code path.
Every case runs on synthetic data whose groups mix four kinds of input: zero mean, per-channel offsets of both signs, groups offset
to mean / std = 1, 4, 16, 64 and 256, and near-constant groups (every value c or one fp32 ulp away, c = 1 or 100: the true variance is
below eps).  The reference is torch's group_norm in float64, then the adaptive scale / shift, SiLU and the resample; the un-normalised
(raw) outputs are compared bit for bit with a torch emulation of the kernels' roundings.  Every output buffer has 0xFF guard bytes
before and after it and is itself pre-filled with 0xFF (NaN in fp32, fp16 and e4m3): the guards must survive and every element must
be written with a finite value.

Error bounds, per (sample, group), with scale = max(1, max |y|, max |(x - mean) a|) over the group:
  * mean / std <= 16: 2e-5 x scale (4e-5 for the f8 operand image: TOL_F8_SUM), the bound of the kernel unit tests.
  * mean / std = r > 16: both statistics sources add fp32 partial sums in fp64, and the sums they produce are held to the bound of
    the plan replay (tests/test_gpu_plan_ops.py): |d sum x| <= 16 u sqrt(n sum x^2), |d sum x^2| <= 16 u sum x^2 (u = 2^-24, the
    1e-6 there).  var = sum x^2 / n - mean^2 then errs by at most 16 u (mean^2 + var) + 2 |mean| 16 u sqrt(mean^2 + var)
    <= 48 u var (1 + r^2), which moves the normalised value by a relative 24 u (1 + r^2): K_OFFSET = 24.
  * near-constant groups (var < eps, so a = gamma' / sqrt(eps)): the fp32 fold b' = b - mean a rounds by u |mean a|, the fp32 mean by
    u |mean|, the fp32 partial sums lose at most one ulp (2u |mean|) of the mean, and a variance estimate the cancellation makes wrong
    moves (x - mean) a by at most 8 u |mean| a (x and mean lie within two ulps of each other): K_CONST = 12, times u |mean| max |a|.
"""
import collections
import functools
import os
import sys
import time
import zlib
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

from diff_sampler_b200 import _cstructs as S

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

U = 2.0 ** -24
EPS = 1e-6
TOL_ACT = 2e-5
TOL_F8_SUM = 4e-5               # tests/test_gpu_plan_ops.py: hi + lo8 of the f8 operand image carries 2^-15 of |v|
R_EXACT_LIMIT = 16.0            # up to this mean / std the plain bound holds
K_OFFSET = 24                   # see the module docstring
K_CONST = 12
OFFSET_RATIOS = (1.0, 4.0, 16.0, 64.0, 256.0)
CONST_LEVELS = (1.0, 100.0)
KINDS = ['zero', 'chan'] + [('offset', r) for r in OFFSET_RATIOS] + [('const', c) for c in CONST_LEVELS]
GUARD = 4096                    # guard bytes before and after every output
MAX_ELEMS = 1 << 26             # per case: inputs beyond this run at batch 1 only

RESULTS = collections.Counter()                 # (kernel, fmt) -> cases run
PEAK = [0]                                      # largest peak device memory of one apply case


class StatsKey(NamedTuple):
    C0: int
    C1: int
    HW: int
    groups: int


class FinalizeKey(NamedTuple):
    C0: int
    C1: int
    groups: int
    unit0: int                  # 0: from fp64 sums (no partials); 4 quads / 2 pairs
    unit1: int                  # 0 without a second source
    slabs: int
    HW: int
    coef: bool
    ada: str                    # 'none', 'shared' (stride 0) or 'per-sample'


class ApplyKey(NamedTuple):
    C0: int
    C1: int
    H: int
    W: int
    groups: int
    resample: int
    fmt: int
    nplanes: int
    silu: int
    ada: str
    act: bool
    raw: bool
    rawf: bool
    stat: str                   # 'sums', 'coef' or 'none'


def _seed(key, B):
    return zlib.crc32(f'{key} B{B}'.encode())


def _ada_kind(d):
    return 'none' if not d.ada else ('shared' if int(d.ada_stride) == 0 else 'per-sample')


# --------------------------------------------------------------------------------------------- the harvest (host only)
def _plans():
    import plan_digest
    for gen in (plan_digest._edm_variants(), plan_digest._small_variants(), plan_digest._benchmarked()):
        for name, pl, _ in gen:
            yield name, pl
    from diff_sampler_b200 import cm_net, plan as planner
    spec, params = cm_net.convert(cm_net.init_state_dict(None, seed=0))
    for f8 in (False, True):
        wb, info = planner.pack_weights(spec, params, f8=f8)
        yield f'cm/lsun256/f8={int(f8)}', planner.compile_plan(spec, wb, info, 2, 1, 0, npass=3, f8=f8)
    from diff_sampler_b200 import vae_plan
    import vq_ref as VQ
    P, _ = VQ.make_params('vq_f4')
    mods, meta = vae_plan.vae_structure(P)
    yield 'vq/vq_f4', vae_plan.compile_vae_plan(mods, meta, vae_plan.pack_vae_weights(mods, meta, P), 1, 64, quantize=True)


@functools.lru_cache(maxsize=None)
def harvest():
    """{'stats' | 'finalize' | 'apply': sorted distinct keys} over the GroupNorm ops of every harvested plan."""
    out = {'stats': set(), 'finalize': set(), 'apply': set()}
    for _, pl in _plans():
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            if op.type == S.DS_OP_GN_STATS:
                d = op.u.gn_stats
                out['stats'].add(StatsKey(d.C0, d.C1, d.HW, d.groups))
            elif op.type == S.DS_OP_GN_FINALIZE:
                d = op.u.gn_finalize
                q = bool(d.quads0)
                out['finalize'].add(FinalizeKey(d.C0, d.C1, d.groups, (2 if d.unit0 == 2 else 4) if q else 0,
                                                (2 if d.unit1 == 2 else 4) if q and d.C1 else 0, d.slabs_per_sample if q else 0,
                                                d.HW if d.coef else d.slabs_per_sample * 32, bool(d.coef), _ada_kind(d)))
            elif op.type == S.DS_OP_GN_APPLY:
                d = op.u.gn_apply
                out['apply'].add(ApplyKey(d.C0, d.C1, d.H, d.W, d.groups, d.resample, d.fmt, d.nplanes, d.silu, _ada_kind(d),
                                          bool(d.out_act), bool(d.out_raw), bool(d.out_raw_f32),
                                          'sums' if d.sums else ('coef' if d.coef else 'none')))
    return {k: sorted(v) for k, v in out.items()}


# the branches of the kernels the harvest does not reach (or reaches only by chance)
EXTRA_APPLY = [
    # (key, batches)
    (ApplyKey(192, 0, 16, 16, 32, 0, 0, 2, 1, 'none', True, True, False, 'coef'), (1, 3)),     # v3: rows = 10, the last unit partial
    (ApplyKey(64, 0, 4, 4, 16, 0, 0, 2, 1, 'none', True, False, False, 'coef'), (1, 3)),       # npix = 16 < rows = 32
    (ApplyKey(64, 0, 4, 4, 16, 0, 0, 2, 1, 'none', True, False, False, 'sums'), (1, 3)),
    (ApplyKey(8, 0, 8, 8, 2, 0, 0, 2, 1, 'per-sample', True, True, False, 'coef'), (1, 3)),    # C = 8: one column, 256 rows
    (ApplyKey(8, 0, 8, 8, 2, 1, 0, 2, 1, 'none', True, True, True, 'sums'), (1, 3)),
    (ApplyKey(2048, 0, 8, 8, 32, 0, 0, 2, 1, 'per-sample', True, False, False, 'coef'), (1, 3)),  # the widest v3
    (ApplyKey(2048, 0, 8, 8, 32, 0, 1, 2, 1, 'none', True, False, False, 'coef'), (3,)),
    (ApplyKey(2056, 0, 8, 8, 8, 0, 0, 2, 1, 'none', True, True, False, 'sums'), (1, 3)),        # nc8 = 257, 257-channel groups
    (ApplyKey(2560, 0, 8, 8, 32, 0, 0, 2, 1, 'shared', True, False, False, 'sums'), (1, 3)),    # 80-channel groups
    (ApplyKey(2048, 2048, 4, 4, 32, 0, 0, 2, 1, 'none', True, False, True, 'sums'), (1, 3)),    # nc8 = 512
    (ApplyKey(2560, 1536, 4, 4, 32, 2, 0, 2, 1, 'none', True, True, False, 'sums'), (1,)),
    (ApplyKey(192, 0, 16, 16, 32, 1, 0, 2, 1, 'per-sample', True, True, True, 'sums'), (1, 3)),  # 6-channel groups
    (ApplyKey(320, 0, 16, 16, 32, 0, 0, 2, 1, 'none', True, True, False, 'coef'), (1, 3)),      # 10-channel groups
    (ApplyKey(576, 0, 8, 8, 32, 2, 1, 2, 1, 'per-sample', True, True, False, 'sums'), (1, 3)),   # 18-channel groups
    (ApplyKey(1344, 0, 8, 8, 32, 0, 1, 2, 1, 'none', True, True, False, 'coef'), (1, 3)),       # 42-channel groups
    (ApplyKey(128, 64, 8, 8, 32, 0, 0, 1, 1, 'none', True, True, False, 'coef'), (1, 3)),       # one fp16 plane
    (ApplyKey(128, 64, 8, 8, 32, 1, 0, 1, 0, 'none', True, True, True, 'sums'), (1, 3)),
    (ApplyKey(128, 0, 8, 8, 32, 3, 0, 1, 1, 'none', True, True, True, 'sums'), (1, 3)),         # space-to-depth, normalised
    (ApplyKey(96, 0, 6, 10, 32, 3, 0, 2, 0, 'none', False, True, True, 'none'), (1, 3)),
    (ApplyKey(256, 0, 16, 16, 32, 0, 0, 2, 1, 'none', True, False, False, 'coef'), (131,)),      # total_chunks > the persistent grid
]
EXTRA_STATS = [StatsKey(128, 0, 4096, 32), StatsKey(64, 64, 1024, 32), StatsKey(2056, 0, 64, 8), StatsKey(192, 144, 64, 28),
               StatsKey(12, 0, 256, 2), StatsKey(4096, 0, 16, 64)]
EXTRA_FINALIZE = [
    FinalizeKey(256, 0, 32, 4, 0, 8, 256, True, 'per-sample'),          # SG > 1
    FinalizeKey(2048, 0, 32, 4, 0, 2, 64, True, 'none'),                # cols = 1024: SG = 1
    FinalizeKey(1024, 1024, 32, 2, 2, 2, 64, False, 'none'),            # cols = 2048
    FinalizeKey(192, 0, 32, 2, 0, 1, 32, True, 'shared'),               # slabs_per_sample = 1
    FinalizeKey(192, 144, 28, 2, 4, 4, 128, True, 'none'),              # 12-channel groups straddling the sources, mixed units
    FinalizeKey(128, 64, 32, 2, 2, 4, 128, True, 'per-sample'),
    FinalizeKey(320, 0, 32, 0, 0, 0, 256, True, 'per-sample'),         # the table from the separate pass's sums
    FinalizeKey(256, 128, 32, 0, 0, 0, 64, True, 'shared'),
]


def _apply_cases():
    cases = []
    for key in harvest()['apply']:
        big = key.H * key.W * (key.C0 + key.C1) * (4 if key.resample == 2 else 1) * 3 > MAX_ELEMS
        cases += [(key, 1)] + ([] if big else [(key, 3)])
    for key, batches in EXTRA_APPLY:
        cases += [(key, b) for b in batches]
    return cases


def _kernel_of(key):
    if key.resample:
        return f'apply<{key.resample}>'
    return 'v3' if key.stat == 'coef' and key.C0 + key.C1 <= 2048 else 'v2'


def test_harvest_covers_every_gn_path():
    """The harvested GroupNorm ops (plus the extra cases) reach every apply kernel, both operand formats, both plane counts, both
    statistics sources (pairs and quads), a group straddling a virtual concat, every optional output and both adaptive-scale kinds."""
    h = harvest()
    assert h['stats'] and h['finalize'] and h['apply']
    keys = h['apply'] + [k for k, _ in EXTRA_APPLY]
    assert {_kernel_of(k) for k in keys} == {'v2', 'v3', 'apply<1>', 'apply<2>', 'apply<3>'}
    assert {_kernel_of(k) for k in h['apply']} >= {'v2', 'v3', 'apply<1>', 'apply<2>', 'apply<3>'}
    assert {k.fmt for k in h['apply']} == {0, 1} and {k.nplanes for k in keys} == {1, 2}
    assert {k.stat for k in h['apply']} == {'sums', 'coef', 'none'}
    assert all(any(getattr(k, o) for k in h['apply']) for o in ('act', 'raw', 'rawf'))
    assert {k.ada for k in keys} == {'none', 'shared', 'per-sample'}
    fin = h['finalize']
    assert {k.unit0 for k in fin} == {2, 4} and h['stats']                      # epilogue pairs and quads; the separate pass
    straddle = [k for k in fin if k.unit0 and k.C1 and k.C0 % ((k.C0 + k.C1) // k.groups)]
    assert straddle, 'no virtual concat with a group across the two sources'
    assert any(k.coef for k in fin) and any(not k.coef for k in fin)
    print(f"harvest: {len(h['stats'])} gn_stats, {len(fin)} gn_finalize, {len(h['apply'])} gn_apply keys "
          f"({len(_apply_cases())} apply cases with the extras)")


# --------------------------------------------------------------------------------------------- device helpers
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


class Guarded:
    """nbytes of device memory pre-filled with 0xFF, between two 0xFF guard regions."""

    def __init__(self, nbytes, fill=255):
        self.n = nbytes
        self.buf = torch.full((nbytes + 2 * GUARD,), 255, dtype=torch.uint8, device=dev())
        self.body = self.buf[GUARD:GUARD + nbytes]
        if fill != 255:
            self.body.fill_(fill)

    @property
    def ptr(self):
        return self.body.data_ptr()

    def guards_intact(self):
        return bool((self.buf[:GUARD] == 255).all()) and bool((self.buf[GUARD + self.n:] == 255).all())


def _group_kinds(B, G):
    """Kind of every (sample, group): the KINDS list dealt round-robin, shifted by one per sample."""
    return [[KINDS[(n + g) % len(KINDS)] for g in range(G)] for n in range(B)]


def make_input(B, npix, C, G, kinds, gen):
    """fp32 [B, npix, C] whose group g of sample n follows kinds[n][g]."""
    cpg = C // G
    x = torch.randn(B, npix, C, generator=gen, dtype=torch.float64)
    for n in range(B):
        for g in range(G):
            k = kinds[n][g]
            sl = slice(g * cpg, (g + 1) * cpg)
            if k == 'zero':
                continue
            if k == 'chan':
                s = torch.rand(cpg, generator=gen, dtype=torch.float64) * 1.5 + 0.5
                o = (torch.rand(cpg, generator=gen, dtype=torch.float64) * 6 - 3)
                x[n, :, sl] = x[n, :, sl] * s + o
            elif k[0] == 'offset':
                std = float(torch.rand(1, generator=gen)) * 1.5 + 0.5
                sign = 1.0 if (n + g) % 2 == 0 else -1.0
                x[n, :, sl] = x[n, :, sl] * std + sign * k[1] * std
    x = x.float()
    for n in range(B):
        for g in range(G):
            k = kinds[n][g]
            if k != 'zero' and k != 'chan' and k[0] == 'const':
                c = torch.tensor(k[1], dtype=torch.float32)
                step = torch.randint(-1, 2, (npix, cpg), generator=gen)
                v = torch.where(step > 0, torch.nextafter(c, torch.tensor(float('inf'))),
                                torch.where(step < 0, torch.nextafter(c, torch.tensor(float('-inf'))), c))
                x[n, :, g * cpg:(g + 1) * cpg] = v
    return x.to(dev())


def exact_sums(x, G):
    """float64 {sum, sum of squares} [B, G, 2] of fp32 x [B, npix, C]."""
    B, npix, C = x.shape
    xd = x.double().reshape(B, npix, G, C // G)
    return torch.stack([xd.sum(dim=(1, 3)), (xd * xd).sum(dim=(1, 3))], dim=-1)


def sums_bound(want, n):
    """The plan replay's gn_stats bound: 16 u of sqrt(n sum x^2) for the sums, of sum x^2 for the squares."""
    q = want[..., 1].clamp_min(0)
    return torch.stack([(q * n).sqrt(), q], dim=-1) * 1e-6 + 1e-12


def resample_f32(v, rs):
    """fp32 [B, H, W, C] -> what the kernel stores as the raw value, bit for bit (pool: 0.25 e_t added in the kernel's t order)."""
    if rs == 1:
        acc = torch.zeros_like(v[:, 0::2, 0::2])
        for t in range(4):
            acc = acc + 0.25 * v[:, (t >> 1)::2, (t & 1)::2]
        return acc
    if rs == 2:
        return v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return v


def resample_f64(v, rs):
    if rs == 1:
        return (v[:, 0::2, 0::2] + v[:, 0::2, 1::2] + v[:, 1::2, 0::2] + v[:, 1::2, 1::2]) / 4
    return resample_f32(v, rs)


def s2d(v):
    """[B, H, W, C] -> the space-to-depth phase layout [B, H/2, W/2, 4 C] (phase = 2 (h & 1) + (w & 1))."""
    B, H, W, C = v.shape
    return v.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4 * C)


def planes_bytes(v, nplanes):
    hi = v.half()
    parts = [hi.reshape(-1).view(torch.uint8)]
    if nplanes == 2:
        parts.append((v - hi.float()).half().reshape(-1).view(torch.uint8))
    return torch.cat(parts)


def f8_image_bytes(v):
    """The f8 operand image as the kernels store it: fp16 of v 2^6 clamped to +-65504; e4m3 of the fp32 of the exact v 2^13 - hi 2^7,
    clamped to +-448; e4m3 of hi 2^-4 (an fp16 product) clamped to +-448."""
    e4 = torch.float8_e4m3fn
    hi = (v * 2.0 ** S.DS_F8_SH_A16).clamp(-65504.0, 65504.0).half()
    lo8 = (v.double() * 2.0 ** S.DS_F8_SH_LO8 - hi.double() * 2.0 ** (S.DS_F8_SH_LO8 - S.DS_F8_SH_A16)).float().clamp(-448.0, 448.0).to(e4)
    hi8 = (hi.float() * 2.0 ** (S.DS_F8_SH_HI8 - S.DS_F8_SH_A16)).half().float().clamp(-448.0, 448.0).to(e4)
    return torch.cat([hi.reshape(-1).view(torch.uint8), lo8.reshape(-1).view(torch.uint8), hi8.reshape(-1).view(torch.uint8)])


def decode_values(body, key, n):
    """(float64 values of the n elements, all finite) of an act / raw buffer: planes summed, the f8 image decoded to hi + lo8."""
    if key.fmt == 1:
        hi = body[:2 * n].view(torch.float16).double() / 2.0 ** S.DS_F8_SH_A16
        lo8 = body[2 * n:3 * n].view(torch.float8_e4m3fn).double() / 2.0 ** S.DS_F8_SH_LO8
        hi8 = body[3 * n:4 * n].view(torch.float8_e4m3fn).double()
        return hi + lo8, bool(torch.isfinite(hi).all() and torch.isfinite(lo8).all() and torch.isfinite(hi8).all())
    h = body.view(torch.float16)
    v = h[:n].double()
    if key.nplanes == 2:
        v = v + h[n:2 * n].double()
    return v, bool(torch.isfinite(v).all())


def gn_reference(x, key, B, gamma, beta, ada):
    """float64 (y, (x - mean) a, exact mean, var) of fp32 x [B, H, W, C] at the input resolution."""
    C, G = key.C0 + key.C1, key.groups
    xd = x.double()
    y = F.group_norm(xd.permute(0, 3, 1, 2), G, gamma.double(), beta.double(), eps=EPS).permute(0, 2, 3, 1)
    xg = xd.reshape(B, -1, G, C // G)
    mu, var = xg.mean(dim=(1, 3)), xg.var(dim=(1, 3), unbiased=False)
    a = (1.0 / torch.sqrt(var + EPS)).repeat_interleave(C // G, dim=1) * gamma.double()[None]
    if ada is not None:
        sc, sh = ada[:, :C].double() + 1, ada[:, C:2 * C].double()
        y = y * sc[:, None, None, :] + sh[:, None, None, :]
        a = a * sc
    pre = (xd - mu.repeat_interleave(C // G, dim=1)[:, None, None, :]) * a[:, None, None, :]
    if key.silu:
        y = F.silu(y)
    return y, pre, a, mu, var


def group_bounds(y, pre, a, mu, var, G, base):
    """Per-(sample, group) error bound (see the module docstring) and the ratio r = |mean| / std."""
    B, C = a.shape
    scale = torch.maximum(y.abs(), pre.abs()).reshape(B, -1, G, C // G).amax(dim=(1, 3)).clamp_min(1.0)
    r = mu.abs() / var.sqrt().clamp_min(1e-300)
    const = var < EPS
    amax = a.abs().reshape(B, G, C // G).amax(dim=2)
    bound = base * scale + torch.where(r > R_EXACT_LIMIT, K_OFFSET * U * (1 + r * r) * scale, torch.zeros_like(r))
    bound = torch.where(const, base * scale + K_CONST * U * mu.abs() * amax, bound)
    return bound, r, const, scale


# --------------------------------------------------------------------------------------------- launches
def run_stats(lib, x0, x1, key, B):
    """gn_stats into a zeroed fp64 buffer between guards; returns the sums [B, G, 2]."""
    G = key.groups
    buf = Guarded(B * G * 2 * 8, fill=0)
    lib.op_launch(S.GnStatsDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if x1 is not None else 0, C0=key.C0, C1=key.C1, HW=key.HW,
                                B=B, groups=G, sums=buf.ptr))
    torch.cuda.synchronize()
    assert buf.guards_intact(), 'gn_stats wrote outside its sums'
    return buf.body.view(torch.float64).reshape(B, G, 2).clone()


def run_finalize(lib, sums, C0, C1, G, B, HW, gamma, beta, ada, ada_stride, quads=None, units=(4, 4), slabs=0):
    """gn_finalize; returns (sums [B, G, 2], coef [B, C, 2] or None).  quads: (partials0, partials1 or None) -> fold them into the
    (pre-filled) sums; else the coefficient table from `sums`."""
    C = C0 + C1
    sbuf = Guarded(B * G * 2 * 8)
    if quads is None:
        sbuf.body.view(torch.float64).copy_(sums.reshape(-1))
    cbuf = Guarded(B * C * 2 * 4) if gamma is not None else None
    d = S.GnFinalizeDesc(quads0=quads[0].data_ptr() if quads else 0, quads1=quads[1].data_ptr() if quads and quads[1] is not None else 0,
                         C0=C0, C1=C1, slabs_per_sample=slabs, B=B, groups=G, unit0=units[0], unit1=units[1], sums=sbuf.ptr)
    if gamma is not None:
        d.gamma, d.beta, d.eps, d.HW, d.coef = gamma.data_ptr(), beta.data_ptr(), EPS, HW, cbuf.ptr
        d.ada, d.ada_stride = (ada.data_ptr(), ada_stride) if ada is not None else (0, 0)
    lib.op_launch(d)
    torch.cuda.synchronize()
    assert sbuf.guards_intact() and (cbuf is None or cbuf.guards_intact()), 'gn_finalize wrote outside its outputs'
    got = sbuf.body.view(torch.float64).reshape(B, G, 2).clone()
    coef = None
    if cbuf is not None:
        coef = cbuf.body.view(torch.float32).reshape(B, C, 2).clone()
        assert torch.isfinite(coef).all(), 'coefficient table not written or not finite'
    return got, coef


def coef_reference(sums, C, G, HW, gamma, beta, ada):
    """float64 {a, b - mean a} from fp64 sums, with rstd rounded to fp32 as the kernel keeps it."""
    cnt = (C // G) * HW
    mu = sums[..., 0] / cnt
    var = (sums[..., 1] / cnt - mu * mu).clamp_min(0)
    rstd = (1.0 / torch.sqrt(var + EPS)).float().double().repeat_interleave(C // G, dim=1)
    a = rstd * gamma.double()[None]
    b = beta.double()[None].expand_as(a)
    if ada is not None:
        sc = ada[:, :C].double() + 1
        a, b = a * sc, b * sc + ada[:, C:2 * C].double()
    return a, b - mu.repeat_interleave(C // G, dim=1) * a


def apply_out_elems(key, B):
    C = key.C0 + key.C1
    if key.resample == 1:
        return B * (key.H // 2) * (key.W // 2) * C
    if key.resample == 2:
        return B * key.H * key.W * 4 * C
    return B * key.H * key.W * C


def run_apply(lib, key, B, x0, x1, gamma, beta, ada, ada_stride, sums=None, coef=None):
    """gn_apply with guarded, 0xFF-filled outputs; returns {name: body bytes} of the outputs the key asks for."""
    n = apply_out_elems(key, B)
    op_bytes = 4 * n if key.fmt == 1 else 2 * key.nplanes * n
    outs = {name: Guarded(nb) for name, want, nb in (('act', key.act, op_bytes), ('raw', key.raw, op_bytes), ('rawf', key.rawf, 4 * n)) if want}
    C = key.C0 + key.C1
    lib.op_launch(S.GnApplyDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if x1 is not None else 0, C0=key.C0, C1=key.C1, H=key.H, W=key.W,
                                B=B, groups=key.groups, sums=sums.data_ptr() if sums is not None else 0,
                                coef=coef.data_ptr() if coef is not None else 0,
                                gamma=gamma.data_ptr() if gamma is not None else 0, beta=beta.data_ptr() if beta is not None else 0,
                                eps=EPS, silu=key.silu, ada=ada.data_ptr() if ada is not None else 0, ada_stride=ada_stride,
                                resample=key.resample, nplanes=key.nplanes, fmt=key.fmt,
                                out_act=outs['act'].ptr if 'act' in outs else 0, out_raw=outs['raw'].ptr if 'raw' in outs else 0,
                                out_raw_f32=outs['rawf'].ptr if 'rawf' in outs else 0))
    torch.cuda.synchronize()
    for name, g in outs.items():
        assert g.guards_intact(), f'{name}: a store outside the output'
    return {name: g.body.clone() for name, g in outs.items()}


def _params(C, B, ada_kind, gen):
    gamma = torch.randn(C, generator=gen).to(dev())
    beta = torch.randn(C, generator=gen).to(dev())
    if ada_kind == 'none':
        return gamma, beta, None, 0, None
    rows = 1 if ada_kind == 'shared' else B
    stride = 0 if ada_kind == 'shared' else 2 * C + 8
    ada = (torch.randn(rows, max(stride, 2 * C), generator=gen) * 0.3).to(dev())
    ada_full = ada[:, :2 * C].expand(B, 2 * C) if rows == 1 else ada[:, :2 * C]
    return gamma, beta, ada, stride, ada_full


# --------------------------------------------------------------------------------------------- gn_stats
@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('key', harvest()['stats'] + EXTRA_STATS, ids=str)
def test_gn_stats(lib, key, B):
    gen = torch.Generator().manual_seed(_seed(key, B))
    C, G = key.C0 + key.C1, key.groups
    x = make_input(B, key.HW, C, G, _group_kinds(B, G), gen)
    x0 = x[..., :key.C0].contiguous()
    x1 = x[..., key.C0:].contiguous() if key.C1 else None
    got = run_stats(lib, x0, x1, key, B)
    want = exact_sums(x, G)
    ratio = ((got - want).abs() / sums_bound(want, (C // G) * key.HW)).max().item()
    RESULTS[('gn_stats', 'f64')] += 1
    print(f'gn_stats {key} B{B}: worst error / bound {ratio:.3f}')
    assert ratio <= 1.0


# --------------------------------------------------------------------------------------------- gn_finalize
@pytest.mark.gpu
@pytest.mark.parametrize('key', harvest()['finalize'] + EXTRA_FINALIZE, ids=str)
def test_gn_finalize(lib, key):
    """The fold of fp32 slab partials (pairs / quads, one or two sources) into fp64 sums, and the coefficient table, at batch 1 and 3."""
    for B in (1, 3):
        gen = torch.Generator().manual_seed(_seed(key, B))
        C, G = key.C0 + key.C1, key.groups
        x = make_input(B, key.HW, C, G, _group_kinds(B, G), gen)
        gamma, beta, ada, stride, ada_full = _params(C, B, key.ada, gen)
        if key.unit0:
            parts = []
            for lo, hi, u in ((0, key.C0, key.unit0), (key.C0, C, key.unit1)):
                if hi == lo:
                    parts.append(None)
                    continue
                xs = x[..., lo:hi].double().reshape(B * key.slabs, 32, (hi - lo) // u, u)
                parts.append(torch.stack([xs.sum(dim=(1, 3)), (xs * xs).sum(dim=(1, 3))], dim=-1).float().contiguous())
            fold = []
            for p, u, cc in ((parts[0], key.unit0, key.C0), (parts[1], key.unit1, key.C1)):
                if p is not None:
                    fold.append(p.double().reshape(B, key.slabs, cc // u, 2).sum(dim=1).repeat_interleave(u, dim=1) / u)
            per_ch = torch.cat(fold, dim=1)                                      # [B, C, 2]: each unit's share spread over its channels
            want = per_ch.reshape(B, G, C // G, 2).sum(dim=2)
            got, coef = run_finalize(lib, None, key.C0, key.C1, G, B, key.HW, gamma if key.coef else None, beta, ada, stride,
                                     quads=parts, units=(key.unit0, key.unit1 or 4), slabs=key.slabs)
            e = (got - want).abs().max().item()
            assert e <= 1e-12 * max(1.0, want.abs().max().item()), ('fold', B, e)
        else:
            got = exact_sums(x, G)
            _, coef = run_finalize(lib, got, key.C0, key.C1, G, B, key.HW, gamma, beta, ada, stride)
        if coef is not None:
            a, b = coef_reference(got, C, G, key.HW, gamma, beta, ada_full)
            ea, eb = (coef[..., 0].double() - a).abs().max().item(), (coef[..., 1].double() - b).abs().max().item()
            assert ea <= 1e-5 * a.abs().max().item() and eb <= 1e-5 * max(1.0, b.abs().max().item()), (B, ea, eb)
        RESULTS[('gn_finalize', 'quads' if key.unit0 == 4 else ('pairs' if key.unit0 else 'sums'))] += 1


# --------------------------------------------------------------------------------------------- gn_apply
def _check_apply(key, B, outs, x, y_out, pre_out, bnd_args, G):
    """act within the per-group bound, raw / rawf bit-exact; returns the worst act error / bound."""
    C = key.C0 + key.C1
    n = apply_out_elems(key, B)
    Ho, Wo = (key.H // 2, key.W // 2) if key.resample == 1 else ((2 * key.H, 2 * key.W) if key.resample == 2 else (key.H, key.W))
    xr = resample_f32(x, key.resample)
    lay = s2d if key.resample == 3 else (lambda v: v)
    worst = 0.0
    if 'act' in outs:
        v, finite = decode_values(outs['act'], key, n)
        assert finite, 'act: an element not written or not finite'
        v = v.reshape(B, Ho // 2, Wo // 2, 4 * C) if key.resample == 3 else v.reshape(B, Ho, Wo, C)
        if key.resample == 3:
            v = v.reshape(B, Ho // 2, Wo // 2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Ho, Wo, C)
        err = (v - y_out).abs().reshape(B, -1, G, C // G).amax(dim=(1, 3))
        # one fp16 plane: the hi plane alone rounds y to 2^-11 relative
        base = TOL_F8_SUM if key.fmt == 1 else (TOL_ACT if key.nplanes == 2 else TOL_ACT + 2.0 ** -11)
        y_, pre_, a_, mu_, var_ = bnd_args
        bound = group_bounds(y_, pre_, a_, mu_, var_, G, base)[0]
        worst = (err / bound).max().item()
        assert worst <= 1.0, f'act: worst (sample, group) error / bound {worst:.3f}'
    want_raw = lay(xr)
    if 'raw' in outs:
        want = f8_image_bytes(want_raw) if key.fmt == 1 else planes_bytes(want_raw, key.nplanes)
        assert torch.equal(outs['raw'], want), 'raw operand differs from the emulation'
    if 'rawf' in outs:
        assert torch.equal(outs['rawf'].view(torch.float32), want_raw.reshape(-1)), 'raw fp32 differs from the emulation'
    return worst


def _apply_case(lib, key, B, seed):
    gen = torch.Generator().manual_seed(seed)
    C, G = key.C0 + key.C1, key.groups
    norm = key.stat != 'none'
    if norm:
        x = make_input(B, key.H * key.W, C, G, _group_kinds(B, G), gen)
    else:                                       # no groups to speak of: per-channel offsets of both signs
        x = make_input(B, key.H * key.W, C, 1, [['chan']] * B, gen)
    x = x.reshape(B, key.H, key.W, C)
    x0 = x[..., :key.C0].contiguous()
    x1 = x[..., key.C0:].contiguous() if key.C1 else None
    gamma, beta, ada, stride, ada_full = _params(C, B, key.ada, gen) if norm else (None, None, None, 0, None)
    sums = coef = None
    if norm:
        sums = run_stats(lib, x0, x1, StatsKey(key.C0, key.C1, key.H * key.W, G), B)
        if key.stat == 'coef' or (key.resample == 0 and C <= 2048):
            _, coef = run_finalize(lib, sums, key.C0, key.C1, G, B, key.H * key.W, gamma, beta, ada, stride)
    y_out = pre_out = bnd = None
    if key.act:
        y, pre, a, mu, var = gn_reference(x, key, B, gamma, beta, ada_full)
        y_out, pre_out = resample_f64(y, key.resample), resample_f64(pre, key.resample)
        bnd = (y_out, pre_out, a, mu, var)
    runs = []
    if not norm:
        runs.append(('none', run_apply(lib, key, B, x0, x1, None, None, None, 0)))
    else:
        if key.stat == 'sums' or key.resample == 0:
            runs.append(('sums', run_apply(lib, key, B, x0, x1, gamma, beta, ada, stride, sums=sums)))
        if coef is not None and key.resample == 0 and C <= 2048:
            runs.append(('coef', run_apply(lib, key, B, x0, x1, gamma, beta, ada, stride, coef=coef)))
    worst = 0.0
    for stat, outs in runs:
        worst = max(worst, _check_apply(key, B, outs, x, y_out, pre_out, bnd, G))
        kern = _kernel_of(key._replace(stat=stat))
        RESULTS[(kern, f'fmt{key.fmt}/p{key.nplanes}')] += 1
    if len(runs) == 2:                      # v2 (sums) and v3 (coefficient table): the same bytes
        for name in runs[0][1]:
            assert torch.equal(runs[0][1][name], runs[1][1][name]), f'{name}: v2 and v3 outputs differ'
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize('key,B', _apply_cases(), ids=lambda v: str(v) if isinstance(v, ApplyKey) else f'B{v}')
def test_gn_apply(lib, key, B):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    worst = _apply_case(lib, key, B, _seed(key, B))
    peak = torch.cuda.max_memory_allocated()
    PEAK[0] = max(PEAK[0], peak)
    print(f'gn_apply {key} B{B}: worst act error / bound {worst:.3f}, {time.time() - t0:.2f} s, peak {peak / 2 ** 30:.2f} GiB')


# --------------------------------------------------------------------------------------------- the mean / std sweep
@pytest.mark.gpu
def test_statistics_sources_against_offset_groups(lib):
    """C = 128 in 4-channel groups at 32 x 32, batch 2: offset groups at each mean / std, with statistics from the separate pass,
    from the GEMM epilogue's quads and from its pairs (real conv_gemm launches with st_quads / st_unit), normalised by v2 (sums) and
    v3 (coefficient table).  Prints the worst error / scale per source and mean / std; near-constant groups from the separate pass."""
    from diff_sampler_b200 import gemm_desc as G_
    gen = torch.Generator().manual_seed(77)
    B, H, W, C, G, Cin = 2, 32, 32, 128, 32, 64
    key = ApplyKey(C, 0, H, W, G, 0, 0, 2, 0, 'none', True, False, False, 'sums')
    gamma = torch.randn(C, generator=gen).to(dev())
    beta = torch.randn(C, generator=gen).to(dev())
    kinds = [[KINDS[(n + g) % len(KINDS)] for g in range(G)] for n in range(B)]
    table = collections.defaultdict(float)
    xin = torch.randn(B, Cin, H, W, generator=gen).to(dev())
    w = (torch.randn(C, Cin, 3, 3, generator=gen) / (3 * Cin ** 0.5)).to(dev())
    conv = F.conv2d(xin.double(), w.double(), padding=1)
    sd = conv.reshape(B, G, -1).std(dim=2).mean(dim=0)                                   # per group
    r_of = torch.tensor([OFFSET_RATIOS[g % len(OFFSET_RATIOS)] * (1 if g % 2 == 0 else -1) for g in range(G)], device=dev(), dtype=torch.float64)
    bias = (r_of * sd).repeat_interleave(C // G).float()
    for source in ('stats', 'quads', 'pairs'):
        if source == 'stats':
            x = make_input(B, H * W, C, G, kinds, gen).reshape(B, H, W, C)
            sums = run_stats(lib, x, None, StatsKey(C, 0, H * W, G), B)
        else:
            unit = 4 if source == 'quads' else 2
            xa = G_.split_planes(xin.permute(0, 2, 3, 1).contiguous())
            out = torch.zeros(B * H * W, C, device=dev())
            part = torch.full((B * H * W // 32, C // unit, 2), float('nan'), device=dev())
            d, _ = G_.conv_gemm(xa.data_ptr(), B, H, W, Cin, G_.pack_conv_weight(w.cpu()).to(dev()).data_ptr(), C, taps=9, npass=3,
                                out_f32=out.data_ptr(), bias=bias.data_ptr())
            d.st_quads, d.st_unit = part.data_ptr(), unit
            lib.op_launch(d)
            torch.cuda.synchronize()
            x = out.reshape(B, H, W, C)
            sums, _ = run_finalize(lib, None, C, 0, G, B, H * W, None, None, None, 0, quads=(part, None), units=(unit, 4), slabs=H * W // 32)
        _, coef = run_finalize(lib, sums, C, 0, G, B, H * W, gamma, beta, None, 0)
        y, pre, a, mu, var = gn_reference(x, key, B, gamma, beta, None)
        bound, r, const, scale = group_bounds(y, pre, a, mu, var, G, TOL_ACT)
        outs = [run_apply(lib, key, B, x, None, gamma, beta, None, 0, sums=sums)['act'],
                run_apply(lib, key, B, x, None, gamma, beta, None, 0, coef=coef)['act']]
        assert torch.equal(outs[0], outs[1]), f'{source}: v2 and v3 outputs differ'
        v, finite = decode_values(outs[0], key, B * H * W * C)
        assert finite
        err = (v.reshape(B, H, W, C) - y).abs().reshape(B, -1, G, C // G).amax(dim=(1, 3))
        ratio = err / bound
        for n in range(B):
            for g in range(G):
                k = kinds[n][g] if source == 'stats' else ('offset', OFFSET_RATIOS[g % len(OFFSET_RATIOS)])
                if k in ('zero', 'chan'):
                    k = (k, 0.0)
                rr = float(r[n, g])
                cell = (source, k[0], k[1])
                table[cell] = max(table[cell], float(err[n, g] / scale[n, g]))
                table[cell + ('r',)] = max(table.get(cell + ('r',), 0.0), rr if not const[n, g] else 0.0)
                table[cell + ('ratio',)] = max(table.get(cell + ('ratio',), 0.0), float(ratio[n, g]))
    print(f"\n{'source':7s} {'kind':7s} {'nominal':>8s} {'mean/std':>9s} {'err/scale':>10s} {'err/bound':>10s}")
    for cell in sorted(c for c in table if len(c) == 3):
        print(f'{cell[0]:7s} {cell[1]:7s} {cell[2]:8g} {table[cell + ("r",)]:9.1f} {table[cell]:10.3e} {table[cell + ("ratio",)]:10.3f}')
    bad = {c: table[c + ('ratio',)] for c in table if len(c) == 3 and table[c + ('ratio',)] > 1.0}
    assert not bad, bad


# --------------------------------------------------------------------------------------------- launcher contract
@pytest.mark.gpu
def test_launcher_rejects_what_its_kernels_get_wrong(lib):
    """Descriptors the GroupNorm kernels cannot run correctly are refused (rc -2, DsError) before any kernel runs, and nothing is written:
    the coefficient table with a resample, a normalised output without statistics, one-channel groups in gn_stats, pooling and
    space-to-depth over an odd height or width."""
    gen = torch.Generator().manual_seed(5)
    B, H, W, C = 2, 8, 8, 64
    x = torch.randn(B, H, W, C, generator=gen).to(dev())
    gamma, beta = torch.ones(C, device=dev()), torch.zeros(C, device=dev())
    sums = torch.zeros(B, 32, 2, dtype=torch.float64, device=dev())
    coef = torch.zeros(B, C, 2, device=dev())
    out = Guarded(2 * 2 * B * 4 * H * W * C)

    def apply_desc(**kw):
        base = dict(src0=x.data_ptr(), src1=0, C0=C, C1=0, H=H, W=W, B=B, groups=32, sums=0, coef=0, gamma=gamma.data_ptr(), beta=beta.data_ptr(),
                    eps=EPS, silu=1, ada=0, ada_stride=0, resample=0, nplanes=2, fmt=0, out_act=out.ptr, out_raw=0, out_raw_f32=0)
        base.update(kw)
        return S.GnApplyDesc(**base)
    bad = [('coef + pool', apply_desc(coef=coef.data_ptr(), resample=1)),
           ('coef + nearest x2', apply_desc(coef=coef.data_ptr(), resample=2)),
           ('act without statistics', apply_desc()),
           ('act without statistics, pool', apply_desc(resample=1)),
           ('pool, odd H', apply_desc(sums=sums.data_ptr(), resample=1, H=7, W=8)),
           ('pool, odd W', apply_desc(sums=sums.data_ptr(), resample=1, H=8, W=7))]
    for name, d in bad:
        with pytest.raises(lib.DsError):
            lib.op_launch(d)
    # space-to-depth over 7 rows: a stray store would land one output row past the buffer, which here still lies inside this
    # allocation (the whole 7 x 8 input's planes plus a guard region of more than one output row of every plane)
    Hs = 7
    xs = torch.randn(B, Hs, W, C, generator=gen).to(dev())
    plane = B * Hs * W * C
    s2d_out = Guarded(2 * (2 * plane + (W // 2) * 4 * C))
    with pytest.raises(lib.DsError):
        lib.op_launch(S.GnApplyDesc(src0=xs.data_ptr(), src1=0, C0=C, C1=0, H=Hs, W=W, B=B, groups=32, sums=0, coef=0, gamma=0, beta=0, eps=0.0,
                                    silu=0, ada=0, ada_stride=0, resample=3, nplanes=2, fmt=0, out_act=0, out_raw=s2d_out.ptr, out_raw_f32=0))
    st = Guarded(B * 64 * 2 * 8, fill=0)
    with pytest.raises(lib.DsError):
        lib.op_launch(S.GnStatsDesc(src0=x.data_ptr(), src1=0, C0=C, C1=0, HW=H * W, B=B, groups=64, sums=st.ptr))
    torch.cuda.synchronize()
    assert bool((out.buf == 255).all()) and bool((s2d_out.buf == 255).all()), 'a refused launch wrote its output'
    assert bool((st.body == 0).all()) and st.guards_intact()
    # the neighbours of the refused descriptors still run: two-channel groups, even sizes, the table at resample 0
    ok = Guarded(B * 32 * 2 * 8, fill=0)
    lib.op_launch(S.GnStatsDesc(src0=x.data_ptr(), src1=0, C0=C, C1=0, HW=H * W, B=B, groups=32, sums=ok.ptr))
    lib.op_launch(apply_desc(sums=ok.ptr, resample=1))
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gn_report():
    if not RESULTS:
        pytest.skip('no GroupNorm case of this module ran')
    print('\ncases per kernel and format')
    for (kern, fmt), n in sorted(RESULTS.items()):
        print(f'{kern:12s} {fmt:10s} {n:5d}')
    print(f'largest peak device memory of one apply case: {PEAK[0] / 2 ** 30:.2f} GiB')

"""Every op of the benchmarked plans, launched alone on the GPU on the activations the plan itself produced, against the float64
plan interpreter (oracle/plan_interp.py, pinned to the network oracles by tests/test_plan_interp.py).

For each op in plan order, on one live device arena: the spans the op stores to (tests/plan_spans.writes) are filled with 0xFF
(NaN in fp32, fp16, e4m3 and fp64), the arena is snapshotted and the interpreter runs the op on the snapshot in float64 on the GPU,
then the kernel runs on the live arena through _lib.op_launch.  Inside the spans an element the reference left NaN must still be
NaN (stray stores inside strided windows: head padding, ldo gaps, padded pitches), an element it wrote must be finite and within
the op class's tolerance; outside the spans arena and io slots must equal the snapshot byte for byte.  The pre-fill bytes then go
back wherever the op did not write, so the next op reads the GPU's own output and errors do not compound.

The EDM nets run at batch 11 (odd; the descriptors encode per-sample geometry, and the benchmark batch would not leave room for a
snapshot and the float64 temporaries on a shared card); SD-1.5 (16 contexts under guidance), its VAE decoder (batch 1) and the
CLIP-L text encoder (batch 2) run at the benchmark batch."""
import collections
import time

import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from oracle import plan_interp as PI
from plan_spans import reads_own_output, resolve, writes
from test_gpu_gemm_tiles import TOL_1P, TOL_EDM, TOL_PLANES, TOL_STATS, TOL_X3, bench_plan_weights, f8_model_tol

pytestmark = pytest.mark.gpu

WORKLOADS = ['cifar10', 'ffhq', 'imagenet64', 'sd15', 'sd_vae', 'clip_l']
EDM_BATCH = 11
EDM_SIGMA = 2.5
CHUNK = 1 << 28                  # bytes per chunk of the byte-for-byte comparison outside the spans

# f8 operand image (fp16 hi = v rounded at 2^-11 relative; lo8 = (v - hi) * 2^13 in e4m3, 3 mantissa bits): |v - hi| <= 2^-11 |v|
# and e4m3 rounds that residual to within 2^-4 of itself, so hi + lo8 carries |v| to 2^-15 = 3.05e-5 relative, plus half the
# smallest e4m3 subnormal (2^-10) over the 2^13 scale, 2^-23 absolute.  A raw (copied) value has no other error; a computed one
# adds its fp32 arithmetic, and the bound of the unit tests (test_groupnorm_apply_f8_layout, test_layernorm_geglu_f8_image),
# 4e-5 x max(1, max|v|), leaves ~1e-5 for it.  hi alone: 6e-4 (fp16), hi8: 2^-4 relative (e4m3), as those tests.
F8_LO_QUANTUM = 2.0 ** -15
F8_SUBNORMAL = 2.0 ** -23
TOL_F8_SUM = 4e-5
TOL_F8_HI, TOL_F8_HI8 = 6e-4, 0.07

# f8 GEMMs beyond K = 13824 (the SD-1.5 3x3 convolutions over 1920 and 2560 channels): f8_model_tol's 3e-5 was measured on the
# zero-mean operands of gemm_replay (2.1e-5 at K = 23040).  The plan's own activations are GroupNorm + SiLU outputs, mostly positive,
# so the hi x hi product's fp32 accumulation error (linear in K on H100, see f8_model_tol) adds up coherently: measured on an H100
# 80GB HBM3, 2.3e-5 at K = 17280 and 3.03e-5 at K = 23040 of max |output|.
K_F8_PLAN_LONG = 13824
TOL_F8_PLAN_LONG_K = 4e-5

RESULTS = {}                     # workload -> dict(rows=[...], skips=[...], seconds, peak)


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


def dev():
    return torch.device('cuda:0')


# --------------------------------------------------------------------------------------------- workloads and their io
def workload(name):
    """(plan, weight blob bytes, {io slot: host tensor}) with seeded inputs as tests/test_plan_interp.py builds them per plan kind."""
    g = torch.Generator().manual_seed(11)
    if name == 'clip_l':
        from diff_sampler_b200 import clip_plan
        from oracle import clip_oracle as CO
        P, cfg = CO.make_params('clip_l', seed=0)
        ccfg = clip_plan.clip_config(P)
        wb = clip_plan.pack_clip_weights(P, ccfg)
        B, T = 2, 77
        ids = torch.randint(0, cfg['vocab_size'], (B, T), generator=g)
        ids[:, 0] = 49406
        ids[0, 9:] = 49407
        pl = clip_plan.compile_clip_plan(ccfg, wb, B, T, num_heads=cfg['num_attention_heads'])
        return pl, wb.bytes(), {S.DS_IO_X: ids.to(torch.int32), S.DS_IO_D: torch.zeros(B, T, cfg['hidden_size'])}
    if name == 'sd15':
        pl, wb, cfg = bench_plan_weights(name)
        B, R, C = 8, cfg['img_resolution'], cfg['in_channels']
        return pl, wb, {S.DS_IO_X: torch.randn(B, C, R, R, generator=g), S.DS_IO_D: torch.zeros(2 * B, C, R, R),
                        S.DS_IO_SIGMA: torch.tensor([417.0]), S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 0.37, 0.0]]),
                        S.DS_IO_BOTTLENECK: torch.zeros(2 * B, 64), S.DS_IO_CTX: torch.randn(2 * B, 77, cfg['context_dim'], generator=g)}
    if name == 'sd_vae':
        pl, wb, cfg = bench_plan_weights(name)
        R, sf = 64, cfg['scale_factor']
        z = torch.randn(1, cfg['z_channels'], R, R, generator=g) * sf * 1.3
        up = R * cfg['upscale']
        return pl, wb, {S.DS_IO_X: z, S.DS_IO_D: torch.zeros(1, cfg['out_ch'], up, up), S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0 / sf, 0.0]])}
    pl, wb, cfg = bench_plan_weights(name, batch=EDM_BATCH)
    B, R, C, nl = EDM_BATCH, cfg['img_resolution'], cfg['img_channels'], cfg.get('label_dim', 0)
    lab = torch.eye(nl)[torch.randint(0, nl, (B,), generator=g)] if nl else None
    return pl, wb, {S.DS_IO_X: torch.randn(B, C, R, R, generator=g) * EDM_SIGMA, S.DS_IO_D: torch.zeros(B, C, R, R),
                    S.DS_IO_SIGMA: torch.tensor([EDM_SIGMA]), S.DS_IO_LABELS: lab, S.DS_IO_BOTTLENECK: torch.zeros(B, 64)}


# --------------------------------------------------------------------------------------------- span bytes as values
def _elements(span, raw):
    """raw: the span's bytes -> (fill pattern per element slot of the whole span, the slots as typed values; None for the f8 image)."""
    if span.fmt in ('f32', 'stats', 'nchw'):
        return raw.view(torch.int32) == -1, raw.view(torch.float32)
    if span.fmt == 'f64':
        return raw.view(torch.int64) == -1, raw.view(torch.float64)
    if span.fmt == 'zero':
        return raw == 255, raw
    if span.fmt == 'f16':
        return raw.view(torch.int16) == -1, raw.view(torch.float16)
    p = span.plane                                             # f8: one fp16 plane, then two e4m3 byte planes
    return torch.cat([raw[:2 * p].view(torch.int16) == -1, raw[2 * p:] == 255]), None


def _f16_values(span, raw):
    h = raw.view(torch.float16)
    n = h.numel() - span.plane if span.nplanes == 2 else h.numel()
    v = h[:n].double()
    if span.nplanes == 2:
        v = v + h[span.plane:span.plane + n].double()
    return v, n


def _f8_decode(span, raw):
    p = span.plane
    hi = raw[:2 * p].view(torch.float16).double() / 2.0 ** S.DS_F8_SH_A16
    lo8 = raw[2 * p:3 * p].view(torch.float8_e4m3fn).double() / 2.0 ** S.DS_F8_SH_LO8
    hi8 = raw[3 * p:].view(torch.float8_e4m3fn).double() / 2.0 ** S.DS_F8_SH_HI8
    return hi, lo8, hi8


def _unwritten_bytes(span, raw):
    """Byte mask of the element slots still holding the fill pattern."""
    pat, _ = _elements(span, raw)
    if span.fmt == 'f8':
        p = span.plane
        return torch.cat([pat[:p].repeat_interleave(2), pat[p:]])
    return pat.repeat_interleave(raw.numel() // pat.numel())


# --------------------------------------------------------------------------------------------- tolerances per op class
def _max(t):
    return t.abs().max().item() if t.numel() else 0.0


def _check_span(op, span, got, want, written, stored, spans, got_all, want_all):
    """(error, bound, ratio) of one span of op.  got / want: the span's bytes after the kernel / the interpreter; written: bool per
    value slot the comparison covers (what the reference wrote)."""
    t = op.type
    d = getattr(op.u, S.UNION_FIELD[t])

    def absdiff(g, w, m):
        return (g[m].double() - w[m].double()).abs()

    def bounded(e, b):
        e = _max(e) if torch.is_tensor(e) else e
        if e != e:                                             # NaN: never a pass
            return e, b, float('inf')
        return e, b, (e / b if b > 0 else (0.0 if e == 0 else float('inf')))

    if span.fmt == 'zero':
        return bounded(float((got != 0).sum().item()), 0.0)
    if span.fmt == 'f8':
        v = next(val for ref, fmt, val, idx in stored if ref == span.ref and fmt == 1)
        hi, lo8, hi8 = _f8_decode(span, got)
        m = written[:span.plane]
        v = v[m]
        hi, lo8, hi8 = hi[m], lo8[m], hi8[m]
        mag = _max(v)
        raw_copy = t == S.DS_OP_GN_APPLY and span.ref == int(d.out_raw)
        b_sum = F8_LO_QUANTUM * mag + F8_SUBNORMAL if raw_copy else TOL_F8_SUM * max(1.0, mag)
        e_sum = _max(hi + lo8 - v)
        # the fp16 plane alone and the e4m3 copy of it (the operand of the lo x hi8 pass) have their own, coarser bounds
        if _max(hi - v) > TOL_F8_HI * max(1.0, mag) or not _max((hi8 - hi).abs() / hi.abs().clamp_min(2.0 ** -8)) <= TOL_F8_HI8:
            return e_sum, b_sum, float('inf')
        return bounded(e_sum, b_sum)
    if span.fmt == 'f16':
        g, n = _f16_values(span, got)
        w, _ = _f16_values(span, want)
        m = written[:n]
    else:
        _, g = _elements(span, got)
        _, w = _elements(span, want)
        m = written
    e = absdiff(g, w, m)
    wm = w[m].double()
    if t == S.DS_OP_GEMM:
        from diff_sampler_b200.gemm_replay import cfg_of
        from test_gpu_gemm_tiles import contraction
        cfg = cfg_of(d)
        tol = f8_model_tol(cfg) if cfg.f8 else (TOL_X3 if cfg.npass == 3 else TOL_1P)
        if cfg.f8 and contraction(cfg) > K_F8_PLAN_LONG:
            tol = TOL_F8_PLAN_LONG_K
        scale = max(_max(_values(s, wa).nan_to_num(0.0)) for s, wa in zip(spans, want_all) if s.fmt in ('f32', 'f16', 'nchw'))
        if span.fmt == 'f32':
            return bounded(e, tol * scale)
        if span.fmt == 'f16':
            return bounded(e, (TOL_PLANES if span.nplanes == 2 else 1e-3) * scale)
        if span.fmt == 'nchw':
            return bounded(e, (TOL_EDM if int(d.edm_out) == 1 else tol) * scale)
        # statistics partials: against sums of the kernel's own fp32 output of this launch (test_gpu_gemm_tiles.py does the same)
        k32 = next(i for i, s in enumerate(spans) if s.fmt == 'f32')
        y = got_all[k32].view(torch.float32)
        M, N, ldo, u = int(d.m_valid), int(d.n_valid), int(d.ldo), span.plane
        y = torch.as_strided(y, (M, N), (ldo, 1)).double().reshape(M // 32, 32, N // u, u)
        ref = torch.stack([y.sum(dim=(1, 3)), (y * y).sum(dim=(1, 3))], dim=-1).reshape(-1)
        return bounded((g.double() - ref).abs(), TOL_STATS * max(1.0, _max(ref)))
    if t == S.DS_OP_GN_APPLY:
        if span.ref == int(d.out_act):
            return bounded(e, 2e-5 * max(1.0, _max(wm)))
        return bounded(e, 1e-5 if span.fmt == 'f16' else 1e-6)
    if t == S.DS_OP_GN_STATS:
        # fp32 partial sums of a few pixels per thread, added in fp64: ~8 fp32 ulps of sum |x| (<= sqrt(count * sum x^2)) and of sum x^2
        C, G = int(d.C0) + int(d.C1), int(d.groups)
        q = w.double().reshape(-1, 2)[:, 1].clamp_min(0)
        bnd = torch.stack([(q * (C // G) * int(d.HW)).sqrt(), q], dim=1).reshape(-1) * 1e-6 + 1e-12
        return bounded(((g.double() - w.double()).abs() / bnd).max().item(), 1.0)
    if t == S.DS_OP_GN_FINALIZE:
        if span.fmt == 'f64':                                  # the same fp32 partials added in another order, in fp64
            return bounded(e, 1e-12 * max(1.0, _max(wm)))
        a_g, a_w = g.view(-1, 2)[:, 0].double(), w.view(-1, 2)[:, 0].double()
        b_g, b_w = g.view(-1, 2)[:, 1].double(), w.view(-1, 2)[:, 1].double()
        ea, eb = _max(a_g - a_w), _max(b_g - b_w)
        ba, bb = 1e-5 * _max(a_w), 1e-5 * max(1.0, _max(b_w))
        return (ea, ba, ea / ba) if ea / ba >= eb / bb else (eb, bb, eb / bb)
    if t == S.DS_OP_ATTN:
        return bounded(e, 2e-5 * max(1.0, _max(wm)))
    if t == S.DS_OP_SOFTMAX:
        return bounded(e, 2e-6)
    if t == S.DS_OP_POSEMB:
        if span.ref == int(d.coef):
            r = (e / w[m].double().abs().clamp_min(1e-3))
            return bounded(r, 1e-6)
        return bounded(e, 2e-6 if int(d.mode) == 0 else 2e-4)
    if t in (S.DS_OP_LAYERNORM, S.DS_OP_GEGLU):
        return bounded(e, 2e-5)
    if t == S.DS_OP_EMBED:
        return bounded(e, 1e-6)
    return bounded(e, 1e-5)                                    # linear, prep_input, chanmean


def _values(span, raw):
    """float64 value per element of the span: planes summed, the f8 image decoded to hi + lo8."""
    if span.fmt == 'f16':
        return _f16_values(span, raw)[0]
    if span.fmt == 'f8':
        hi, lo8, _ = _f8_decode(span, raw)
        return hi + lo8
    return _elements(span, raw)[1].double()


# --------------------------------------------------------------------------------------------- the replay
def shape_of(op):
    d = getattr(op.u, S.UNION_FIELD[op.type])
    t = op.type
    if t == S.DS_OP_GEMM:
        f = ('f8' if d.f8 else f'x{d.npass}') + f' BN{d.BN}'
        if d.a_mode == 0:
            return f'conv{d.taps} {d.conv_H}x{d.conv_W} K{int(d.b_dims[0])} N{d.n_valid} {f}'
        return f'rows z{d.num_z}/{d.nh} {d.m_valid}x{d.n_valid}x{d.cpb * 64} {f}'
    if t == S.DS_OP_ATTN:
        return f'B{d.B} h{d.nh} L{d.L} Lk{d.Lk}' + (' causal' if d.causal else '') + f' vt{d.vt_pitch}'
    if t == S.DS_OP_SOFTMAX:
        return f'{d.rows}x{d.L} pitch {d.pitch_in or d.L}/{d.pitch_out or d.L}'
    if t in (S.DS_OP_GN_APPLY, S.DS_OP_GN_STATS):
        extra = f' rs{d.resample} fmt{d.fmt}' if t == S.DS_OP_GN_APPLY else ''
        return f'B{d.B} {getattr(d, "H", "")}{"x" if t == S.DS_OP_GN_APPLY else ""}{getattr(d, "W", d.HW if t == S.DS_OP_GN_STATS else "")} C{d.C0}+{d.C1} G{d.groups}' + extra
    if t == S.DS_OP_GN_FINALIZE:
        return f'B{d.B} C{d.C0}+{d.C1} G{d.groups}' + (' quads' if d.quads0 else '') + (' coef' if d.coef else '')
    if t in (S.DS_OP_LAYERNORM, S.DS_OP_GEGLU):
        return f'{d.rows}x{getattr(d, "C", None) or getattr(d, "I", None)} fmt{d.fmt}' + (f' mode{d.mode}' if t == S.DS_OP_GEGLU else '')
    if t == S.DS_OP_LINEAR:
        return f'{d.n_rows}x{d.in_f}->{d.out_f}'
    if t == S.DS_OP_MEMSET:
        return f'{d.bytes} B'
    return ''


def _equal_chunked(a, b):
    for o in range(0, a.numel(), CHUNK):
        if not torch.equal(a[o:o + CHUNK], b[o:o + CHUNK]):
            diff = (a[o:o + CHUNK] != b[o:o + CHUNK]).nonzero()
            return o + int(diff[0])
    return None


def replay(lib, name):
    pl, wb, io_host = workload(name)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    arena = torch.zeros(pl.arena_bytes, dtype=torch.uint8, device=dev())
    weights = torch.frombuffer(bytearray(wb), dtype=torch.uint8).to(dev())
    io = {k: v.contiguous().to(dev()) for k, v in io_host.items() if v is not None}
    rows, skips = [], []

    def regions(ar, iod):
        r = {S.SPACE_ARENA: ar}
        r.update({(S.SPACE_IO, k): v.reshape(-1).view(torch.uint8) for k, v in iod.items()})
        return r

    def locate(reg, span):
        space, off = span.ref >> 60, span.ref & PI.MASK60
        if space == S.SPACE_ARENA:
            return reg[S.SPACE_ARENA][off:off + span.nbytes]
        t = reg[(space, off)]
        assert span.nbytes <= t.numel(), (span, t.numel())
        return t[:span.nbytes]

    live = regions(arena, io)
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        spans = writes(op)
        fill = not reads_own_output(op)
        pre = [locate(live, s).clone() for s in spans]
        if fill:
            for s in spans:
                locate(live, s).fill_(255)
        else:
            skips.append(i)
        snap_arena, snap_io = arena.clone(), {k: v.clone() for k, v in io.items()}
        ref = PI.Memory(0, None, snap_io, device=dev(), arena=snap_arena, weights=weights)
        ref.stored = []
        PI.run_op(ref, op)
        lib.op_launch(resolve(op, arena, weights, io))
        torch.cuda.synchronize()
        snap = regions(snap_arena, snap_io)
        got = [locate(live, s).clone() for s in spans]
        want = [locate(snap, s) for s in spans]
        # outside the spans: byte for byte (the spans are set to the reference's bytes, then the whole memory is compared)
        for s, w in zip(spans, want):
            locate(live, s).copy_(w)
        for key in live:
            at = _equal_chunked(live[key], snap[key])
            assert at is None, f'{name} op {i} ({S.UNION_FIELD[op.type]} tag {op.tag}): store outside its spans, {key} byte {at}'
        worst, problems = (0.0, 0.0, 0.0), []
        for k, s in enumerate(spans):
            pat_g, _ = _elements(s, got[k])
            pat_w, _ = _elements(s, want[k])
            if fill:
                if (pat_w & ~pat_g).any():
                    problems.append(f'span {k} ({s.fmt}): a store where the reference wrote nothing')
                if (~pat_w & pat_g).any():
                    problems.append(f'span {k} ({s.fmt}): an element the reference wrote was not written')
                written = ~pat_w
            else:                                              # only GroupNorm statistics (asserted below): every slot is written
                written = torch.ones_like(pat_w)
            if s.fmt != 'zero':
                vals = _values(s, got[k])
                if not torch.isfinite(vals[written[:vals.numel()]]).all():
                    problems.append(f'span {k} ({s.fmt}): non-finite value where the reference wrote one')
            r = _check_span(op, s, got[k], want[k], written, ref.stored, spans, got, want)
            if r[2] >= worst[2]:
                worst = r
        # back to the pre-fill bytes wherever the op did not write; elsewhere the GPU's output stays for the next op
        for s, p, g in zip(spans, pre, got):
            dst = locate(live, s)
            dst.copy_(torch.where(_unwritten_bytes(s, g), p, g) if fill else g)
        del snap_arena, snap_io, ref, snap, got, want, pre
        row = dict(i=i, type=S.UNION_FIELD[op.type], tag=op.tag, shape=shape_of(op), err=worst[0], bound=worst[1], ratio=worst[2],
                   fill=fill, problems=problems)
        rows.append(row)
    torch.cuda.synchronize()
    res = dict(rows=rows, skips=skips, seconds=time.time() - t0, peak=torch.cuda.max_memory_allocated(), n_ops=pl.n_ops,
               types={S.UNION_FIELD[pl.ops_array[i].type] for i in range(pl.n_ops)})
    del arena, weights, io, live
    torch.cuda.empty_cache()
    return res


def _fmt(name, r):
    flag = '' if r['ratio'] <= 1.0 and not r['problems'] else '  !!'
    return (f"{name:10s} {r['i']:4d} {r['type']:11s} {r['tag']:5d} {r['shape']:44s} {r['err']:10.3e} {r['bound']:10.3e} {r['ratio']:7.3f}"
            + ('' if r['fill'] else ' (no fill)') + flag + (' ' + '; '.join(r['problems']) if r['problems'] else ''))


@pytest.mark.parametrize('name', WORKLOADS)
def test_plan_ops_against_the_interpreter(lib, name):
    res = replay(lib, name)
    RESULTS[name] = res
    print(f"\n{'workload':10s} {'op':>4s} {'type':11s} {'tag':>5s} {'shape':44s} {'max err':>10s} {'bound':>10s} {'ratio':>7s}")
    for r in res['rows']:
        print(_fmt(name, r))
    compared = {r['type'] for r in res['rows']}
    print(f"{name}: {res['n_ops']} ops, {len(res['skips'])} without NaN fill ({', '.join(sorted({res['rows'][i]['type'] for i in res['skips']}))}), "
          f"{res['seconds']:.1f} s, peak device memory {res['peak'] / 2 ** 30:.2f} GiB")
    bad = [r for r in res['rows'] if r['ratio'] > 1.0 or r['problems']]
    assert len(res['rows']) == res['n_ops'] and compared == res['types'], sorted(res['types'] - compared)
    assert all(res['rows'][i]['type'] == 'gn_stats' for i in res['skips'])
    assert not bad, '\n'.join(_fmt(name, r) for r in bad[:20])


def test_plan_ops_report():
    if not RESULTS:
        pytest.skip('no workload of this module ran')
    print('\nworst ratio (error / bound) per op type')
    types = sorted({t for res in RESULTS.values() for t in res['types']})
    print(f"{'workload':10s} {'ops':>4s} {'secs':>6s} {'GiB':>6s} " + ' '.join(f'{t:>11s}' for t in types))
    for name, res in RESULTS.items():
        worst = collections.defaultdict(float)
        for r in res['rows']:
            worst[r['type']] = max(worst[r['type']], r['ratio'])
        print(f"{name:10s} {res['n_ops']:4d} {res['seconds']:6.1f} {res['peak'] / 2 ** 30:6.2f} "
              + ' '.join(f'{worst[t]:11.3f}' if t in res['types'] else f"{'-':>11s}" for t in types))
        assert {r['type'] for r in res['rows']} == res['types']

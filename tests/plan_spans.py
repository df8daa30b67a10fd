"""What a plan op touches, as data: `resolve` maps a descriptor's plan references to device addresses, `writes` lists the spans an op
stores to.  Both follow csrc/ops.h (pointer fields are exactly the c_uint64 fields of the _cstructs mirrors; the spans are the store
extents the kernels in csrc/*.cu implement).  Used by tests/test_gpu_plan_ops.py (replay of every op against the float64
interpreter) and checked on the CPU interpreter by tests/test_host_logic.py."""
import collections

from diff_sampler_b200 import _cstructs as S

MASK60 = (1 << 60) - 1

# One contiguous byte range an op may store to, starting at plan reference `ref`.
#   fmt 'f32'    fp32 elements
#        'f16'    fp16 planes: `nplanes` (1 or 2: hi, then lo at +`plane` elements); the span covers both planes and any gap between
#        'f8'     f8 GEMM operand image of `plane` elements: fp16 (v * 2^A16), e4m3 ((v - hi) * 2^LO8), e4m3 (hi * 2^HI8)
#        'f64'    fp64 GroupNorm sums [B][groups][2]
#        'stats'  fp32 GroupNorm partials of a GEMM epilogue [slabs][n_valid / unit][2] (`plane` = unit)
#        'nchw'   fp32 NCHW image store of a GEMM epilogue (EDM fold or plain eps output)
#        'zero'   bytes a memset clears
Span = collections.namedtuple('Span', ['ref', 'nbytes', 'fmt', 'nplanes', 'plane'])


def _field_names(desc):
    return [name for name, typ in type(desc)._fields_ if typ is S.P]


def resolve(op, arena, weights, io):
    """A copy of op's descriptor (the typed union member) with every pointer field mapped from a plan reference to a device address.
    arena / weights: uint8 device tensors; io: {slot: device tensor or None} (a missing slot resolves to NULL, as in the executor)."""
    src = getattr(op.u, S.UNION_FIELD[op.type])
    desc = type(src).from_buffer_copy(src)
    for name in _field_names(desc):
        ref = int(getattr(desc, name))
        space, off = ref >> 60, ref & MASK60
        if space == S.SPACE_ABS:
            continue
        if space == S.SPACE_ARENA:
            assert off < arena.numel(), (name, off)
            addr = arena.data_ptr() + off
        elif space == S.SPACE_WEIGHTS:
            assert off < weights.numel(), (name, off)
            addr = weights.data_ptr() + off
        elif space == S.SPACE_IO:
            t = io.get(off)
            addr = t.data_ptr() if t is not None else 0
        else:
            raise ValueError(f'{name}: bad pointer reference {ref:#x}')
        setattr(desc, name, addr)
    for name in _field_names(desc):
        assert int(getattr(desc, name)) >> 60 == 0, f'{name} still holds a plan reference'
    return desc


def _planes(ref, n, nplanes, fmt=0):
    if fmt == 1:
        return Span(int(ref), 4 * n, 'f8', 2, n)
    return Span(int(ref), 2 * n * nplanes, 'f16', nplanes, n)


def _gemm(d):
    out = []
    m, n = int(d.m_valid), int(d.n_valid)
    if d.st_quads:
        u = 2 if int(d.st_unit) == 2 else 4
        out.append(Span(int(d.st_quads), 4 * (m // 32) * (n // u) * 2, 'stats', 1, u))
    if d.edm_out:
        hw = int(d.rows_per_sample)
        out.append(Span(int(d.edm_D), 4 * (m // hw) * int(d.edm_C) * hw, 'nchw', 1, 0))
        return out
    nh = max(int(d.nh), 1)
    bases = [zb * int(d.o_zb) + zh * int(d.o_zh) for zb, zh in (divmod(z, nh) for z in range(int(d.num_z)))]
    lo, hi = min(bases), max(bases) + (m - 1) * int(d.ldo) + n               # elements: the union of the z windows
    if d.out_f32:
        out.append(Span(int(d.out_f32) + 4 * lo, 4 * (hi - lo), 'f32', 1, 0))
    if d.out_h16:
        if d.o_plane:
            assert int(d.o_plane) >= hi - lo, 'the lo plane of a GEMM output overlaps its hi plane'
            out.append(Span(int(d.out_h16) + 2 * lo, 2 * (int(d.o_plane) + hi - lo), 'f16', 2, int(d.o_plane)))
        else:
            out.append(Span(int(d.out_h16) + 2 * lo, 2 * (hi - lo), 'f16', 1, hi - lo))
    return out


def _gn_apply(d):
    C = int(d.C0) + int(d.C1)
    rs = int(d.resample)
    H, W = int(d.H), int(d.W)
    Ho, Wo = (H // 2, W // 2) if rs == 1 else ((2 * H, 2 * W) if rs == 2 else (H, W))
    n = int(d.B) * Ho * Wo * C                                 # space-to-depth keeps the element count
    out = [_planes(p, n, int(d.nplanes), int(d.fmt)) for p in (d.out_act, d.out_raw) if p]
    if d.out_raw_f32:
        out.append(Span(int(d.out_raw_f32), 4 * n, 'f32', 1, 0))
    return out


def _gn_finalize(d):
    out = []
    if d.quads0:
        out.append(Span(int(d.sums), 8 * int(d.B) * int(d.groups) * 2, 'f64', 1, 0))
    if d.coef:
        out.append(Span(int(d.coef), 4 * int(d.B) * (int(d.C0) + int(d.C1)) * 2, 'f32', 1, 0))
    return out


def _layer_out(d, n):
    if int(d.fmt) == 2:
        return [Span(int(d.out), 4 * n, 'f32', 1, 0)]
    return [_planes(d.out, n, int(d.nplanes), int(d.fmt))]


_WRITES = {
    S.DS_OP_GEMM: _gemm,
    S.DS_OP_GN_STATS: lambda d: [Span(int(d.sums), 8 * int(d.B) * int(d.groups) * 2, 'f64', 1, 0)],
    S.DS_OP_GN_APPLY: _gn_apply,
    S.DS_OP_SOFTMAX: lambda d: [_planes(d.P, int(d.rows) * (int(d.pitch_out) or int(d.L)), int(d.nplanes))],
    S.DS_OP_POSEMB: lambda d: [Span(int(d.emb), 4 * int(d.nsig) * int(d.num_channels), 'f32', 1, 0)]
                              + ([Span(int(d.coef), 4 * int(d.nsig) * 4, 'f32', 1, 0)] if int(d.mode) == 0 else []),
    S.DS_OP_LINEAR: lambda d: [Span(int(d.out), 4 * int(d.n_rows) * int(d.out_f), 'f32', 1, 0)],
    S.DS_OP_PREP_INPUT: lambda d: [_planes(d.out, int(d.B) * int(d.HW) * 64, int(d.nplanes))],
    S.DS_OP_CHANMEAN: lambda d: [Span(int(d.out), 4 * int(d.rows), 'f32', 1, 0)] if d.out else [],
    S.DS_OP_MEMSET: lambda d: [Span(int(d.ptr), int(d.bytes), 'zero', 1, 0)],
    S.DS_OP_LAYERNORM: lambda d: _layer_out(d, int(d.rows) * int(d.C)),
    S.DS_OP_GEGLU: lambda d: _layer_out(d, int(d.rows) * int(d.I)),
    S.DS_OP_GN_FINALIZE: _gn_finalize,
    S.DS_OP_ATTN: lambda d: [_planes(d.out, int(d.B) * int(d.L) * int(d.o_pitch), 2)],
    S.DS_OP_EMBED: lambda d: [Span(int(d.out), 4 * int(d.rows) * int(d.C), 'f32', 1, 0)],
}


def writes(op):
    """The spans op stores to (plan references), as Span records; io slots included (the EDM / eps image D, the bottleneck)."""
    return _WRITES[op.type](getattr(op.u, S.UNION_FIELD[op.type]))


def reads_own_output(op):
    """True when an op reads bytes of its own output spans, so those cannot be pre-filled: GroupNorm statistics accumulate into
    their sums, and a GEMM may add a residual it then overwrites in place."""
    if op.type == S.DS_OP_GN_STATS:
        return True
    if op.type != S.DS_OP_GEMM:
        return False
    d = op.u.gemm
    reads = []
    if d.residual:
        reads.append((int(d.residual), 4 * ((int(d.m_valid) - 1) * int(d.ldr) + int(d.n_valid))))
    if d.edm_out == 1:
        reads.append((int(d.edm_x), 4 * int(d.edm_C) * int(d.m_valid)))
    return any(overlap(a, n, s.ref, s.nbytes) for a, n in reads for s in writes(op))


def overlap(a, na, b, nb):
    """Whether byte ranges [a, a + na) and [b, b + nb) (plan references) share a byte; an io reference names a whole slot."""
    if a >> 60 != b >> 60:
        return False
    if a >> 60 == S.SPACE_IO:
        return a == b
    return a < b + nb and b < a + na

"""The float64 plan interpreter (oracle/plan_interp.py) and the write spans (tests/plan_spans.py) for the ops the Inception-v3 feature
extractor plans add (test infrastructure):
  * a GEMM with the ReLU epilogue (ds_gemm_desc.relu);
  * the TF1 legacy resize of uint8 images (ds_img_input), im2col (ds_im2col) and pooling (ds_pool).
Every other op, and a GEMM without relu, runs exactly as plan_interp runs it.  `install(monkeypatch)` adds these entries to
plan_interp's dispatch table, plan_spans' write table and the union-field table plan_spans and tests/test_gpu_plan_ops.py read, for
the duration of one test.
"""
import torch

from diff_sampler_b200 import _cstructs as S

from oracle import plan_interp as PI
import plan_spans as PS


# ------------------------------------------------------------------------------------------------ interpreter
def gemm(mem, d):
    if not int(d.relu):
        return PI._gemm(mem, d)
    # plan_interp rounds the float64 epilogue value once to fp32 and splits that into the fp16 planes; max(v, 0) commutes with that
    # rounding, so the fp32 output with relu applied in place, then split, is what the kernel's epilogue stores
    assert d.out_f32 and not d.st_quads and not d.edm_out and int(d.num_z) == 1
    d2 = type(d).from_buffer_copy(d)
    d2.relu, d2.out_h16, d2.o_plane = 0, 0, 0
    PI._gemm(mem, d2)
    m, n, ldo = int(d.m_valid), int(d.n_valid), int(d.ldo)
    o = PI._strided(mem.view(d.out_f32, torch.float32, (m - 1) * ldo + n), (m, n), (ldo, 1))
    o.clamp_(min=0.0)
    if d.out_h16:
        hi, lo = PI._split16(o.clone())
        PI._strided(mem.view(d.out_h16, torch.float16, (m - 1) * ldo + n), (m, n), (ldo, 1))[:] = hi
        if d.o_plane:
            PI._strided(mem.view(d.out_h16, torch.float16, (m - 1) * ldo + n, byte_offset=2 * int(d.o_plane)), (m, n), (ldo, 1))[:] = lo


def img_input(mem, d):
    B, C, H, W, Ho, Wo = (int(v) for v in (d.B, d.C, d.H, d.W, d.Ho, d.Wo))
    st = [int(v) for v in (d.sn, d.sc, d.sy, d.sx)]
    u8 = mem.view(d.src, torch.uint8, 1 + sum((n - 1) * s for n, s in zip((B, C, H, W), st)))
    x = PI._strided(u8, (B, C, H, W), st).double()

    def axis(n, no):
        f = torch.arange(no, dtype=torch.float64, device=mem.device) * n / no
        i0 = f.floor().long()
        return i0, (i0 + 1).clamp(max=n - 1), f - i0
    y0, y1, dy = axis(H, Ho)
    x0, x1, dx = axis(W, Wo)
    top = x[:, :, y0][..., x0] + (x[:, :, y0][..., x1] - x[:, :, y0][..., x0]) * dx
    bot = x[:, :, y1][..., x0] + (x[:, :, y1][..., x1] - x[:, :, y1][..., x0]) * dx
    v = (top + (bot - top) * dy[:, None] - 128.0) / 128.0
    mem.view(d.out, torch.float32, B * Ho * Wo * C)[:] = v.permute(0, 2, 3, 1).reshape(-1).float()


def _nhwc_in(mem, d):
    B, H, W, C, pitch, c0 = int(d.B), int(d.H), int(d.W), int(d.C), int(d.src_pitch), int(d.src_c0)
    return mem.view(d.src, torch.float32, B * H * W * pitch).reshape(B, H, W, pitch)[..., c0:c0 + C].double()


def im2col(mem, d):
    B, H, W, C = int(d.B), int(d.H), int(d.W), int(d.C)
    kh, kw, sh, sw, ph, pw, K64 = (int(v) for v in (d.kh, d.kw, d.sh, d.sw, d.ph, d.pw, d.K64))
    x = torch.nn.functional.pad(_nhwc_in(mem, d), (0, 0, pw, pw, ph, ph))
    Ho, Wo = (H + 2 * ph - kh) // sh + 1, (W + 2 * pw - kw) // sw + 1
    cols = [x[:, i:i + sh * (Ho - 1) + 1:sh, j:j + sw * (Wo - 1) + 1:sw, :] for i in range(kh) for j in range(kw)]
    rows = torch.zeros(B * Ho * Wo, K64, dtype=torch.float64, device=mem.device)
    rows[:, :kh * kw * C] = torch.cat(cols, dim=3).reshape(B * Ho * Wo, kh * kw * C)
    PI._store_planes(mem, d.out, rows, int(d.nplanes))


def pool(mem, d):
    x = _nhwc_in(mem, d)
    B, C = int(d.B), int(d.C)
    if int(d.mode) == S.DS_POOL_MEAN:
        o = mem.view(d.out_f32, torch.float32, (B - 1) * int(d.out_pitch) + int(d.out_c0) + C)
        PI._strided(o, (B, C), (int(d.out_pitch), 1), int(d.out_c0))[:] = x.mean(dim=(1, 2)).float()
        return
    k, s, p = int(d.k), int(d.stride), int(d.pad)
    xc = x.permute(0, 3, 1, 2)
    if int(d.mode) == S.DS_POOL_MAX:
        y = torch.nn.functional.max_pool2d(xc, k, s, p)
    else:
        y = torch.nn.functional.avg_pool2d(xc, k, s, p, count_include_pad=False)
    y = y.permute(0, 2, 3, 1)
    rows, pitch, c0 = y.shape[0] * y.shape[1] * y.shape[2], int(d.out_pitch), int(d.out_c0)
    y = y.reshape(rows, C)
    idx = (torch.arange(rows, device=mem.device)[:, None] * pitch + c0 + torch.arange(C, device=mem.device)[None, :]).reshape(-1)
    if d.out_f32:
        mem.view(d.out_f32, torch.float32, rows * pitch)[idx] = y.reshape(-1).float()
    if d.out_h16:
        PI._store_planes(mem, d.out_h16, y, int(d.nplanes), plane_elems=rows * pitch, index=idx)


# plan_interp._DISPATCH entries
DISPATCH = {S.DS_OP_GEMM: ('gemm', gemm), S.DS_OP_IMG_INPUT: ('img_input', img_input), S.DS_OP_IM2COL: ('im2col', im2col),
            S.DS_OP_POOL: ('pool', pool)}


def run_op(mem, op):
    if op.type in DISPATCH:
        field, fn = DISPATCH[op.type]
        with torch.no_grad():
            fn(mem, getattr(op.u, field))
        return
    PI.run_op(mem, op)


def run_plan(plan, weight_blob, io):
    mem = PI.Memory(plan.arena_bytes, weight_blob, io)
    for i in range(plan.n_ops):
        run_op(mem, plan.ops_array[i])
    return mem


# ------------------------------------------------------------------------------------------------ write spans
def _im2col_rows(d):
    return ((int(d.H) + 2 * int(d.ph) - int(d.kh)) // int(d.sh) + 1) * ((int(d.W) + 2 * int(d.pw) - int(d.kw)) // int(d.sw) + 1)


def _pool_spans(d):
    """Pool outputs: the channel window c0 .. c0 + C of every output row at the row pitch (fp32 and / or fp16 planes)."""
    B, C, pitch, c0 = int(d.B), int(d.C), int(d.out_pitch), int(d.out_c0)
    if int(d.mode) == S.DS_POOL_MEAN:
        return [PS.Span(int(d.out_f32) + 4 * c0, 4 * ((B - 1) * pitch + C), 'f32', 1, 0)]
    k, s, p = int(d.k), int(d.stride), int(d.pad)
    rows = B * ((int(d.H) + 2 * p - k) // s + 1) * ((int(d.W) + 2 * p - k) // s + 1)
    n = (rows - 1) * pitch + C
    out = []
    if d.out_f32:
        out.append(PS.Span(int(d.out_f32) + 4 * c0, 4 * n, 'f32', 1, 0))
    if d.out_h16:
        npl = int(d.nplanes)
        out.append(PS.Span(int(d.out_h16) + 2 * c0, 2 * (rows * pitch * (npl - 1) + n), 'f16', npl, rows * pitch if npl == 2 else n))
    return out


# plan_spans._WRITES entries
WRITES = {
    S.DS_OP_IMG_INPUT: lambda d: [PS.Span(int(d.out), 4 * int(d.B) * int(d.Ho) * int(d.Wo) * int(d.C), 'f32', 1, 0)],
    S.DS_OP_IM2COL: lambda d: [PS._planes(d.out, int(d.B) * _im2col_rows(d) * int(d.K64), int(d.nplanes))],
    S.DS_OP_POOL: _pool_spans,
}


def install(monkeypatch):
    """The entries above in plan_interp, plan_spans and the union-field table, until the test ends."""
    for t, entry in DISPATCH.items():
        monkeypatch.setitem(PI._DISPATCH, t, entry)
    for t, fn in WRITES.items():
        monkeypatch.setitem(PS._WRITES, t, fn)
    for t, f in S.INCEPTION_UNION_FIELD.items():
        monkeypatch.setitem(S.UNION_FIELD, t, f)

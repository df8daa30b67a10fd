"""The float64 plan interpreter (oracle/plan_interp.py) and the write spans (tests/plan_spans.py) for the ops the CLIP-score plans add
(test infrastructure):
  * the image input (ds_clip_input: the integer Pillow resample from the plan's tables, then ToTensor / Normalize in fp32);
  * the pooled heads (ds_clip_head: gather, L2 normalisation, score);
  * exact GELU (ds_geglu_desc.mode 2) and attention over heads of width 72 .. 128 (ds_attn_desc.pad0).
The image plan's im2col runs as tests/inception_interp.py runs it; every other op exactly as plan_interp runs it.  `install(monkeypatch)` adds these entries to plan_interp's dispatch table,
plan_spans' write table and the union-field table for the duration of one test.
"""
import torch

from diff_sampler_b200 import _cstructs as S

from oracle import plan_interp as PI
import inception_interp as II
import plan_spans as PS


def clip_input(mem, d):
    B, H, W, Sz, ky, kx = (int(v) for v in (d.B, d.H, d.W, d.S, d.ky, d.kx))
    st = [int(v) for v in (d.sn, d.sc, d.sy, d.sx)]
    u8 = mem.view(d.src, torch.uint8, 1 + sum((n - 1) * s for n, s in zip((B, 3, H, W), st)))
    x = PI._strided(u8, (B, 3, H, W), st).long()
    tab = mem.view(d.tab, torch.int32, 4 * Sz + Sz * (ky + kx)).long()
    y0, ny, x0, nx = (tab[i * Sz:(i + 1) * Sz] for i in range(4))
    wy = tab[4 * Sz:4 * Sz + Sz * ky].reshape(Sz, ky)
    wx = tab[4 * Sz + Sz * ky:].reshape(Sz, kx)

    def clip8(v):
        return torch.where(v >= 1 << 30, 255, torch.where(v <= 0, 0, v >> 22))

    def gather(n0, n, k, ks):      # [Sz][ks] source indices (clamped where the weight is 0) and weights
        j = torch.arange(ks, device=mem.device)[None, :]
        valid = j < n[:, None]
        return torch.where(valid, n0[:, None] + j, n0[:, None]), torch.where(valid, k, 0)
    iy, ky_ = gather(y0, ny, wy, ky)
    ix, kx_ = gather(x0, nx, wx, kx)
    # horizontal pass on every source row, rounded to uint8, then the vertical pass
    h = clip8((1 << 21) + (x[:, :, :, ix] * kx_).sum(-1))                          # [B][3][H][Sz]
    v = clip8((1 << 21) + (h[:, :, iy, :] * ky_[:, :, None]).sum(3))              # [B][3][Sz][Sz]
    mean = torch.tensor(list(d.mean), dtype=torch.float32, device=mem.device)[:, None, None]
    std = torch.tensor(list(d.std), dtype=torch.float32, device=mem.device)[:, None, None]
    # ToTensor's x / 255 as a true fp32 division on every device: CUDA tensors divide by a CPU scalar as a multiplication by its
    # rounded reciprocal, one ulp off for half of the 256 values
    y = (v.float() / torch.tensor(255.0, device=mem.device) - mean) / std
    mem.view(d.out, torch.float32, B * Sz * Sz * 3)[:] = y.permute(0, 2, 3, 1).reshape(-1)


def clip_head(mem, d):
    B, C, mode = int(d.B), int(d.C), int(d.mode)
    if mode == S.DS_CLIP_GATHER:
        ss, os_, T = int(d.src_stride), int(d.out_stride), int(d.T)
        rows = mem.view(d.ids, torch.int32, B * T).reshape(B, T).long().argmax(dim=1) if d.ids else torch.full((B,), int(d.row))
        src = mem.view(d.src, torch.float32, (B - 1) * ss + (int(rows.max()) + 1) * C)
        out = mem.view(d.out, torch.float32, (B - 1) * os_ + C)
        for n in range(B):
            out[n * os_:n * os_ + C] = src[n * ss + int(rows[n]) * C:n * ss + (int(rows[n]) + 1) * C]
        return
    a = mem.view(d.src, torch.float32, B * C).reshape(B, C).double()
    if mode == S.DS_CLIP_L2NORM:
        mem.view(d.out, torch.float32, B * C)[:] = (a / a.norm(dim=1, keepdim=True).clamp(min=1e-12)).reshape(-1).float()
        return
    b = mem.view(d.src2, torch.float32, B * C).reshape(B, C).double()
    mem.view(d.out, torch.float32, B)[:] = (float(d.scale) * (a * b).sum(1)).float()


def geglu(mem, d):
    if int(d.mode) != 2:
        return PI._geglu(mem, d)
    rows, I = int(d.rows), int(d.I)
    x = mem.view(d.src, torch.float32, rows * I).reshape(rows, I).double()
    PI._store_planes(mem, d.out, torch.nn.functional.gelu(x), int(d.nplanes), 0)


def attn(mem, d):
    hd = int(d.pad0)
    if hd in (0, 64, 32):
        return PI._attn(mem, d)
    B, nh, L, Lk = int(d.B), int(d.nh), int(d.L), int(d.Lk)
    qp, kp, vp, op = int(d.q_pitch), int(d.k_pitch), int(d.vt_pitch), int(d.o_pitch)
    q = PI._planes_f16(mem, d.q, B * L * qp, 2).reshape(B, L, qp)
    k = PI._planes_f16(mem, d.k, B * Lk * kp, 2).reshape(B, Lk, kp)
    vt = PI._planes_f16(mem, d.vt, B * nh * hd * vp, 2).reshape(B, nh * hd, vp)
    assert op == nh * hd and not int(d.causal)
    out = torch.zeros(B, L, op, dtype=torch.float64, device=mem.device)
    for h in range(nh):
        qs = q[:, :, int(d.q_c0) + h * hd:int(d.q_c0) + (h + 1) * hd]
        ks = k[:, :, int(d.k_c0) + h * hd:int(d.k_c0) + (h + 1) * hd]
        p = torch.softmax(float(d.scale) * qs @ ks.transpose(1, 2), dim=2)
        out[:, :, h * hd:(h + 1) * hd] = p @ vt[:, h * hd:(h + 1) * hd, :Lk].transpose(1, 2)
    PI._store_planes(mem, d.out, out, 2)


DISPATCH = {**II.DISPATCH, S.DS_OP_CLIP_INPUT: ('clip_input', clip_input), S.DS_OP_CLIP_HEAD: ('clip_head', clip_head),
            S.DS_OP_GEGLU: ('geglu', geglu), S.DS_OP_ATTN: ('attn', attn)}


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


def _head_spans(d):
    B, C, mode = int(d.B), int(d.C), int(d.mode)
    if mode == S.DS_CLIP_GATHER:
        return [PS.Span(int(d.out), 4 * ((B - 1) * int(d.out_stride) + C), 'f32', 1, 0)]
    return [PS.Span(int(d.out), 4 * (B * C if mode == S.DS_CLIP_L2NORM else B), 'f32', 1, 0)]


WRITES = {
    **II.WRITES,
    S.DS_OP_CLIP_INPUT: lambda d: [PS.Span(int(d.out), 4 * int(d.B) * int(d.S) * int(d.S) * 3, 'f32', 1, 0)],
    S.DS_OP_CLIP_HEAD: _head_spans,
}


def install(monkeypatch):
    """The entries above in plan_interp, plan_spans and the union-field table, until the test ends."""
    for t, entry in DISPATCH.items():
        monkeypatch.setitem(PI._DISPATCH, t, entry)
    for t, fn in WRITES.items():
        monkeypatch.setitem(PS._WRITES, t, fn)
    for t, f in {**S.INCEPTION_UNION_FIELD, **S.OPENCLIP_UNION_FIELD}.items():
        monkeypatch.setitem(S.UNION_FIELD, t, f)

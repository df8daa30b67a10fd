"""The float64 plan interpreter (oracle/plan_interp.py) for the ops the unconditional latent-diffusion plans add (test infrastructure):
  * a conv GEMM whose 1x1 skip operand has a channel count that is not a multiple of 64 (the K loop's last aux block zero-filled);
  * the space-to-depth repack at a phase pitch (ds_gn_apply_desc.pad0): each phase at pad0 channels, the gap zero;
  * attention over 32-wide heads in pairs (ds_attn_desc.pad0 = 32).
Every other op, and these ops without the new fields, run exactly as plan_interp runs them.  A main-operand channel remainder needs
nothing here: plan_interp's im2col already zero-fills past the tensor's channel extent.
"""
import ctypes

import torch

from diff_sampler_b200 import _cstructs as S

from oracle import plan_interp as PI

_TMP_SLOT = 1 << 20             # an io slot no plan uses: the zero-padded copy of a skip operand


def gemm(mem, d):
    c2 = int(d.a2_c)
    if int(d.a_mode) != 0 or c2 % 64 == 0:
        return PI._gemm(mem, d)
    # plan_interp reads an aux operand of whole 64-channel blocks: hand it a zero-padded copy of the skip planes
    H, W, Bn = int(d.conv_H), int(d.conv_W), int(d.a2_plane_n)
    npl = 2 if int(d.npass) == 3 else 1
    src = mem.view(d.a2_ptr, torch.float16, npl * Bn * H * W * c2).reshape(npl, Bn, H, W, c2)
    c2p = -(-c2 // 64) * 64
    pad = torch.zeros(npl, Bn, H, W, c2p, dtype=torch.float16, device=mem.device)
    pad[..., :c2] = src
    d2 = type(d).from_buffer_copy(d)
    d2.a2_ptr, d2.a2_c = S.ref(S.SPACE_IO, _TMP_SLOT), c2p
    mem.io[_TMP_SLOT] = pad
    try:
        PI._gemm(mem, d2)
    finally:
        del mem.io[_TMP_SLOT]


def gn_apply(mem, d):
    C = int(d.C0) + int(d.C1)
    cp = int(d.pad0)
    if int(d.resample) != 3 or cp in (0, C):
        return PI._gn_apply(mem, d)
    # the plans use the pitched repack for the raw pass-through only (the Downsample's operand)
    assert not d.out_act and not d.out_raw_f32 and d.out_raw
    B, H, W = int(d.B), int(d.H), int(d.W)
    x = PI._src_cat(mem, d, B * H * W).reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4, C)
    y = torch.zeros(B, H // 2, W // 2, 4, cp, dtype=x.dtype, device=x.device)
    y[..., :C] = x
    PI._store_planes(mem, d.out_raw, y.reshape(B, H // 2, W // 2, 4 * cp), int(d.nplanes), int(d.fmt))


def attn(mem, d):
    if int(d.pad0) != 32:
        return PI._attn(mem, d)
    B, nh, L, Lk = int(d.B), int(d.nh), int(d.L), int(d.Lk)
    qp, kp, vp, op = int(d.q_pitch), int(d.k_pitch), int(d.vt_pitch), int(d.o_pitch)
    q = PI._planes_f16(mem, d.q, B * L * qp, 2).reshape(B, L, qp)
    k = PI._planes_f16(mem, d.k, B * Lk * kp, 2).reshape(B, Lk, kp)
    vt = PI._planes_f16(mem, d.vt, B * nh * 32 * vp, 2).reshape(B, nh * 32, vp)
    assert op == nh * 32
    out = torch.zeros(B, L, op, dtype=torch.float64, device=mem.device)
    for h in range(nh):
        qs = q[:, :, int(d.q_c0) + h * 32:int(d.q_c0) + (h + 1) * 32]
        ks = k[:, :, int(d.k_c0) + h * 32:int(d.k_c0) + (h + 1) * 32]
        sc = float(d.scale) * qs @ ks.transpose(1, 2)
        if int(d.causal):
            sc = sc + torch.full((L, Lk), float('-inf'), dtype=torch.float64, device=mem.device).triu(1)
        out[:, :, h * 32:(h + 1) * 32] = torch.softmax(sc, dim=2) @ vt[:, h * 32:(h + 1) * 32, :Lk].transpose(1, 2)
    PI._store_planes(mem, d.out, out, 2)


# plan_interp._DISPATCH entries for a run that replays ops through plan_interp (tests/test_gpu_plan_ops.replay)
DISPATCH = {S.DS_OP_GEMM: ('gemm', gemm), S.DS_OP_GN_APPLY: ('gn_apply', gn_apply), S.DS_OP_ATTN: ('attn', attn)}


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


def gn_apply_spans(span_fn):
    """plan_spans' gn_apply writes for a descriptor with a phase pitch: the repack covers B (H/2) (W/2) 4 pad0 elements."""
    def spans(d):
        cp, C = int(d.pad0), int(d.C0) + int(d.C1)
        if int(d.resample) != 3 or cp in (0, C):
            return span_fn(d)
        d2 = type(d).from_buffer_copy(d)
        d2.C0, d2.C1 = cp, 0
        return span_fn(d2)
    return spans

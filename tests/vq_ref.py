"""Float64 restatements for the VQ first-stage decode (VQModelInterface.decode, models/ldm/models/autoencoder.py:274-282).

The reference's quantizer is taming-transformers' VectorQuantizer2, which is not part of the reference tree; its inference path is
restated here, not pinned: z_q = e[argmin_j |z - e_j|^2] per pixel (the reference evaluates |z|^2 + |e_j|^2 - 2 z.e_j in fp32 and
returns z + (z_q - z).detach(), i.e. z_q up to an fp32 rounding).  What follows the quantizer -- post_quant_conv and the Decoder -- is
oracle/vae_oracle.py, pinned to the reference Decoder by tests/golden/ref_vae.npz.

Note that the kernel takes sum_c (v_c - e_c)^2 directly, while the reference takes the expanded form; both are fp32, so a pixel whose
two nearest rows are within fp32 rounding of each other may resolve differently between them (and from float64).  The tests compare
indices only where the float64 gap exceeds MIN_GAP.

Also: the quantizing prep_input op restated for the plan interpreter (oracle/plan_interp.py runs every other op; use run_op /
run_plan below for plans that quantize), and the extra span the op stores to when it keeps the chosen indices."""
from unittest import mock

import torch

from diff_sampler_b200 import _cstructs as S
from oracle import plan_interp as PI
from oracle import vae_oracle as VO
from plan_spans import Span, writes

CONFIGS = {
    # models/ldm/configs/latent-diffusion/lsun_bedrooms-ldm-vq-4.yaml:44-63 (first_stage_config; the same in ffhq-ldm-vq-4.yaml);
    # scale_factor is the LatentDiffusion default 1.0 (the configs do not set it); latents 64x64 -> images 256x256
    'vq_f4': dict(ch=128, out_ch=3, ch_mult=(1, 2, 4), num_res_blocks=2, z_channels=3, embed_dim=3, scale_factor=1.0, n_embed=8192),
    # reduced net of the same structure
    'tiny_vq': dict(ch=64, out_ch=3, ch_mult=(1, 2), num_res_blocks=1, z_channels=3, embed_dim=3, scale_factor=1.0, n_embed=512),
}

# Smallest float64 best-to-second squared-distance gap at which the kernel's fp32 distances must pick the same row: with |v|, |e| of a
# few units (randn), sum_c (v_c - e_c)^2 is at most ~100 and carries an fp32 error below 4 ulp of that, 2.4e-5.
MIN_GAP = 1e-4


def make_params(name, seed=0):
    """vae_oracle's seeded Decoder + post_quant_conv parameters, plus a codebook `quantize.embedding.weight` of O(1) spread (randn):
    the stock uniform(+-1/n_embed) init would map nearly every latent to the same few rows and test nothing."""
    cfg = dict(CONFIGS[name])
    with mock.patch.dict(VO.CONFIGS, {name: cfg}):
        P, _ = VO.make_params(name, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    P['quantize.embedding.weight'] = torch.randn(cfg['n_embed'], cfg['embed_dim'], generator=g)
    return P, cfg


def nearest(v, codebook):
    """v [N, C], codebook [n_embed, C] -> (index of the nearest row, float64 distance to it, to the second nearest), by brute force."""
    v, e = v.double(), codebook.double().to(v.device)
    d = (v * v).sum(1, keepdim=True) + (e * e).sum(1)[None, :] - 2.0 * v @ e.T
    two = d.topk(min(2, e.shape[0]), dim=1, largest=False).values
    best = d.argmin(dim=1)                                          # lowest index on exact ties, as torch.argmin
    return best, two[:, 0], two[:, 1] if e.shape[0] > 1 else torch.full_like(two[:, 0], float('inf'))


def latents_near_codes(P, cfg, B, R, seed=3, spread=0.05, min_gap=MIN_GAP):
    """Latents [B, C, R, R] scattered around random codebook rows (times scale_factor), and the float64 best-to-second distance gap
    of every pixel, so a test can check first that no pixel is a near tie.  Pixels closer to a tie than min_gap are drawn again,
    nearer to their row."""
    e = P['quantize.embedding.weight']
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, e.shape[0], (B * R * R,), generator=g)
    v = e[idx] + spread * torch.randn(B * R * R, e.shape[1], generator=g)
    for _ in range(8):
        _, d1, d2 = nearest(v, e)
        tie = (d2 - d1) <= min_gap
        if not tie.any():
            break
        spread *= 0.25
        v[tie] = e[idx[tie]] + spread * torch.randn(int(tie.sum()), e.shape[1], generator=g)
    _, d1, d2 = nearest(v, e)
    z = v.reshape(B, R, R, -1).permute(0, 3, 1, 2).contiguous() * cfg['scale_factor']
    return z, (d2 - d1)


def quantize(P, cfg, z):
    """VectorQuantizer2 inference on z / scale_factor: every pixel's channel vector replaced by its nearest codebook row (float64)."""
    e = P['quantize.embedding.weight'].double()
    B, C, H, W = z.shape
    v = (z.double() / cfg['scale_factor']).permute(0, 2, 3, 1).reshape(-1, C)
    best, _, _ = nearest(v, e)
    return e.to(v.device)[best].reshape(B, H, W, C).permute(0, 3, 1, 2), best.reshape(B, H * W)


def decode(P, cfg, z, taps=None, force_not_quantize=False):
    """VQModelInterface.decode after z / scale_factor (ddpm.py:714, :761-762): quantize, post_quant_conv, Decoder (float64 if z is)."""
    q = z.double() / cfg['scale_factor'] if force_not_quantize else quantize(P, cfg, z)[0]
    Pd = {k: v.double().to(q.device) for k, v in P.items()}
    return VO.decode(Pd, dict(cfg, scale_factor=1.0), q, taps=taps)


# --------------------------------------------------------------------------------------------- the plan op
def run_prep_input_vq(mem, d):
    """Float64 restatement of the quantizing prep_input (csrc/elementwise.cu vq_prep_input_kernel) on a plan_interp.Memory."""
    B, C, HW, n_embed = int(d.B), int(d.C), int(d.HW), int(d.n_embed)
    xb = int(d.x_batch) if d.x_batch > 0 else B
    x = mem.view(d.x, torch.float32, xb * C * HW).reshape(xb, C, HW)
    cst = int(d.coef_stride)
    coef = mem.view(d.coef, torch.float32, (xb - 1) * cst + 4)
    e = mem.view(d.codebook, torch.float32, n_embed * C).reshape(n_embed, C)
    out = torch.zeros(B, HW, 64, dtype=torch.float64, device=mem.device)
    idx = torch.zeros(B, HW, dtype=torch.int32, device=mem.device)
    for n in range(B):
        nx = n % xb
        v = (coef[nx * cst + 2] * x[nx]).T                             # the fp32 product the kernel forms
        best, _, _ = nearest(v, e)
        out[n, :, :C] = e[best].double()
        idx[n] = best.to(torch.int32)
    PI._store_planes(mem, d.out, out, int(d.nplanes))
    if d.idx:
        mem.view(d.idx, torch.int32, B * HW)[:] = idx.reshape(-1)


def is_vq(op):
    return op.type == S.DS_OP_PREP_INPUT and bool(op.u.prep_input.codebook)


def run_op(mem, op):
    if is_vq(op):
        with torch.no_grad():
            run_prep_input_vq(mem, op.u.prep_input)
    else:
        PI.run_op(mem, op)


def run_plan(plan, weight_blob, io):
    """plan_interp.run_plan for plans that may hold a quantizing prep_input (plan_interp's own _prep_input has no codebook search)."""
    mem = PI.Memory(plan.arena_bytes, weight_blob, io)
    for i in range(plan.n_ops):
        run_op(mem, plan.ops_array[i])
    return mem


def vq_writes(op):
    """plan_spans.writes, plus the index buffer of a quantizing prep_input that keeps its indices: fmt 'i32', int32 elements."""
    spans = writes(op)
    if is_vq(op) and op.u.prep_input.idx:
        d = op.u.prep_input
        spans.append(Span(int(d.idx), 4 * int(d.B) * int(d.HW), 'i32', 1, 0))
    return spans

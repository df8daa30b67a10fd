"""ORACLE — test infrastructure, not product code (see oracle/edm_oracle.py header).

The plan interpreter (oracle/plan_interp.py) for plans whose embedding op carries a noise scale: the Consistency-Models nets embed
noise_scale * ln(sigma) / 4 (ds_posemb_desc.noise_scale = 1000, CMPrecond networks_edm.py:539-540).  Every other op, and a posemb
op whose noise_scale is 0 (= 1), runs exactly as plan_interp runs it.
"""
import torch

from diff_sampler_b200 import _cstructs as S

from . import plan_interp as PI


def posemb(mem, d):
    """plan_interp's posemb, then the embedding rewritten from the scaled argument in float64 when noise_scale is not 1."""
    PI._posemb(mem, d)
    scale = float(d.noise_scale) or 1.0
    if d.mode != 0 or scale == 1.0:
        return
    n, ch = int(d.nsig), int(d.num_channels)
    half = ch // 2
    sig = mem.view(d.sigma, torch.float32, n).double()
    i = torch.arange(half, dtype=torch.float64, device=mem.device)
    a = (scale * torch.log(sig) / 4)[:, None] * ((1.0 / 10000.0) ** (i / (half - (1 if d.endpoint else 0))))[None, :]
    cs, sn = torch.cos(a).float(), torch.sin(a).float()
    emb = mem.view(d.emb, torch.float32, n * ch).reshape(n, ch)
    if d.swap_sincos:
        emb[:, :half], emb[:, half:] = sn, cs
    else:
        emb[:, :half], emb[:, half:] = cs, sn


DISPATCH_ENTRY = ('posemb', posemb)          # plan_interp._DISPATCH[S.DS_OP_POSEMB] for a run that replays ops through plan_interp


def run_op(mem, op):
    if op.type == S.DS_OP_POSEMB:
        with torch.no_grad():
            posemb(mem, op.u.posemb)
        return
    PI.run_op(mem, op)


def run_plan(plan, weight_blob, io):
    """plan_interp.run_plan with the noise-scaled embedding."""
    mem = PI.Memory(plan.arena_bytes, weight_blob, io)
    for i in range(plan.n_ops):
        run_op(mem, plan.ops_array[i])
    return mem


"""Float64 restatement of diff-analyzer's optimal denoiser (diff-analyzer-main/solvers.py:19-28), its Euler sampler (:773-868) and the
k-nearest-neighbour read-out, the seeded datasets the tests use, and the float64 plan-interpreter ops of csrc/optimal.cu (registered
into oracle/plan_interp on import).  Test infrastructure: only tests/ and tools/ import this; it is pinned to tests/golden/ref_opt.npz,
which tools/gen_opt_golden.py writes from the reference's own functions."""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from diff_sampler_b200 import _cstructs as S      # noqa: E402
from oracle import plan_interp as PI               # noqa: E402

# ------------------------------------------------------------------------------------------------ seeded data
GOLDEN_SIGMAS = (80.0, 5.0, 1.0, 0.2, 0.05, 0.01, 0.002)
GOLDEN_SAMPLER_RUNS = {
    'plain': dict(num_steps=6, return_inters=True, return_denoised=True, return_eps=True),
    'dtz': dict(num_steps=6, denoise_to_zero=True, return_inters=True, return_denoised=True, return_eps=True),
    'dtz_x': dict(num_steps=5, denoise_to_zero=True),
    'afs': dict(num_steps=6, afs=True),
    'tsteps': dict(t_steps=[40.0, 10.0, 2.0, 0.5, 0.1, 0.02], return_inters=True, return_denoised=True, return_eps=True),
}


def uint8_images(n, c, h, w, seed, smooth=True):
    """Seeded images as uint8 levels / 127.5 - 1 (utils.cifar10_prepare's scaling): a random low-frequency field per image plus a
    little pixel noise, so that images have spatial structure and distinct nearest neighbours (not white noise)."""
    g = torch.Generator().manual_seed(seed)
    if smooth:
        lo = torch.rand(n, c, max(1, h // 4), max(1, w // 4), generator=g) * 2 - 1
        img = torch.nn.functional.interpolate(lo, size=(h, w), mode='bilinear', align_corners=False)
        img = img + 0.15 * torch.randn(n, c, h, w, generator=g)
    else:
        img = torch.rand(n, c, h, w, generator=g) * 2 - 1
    lv = ((img.clamp(-1, 1) + 1) * 127.5).round().clamp(0, 255)
    return lv.to(torch.float32) / 127.5 - 1


def near_duplicates(n, c, h, w, seed):
    """Pairs one level apart in 1..16 values, plus exact duplicates (rows 2k, 2k+1)."""
    base = uint8_images(n // 2, c, h, w, seed)
    lv = ((base + 1) * 127.5).round()
    twin = lv.clone().reshape(n // 2, -1)
    g = torch.Generator().manual_seed(seed + 1)
    for k in range(n // 2):
        m = int(k % 17)                       # 0: exact duplicate, else 1..16 values one level apart
        idx = torch.randperm(twin.shape[1], generator=g)[:m]
        step = torch.where(twin[k, idx] >= 255, -1.0, 1.0)
        twin[k, idx] += step
    both = torch.stack([lv.reshape(n // 2, -1), twin], dim=1).reshape(n - n % 2, c, h, w)
    return both / 127.5 - 1


def golden_dataset():
    return uint8_images(300, 3, 8, 8, seed=7)


def golden_latents():
    return torch.randn(4, 3, 8, 8, generator=torch.Generator().manual_seed(11))


# ------------------------------------------------------------------------------------------------ float64 oracle
def denoise_opt(x, sigma, dataset, return_logits=False):
    """D*(x; sigma) in float64: softmax_i(-||x - y_i||^2 / (2 sigma^2)) weighted sum of y_i.  sigma: scalar or [B]."""
    x64 = x.double().reshape(x.shape[0], -1)
    y64 = dataset.to(x64.device).double().reshape(dataset.shape[0], -1)
    s = torch.as_tensor(sigma, dtype=torch.float64, device=x64.device).reshape(-1, 1)
    d2 = (x64 * x64).sum(1, keepdim=True) - 2 * x64 @ y64.T + (y64 * y64).sum(1)[None]
    d2 = d2.clamp_min(0)
    logits = -d2 / (2 * s * s)
    w = torch.softmax(logits, dim=1)
    D = (w @ y64).reshape(x.shape)
    return (D, logits) if return_logits else D


def exact_dist2(x, dataset):
    """Squared distances [B, N] from the differences in float64 (no cancellation)."""
    x64 = x.double().reshape(x.shape[0], 1, -1)
    y64 = dataset.to(x64.device).double().reshape(1, dataset.shape[0], -1)
    out = torch.empty(x64.shape[0], y64.shape[1], dtype=torch.float64, device=x64.device)
    step = max(1, (1 << 26) // max(1, y64.shape[1] * y64.shape[2]))
    for b0 in range(0, x64.shape[0], step):
        out[b0:b0 + step] = ((x64[b0:b0 + step] - y64) ** 2).sum(-1)
    return out


def knn(x, dataset, k):
    """(distances, indices) of the k nearest rows, ascending, ties to the lower index; also the sorted float64 distances."""
    d2 = exact_dist2(x, dataset)
    order = torch.argsort(d2, dim=1, stable=True)                            # stable: equal distances keep index order
    sd = torch.gather(d2, 1, order)
    return sd[:, :k].sqrt(), order[:, :k], sd


def polynomial_schedule(num_steps, sigma_min=0.002, sigma_max=80.0, rho=7):
    i = torch.arange(num_steps, dtype=torch.float64)
    return (sigma_max ** (1 / rho) + i / (num_steps - 1) * (sigma_min ** (1 / rho) - sigma_max ** (1 / rho))) ** rho


def optimal_sampler(latents, dataset, num_steps=None, sigma_min=0.002, sigma_max=80.0, afs=False, denoise_to_zero=False,
                    return_inters=False, t_steps=None, denoiser=None):
    """diff-analyzer's optimal_sampler in float64 (its quirks included: denoise_to_zero evaluates at the last step's input and
    sigma, divides by t_N; without return_inters it returns x_N).  Returns x_N, or (trajectory, denoised, eps)."""
    den = denoiser or (lambda x, s: denoise_opt(x, s, dataset))
    t = polynomial_schedule(num_steps, sigma_min, sigma_max) if t_steps is None else torch.as_tensor(t_steps, dtype=torch.float64)
    t = t.to(torch.float32).double().tolist()                               # the samplers run on the fp32 grid
    x = latents.double() * t[0]
    xt, dens, eps = [x], [], []
    D = None
    x_cur = x
    for i in range(len(t) - 1):
        x_cur = x
        if afs and i == 0:
            d = x_cur / math.sqrt(1 + t[i] ** 2)
        else:
            D = den(x_cur, t[i])
            d = (x_cur - D) / t[i]
        x = x_cur + (t[i + 1] - t[i]) * d
        xt.append(x)
        dens.append(D)
        eps.append(d)
    if denoise_to_zero:
        D = den(x_cur, t[-2])
        xt.append(D)
        dens.append(D)
        eps.append((x - D) / t[-1])
    if return_inters:
        return torch.stack(xt), torch.stack(dens), torch.stack(eps)
    return x


# ------------------------------------------------------------------------------------------------ plan interpreter ops
def _u(mem, d):
    B, N, ldp, ns = int(d.B), int(d.N), int(d.ldp), int(d.nslice)
    part = mem.view(d.part, torch.float32, ns * B * ldp).reshape(ns, B, ldp)[:, :, :N].double().sum(0)
    return part - mem.view(d.hy2, torch.float64, N)[None, :]


def _rows(mem, d):
    B, N, D = int(d.B), int(d.N), int(d.D)
    x = mem.view(d.x, torch.float32, B * D).reshape(B, D).double()
    y = mem.view(d.y, torch.float32, N * D).reshape(N, D).double()
    return x, y


def _opt_prep(mem, d):
    B, D, pitch = int(d.B), int(d.D), int(d.pitch)
    x = mem.view(d.x, torch.float32, B * D).reshape(B, D).double()
    xp = torch.zeros(B, pitch, dtype=torch.float64, device=mem.device)
    xp[:, :D] = x
    PI._store_planes(mem, d.planes, xp, 2)
    mem.view(d.xn2, torch.float64, B)[:] = (x * x).sum(1)


def _opt_softmax(mem, d):
    """The op's arithmetic in float64: logits u_i / sigma^2, the same band rule, exact distances for rescored rows."""
    B, N, ldP = int(d.B), int(d.N), int(d.ldP)
    u = _u(mem, d)
    x, y = _rows(mem, d)
    sig = mem.view(d.sigma, torch.float32, int(d.nsig)).double()
    s2 = (sig * sig).reshape(-1, 1).expand(B, 1)
    logits = u / s2
    xn = mem.view(d.xn2, torch.float64, B).sqrt()
    E = (xn + float(d.ymax)) * (S.DS_OPT_EPS * float(d.ymax) + math.sqrt(int(d.D)) * 2.0 ** -25) / s2[:, 0]
    P = torch.zeros(B, ldP, dtype=torch.float64, device=mem.device)
    status = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        lg = logits[b]
        if E[b] > S.DS_OPT_TAU:
            band = torch.nonzero(lg >= lg.max() - (2 * E[b] + S.DS_OPT_BAND_NATS)).reshape(-1)
            if band.numel() <= S.DS_OPT_CAP:
                ex = -0.5 * ((x[b][None] - y[band]) ** 2).sum(1) / s2[b, 0]
                P[b, band] = torch.softmax(ex, 0)
                status[b] = S.DS_OPT_RESCORED
                continue
            status[b] = S.DS_OPT_UNREFINED
        P[b, :N] = torch.softmax(lg, 0)
    PI._store_planes(mem, d.P, P * 2.0 ** S.DS_OPT_P_SHIFT, 2)
    if d.status:
        mem.view(d.status, torch.int32, B)[:] = status.to(mem.device)


def _opt_reduce(mem, d):
    rows, cols, ld, ns = int(d.rows), int(d.cols), int(d.ld), int(d.nsplit)
    part = mem.view(d.part, torch.float32, ns * rows * ld).reshape(ns, rows, ld)[:, :, :cols].double().sum(0)
    mem.view(d.out, torch.float32, rows * cols)[:] = (part * float(d.scale)).reshape(-1).float()


def _opt_knn(mem, d):
    B, k = int(d.B), int(d.k)
    x, y = _rows(mem, d)
    d2 = ((x[:, None, :] - y[None]) ** 2).sum(-1)
    order = torch.argsort(d2, dim=1, stable=True)[:, :k]
    mem.view(d.dist, torch.float32, B * k)[:] = torch.gather(d2, 1, order).sqrt().reshape(-1).float()
    mem.view(d.idx, torch.int32, B * k)[:] = order.reshape(-1).to(torch.int32)


def writes(op):
    """Store spans (tests/plan_spans.Span) of an op of an optimal-denoiser plan: the GEMM's from tests/plan_spans, the others' from
    csrc/optimal.cu (opt_softmax and opt_knn overwrite logits slice 0 with u)."""
    import plan_spans as PS
    if op.type == S.DS_OP_GEMM:
        return PS.writes(op)
    d = getattr(op.u, S.OPT_UNION_FIELD[op.type])
    if op.type == S.DS_OP_OPT_PREP:
        return [PS._planes(d.planes, int(d.B) * int(d.pitch), 2), PS.Span(int(d.xn2), 8 * int(d.B), 'f64', 1, 0)]
    if op.type == S.DS_OP_OPT_REDUCE:
        return [PS.Span(int(d.out), 4 * int(d.rows) * int(d.cols), 'f32', 1, 0)]
    u = PS.Span(int(d.part), 4 * int(d.B) * int(d.ldp), 'f32', 1, 0)
    if op.type == S.DS_OP_OPT_SOFTMAX:
        return [u, PS._planes(d.P, int(d.B) * int(d.ldP), 2)] + ([PS.Span(int(d.status), 4 * int(d.B), 'f32', 1, 0)] if d.status else [])
    return [u, PS.Span(int(d.dist), 4 * int(d.B) * int(d.k), 'f32', 1, 0), PS.Span(int(d.idx), 4 * int(d.B) * int(d.k), 'f32', 1, 0)]


PI._DISPATCH.update({S.DS_OP_OPT_PREP: ('opt_prep', _opt_prep), S.DS_OP_OPT_SOFTMAX: ('opt_softmax', _opt_softmax),
                     S.DS_OP_OPT_REDUCE: ('opt_reduce', _opt_reduce), S.DS_OP_OPT_KNN: ('opt_knn', _opt_knn)})

"""Float64 restatement of sfd-main/prdc.py's compute_prdc (:29-125): distances from explicit float64 differences, every comparison on
float64 distances.  Also the seeded golden inputs (features on a 1/16 grid, where the reference's own distance matrices are exact),
and the float64 plan-interpreter ops of csrc/prdc.cu (registered into oracle/plan_interp on import).  Test infrastructure: only tests/,
tools/ and oracle/gen_prdc_golden.py import this; it is pinned to tests/golden/ref_prdc.npz, which that script writes from the
reference's own compute_prdc."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from diff_sampler_b200 import _cstructs as S      # noqa: E402
from diff_sampler_b200 import prdc as P           # noqa: E402
from oracle import plan_interp as PI               # noqa: E402

KEYS = ('precision', 'recall', 'density', 'coverage')


# ------------------------------------------------------------------------------------------------ seeded data
def _codes(g, n, d, hi=16):
    return torch.randint(0, hi, (n, d), generator=g, dtype=torch.uint8)


def golden_cases():
    """[(name, real uint8 codes [N_r, D], fake codes [N_f, D], nearest_k)]; features are codes / 16."""
    g = torch.Generator().manual_seed(2024)
    cases = []
    # D = 2048, a few hundred rows; fake rows 0..9 copy real rows (zero distances across the sets, and pairs exactly at a real radius),
    # fake rows 20..24 repeat fake row 19 and real rows 30..33 repeat real row 29 (duplicates within each set)
    r, f = _codes(g, 240, 2048), _codes(g, 200, 2048)
    f[:10] = r[:10]
    f[20:25] = f[19]
    r[30:34] = r[29]
    cases.append(('d2048', r, f, 5))
    # D = 64, a few thousand rows, features clustered so that neighbourhoods overlap
    centres = _codes(g, 40, 64, 12)
    r = (centres[torch.randint(0, 40, (2500,), generator=g)] + _codes(g, 2500, 64, 5)).to(torch.uint8)
    f = (centres[torch.randint(0, 40, (1800,), generator=g)] + _codes(g, 1800, 64, 5)).to(torch.uint8)
    f[:50] = r[100:150]
    cases.append(('d64', r, f, 5))
    for k, (nr, nf) in ((1, (300, 350)), (8, (420, 310))):
        r, f = _codes(g, nr, 64, 6), _codes(g, nf, 64, 6)
        f[:30] = r[:30]
        cases.append((f'k{k}', r, f, k))
    # zero radii: real row 0 repeated k + 1 times has radius 0 (below the median); fake rows 0 and 1 equal it, so their realism is
    # 0 / 0 = nan; fake row 2 equals real row 50, whose radius is positive, so its ratio is inf unless a nan wins
    r, f = _codes(g, 150, 32, 8), _codes(g, 120, 32, 8)
    r[1:6] = r[0]
    f[0] = f[1] = r[0]
    f[2] = r[50]
    cases.append(('zero', r, f, 5))
    return cases


def features(codes):
    return codes.to(torch.float64) / 16


# ------------------------------------------------------------------------------------------------ float64 restatement
def exact_d2(X, Y):
    """||X_i - Y_j||^2 [N_x, N_y] in float64 from the differences."""
    X, Y = X.double(), Y.double().to(X.device)
    out = torch.empty(X.shape[0], Y.shape[0], dtype=torch.float64, device=X.device)
    step = max(1, (1 << 24) // max(1, Y.shape[0] * Y.shape[1]))
    for i in range(0, X.shape[0], step):
        out[i:i + step] = ((X[i:i + step, None, :] - Y[None]) ** 2).sum(-1)
    return out


def sqrt(t):
    """Correctly rounded float64 sqrt, as numpy's and the GPU's (torch's vectorised CPU sqrt is not, in the last bit)."""
    return torch.from_numpy(np.sqrt(t.cpu().numpy())).to(t.device)


def radii(X, k):
    """The (k+1)-th smallest distance of each row to its own set (self distance 0 included): (radius, its squared distance)."""
    d2 = exact_d2(X, X).kthvalue(k + 1, dim=1).values
    return sqrt(d2), d2


def prdc(real, fake, k, realism=False):
    """compute_prdc in float64 with explicit differences; returns (the reference's dict, real radii, fake radii)."""
    r = radii(real, k)[0].cpu().numpy()
    s = radii(fake, k)[0].cpu().numpy()
    d = np.sqrt(exact_d2(real, fake).cpu().numpy())
    inside = d < r[:, None]
    out = dict(precision=inside.any(axis=0).mean(), recall=(d < s[None, :]).any(axis=1).mean(),
               density=(1. / float(k)) * inside.sum(axis=0).mean(), coverage=(d.min(axis=1) < r).mean())
    if realism:
        mask = r < np.median(r)
        with np.errstate(divide='ignore', invalid='ignore'):
            out['realism'] = (r[mask][:, None] / d[mask]).max(axis=0)
    return out, r, s


# ------------------------------------------------------------------------------------------------ plan interpreter ops
def _rows(mem, d, N_q):
    D = int(d.D)
    q = mem.view(d.q, torch.float64, N_q * D).reshape(N_q, D)
    t = mem.view(d.t, torch.float64, int(d.N) * D).reshape(int(d.N), D)
    return q, t


def _prdc_kth(mem, d):
    """The op in exact arithmetic: rad2 = the (k+1)-th smallest exact d2, rad = its sqrt; slice 0 of the partials becomes the
    approximate d2 (fp32).  nres (how many pairs the GPU recomputed) depends on the GEMM's rounding and is left as it is."""
    B, N, ldp, ns = int(d.B), int(d.N), int(d.ldp), int(d.nslice)
    q, t = _rows(mem, d, B)
    part = mem.view(d.part, torch.float32, ns * B * ldp).reshape(ns, B, ldp)
    qn2, tn2 = mem.view(d.qn2, torch.float64, B), mem.view(d.tn2, torch.float64, N)
    part[0, :, :N] = (qn2[:, None] + tn2[None] - 2 * part[:, :, :N].double().sum(0) / (float(d.sq) * float(d.st))).float()
    e = exact_d2(q, t).kthvalue(int(d.k) + 1, dim=1).values
    mem.view(d.rad2, torch.float64, B)[:] = e
    mem.view(d.rad, torch.float64, B)[:] = sqrt(e)


def _prdc_count(mem, d):
    B, N = int(d.B), int(d.N)
    q, t = _rows(mem, d, B)
    dist = sqrt(exact_d2(q, t))
    tau = mem.view(d.tau, torch.float64, N)
    mem.view(d.cnt_t, torch.int32, B)[:] = (dist < tau[None]).sum(1).to(torch.int32)
    if d.rho:
        rho = mem.view(d.rho, torch.float64, B)
        mem.view(d.cnt_own, torch.int32, B)[:] = (dist < rho[:, None]).sum(1).to(torch.int32)
    if d.realism:
        m = tau < float(d.med)
        mem.view(d.realism, torch.float64, B)[:] = (tau[m][None] / dist[:, m]).amax(1)      # x / 0 = inf, 0 / 0 = nan; amax keeps nan


PI._DISPATCH.update({S.DS_OP_PRDC_KTH: ('prdc_kth', _prdc_kth), S.DS_OP_PRDC_COUNT: ('prdc_count', _prdc_count)})


# ------------------------------------------------------------------------------------------------ host-side plans
class HostSets:
    """The real and fake sets in one host blob addressed as plan weights, laid out as B200PRDC lays them out on the device, with
    the output arrays; run() executes the radii plan and the score plan of prdc.compile_plan on the float64 interpreter."""

    def __init__(self, real, fake, k):
        self.k, self.D = k, real.shape[1]
        self.off, size = {}, 0
        self.sets = {}
        for name, x in (('r', real), ('f', fake)):
            N = x.shape[0]
            for buf, nbytes in (('planes', 2 * N * P._pad(self.D) * 2), ('rows', N * self.D * 8), ('n2', N * 8), ('rad', N * 8),
                                ('rad2', N * 8), ('cnt', N * 4), ('own', N * 4), ('realism', N * 8)):
                self.off[name + buf] = size
                size += -(-nbytes // 1024) * 1024
        self.blob = torch.zeros(size, dtype=torch.uint8)
        for name, x in (('r', real), ('f', fake)):
            x = x.double()
            scale = P.operand_scale(x)
            self._put(name + 'planes', P.split_rows(x, scale, P._pad(self.D)))
            self._put(name + 'rows', x)
            self._put(name + 'n2', (x * x).sum(1))
            self.sets[name] = P.SetRefs(x.shape[0], self.D, self.ref(name + 'planes'), self.ref(name + 'rows'), self.ref(name + 'n2'),
                                        self.ref(name + 'rad'), self.ref(name + 'rad2'), scale)

    def ref(self, name):
        return S.ref(S.SPACE_WEIGHTS, self.off[name])

    def _put(self, name, t):
        b = t.contiguous().reshape(-1).view(torch.uint8)
        self.blob[self.off[name]:self.off[name] + b.numel()] = b

    def get(self, mem, name, dtype, n):
        return mem.view(self.ref(name), dtype, n).clone()

    def run(self, realism):
        R, F = self.sets['r'], self.sets['f']
        radii_plan = P.compile_plan([('kth', R, 0)], self.D, self.k)
        mem = PI.Memory(0, bytes(self.blob.numpy()), {})
        plans = [radii_plan]
        mem.arena = torch.zeros(radii_plan.arena_bytes, dtype=torch.uint8)
        for i in range(radii_plan.n_ops):
            PI.run_op(mem, radii_plan.ops_array[i])
        rad = self.get(mem, 'rrad', torch.float64, R.N).numpy()
        med = float(np.median(rad))
        score_plan = P.compile_plan([('kth', F, 0),
                                     ('count', F, R, self.ref('fcnt'), 0, self.ref('frealism') if realism else 0, med, 0),
                                     ('count', R, F, self.ref('rcnt'), self.ref('rown'), 0, 0.0, 0)], self.D, self.k)
        plans.append(score_plan)
        mem.arena = torch.zeros(score_plan.arena_bytes, dtype=torch.uint8)
        for i in range(score_plan.n_ops):
            PI.run_op(mem, score_plan.ops_array[i])
        out = dict(radii=rad, fake_radii=self.get(mem, 'frad', torch.float64, F.N).numpy(),
                   cnt_f=self.get(mem, 'fcnt', torch.int32, F.N).numpy(), cnt_r=self.get(mem, 'rcnt', torch.int32, R.N).numpy(),
                   own_r=self.get(mem, 'rown', torch.int32, R.N).numpy(), plans=plans)
        if realism:
            out['realism'] = self.get(mem, 'frealism', torch.float64, F.N).numpy()
        return out

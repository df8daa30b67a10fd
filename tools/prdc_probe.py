"""Time B200PRDC on seeded Inception-like features (|randn|, D = 2048) at 10 000 and 50 000 rows per set, with a float64 eager-torch
comparator on the same card at 10 000 (torch.cdist in its direct-difference mode, kthvalue and the same comparisons).  Prints one JSON
line: the card (name, power limit, max SM clock, read in this run), per size the radii time, the score time, time per op type, GEMM
TFLOP/s in algorithmic FLOPs (2 N_q N_t D per product) and the rescored-pair count.

    python tools/prdc_probe.py [--sizes 10000,50000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diff_sampler_b200 import _cstructs as S    # noqa: E402
from diff_sampler_b200 import prdc as P         # noqa: E402

D, K = 2048, 5
OP_NAMES = {S.DS_OP_GEMM: 'gemm', S.DS_OP_PRDC_KTH: 'prdc_kth', S.DS_OP_PRDC_COUNT: 'prdc_count'}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, min_s=0.5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 0, 0.0
    while total < min_s * 1e3:
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
        n += 1
    return total / n, n


def features(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(n, D, generator=g, device='cuda').abs()


def eager(real, fake):
    """The reference's arithmetic in float64 eager torch: direct-difference distances, kthvalue radii, the same comparisons."""
    R, F = real.double(), fake.double()
    cd = lambda a, b: torch.cdist(a, b, compute_mode='donot_use_mm_for_euclid_dist')
    r = cd(R, R).kthvalue(K + 1, dim=1).values
    s = cd(F, F).kthvalue(K + 1, dim=1).values
    d = cd(R, F)
    inside = d < r[:, None]
    out = [inside.any(0).double().mean(), (d < s[None]).any(1).double().mean(), (1.0 / K) * inside.sum(0).double().mean(),
           (d.min(1).values < r).double().mean()]
    return [float(v) for v in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='10000,50000')
    args = ap.parse_args()
    res = dict(card=card(), D=D, nearest_k=K, sizes={})
    for n in (int(v) for v in args.sizes.split(',')):
        real, fake = features(n, 1), features(n, 2) * 1.02
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = P.B200PRDC(real, K)
        torch.cuda.synchronize()
        radii_s = time.perf_counter() - t0
        radii_pairs = m.last_rescored_pairs
        ms, reps = timed(lambda: m.score(fake))
        got = m.score(fake)
        per_op = {}
        for t, v in m.profile_score(fake):
            per_op[OP_NAMES.get(t, str(t))] = per_op.get(OP_NAMES.get(t, str(t)), 0.0) + v
        flops = 3 * 2.0 * n * n * D
        row = dict(radii_s=round(radii_s, 4), radii_rescored_pairs=radii_pairs, score_ms=round(ms, 3), score_reps=reps,
                   per_op_ms={k: round(v, 3) for k, v in per_op.items()}, gemm_tflops=round(flops / (per_op['gemm'] * 1e-3) / 1e12, 1),
                   rescored_pairs=m.last_rescored_pairs, scores={k: float(v) for k, v in got.items()})
        if n <= 10000:
            e_ms, e_reps = timed(lambda: eager(real, fake), min_s=0.5)
            ev = eager(real, fake)
            row['eager_fp64_ms'] = round(e_ms, 2)
            row['eager_reps'] = e_reps
            row['eager_scores'] = ev
        res['sizes'][n] = row
        del m, real, fake
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()

"""Measure the optimal denoiser (diff_sampler_b200.optimal) on a seeded synthetic CIFAR-shaped dataset: 50 000 structured images of
3 x 32 x 32 uint8 levels / 127.5 - 1 (tests/opt_ref.uint8_images).  Needs a CUDA device; prints one JSON document at the end (and
writes it to --out if given).

    python tools/optimal_probe.py [--out results.json] [--n 50000]

Reports, with the card name and power limit read in the same run:
  * ms per evaluation at B in {8, 64, 512} and sigma in {80, 5, 1, 0.002} (CUDA events over repeated calls, after warm-up), the
    algorithmic TFLOP/s of the two contractions (4 B N D / time) and the per-row status counts (GEMM logits / rescored / unrefined);
  * the per-op split of one evaluation from the plan profiler;
  * the status counts over a sigma sweep (where rescoring takes over from the GEMM logits), and the largest error against the float64
    oracle with the logit error bound E_row per sigma;
  * the same status / error sweep on a clustered set (500 prototypes x 100 variants within +-6 levels), where many keys compete;
  * optimal_sampler images/s at num_steps = 18;
  * an eager-PyTorch restatement of the reference's per-image loop (diff-analyzer-main/solvers.py:19-28) at B = 8 and 64, same GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from diff_sampler_b200 import _cstructs as S      # noqa: E402
from diff_sampler_b200 import optimal as OPT        # noqa: E402
import opt_ref as O                                 # noqa: E402

OP_NAMES = {S.DS_OP_OPT_PREP: 'opt_prep', S.DS_OP_GEMM: 'gemm', S.DS_OP_OPT_SOFTMAX: 'opt_softmax', S.DS_OP_OPT_REDUCE: 'opt_reduce'}


def card():
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        info['power_limit_and_max_sm_clock'] = q.stdout.strip()
    except Exception as e:                       # the measurement stands; the card line says why it is missing
        info['power_limit_and_max_sm_clock'] = f'unavailable: {e}'
    return info


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def reference_loop(x, t, ds):
    """The reference's get_denoised_opt, restated in eager PyTorch (per image: dataset - x[j], norms, softmax, weighted sum)."""
    out = []
    for j in range(x.shape[0]):
        l2 = torch.norm(ds - x[j].unsqueeze(0), p=2, dim=(1, 2, 3))
        w = torch.softmax(-l2 ** 2 / (2 * t ** 2), dim=0).reshape(-1, 1, 1, 1)
        out.append((ds * w).sum(dim=0))
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--n', type=int, default=50000)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    res = {'card': card()}
    y = O.uint8_images(args.n, 3, 32, 32, seed=1234).to(dev)
    N, D = y.shape[0], y[0].numel()
    t0 = time.time()
    den = OPT.B200OptimalDenoiser(y, device=dev)
    torch.cuda.synchronize()
    res['pack_s'] = time.time() - t0
    res['dataset'] = dict(N=N, D=D, packed_bytes=den.weight_bytes, chunk=den.chunk)
    g = torch.Generator(device=dev).manual_seed(0)
    evals = []
    for B in (8, 64, 512):
        idx = torch.randint(0, N, (B,), generator=g, device=dev)
        for sigma in (80.0, 5.0, 1.0, 0.002):
            x = (y[idx] + sigma * torch.randn(y[idx].shape, generator=g, device=dev)).contiguous()
            out = torch.empty_like(x)
            ms = time_ms(lambda: den(x, sigma, out=out), reps=20 if B < 512 else 10)
            st = den.last_row_status
            evals.append(dict(B=B, sigma=sigma, ms=ms, tflops=4.0 * B * N * D / (ms * 1e-3) / 1e12,
                              plain=int((st == 0).sum()), rescored=int((st == 1).sum()), unrefined=int((st == 2).sum())))
            print(evals[-1], flush=True)
    res['evals'] = evals
    prof = {}
    for B, sigma in ((64, 1.0), (512, 1.0), (512, 0.002)):
        x = (y[:B] + sigma * torch.randn(y[:B].shape, generator=g, device=dev)).contiguous()
        ops = den.profile_forward(x, sigma)
        prof[f'B{B}_sigma{sigma}'] = [(OP_NAMES.get(t, str(t)), ms) for t, ms in ops]
    res['per_op_ms'] = prof
    print(prof, flush=True)
    sweep = []
    idx = torch.randint(0, N, (512,), generator=g, device=dev)
    for sigma in (80.0, 30.0, 10.0, 5.0, 3.0, 2.0, 1.5, 1.0, 0.7, 0.5, 0.3, 0.2, 0.1, 0.05, 0.02, 0.01, 0.002):
        x = (y[idx] + sigma * torch.randn(y[idx].shape, generator=g, device=dev)).contiguous()
        den(x, sigma)
        st = den.last_row_status
        sweep.append(dict(sigma=sigma, plain=int((st == 0).sum()), rescored=int((st == 1).sum()), unrefined=int((st == 2).sum())))
    res['status_sweep_B512'] = sweep
    print(sweep, flush=True)
    errs = []
    idx = torch.randint(0, N, (64,), generator=g, device=dev)
    for sigma in (80.0, 10.0, 5.0, 2.0, 1.5, 1.0, 0.2, 0.05, 0.002):
        x = (y[idx] + sigma * torch.randn(y[idx].shape, generator=g, device=dev)).contiguous()
        got = den(x, sigma)
        st = den.last_row_status
        err = (got.double() - O.denoise_opt(x, sigma, y)).reshape(64, -1).abs().amax(dim=1)
        xn = x.double().reshape(64, -1).norm(dim=1)
        E = (xn + den.ymax) * (S.DS_OPT_EPS * den.ymax + D ** 0.5 * 2.0 ** -25) / sigma ** 2
        errs.append(dict(sigma=sigma, max_abs_err=err.max().item(), rescored=int((st == 1).sum()), E_row_max=E.max().item(),
                         E_row_min=E.min().item()))
    res['max_abs_err_vs_float64_B64'] = errs
    print(errs, flush=True)
    # clustered set: 500 structured prototypes x 100 variants within +-6 levels per value, so that many keys compete at mid sigma
    proto = O.uint8_images(500, 3, 32, 32, seed=99).to(dev)
    gv = torch.Generator(device=dev).manual_seed(98)
    lv = ((proto + 1) * 127.5).round().repeat_interleave(100, dim=0)
    lv = (lv + torch.randint(-6, 7, lv.shape, generator=gv, device=dev)).clamp(0, 255)
    yc = (lv / 127.5 - 1).contiguous()
    del lv
    denc = OPT.B200OptimalDenoiser(yc, device=dev)
    clus = []
    idx = torch.randint(0, yc.shape[0], (64,), generator=g, device=dev)
    for sigma in (80.0, 10.0, 5.0, 2.0, 1.0, 0.5, 0.3, 0.2, 0.1, 0.05, 0.02, 0.002):
        x = (yc[idx] + sigma * torch.randn(yc[idx].shape, generator=g, device=dev)).contiguous()
        got = denc(x, sigma)
        st = denc.last_row_status
        err = (got.double() - O.denoise_opt(x, sigma, yc)).reshape(64, -1).abs().amax(dim=1)
        un = st == 2
        clus.append(dict(sigma=sigma, plain=int((st == 0).sum()), rescored=int((st == 1).sum()), unrefined=int(un.sum()),
                         max_abs_err=err.max().item(), max_abs_err_unrefined=err[un].max().item() if un.any() else None))
    res['clustered_sweep_B64'] = clus
    print(clus, flush=True)
    del denc, yc
    samp = {}
    for B in (64, 512):
        lat = torch.randn(B, 3, 32, 32, generator=g, device=dev)
        OPT._CACHE.clear()
        OPT._CACHE[OPT._dataset_key(y) + (str(dev),)] = den
        ms = time_ms(lambda: OPT.optimal_sampler(None, lat, y, num_steps=18), reps=2)
        samp[B] = dict(ms=ms, images_per_s=B / (ms * 1e-3))
    res['optimal_sampler_18_steps'] = samp
    print(samp, flush=True)
    ref = {}
    for B in (8, 64):
        idx = torch.randint(0, N, (B,), generator=g, device=dev)
        x = (y[idx] + 1.0 * torch.randn(y[idx].shape, generator=g, device=dev)).contiguous()
        t = torch.tensor(1.0, device=dev)
        ms_ref = time_ms(lambda: reference_loop(x, t, y), reps=2)
        ms_nat = time_ms(lambda: den(x, 1.0), reps=10)
        err = (reference_loop(x, t, y) - den(x, 1.0)).abs().max().item()
        ref[B] = dict(eager_ms=ms_ref, native_ms=ms_nat, speedup=ms_ref / ms_nat, max_abs_diff=err)
    res['eager_reference_loop_sigma1'] = ref
    print(ref, flush=True)
    free, total = torch.cuda.mem_get_info(dev)
    res['device_memory_used_gib'] = (total - free) / 2 ** 30
    res['card_after'] = card()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()

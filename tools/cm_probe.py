#!/usr/bin/env python
"""Throughput of the Consistency-Models LSUN-256 denoiser (lsun_setting: the lsun_bedroom / lsun_cat nets) on seeded random weights.

    python tools/cm_probe.py [--batches 8,32] [--precisions fp16x3,fp16,fp16f8] [--seconds 1.0]

Prints the card (name, power limit, max SM clock, read in the same run), the algorithmic FLOPs of one forward computed from the
spec, and per (precision, batch): the plan's arena bytes, images/s of one forward and of a Heun sample (num_steps=6, its NFE
counted), from CUDA events around >= --seconds of back-to-back calls after warm-up.  One JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = 'name,power.limit,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(','), [x.strip() for x in out.splitlines()[0].split(',')]))
    except Exception as e:                       # the timings stand without it; say why it is missing
        return dict(error=repr(e))


def time_ms(fn, seconds):
    import torch
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 1
    while True:
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        total = a.elapsed_time(b)
        if total >= 1000 * seconds:
            return total / n
        n *= 2


def forward_flops(spec):
    """Multiply-adds x 2 of the convolutions, attention products and embedding layers of one image's forward."""
    R = spec.img_resolution
    f = 2 * R * R * 9 * spec.img_channels * spec.stem_cout
    for b in spec.enc + spec.dec:
        hw = b.res_out ** 2
        f += 2 * hw * 9 * (b.cin * b.cout + b.cout * b.cout)
        if b.skip == 'conv':
            f += 2 * hw * b.cin * b.cout
        if b.heads:
            f += 2 * hw * (3 * b.cout * b.cout + b.cout * b.cout) + 2 * 2 * hw * hw * b.cout
    f += 2 * R * R * 9 * spec.stem_cout * spec.img_channels
    f += 2 * (spec.noise_channels * spec.emb_channels + spec.emb_channels ** 2 + spec.emb_channels * spec.aff_total)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='8,32')
    ap.add_argument('--precisions', default='fp16x3,fp16,fp16f8')
    ap.add_argument('--seconds', type=float, default=1.0)
    ap.add_argument('--steps', type=int, default=6)
    args = ap.parse_args()
    import torch
    from diff_sampler_b200 import cm_net, solvers
    from diff_sampler_b200.net import B200Net
    assert torch.cuda.is_available(), 'this probe measures on a CUDA device'
    dev = torch.device('cuda:0')
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    spec, params = cm_net.convert(cm_net.init_state_dict(None, seed=0))
    flops = forward_flops(spec)
    print(json.dumps(dict(net='cm lsun_setting', gflop_per_image_forward=round(flops / 1e9, 1))), flush=True)
    for prec in args.precisions.split(','):
        net = B200Net(params, spec.img_resolution, spec.img_channels, 0, precision=prec, device=dev, spec=spec)
        for B in (int(b) for b in args.batches.split(',')):
            g = torch.Generator(device=dev).manual_seed(0)
            x = torch.randn(B, 3, 256, 256, device=dev, generator=g)
            sig = torch.tensor(2.5, device=dev)
            out = torch.empty_like(x)
            _, pl = net._plan(B, 1, 0)
            fwd = time_ms(lambda: net(x * 2.5, sig, out=out), args.seconds)
            calls = [0]

            class Counted:
                def __getattr__(self, k):
                    return getattr(net, k)

                def __call__(self, *a, **k):
                    calls[0] += 1
                    return net(*a, **k)
            solvers.heun_sampler(Counted(), x, num_steps=args.steps)
            nfe = calls[0]
            smp = time_ms(lambda: solvers.heun_sampler(net, x, num_steps=args.steps), args.seconds)
            print(json.dumps(dict(precision=prec, batch=B, arena_gib=round(pl.arena_bytes / 2 ** 30, 2), forward_ms=round(fwd, 2),
                                  forward_img_s=round(B / fwd * 1000, 1), forward_tflops=round(flops * B / fwd / 1e9, 1),
                                  heun_steps=args.steps, heun_nfe=nfe, sample_ms=round(smp, 1), sample_img_s=round(B / smp * 1000, 2))),
                  flush=True)
        del net
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()

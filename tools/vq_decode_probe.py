#!/usr/bin/env python
"""Timing of the VQ-f4 first-stage decode (the decoder of lsun_bedroom_ldm / ffhq_ldm: 3 x 64 x 64 latents -> 256 x 256 images,
8192 codes) on seeded weights.

    python tools/vq_decode_probe.py [--batch 16] [--seconds 0.5]

Prints the card, then per measurement ms per call from CUDA events around >= --seconds of back-to-back calls after warm-up:
the codebook search alone (the quantizing input op, one launch), and the whole decode with and without quantization, alternated
in rounds so that both see the same card state."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def gpu_info():
    q = 'name,power.limit,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(','), [x.strip() for x in out.splitlines()[0].split(',')]))
    except Exception as e:                       # the timings stand without it; say why it is missing
        return dict(error=repr(e))


def time_ms(fn, seconds):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 1, 0.0
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--seconds', type=float, default=0.5)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    import vq_ref as VQ
    from diff_sampler_b200 import _cstructs as S, _lib
    from diff_sampler_b200.vae_net import B200VAEDecoder
    assert torch.cuda.is_available(), 'this probe measures on a CUDA device'
    dev = torch.device('cuda:0')
    B, R = args.batch, 64
    P, cfg = VQ.make_params('vq_f4')
    vae = B200VAEDecoder(P, scale_factor=cfg['scale_factor'], device=dev)
    z = VQ.latents_near_codes(P, cfg, B, R, min_gap=0.0)[0].to(dev)

    x = z.reshape(B, 3, R * R)
    coef = torch.tensor([[0.0, 0.0, 1.0, 0.0]], device=dev)
    e = P['quantize.embedding.weight'].to(dev)
    o = torch.empty(2 * B * R * R * 64, dtype=torch.float16, device=dev)
    desc = S.PrepInputDesc(x=x.data_ptr(), coef=coef.data_ptr(), coef_stride=0, B=B, C=3, HW=R * R, nplanes=2, out=o.data_ptr(),
                           codebook=e.data_ptr(), n_embed=e.shape[0])
    res = dict(gpu=gpu_info(), batch=B, latent=R, n_embed=e.shape[0], quantize_op_ms=time_ms(lambda: _lib.op_launch(desc), args.seconds))
    res['quantize_op_gdist_per_s'] = B * R * R * e.shape[0] / (res['quantize_op_ms'] * 1e6)
    out = torch.empty(B, 3, 256, 256, device=dev)
    runs = {'decode_ms': [], 'decode_not_quantized_ms': []}
    for _ in range(args.rounds):
        runs['decode_ms'].append(time_ms(lambda: vae.decode(z, out=out), args.seconds))
        runs['decode_not_quantized_ms'].append(time_ms(lambda: vae.decode(z, out=out, force_not_quantize=True), args.seconds))
    for k, v in runs.items():
        res[k] = min(v)
        res[k + '_all'] = [round(t, 3) for t in v]
    res['images_per_s'] = B / (res['decode_ms'] / 1e3)
    print(json.dumps(res))


if __name__ == '__main__':
    main()

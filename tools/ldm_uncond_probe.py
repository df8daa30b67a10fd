"""Timing of the unconditional LSUN-Bedroom / FFHQ LDM-VQ-f4 eps-net (seeded weights of tests/ldm_uncond_ref.py; time does not depend
on their values) with CUDA events: forward images/s at batch 8 and 32 in fp16x3 and fp16, the per-op-type split, each attention launch
with head pairs against 64-padded heads, and a 224- against a 256-channel 3x3 convolution (the cost of the zero-filled channels).
Prints one JSON line with the card name, power limit and max SM clock read in the same run.

    python tools/ldm_uncond_probe.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import torch  # noqa: E402


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the probe measures on a CUDA device'
    import ldm_uncond_ref as U
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    from diff_sampler_b200 import gemm_desc as G
    from diff_sampler_b200.ldm_net import B200LDMNet
    dev = torch.device('cuda:0')
    P, cfg = U.make_params('ldm_vq4')
    res = dict(card=_card())
    names = {v: k for k, v in vars(S).items() if k.startswith('DS_OP_') and isinstance(v, int)}
    for prec in ('fp16x3', 'fp16'):
        for pairs in ((True, False) if prec == 'fp16x3' else (True,)):
            net = B200LDMNet(P, img_resolution=64, img_channels=3, guidance_type='uncond', num_head_channels=32, precision=prec,
                             head_pairs=pairs, device=dev)
            tag = f"{prec}{'' if pairs else ' padded heads'}"
            for B in (8, 32):
                x = torch.randn(B, 3, 64, 64, device=dev)
                sig = torch.tensor([2.0], device=dev)
                ms = _time(lambda: net(x, sig), args.iters)
                res[f'{tag} B{B} images/s'] = round(B / ms * 1e3, 1)
            split, per_op = net.profile_call(x, sig, None)
            res[f'{tag} B32 ms by op'] = {names.get(t, str(t)): [c, round(v, 3)] for t, (c, v) in split.items()}
            res[f'{tag} B32 attention launches ms'] = [round(ms_, 4) for t, _, ms_ in per_op if t == S.DS_OP_ATTN]
            del net
    # 3x3 conv at 32 x 32, batch 32: 224 channels (4 K blocks, the last half zero-filled) against 256
    for C in (224, 256):
        x = torch.randn(32, 32, 32, C, device=dev)
        xp = G.split_planes(x)
        wp = G.pack_conv_weight(torch.randn(224, C, 3, 3) * 0.02).to(dev)
        out = torch.empty(32 * 32 * 32, 224, device=dev)
        d, _ = G.conv_gemm(xp.data_ptr(), 32, 32, 32, C, wp.data_ptr(), 224, taps=9, out_f32=out.data_ptr())
        res[f'conv3x3 {C}->224 @32x32 x32 ms'] = round(_time(lambda: _lib.op_launch(d), args.iters * 5), 4)
    print(json.dumps(res))


if __name__ == '__main__':
    main()

"""Throughput of the native FID feature extractor (diff_sampler_b200.inception_net.B200InceptionV3) with CUDA events: images/s at
batch 250 for 32^2, 64^2, 256^2 and 512^2 uint8 inputs in fp16x3 and fp16, the same for torchvision's Inception3 with the TF graph's
pools (pytorch-fid's patches) in fp32 eager on the same GPU, and the arena of one 64-image chunk.  Prints one JSON line with the card
name, power limit and max SM clock read in the same run.

    python tools/inception_probe.py [--iters 5] [--weights pt_inception.pth] [--detector inception-2015-12-05.pkl]

--weights: a torchvision-layout state dict (pytorch-fid's pt_inception-2015-12-05-*.pth); default: seeded random weights (time does
not depend on their values).  --detector: NVIDIA's pickle; with --weights holding the same network, the max feature difference
between it and the native extractor is reported.
"""
import argparse
import json
import os
import pickle
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

SIZES = (32, 64, 256, 512)


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


def torch_detector(sd, dev):
    """torchvision Inception3 in fp32 eager with the TF graph's pools (averages without the padding, Mixed_7c's a max pool) and
    NVIDIA's resize (affine_grid / grid_sample): uint8 [B, 3, H, W] -> [B, 2048]."""
    import torchvision
    m = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=False, transform_input=False)
    m.load_state_dict(sd, strict=False)
    m.fc = torch.nn.Identity()
    m = m.to(dev).eval()
    state, avg = {'max': False}, F.avg_pool2d

    def pool(x, kernel_size, stride=None, padding=0, **kw):
        return F.max_pool2d(x, kernel_size, stride, padding) if state['max'] else avg(x, kernel_size, stride, padding, count_include_pad=False)
    m.Mixed_7c.register_forward_pre_hook(lambda *a: state.update(max=True))
    m.Mixed_7c.register_forward_hook(lambda *a: state.update(max=False))

    def run(x):
        B, C, H, W = x.shape
        theta = torch.eye(2, 3, device=dev)
        theta[0, 2] += 1.0 / W - 1.0 / 299
        theta[1, 2] += 1.0 / H - 1.0 / 299
        grid = F.affine_grid(theta.unsqueeze(0).repeat(B, 1, 1), [B, C, 299, 299], align_corners=False)
        y = (F.grid_sample(x.float(), grid, mode='bilinear', padding_mode='border', align_corners=False) - 128) / 128
        F.avg_pool2d, saved = pool, F.avg_pool2d
        try:
            with torch.no_grad():
                return m(y)
        finally:
            F.avg_pool2d = saved
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--batch', type=int, default=250)
    ap.add_argument('--weights', default=None)
    ap.add_argument('--detector', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the probe measures on a CUDA device'
    from diff_sampler_b200 import inception_plan as IP
    from diff_sampler_b200.inception_net import B200InceptionV3
    dev = torch.device('cuda:0')
    if args.weights:
        sd = torch.load(args.weights, map_location='cpu', weights_only=True)
    else:
        from oracle import inception_oracle as O
        sd = O.make_state_dict(0)
    res = dict(card=_card(), batch=args.batch, images_per_s={})
    g = torch.Generator().manual_seed(0)
    xs = {s: torch.randint(0, 256, (args.batch, 3, s, s), generator=g, dtype=torch.uint8).to(dev) for s in SIZES}
    for prec in ('fp16x3', 'fp16'):
        det = B200InceptionV3(sd, precision=prec)
        for s in SIZES:
            ms = _time(lambda: det(xs[s]), args.iters)
            res['images_per_s'][f'{prec} {s}'] = round(args.batch / ms * 1e3, 1)
        res[f'arena_MiB_per_64_images {prec}'] = round(det.arena_bytes(64, 256, 256) / 2 ** 20, 1)
        del det
        torch.cuda.empty_cache()
    ref = torch_detector(sd, dev)
    for s in SIZES:
        ms = _time(lambda: ref(xs[s]), args.iters)
        res['images_per_s'][f'torch fp32 {s}'] = round(args.batch / ms * 1e3, 1)
    if args.detector:
        if not args.weights:
            res['detector'] = 'skipped: --detector needs --weights holding the same network'
        elif not os.path.exists(args.detector):
            res['detector'] = f'skipped: {args.detector} not found'
        else:
            with open(args.detector, 'rb') as f:
                nv = pickle.load(f).to(dev)
            det = B200InceptionV3(sd)
            x = xs[256][:32]
            with torch.no_grad():
                want = nv(x, return_features=True).float()
            res['detector_max_abs_diff'] = (det(x) - want).abs().max().item()
            res['detector_max_abs_feature'] = want.abs().max().item()
    print(json.dumps(res))


if __name__ == '__main__':
    main()

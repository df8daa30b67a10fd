#!/usr/bin/env python
"""Per-shape timing of the GEMM kernel on the flagship plan (EDM CIFAR-10 DDPM++, batch 512, fp16f8).

    python tools/gemm_probe.py [--root TREE] [--batch 512] [--seconds 0.5] [--out FILE.json]

Every distinct GEMM configuration of the compiled plan is rebuilt by gemm_replay.make_desc on seeded device buffers and launched
alone, CUDA events around >= --seconds of back-to-back launches after warm-up.  Per shape: ms per launch, algorithmic TFLOP/s
(2 M N K), and the bytes the CTAs request from L2 into shared memory per launch (every ring stage of every tile: one A box and one
B box), with their rate.  The dominant shape is also run at BN = 128 and BN = 256: if its time followed those bytes rather than its
FLOPs, L2 bandwidth would be the limit.  --root imports the package and library from another checkout of this project (to compare
builds in one run); the configurations are always rebuilt by this checkout's gemm_replay, on top of that checkout's gemm_desc."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = 'name,power.limit,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(','), [x.strip() for x in out.splitlines()[0].split(',')]))
    except Exception as e:                       # the timings stand without it; say why it is missing
        return dict(error=repr(e))


def replay_module():
    """This checkout's gemm_replay, loaded into the imported package (which --root may take from an older checkout without it)."""
    import importlib.util
    name = 'diff_sampler_b200.gemm_replay'
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'diff-sampler_b200', 'gemm_replay.py'))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
    return sys.modules[name]


def plan_shapes(net, B, dev):
    """Distinct GEMM configurations of one forward (gemm_replay.GemmCfg -> launches per forward)."""
    import torch
    gemm_replay = replay_module()
    x = torch.randn(B, net.img_channels, net.img_resolution, net.img_resolution, device=dev)
    net(x, torch.tensor(2.0, device=dev))
    _, pl = next(iter(net._plans.values()))
    return gemm_replay.plan_configs(pl)


def l2_bytes(d):
    """Bytes the CTAs of one launch request from L2 into shared memory: per tile and ring stage one A box (128 rows x 128 B) and
    one B box (BN rows x 128 B)."""
    taps, cpb, c2 = int(d.taps), int(d.cpb), int(d.a2_c)
    nkb = taps * cpb + c2 // 64
    if d.f8 & 1:
        stages = 2 * (taps * ((cpb + 1) // 2) + (c2 + 127) // 128) + nkb
    else:
        stages = int(d.npass) * nkb
    tiles = int(d.m_tiles) * int(d.n_tiles) * max(int(d.num_z), 1)
    return tiles * stages * (128 * 128 + int(d.BN) * 128), stages


def time_launch(lib, d, seconds):
    import torch
    for _ in range(10):
        lib.op_launch(d)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        lib.op_launch(d)
    e1.record()
    torch.cuda.synchronize()
    n = max(20, int(seconds / (e0.elapsed_time(e1) / 10 / 1e3)) + 1)
    e0.record()
    for _ in range(n):
        lib.op_launch(d)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', default=ROOT, help='checkout whose package and library are probed')
    ap.add_argument('--batch', type=int, default=512)
    ap.add_argument('--seconds', type=float, default=0.5)
    ap.add_argument('--out', default=None, help='also write the rows as JSON here')
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from diff_sampler_b200 import _lib as L
    from diff_sampler_b200 import gemm_desc as G
    from diff_sampler_b200.net import B200Net
    make_desc = replay_module().make_desc
    assert torch.cuda.is_available(), 'the probe times kernels on a CUDA device'
    dev = torch.device('cuda:0')
    gpu = gpu_info()
    net = B200Net.from_config('cifar10', seed=0, dezero=True, precision='fp16f8', device=dev, fuse_stats=True, f8_min_channels=0)
    shapes = plan_shapes(net, args.batch, dev)
    del net
    torch.cuda.empty_cache()
    rows = []
    dom = None
    for key in shapes:
        d, info, keep = make_desc(key, dev)
        cfg = L.gemm_config(d) if hasattr(L, 'gemm_config') else None
        ms, n = time_launch(L, d, args.seconds)
        r = G.describe(d)
        by, stages = l2_bytes(d)
        row = dict(label=r['label'], BN=int(d.BN), launches_per_forward=shapes[key], ms=ms, timed_launches=n,
                   tflops=r['flops'] / (ms / 1e3) / 1e12, k_stages_per_tile=stages, l2_smem_bytes=by, l2_smem_tbs=by / (ms / 1e3) / 1e12,
                   ring_stages=cfg['stages'] if cfg else None, grid=cfg['grid'] if cfg else None,
                   fwd_ms=ms * shapes[key])
        rows.append(row)
        del keep
        if dom is None or row['fwd_ms'] > dom[1]['fwd_ms']:
            dom = (key, row)
    if dom is not None:
        for bn in (128, 256):
            d, info, keep = make_desc(dom[0], dev, bn)
            cfg = L.gemm_config(d) if hasattr(L, 'gemm_config') else None
            ms, n = time_launch(L, d, args.seconds)
            r = G.describe(d)
            by, stages = l2_bytes(d)
            rows.append(dict(label=r['label'] + f' (dominant, bn={bn})', BN=bn, launches_per_forward=0, ms=ms, timed_launches=n,
                             tflops=r['flops'] / (ms / 1e3) / 1e12, k_stages_per_tile=stages, l2_smem_bytes=by,
                             l2_smem_tbs=by / (ms / 1e3) / 1e12, ring_stages=cfg['stages'] if cfg else None,
                             grid=cfg['grid'] if cfg else None, fwd_ms=0.0,
                             bytes_per_flop=by / r['flops']))
            del keep
    print(json.dumps(dict(gpu=gpu, root=os.path.abspath(args.root), batch=args.batch)))
    hdr = f"{'shape':58s} {'BN':>4s} {'n/fwd':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'L2 MB':>8s} {'TB/s':>6s} {'stg':>4s} {'grid':>5s}"
    print(hdr)
    for r in rows:
        print(f"{r['label'][:58]:58s} {r['BN']:4d} {r['launches_per_forward']:5d} {r['ms']:8.4f} {r['tflops']:8.1f} {r['l2_smem_bytes'] / 1e6:8.1f} "
              f"{r['l2_smem_tbs']:6.2f} {str(r['ring_stages']):>4s} {str(r['grid']):>5s}")
    print(f"sum over the plan's shapes: {sum(r['fwd_ms'] for r in rows):.2f} ms of GEMM time per forward (each shape timed alone)")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(dict(gpu=gpu, root=os.path.abspath(args.root), batch=args.batch, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()

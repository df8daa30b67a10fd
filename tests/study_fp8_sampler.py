"""Numerics study (CPU, not a test): final-image error of the f8 GEMM mode on the configuration that misses the 1e-3 gate on the GPU
(FFHQ-64, iPNDM NFE=6 with every block in f8), emulated inside the CPU oracle, with the f8 mode in
all block convolutions and only in those with at least 256 input and output channels (`B200Net(f8_min_channels=256)`).

    python tests/study_fp8_sampler.py

Measured here (batch 4; the max over 256 images is ~1.45x larger):  fp16x3 4.0e-5,  f8 everywhere 7.5e-4,  f8 >= 256 channels 3.8e-4.
"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import study_fp8_corrections as St
from oracle import edm_oracle as O, solvers_oracle as SO
torch.set_num_threads(8)
name, solver, kw = 'ffhq', 'ipndm', dict(num_steps=7, max_order=4)
P, S = O.make_net(name, seed=0, dezero=True)
net = O.OracleNet(P, S)
B = 4
lat = O.stacked_randn(range(B), (3, 64, 64))
f8c, x3c = St.make_conv('fp16+f8'), St.make_conv('fp16x3')
def mk(thr):
    def conv2d(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
        if groups != 1:
            return St._real_conv2d(x, w, bias, stride, padding, dilation, groups)
        use8 = thr is not None and min(w.shape[0], w.shape[1]) >= thr and w.shape[1] >= 64
        return (f8c if use8 else x3c)(x, w, bias, stride, padding, dilation, groups)
    return conv2d
with torch.no_grad():
    ref = SO.sample(net, lat, solver, **kw)
    for label, thr in (('fp16x3', None), ('f8 all', 0), ('f8 >= 256', 256)):
        O.F.conv2d = mk(thr)
        t0 = time.time()
        got = SO.sample(net, lat, solver, **kw)
        O.F.conv2d = St._real_conv2d
        print(f'{name} {solver} NFE=6 batch {B}: {label:10s} final-image max-abs vs fp32 {(got - ref).abs().max().item():.3e}  ({time.time() - t0:.0f}s)', flush=True)

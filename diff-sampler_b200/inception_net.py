"""B200InceptionV3 — the FID feature extractor, native: TensorFlow's `inception-2015-12-05` graph that fid.py loads as
`inception-2015-12-05.pkl` and calls as `detector_net(images, return_features=True)`, with the same call signature, so
`fid_stats.FeatureStats.append_images(images, det)` and fid.py-style loops take it unchanged.  See inception_plan.py, DESIGN.md 4.10.

    det = B200InceptionV3(state_dict)                      # torchvision Inception3 layout, e.g. pytorch-fid's pt_inception-2015-12-05
    det = B200InceptionV3.from_torchvision(module)         # or straight from a torchvision / pytorch-fid Inception3 module
    feats = det(images_u8)                                 # [B, 3, H, W] uint8 on the GPU -> [B, 2048] fp32
"""
import torch

from . import _lib
from . import inception_plan
from .net import PRECISIONS, default_cuda_graph


class B200InceptionV3:
    def __init__(self, state_dict, precision='fp16x3', max_batch=64, device='cuda', cuda_graph=None):
        """state_dict: torchvision `Inception3` layout (fc.*, AuxLogits.* and num_batches_tracked are ignored).  Batches larger than
        `max_batch` run in chunks of at most that many images, which bounds the arena (arena_bytes())."""
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200InceptionV3 needs a CUDA device (no CPU fallback)')
        if precision not in ('fp16x3', 'fp16'):
            raise ValueError(f'precision {precision!r}: the Inception detector runs fp16x3 or fp16')
        missing = [k for k in inception_plan.required_keys() if k not in state_dict]
        if missing:
            raise KeyError(f'Inception3 state dict lacks {len(missing)} keys: {missing}')
        if max_batch < 1:
            raise ValueError(f'max_batch must be positive, got {max_batch}')
        self.lib = _lib.load()
        self.precision, self.npass, self.max_batch = precision, PRECISIONS[precision], int(max_batch)
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        sd = {k: state_dict[k].detach().cpu() for k in inception_plan.required_keys()}
        self.wb = inception_plan.pack_inception_weights(sd)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self.total_launches = 0

    @classmethod
    def from_torchvision(cls, module, **kw):
        """A torchvision `Inception3` (or pytorch-fid's `FIDInceptionA/C/E` variant of it): its weights; the TF graph's pools are this
        class's own."""
        return cls(module.state_dict(), **kw)

    def plan(self, B, H, W, strides):
        """(handle, plan) for B images of H x W with element strides (sn, sc, sy, sx)."""
        key = (B, H, W, strides)
        return self.native.get(key, lambda: inception_plan.compile_inception_plan(self.wb, B, H, W, self.npass, strides),
                               (lambda pl: (B * 3 * H * W, B * inception_plan.FEATURES * 4, 0, 0, 0, 0)) if self.cuda_graph else None)

    def __call__(self, images, return_features=True):
        """images: uint8 [B, 3, H, W] on the device, any layout whose elements fill one dense block (contiguous NCHW, or the
        permute(0, 3, 1, 2) view of NHWC samples) -> pool3 features [B, 2048] fp32."""
        if not return_features:
            raise NotImplementedError('B200InceptionV3 computes the pool3 features FID uses; the logits (Inception Score) are not implemented')
        if images.device.type != 'cuda':
            raise _lib.DsError('B200InceptionV3: images must live on the CUDA device (no CPU fallback)')
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f'expected uint8 images [B, 3, H, W], got {images.dtype} {tuple(images.shape)}')
        B, _, H, W = images.shape
        if not _dense(images):
            images = images.contiguous()
        out = torch.empty(B, inception_plan.FEATURES, dtype=torch.float32, device=images.device)
        stream = torch.cuda.current_stream(images.device).cuda_stream
        strides = tuple(int(s) for s in images.stride())
        for b0 in range(0, B, self.max_batch):
            n = min(self.max_batch, B - b0)
            h, _ = self.plan(n, H, W, strides)
            io = (images.data_ptr() + b0 * strides[0], out[b0].data_ptr(), None, None, None, None)
            self.total_launches += self.native.run(h, io, stream)
        return out

    def arena_bytes(self, B, H, W):
        """Workspace of the plan for B images of H x W (compiled on first use)."""
        return self.plan(B, H, W, (3 * H * W, H * W, W, 1))[1].arena_bytes


def _dense(x):
    """Whether each image's elements fill one block of C*H*W elements (any order of c, y, x) and the images follow each other, so that
    a chunk of the batch is one byte range (the staged input copy of a CUDA-graph replay takes it whole)."""
    B, Cc, H, W = x.shape
    expect = 1
    for s, n in sorted((s, n) for s, n in zip(x.stride()[1:], x.shape[1:]) if n > 1):
        if s != expect:
            return False
        expect *= n
    return B == 1 or x.stride(0) == Cc * H * W

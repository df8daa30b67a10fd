"""B200Net — the native denoiser behind the reference's `net(x, sigma, class_labels=...)` contract.

Drop-in for models.networks_edm.EDMPrecond (networks_edm.py:459-500): same call signature and the attributes the
samplers and sample.py read (img_resolution, img_channels, label_dim, sigma_min, sigma_max, sigma_data, round_sigma).
All arithmetic runs in hand-written sm_90a kernels through the C ABI; there is no PyTorch/CPU fallback.
"""
import ctypes as C
from collections import OrderedDict

import torch

from . import _lib
from . import edm_nets
from . import plan as planner

# precision -> MMA passes per product.  'fp16f8': the block convolutions (98 % of the FLOPs) run hi x hi in fp16 and the two 2^-11
# correction products as e4m3 MMAs at twice the rate (2 MMA units per product instead of 3, csrc/ops.h); everything else is fp16x3.
PRECISIONS = {'fp16x3': 3, 'fp16': 1, 'fp16f8': 3}


def default_precision():
    """Precision of a B200Net built without an explicit `precision=`; the environment variable DSB_PRECISION overrides it."""
    import os
    p = os.environ.get('DSB_PRECISION', 'fp16x3')
    if p not in PRECISIONS:
        raise ValueError(f'DSB_PRECISION={p!r}: expected one of {sorted(PRECISIONS)}')
    return p


def default_cuda_graph():
    """Replay each denoiser evaluation as ONE CUDA graph (ds_unet_enable_graph) unless DSB_CUDA_GRAPH=0."""
    import os
    return os.environ.get('DSB_CUDA_GRAPH', '1') != '0'


class B200Net:
    def __init__(self, params, img_resolution, img_channels, label_dim=0, sigma_min=0.002, sigma_max=80.0, sigma_data=0.5,
                 precision=None, device='cuda', fuse_stats=True, flash_attn=True, f8_min_channels=None, cuda_graph=None, spec=None):
        self.device = torch.device(device)
        precision = precision or default_precision()
        if self.device.type != 'cuda':
            raise _lib.DsError('B200Net needs a CUDA device (no CPU fallback)')
        self.lib = _lib.load()
        self.img_resolution, self.img_channels, self.label_dim = img_resolution, img_channels, label_dim
        self.sigma_min, self.sigma_max, self.sigma_data = sigma_min, sigma_max, sigma_data
        self.precision = precision
        self.npass = PRECISIONS[precision]
        self.f8 = precision == 'fp16f8'
        if f8_min_channels is None:
            import os
            f8_min_channels = int(os.environ.get('DSB_F8_MIN_CHANNELS', '0'))
        self.f8_min_channels = int(f8_min_channels)          # fp16f8 only: blocks narrower than this stay fp16x3 (plan.pack_weights)
        self.fuse_stats = bool(fuse_stats)
        self.flash_attn = bool(flash_attn)
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        # spec: the block structure when the parameter names cannot carry it (Consistency-Models nets, cm_net.py)
        self.spec = spec if spec is not None else edm_nets.spec_from_params(params, img_resolution, img_channels, label_dim)
        self.spec.sigma_data = sigma_data
        self.wb, self.winfo = planner.pack_weights(self.spec, params, f8=self.f8, f8_min_channels=self.f8_min_channels)
        blob = self.wb.bytes()
        self.native = _lib.NativePlans(blob, self.device)
        self.weight_bytes = len(blob)
        self.launches_last_forward = 0
        self.total_launches = 0

    # ---- construction helpers ---------------------------------------------------------------------------------------
    @classmethod
    def from_config(cls, name, seed=0, dezero=False, **kw):
        params, cfg = edm_nets.init_params(name, seed=seed)
        if dezero:
            edm_nets.dezero_(params, cfg['kind'], seed=seed)
        return cls(params, cfg['img_resolution'], cfg['img_channels'], cfg.get('label_dim', 0), **kw)

    @classmethod
    def from_reference(cls, net, **kw):
        """Compile a reference EDMPrecond module (or anything with the same state_dict layout and attributes)."""
        sd = OrderedDict((k, v) for k, v in net.state_dict().items() if 'resample_filter' not in k)
        return cls(sd, net.img_resolution, net.img_channels, net.label_dim, sigma_min=float(net.sigma_min),
                   sigma_max=float(net.sigma_max), sigma_data=float(getattr(net, 'sigma_data', 0.5)), **kw)

    @classmethod
    def from_pickle(cls, f, key='ema', **kw):
        """Load an EDM `network-snapshot-*.pkl` (what sample.py:81-82 feeds to `pickle.load(f)['ema']`) without the reference's
        torch_utils / dnnlib on the path and without executing the source embedded in the file (checkpoint.py).  The reference then sets
        `net.sigma_min = 0.002; net.sigma_max = 80.0` (sample.py:83-84); pass other values through `kw` if needed."""
        from . import checkpoint
        params, meta = checkpoint.load_edm_pickle(f, key=key)
        kw.setdefault('sigma_min', 0.002)
        kw.setdefault('sigma_max', 80.0)
        kw.setdefault('sigma_data', meta['sigma_data'])
        net = cls(params, meta['img_resolution'], meta['img_channels'], meta['label_dim'], **kw)
        net.checkpoint_meta = meta
        return net

    @classmethod
    def from_cm(cls, net, setting=None, **kw):
        """Compile a reference CMPrecond module (networks_edm.py:504-549) around a Consistency-Models UNetModel built with `setting`
        (default: cm_model_loader.lsun_setting(), the lsun_bedroom / lsun_cat nets)."""
        from . import cm_net
        if getattr(net, 'label_dim', 0):
            raise ValueError('label_dim: class-conditional CM nets are not lowered')
        spec, params = cm_net.convert(net.state_dict(), setting, prefix='model.')
        if int(net.img_resolution) != spec.img_resolution:
            raise ValueError(f'img_resolution={net.img_resolution} does not match the settings ({spec.img_resolution})')
        return cls(params, spec.img_resolution, spec.img_channels, 0, sigma_min=float(net.sigma_min), sigma_max=float(net.sigma_max),
                   sigma_data=float(net.sigma_data), spec=spec, **kw)

    @classmethod
    def from_cm_checkpoint(cls, f, setting=None, **kw):
        """Load a released Consistency-Models checkpoint (edm_bedroom256_ema.pt, edm_cat256_ema.pt: a UNetModel state dict) from a path
        or file object, with torch.load(weights_only=True), and wrap it as sample.py does (CMPrecond defaults: sigma in [0.002, 80],
        sigma_data 0.5)."""
        from . import cm_net
        sd = torch.load(f, map_location='cpu', weights_only=True)
        spec, params = cm_net.convert(sd, setting)
        for k, v in (('sigma_min', 0.002), ('sigma_max', 80.0), ('sigma_data', 0.5)):
            kw.setdefault(k, v)
        return cls(params, spec.img_resolution, spec.img_channels, 0, spec=spec, **kw)

    # ---- plan cache -------------------------------------------------------------------------------------------------
    @property
    def _plans(self):
        return self.native.plans

    def _plan(self, B, nsig, nlab):
        img = B * self.img_channels * self.img_resolution ** 2 * 4
        return self.native.get((B, nsig, nlab),
                               lambda: planner.compile_plan(self.spec, self.wb, self.winfo, B, nsig, nlab, npass=self.npass,
                                                            fuse_stats=self.fuse_stats, flash_attn=self.flash_attn, f8=self.f8),
                               (lambda pl: (img, img, nsig * 4, nlab * self.label_dim * 4, B * 64 * 4, 0)) if self.cuda_graph else None)

    # ---- the reference-facing call ----------------------------------------------------------------------------------
    def __call__(self, x, sigma, class_labels=None, out=None, bottleneck=None, **_):
        if x.device.type != 'cuda':
            raise _lib.DsError('B200Net: input must live on the CUDA device (no CPU fallback)')
        x = x.to(torch.float32).contiguous()
        B = x.shape[0]
        sig = torch.as_tensor(sigma, dtype=torch.float32, device=x.device).reshape(-1)
        if not sig.is_contiguous():
            sig = sig.contiguous()
        if sig.numel() not in (1, B):
            raise ValueError(f'sigma must have 1 or {B} elements, got {sig.numel()}')
        nsig = sig.numel() if sig.numel() == B and B > 1 else 1
        lab = None
        nlab = 0
        if self.label_dim:
            if class_labels is None:
                lab = torch.zeros([1, self.label_dim], device=x.device)          # networks_edm.py:485
            else:
                lab = class_labels.to(torch.float32).reshape(-1, self.label_dim).contiguous()
            nlab = lab.shape[0]
            if nlab not in (1, B):
                raise ValueError('class_labels batch mismatch')
        h, pl = self._plan(B, nsig, nlab)
        if out is None:
            out = torch.empty_like(x)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        self.launches_last_forward = self.native.run(h, (x.data_ptr(), out.data_ptr(), sig.data_ptr(), lab.data_ptr() if lab is not None else None,
                                                         bottleneck.data_ptr() if bottleneck is not None else None, None), stream)
        self.total_launches += self.launches_last_forward
        return out

    def profile_forward(self, x, sigma, class_labels=None):
        """One forward with per-op CUDA-event timing.  Returns {op_type: (count, total_ms)} (bench.py roofline leg)."""
        B = x.shape[0]
        self(x, sigma, class_labels)                                     # make sure the plan exists / warm
        sig = torch.as_tensor(sigma).reshape(-1)
        nsig = sig.numel() if sig.numel() == B and B > 1 else 1
        nlab = 0 if not self.label_dim else (1 if class_labels is None else class_labels.reshape(-1, self.label_dim).shape[0])
        h, pl = self._plan(B, nsig, nlab)
        _lib.check(self.lib.ds_unet_set_profiling(h, 1), 'ds_unet_set_profiling')
        self(x, sigma, class_labels)
        buf = (C.c_float * pl.n_ops)()
        n = self.lib.ds_unet_get_profile(h, buf, pl.n_ops)
        self.lib.ds_unet_set_profiling(h, 0)
        out = {}
        for i in range(n):
            t = self.lib.ds_unet_op_type(h, i)
            c, ms = out.get(t, (0, 0.0))
            out[t] = (c + 1, ms + buf[i])
        self.last_profile = ([float(buf[i]) for i in range(n)], pl)          # per-op milliseconds + the plan they index
        return out

    def round_sigma(self, sigma):
        return torch.as_tensor(sigma)

    def debug_read(self, B, nsig, nlab, name, numel, dtype=torch.float32):
        """Copy a named workspace buffer of the plan for (B, nsig, nlab) to the host (tests only)."""
        self._plan(B, nsig, nlab)
        return self.native.debug_read((B, nsig, nlab), name, numel, dtype)

    # torch.nn.Module-ish conveniences used by sample.py-style callers
    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def requires_grad_(self, *_a, **_k):
        return self

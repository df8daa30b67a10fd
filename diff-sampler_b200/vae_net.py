"""B200VAEDecoder — native `decode_first_stage` of the latent-diffusion models (sample.py:299; ddpm.py:707-760, AutoencoderKL path):
images = Decoder(post_quant_conv(z / scale_factor)).  OPT-IN, not yet run on hardware (see vae_plan.py); SURVEY section 8(f)3.

    vae = B200VAEDecoder.from_reference(net.model)            # net.model: the LatentDiffusion object behind CFGPrecond
    images = vae.decode(latents)                              # instead of net.model.decode_first_stage(latents)
"""
from collections import OrderedDict

import torch

from . import _lib
from . import vae_plan
from .net import PRECISIONS


class B200VAEDecoder:
    def __init__(self, params, scale_factor=0.18215, precision='fp16x3', device='cuda'):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200VAEDecoder needs a CUDA device (no CPU fallback)')
        self.lib = _lib.load()
        self.scale_factor = float(scale_factor)
        if precision not in ('fp16x3', 'fp16'):
            raise ValueError(f'precision {precision!r}: the VAE decoder runs fp16x3 or fp16')
        self.npass = PRECISIONS[precision]
        self.mods, self.meta = vae_plan.vae_structure(params)
        self.wb = vae_plan.pack_vae_weights(self.mods, self.meta, params)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self._coef = torch.tensor([[0.0, 0.0, 1.0 / self.scale_factor, 0.0]], device=self.device)
        self.total_launches = 0

    @classmethod
    def from_reference(cls, ldm_model, **kw):
        """`ldm_model`: the reference LatentDiffusion (has `.first_stage_model` and `.scale_factor`, ddpm.py:424-470)."""
        sd = OrderedDict((k, v) for k, v in ldm_model.first_stage_model.state_dict().items()
                         if k.startswith('decoder.') or k.startswith('post_quant_conv.'))
        return cls(sd, scale_factor=float(ldm_model.scale_factor), **kw)

    def _plan(self, B, R):
        return self.native.get((B, R), lambda: vae_plan.compile_vae_plan(self.mods, self.meta, self.wb, B, R, npass=self.npass))

    def decode(self, z, out=None):
        """z: [B, z_channels, R, R] latents as the samplers return them -> images [B, out_ch, s R, s R] (fp32, NCHW)."""
        if z.device.type != 'cuda':
            raise _lib.DsError('B200VAEDecoder: input must live on the CUDA device (no CPU fallback)')
        z = z.to(torch.float32).contiguous()
        B, Cz, R, R2 = z.shape
        if R != R2 or Cz != self.meta['embed_dim']:
            raise ValueError(f'expected square latents with {self.meta["embed_dim"]} channels, got {tuple(z.shape)}')
        h, pl = self._plan(B, R)
        s = self.meta['upscale']
        if out is None:
            out = torch.empty(B, self.meta['out_ch'], R * s, R * s, device=z.device)
        io = (z.data_ptr(), out.data_ptr(), None, self._coef.data_ptr(), None, None)
        self.total_launches += self.native.run(h, io, torch.cuda.current_stream(z.device).cuda_stream)
        return out

    decode_first_stage = decode          # the reference's method name (ddpm.py:707)

    def debug_read(self, B, R, name, numel, dtype=torch.float32):
        self._plan(B, R)
        return self.native.debug_read((B, R), name, numel, dtype)

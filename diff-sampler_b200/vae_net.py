"""B200VAEDecoder — native `decode_first_stage` of the latent-diffusion models (sample.py:299; ddpm.py:707-760):
images = Decoder(post_quant_conv(z / scale_factor)) for an AutoencoderKL first stage (Stable Diffusion), and
images = Decoder(post_quant_conv(quantize(z / scale_factor))) for a VQModelInterface one (the VQ-f4 of `lsun_bedroom_ldm` / `ffhq_ldm`,
autoencoder.py:274-282), where quantize snaps every latent pixel to its nearest codebook row.  See vae_plan.py; SURVEY section 8(f)3.

    vae = B200VAEDecoder.from_reference(net.model)            # net.model: the LatentDiffusion object behind CFGPrecond
    images = vae.decode(latents)                              # instead of net.model.decode_first_stage(latents)
"""
from collections import OrderedDict

import torch

from . import _lib
from . import vae_plan
from .net import PRECISIONS


class B200VAEDecoder:
    def __init__(self, params, scale_factor=0.18215, precision='fp16x3', device='cuda', debug_indices=False):
        """params: the first stage's state dict (decoder.*, post_quant_conv.* and, for a VQ first stage, quantize.embedding.weight).
        debug_indices: VQ first stages also keep the chosen codebook rows, readable with debug_read(B, R, 'vq_idx', B*R*R, torch.int32)."""
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200VAEDecoder needs a CUDA device (no CPU fallback)')
        self.lib = _lib.load()
        self.scale_factor = float(scale_factor)
        if precision not in ('fp16x3', 'fp16'):
            raise ValueError(f'precision {precision!r}: the VAE decoder runs fp16x3 or fp16')
        self.npass = PRECISIONS[precision]
        self.mods, self.meta = vae_plan.vae_structure(params)
        self.is_vq = 'n_embed' in self.meta
        self.debug_indices = bool(debug_indices)
        self.wb = vae_plan.pack_vae_weights(self.mods, self.meta, params)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self._coef = torch.tensor([[0.0, 0.0, 1.0 / self.scale_factor, 0.0]], device=self.device)
        self.total_launches = 0

    @classmethod
    def from_reference(cls, ldm_model, **kw):
        """`ldm_model`: the reference LatentDiffusion (has `.first_stage_model` and `.scale_factor`, ddpm.py:424-470); its first stage
        may be an AutoencoderKL or a VQModelInterface."""
        sd = OrderedDict((k, v) for k, v in ldm_model.first_stage_model.state_dict().items()
                         if k.startswith('decoder.') or k.startswith('post_quant_conv.') or k == 'quantize.embedding.weight')
        return cls(sd, scale_factor=float(ldm_model.scale_factor), **kw)

    def _plan(self, B, R, force_not_quantize=False):
        q = self.is_vq and not force_not_quantize
        return self.native.get((B, R, q), lambda: vae_plan.compile_vae_plan(self.mods, self.meta, self.wb, B, R, npass=self.npass, quantize=q,
                                                                             debug_indices=q and self.debug_indices))

    def decode(self, z, out=None, force_not_quantize=False):
        """z: [B, z_channels, R, R] latents as the samplers return them -> images [B, out_ch, s R, s R] (fp32, NCHW).
        force_not_quantize: a VQ first stage decodes z as given, without snapping it to the codebook (ddpm.py:761-762); an
        AutoencoderKL has no codebook and ignores it, as the reference does."""
        if z.device.type != 'cuda':
            raise _lib.DsError('B200VAEDecoder: input must live on the CUDA device (no CPU fallback)')
        z = z.to(torch.float32).contiguous()
        B, Cz, R, R2 = z.shape
        if R != R2 or Cz != self.meta['embed_dim']:
            raise ValueError(f'expected square latents with {self.meta["embed_dim"]} channels, got {tuple(z.shape)}')
        h, pl = self._plan(B, R, force_not_quantize)
        s = self.meta['upscale']
        if out is None:
            out = torch.empty(B, self.meta['out_ch'], R * s, R * s, device=z.device)
        io = (z.data_ptr(), out.data_ptr(), None, self._coef.data_ptr(), None, None)
        self.total_launches += self.native.run(h, io, torch.cuda.current_stream(z.device).cuda_stream)
        return out

    decode_first_stage = decode          # the reference's method name (ddpm.py:707)

    def debug_read(self, B, R, name, numel, dtype=torch.float32, force_not_quantize=False):
        q = self.is_vq and not force_not_quantize
        self._plan(B, R, force_not_quantize)
        return self.native.debug_read((B, R, q), name, numel, dtype)

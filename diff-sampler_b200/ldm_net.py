"""B200LDMNet — native drop-in for the reference's `CFGPrecond` wrapper around a latent-diffusion eps-net
(networks_edm.py:630-759) around a latent-diffusion eps-net: Stable Diffusion v1.x with classifier-free guidance, or the unconditional
LSUN-Bedroom / FFHQ LDM-VQ-f4 `UNetModel` (guidance_type='uncond').  Same call contract:
    net(x, sigma, condition=..., unconditional_condition=...) -> D = x - sigma * eps_cfg
and the attributes the samplers / schedules read (guidance_type, guidance_rate, img_resolution, img_channels, label_dim,
sigma_min, sigma_max, sigma(), sigma_inv(), round_sigma()).  The eps-net runs in the hand-written kernels (ldm_plan.py);
the sigma <-> t interpolation over the 1000 log-alpha knots is a few scalar torch ops on the device.
"""
import ctypes as C
from collections import OrderedDict

import torch

from . import _cstructs as S
from . import _lib
from . import ldm_plan
from .net import PRECISIONS, default_cuda_graph, default_precision
from .solver_utils import solver_update


def make_alphas_cumprod(linear_start=0.00085, linear_end=0.0120, n=1000):
    """'linear' beta schedule of v1-inference.yaml:5-6 (sqrt-space linspace, squared)."""
    betas = torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0).to(torch.float32)


UNCOND_BETAS = (0.0015, 0.0195)       # linear_start / linear_end of lsun_bedrooms-ldm-vq-4.yaml and ffhq-ldm-vq-4.yaml


def load_ldm_checkpoint(path):
    """The released LDM `model.ckpt` (a LatentDiffusion state dict under 'state_dict') read with torch.load(weights_only=True), never
    unpickled further -> (eps-net state dict (`model.diffusion_model.*`), VQ first-stage decoder state dict (`first_stage_model.`
    decoder / post_quant_conv / codebook), alphas_cumprod or None, scale_factor)."""
    import pickle
    try:
        ck = torch.load(path, map_location='cpu', weights_only=True)
    except pickle.UnpicklingError as e:
        raise ValueError(f'{path}: not loadable with torch.load(weights_only=True); it is not unpickled any further, since a full '
                         f'unpickle can run arbitrary code.  Re-save its state_dict alone to use it here.  ({e})') from None
    if not isinstance(ck, dict) or not isinstance(ck.get('state_dict'), dict):
        raise ValueError(f'{path}: no state_dict in the checkpoint')
    sd = ck['state_dict']
    unet = OrderedDict((k[len('model.diffusion_model.'):], v) for k, v in sd.items() if k.startswith('model.diffusion_model.'))
    first = OrderedDict((k[len('first_stage_model.'):], v) for k, v in sd.items() if k.startswith('first_stage_model.')
                        and k[len('first_stage_model.'):].startswith(('decoder.', 'post_quant_conv.', 'quantize.embedding.')))
    if not unet or not first:
        raise ValueError(f'{path}: expected model.diffusion_model.* and first_stage_model.* keys of a LatentDiffusion checkpoint')
    sf = sd.get('scale_factor')
    return unet, first, sd.get('alphas_cumprod'), float(sf) if sf is not None else 1.0


class B200LDMNet:
    def __init__(self, params, img_resolution=64, img_channels=4, num_heads=8, alphas_cumprod=None, guidance_type='classifier-free',
                 guidance_rate=1.0, epsilon_t=1e-3, precision=None, device='cuda', flash_attn=True, f8_linear=None, cuda_graph=None,
                 num_head_channels=-1, head_pairs=True):
        """guidance_type 'uncond': the unconditional nets (no context, one pass per call); their legacy attention layers take
        num_head_channels (32 for LDM-VQ-f4) and, with head_pairs, run their 32-wide heads two per CTA."""
        if guidance_type not in ('classifier-free', 'uncond'):
            raise ValueError(f'B200LDMNet: guidance_type {guidance_type!r} is not one of classifier-free, uncond')
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200LDMNet needs a CUDA device (no CPU fallback)')
        self.uncond = guidance_type == 'uncond'
        self.precision = precision or default_precision()
        if self.uncond and self.precision == 'fp16f8':
            raise ValueError('B200LDMNet: fp16f8 is not available for the unconditional nets: the f8 GEMM mode needs channel counts that '
                             'are multiples of 64, and their 224 / 672 / 1120 / 1568-channel convolutions are not')
        self.lib = _lib.load()
        self.img_resolution, self.img_channels = img_resolution, img_channels
        self.label_dim = 0 if self.uncond else True
        self.guidance_type, self.guidance_rate = guidance_type, guidance_rate
        self.npass = PRECISIONS[self.precision]
        self.f8 = self.precision == 'fp16f8'           # ResBlock convolutions in the f8 GEMM mode (csrc/ops.h)
        # with fp16f8, proj_in / attn2.to_q / GEGLU ff / proj_out also run in the f8 GEMM mode (held by the f8 parity tests;
        # DSB_LDM_F8_LINEAR=0 or f8_linear=False keeps them fp16x3)
        if f8_linear is None:
            import os
            f8_linear = os.environ.get('DSB_LDM_F8_LINEAR', '1') != '0'
        self.f8_linear = bool(f8_linear) and self.f8
        self.flash_attn = bool(flash_attn)
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        self.st = ldm_plan.ldm_structure(params, num_heads, num_head_channels)
        self.wb, self.info = ldm_plan.pack_ldm_weights(self.st, params, f8=self.f8, f8_linear=self.f8_linear, head_pairs=head_pairs)
        if self.uncond and self.info['ctx_dim'] is not None:
            raise ValueError('B200LDMNet: guidance_type uncond given for a net with cross-attention')
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self.total_launches = 0
        if alphas_cumprod is None:
            ac = make_alphas_cumprod(*UNCOND_BETAS) if self.uncond else make_alphas_cumprod()
        else:
            ac = torch.as_tensor(alphas_cumprod).detach().float().cpu()
        log_alphas = 0.5 * torch.log(ac)
        self.M = len(log_alphas)
        self.t_array = torch.linspace(0., 1., self.M + 1)[1:].reshape((1, -1))
        self.log_alpha_array = log_alphas.reshape((1, -1))
        self.sigma_min = float(self.sigma(epsilon_t))
        self.sigma_max = float(self.sigma(1))

    @classmethod
    def from_reference(cls, net, num_heads=8, **kw):
        """Compile a reference CFGPrecond (net.model.model.diffusion_model is the UNetModel; net.model.alphas_cumprod the schedule)."""
        unet = net.model.model.diffusion_model if hasattr(net.model, 'model') else net.model.u
        sd = OrderedDict(unet.state_dict())
        nh = getattr(unet, 'num_heads', num_heads)          # openaimodel.py:466 (-1 when the config gives num_head_channels instead)
        if isinstance(nh, int) and nh > 0:
            num_heads = nh
        nhc = getattr(unet, 'num_head_channels', -1)
        return cls(sd, img_resolution=net.img_resolution, img_channels=net.img_channels, num_heads=num_heads,
                   alphas_cumprod=net.model.alphas_cumprod, guidance_type=net.guidance_type, guidance_rate=net.guidance_rate,
                   num_head_channels=nhc if isinstance(nhc, int) else -1, **kw)

    @classmethod
    def from_ldm_checkpoint(cls, path, img_resolution=64, num_head_channels=32, device='cuda', **kw):
        """The unconditional LSUN-Bedroom / FFHQ LDM-VQ-f4 `model.ckpt` -> (eps-net as B200LDMNet(guidance_type='uncond'), its VQ
        decoder as B200VAEDecoder).  The file is read with torch.load(weights_only=True) only (load_ldm_checkpoint)."""
        from .vae_net import B200VAEDecoder
        unet, first, ac, sf = load_ldm_checkpoint(path)
        net = cls(unet, img_resolution=img_resolution, img_channels=unet['input_blocks.0.0.weight'].shape[1], guidance_type='uncond',
                  num_head_channels=num_head_channels, alphas_cumprod=ac, device=device, **kw)
        return net, B200VAEDecoder(first, scale_factor=sf, device=device)

    # ---- VP <-> sigma mapping (networks_edm.py:694-718; piecewise-linear interpolation :720-756) ---------------------------------
    @staticmethod
    def interpolate_fn(x, xp, yp):
        """y = f(x) through the keypoints (xp, yp) [1, K], x [N, 1]; linear extrapolation outside.  Uses searchsorted instead of the
        reference's sort/gather construction (same piecewise-linear function)."""
        xs, ys = xp.reshape(-1), yp.reshape(-1)
        xq = x.reshape(-1)
        K = xs.numel()
        idx = torch.searchsorted(xs.contiguous(), xq.contiguous()).clamp(1, K - 1)
        x0, x1, y0, y1 = xs[idx - 1], xs[idx], ys[idx - 1], ys[idx]
        return (y0 + (xq - x0) * (y1 - y0) / (x1 - x0)).reshape(-1, 1)

    def marginal_log_mean_coeff(self, t):
        t = torch.as_tensor(t, dtype=torch.float32)
        return self.interpolate_fn(t.reshape((-1, 1)), self.t_array.to(t.device), self.log_alpha_array.to(t.device)).reshape((-1))

    def sigma(self, t):
        lm = self.marginal_log_mean_coeff(t)
        return torch.sqrt(1. - torch.exp(2. * lm)) / torch.exp(lm)

    def sigma_inv(self, sigma):
        sigma = torch.as_tensor(sigma, dtype=torch.float32)
        lamb = -(sigma.log())
        log_alpha = -0.5 * torch.logaddexp(torch.zeros((1,), device=lamb.device), -2. * lamb)
        t = self.interpolate_fn(log_alpha.reshape((-1, 1)), torch.flip(self.log_alpha_array.to(lamb.device), [1]),
                                torch.flip(self.t_array.to(lamb.device), [1]))
        return t.reshape((-1,))

    def round_sigma(self, sigma):
        return torch.as_tensor(sigma)

    # ---- plan cache ---------------------------------------------------------------------------------------------------------
    def _plan(self, B, Bt, nT):
        px = self.img_channels * self.img_resolution ** 2 * 4
        ctx_f = self.info['ctx_dim'] or 0
        return self.native.get((B, Bt, nT),
                               lambda: ldm_plan.compile_ldm_plan(self.st, self.wb, self.info, B, Bt, nT, self.img_resolution, npass=self.npass,
                                                                 flash_attn=self.flash_attn, f8=self.f8, f8_linear=self.f8_linear),
                               (lambda pl: (B * px, Bt * px, nT * 4, (B if nT > 1 else 1) * 16, Bt * 64 * 4,
                                            Bt * pl.meta['ctx_tokens'] * ctx_f * 4)) if self.cuda_graph else None)

    def eps(self, x_scaled_src, coef, tvals, context, bottleneck=None):
        """eps-net on Bt = context.shape[0] samples (B without context): inputs x [B,...] (c_in applied in-kernel via coef[:,2]),
        timesteps tvals [1|Bt]."""
        B = x_scaled_src.shape[0]
        Bt = context.shape[0] if context is not None else B
        nT = tvals.numel()
        h, pl = self._plan(B, Bt, nT)
        out = torch.empty((Bt,) + tuple(x_scaled_src.shape[1:]), device=x_scaled_src.device)
        io = (x_scaled_src.data_ptr(), out.data_ptr(), tvals.data_ptr(), coef.data_ptr(), bottleneck.data_ptr() if bottleneck is not None else None,
              context.data_ptr() if context is not None else None)
        self.total_launches += self.native.run(h, io, torch.cuda.current_stream(x_scaled_src.device).cuda_stream)
        return out

    # ---- the reference-facing call (networks_edm.py:670-692) -------------------------------------------------------------------
    def __call__(self, x, sigma, condition=None, unconditional_condition=None, out=None, bottleneck=None, **_):
        if x.device.type != 'cuda':
            raise _lib.DsError('B200LDMNet: input must live on the CUDA device (no CPU fallback)')
        x = x.to(torch.float32).contiguous()
        B = x.shape[0]
        sig = torch.as_tensor(sigma, dtype=torch.float32, device=x.device).reshape(-1)
        c_in = 1 / (sig ** 2 + 1).sqrt()
        c_noise = self.M * self.sigma_inv(sig) - 1.
        coef = torch.zeros(sig.numel(), 4, device=x.device)
        coef[:, 2] = c_in
        cfg = self.guidance_type == 'classifier-free' and not (self.guidance_rate == 1. or unconditional_condition is None)
        if self.uncond:
            ctx, tvals = None, c_noise
        elif cfg:
            ctx = torch.cat([unconditional_condition, condition]).to(torch.float32).contiguous()
            tvals = c_noise if c_noise.numel() == 1 else torch.cat([c_noise] * 2)
        else:
            ctx = condition.to(torch.float32).contiguous()
            tvals = c_noise
        tvals = tvals.contiguous()
        bott = None
        if bottleneck is not None:
            bott = torch.empty(ctx.shape[0] if ctx is not None else B, 64, device=x.device)
        F = self.eps(x, coef.contiguous(), tvals, ctx, bottleneck=bott)
        if bottleneck is not None:
            bottleneck.copy_(bott[-B:])           # the conditional half (solvers_amed.py:24-25), or the whole batch (uncond)
        if out is None:
            out = torch.empty_like(x)
        # D = x - sigma * (eps_u + g (eps_c - eps_u))   [c_skip = 1, c_out = -sigma]; one fused update kernel
        g = float(self.guidance_rate)
        if sig.numel() == 1:
            s = float(sig)      # host scalar: the samplers hold sigma on the host too (one value per step)
            if cfg:
                solver_update(out, x, [1.0, 0.0, -s * (1 - g), -s * g], mode=S.DS_M_NONE, hist=[F[:B], F[B:]])
            else:
                solver_update(out, x, [1.0, 0.0, -s], mode=S.DS_M_NONE, hist=[F])
        else:
            z = torch.zeros_like(sig)
            if cfg:
                cd = torch.stack([torch.ones_like(sig), z, -sig * (1 - g), -sig * g, z, z]).contiguous()
                solver_update(out, x, [0] * 6, mode=S.DS_M_NONE, hist=[F[:B], F[B:]], coef_dev=cd)
            else:
                cd = torch.stack([torch.ones_like(sig), z, -sig, z, z, z]).contiguous()
                solver_update(out, x, [0] * 6, mode=S.DS_M_NONE, hist=[F], coef_dev=cd)
        return out

    def profile_call(self, x, sigma, condition, unconditional_condition=None):
        """One denoiser call with per-op CUDA-event timing -> {op_type: (count, total_ms)} and per-op list [(type, tag, ms)]."""
        self(x, sigma, condition=condition, unconditional_condition=unconditional_condition)
        for (h, pl) in self.native.plans.values():
            self.lib.ds_unet_set_profiling(h, 1)
        self(x, sigma, condition=condition, unconditional_condition=unconditional_condition)
        out, per_op = {}, []
        for (h, pl) in self.native.plans.values():
            buf = (C.c_float * pl.n_ops)()
            n = self.lib.ds_unet_get_profile(h, buf, pl.n_ops)
            self.lib.ds_unet_set_profiling(h, 0)
            if not any(buf[i] > 0 for i in range(n)):          # a cached plan of another (batch, sigma-mode) that this call did not run
                continue
            for i in range(n):
                t = self.lib.ds_unet_op_type(h, i)
                c, ms = out.get(t, (0, 0.0))
                out[t] = (c + 1, ms + buf[i])
                per_op.append((t, pl.ops_array[i].tag, buf[i]))
        return out, per_op

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def requires_grad_(self, *_a, **_k):
        return self

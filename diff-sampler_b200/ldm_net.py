"""B200LDMNet — native drop-in for the reference's `CFGPrecond` wrapper around a latent-diffusion eps-net
(networks_edm.py:630-759; Stable Diffusion v1.x `UNetModel`).  Same call contract:
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


class B200LDMNet:
    def __init__(self, params, img_resolution=64, img_channels=4, num_heads=8, alphas_cumprod=None, guidance_type='classifier-free',
                 guidance_rate=1.0, epsilon_t=1e-3, precision=None, device='cuda', flash_attn=True, f8_linear=None, cuda_graph=None):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200LDMNet needs a CUDA device (no CPU fallback)')
        self.lib = _lib.load()
        self.img_resolution, self.img_channels, self.label_dim = img_resolution, img_channels, True
        self.guidance_type, self.guidance_rate = guidance_type, guidance_rate
        self.precision = precision or default_precision()
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
        self.st = ldm_plan.ldm_structure(params, num_heads)
        self.wb, self.info = ldm_plan.pack_ldm_weights(self.st, params, f8=self.f8, f8_linear=self.f8_linear)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self.total_launches = 0
        ac = make_alphas_cumprod() if alphas_cumprod is None else torch.as_tensor(alphas_cumprod).float()
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
        return cls(sd, img_resolution=net.img_resolution, img_channels=net.img_channels, num_heads=num_heads,
                   alphas_cumprod=net.model.alphas_cumprod, guidance_type=net.guidance_type, guidance_rate=net.guidance_rate, **kw)

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
        return self.native.get((B, Bt, nT),
                               lambda: ldm_plan.compile_ldm_plan(self.st, self.wb, self.info, B, Bt, nT, self.img_resolution, npass=self.npass,
                                                                 flash_attn=self.flash_attn, f8=self.f8, f8_linear=self.f8_linear),
                               (lambda pl: (B * px, Bt * px, nT * 4, (B if nT > 1 else 1) * 16, Bt * 64 * 4,
                                            Bt * pl.meta['ctx_tokens'] * self.info['ctx_dim'] * 4)) if self.cuda_graph else None)

    def eps(self, x_scaled_src, coef, tvals, context, bottleneck=None):
        """eps-net on Bt = context.shape[0] samples: inputs x [B,...] (c_in applied in-kernel via coef[:,2]), timesteps tvals [1|Bt]."""
        B, Bt = x_scaled_src.shape[0], context.shape[0]
        nT = tvals.numel()
        h, pl = self._plan(B, Bt, nT)
        out = torch.empty((Bt,) + tuple(x_scaled_src.shape[1:]), device=x_scaled_src.device)
        io = (x_scaled_src.data_ptr(), out.data_ptr(), tvals.data_ptr(), coef.data_ptr(), bottleneck.data_ptr() if bottleneck is not None else None,
              context.data_ptr())
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
        if self.guidance_type == 'uncond':
            raise NotImplementedError('unconditional latent-diffusion nets are not lowered (no context)')
        if cfg:
            ctx = torch.cat([unconditional_condition, condition]).to(torch.float32).contiguous()
            tvals = c_noise if c_noise.numel() == 1 else torch.cat([c_noise] * 2)
        else:
            ctx = condition.to(torch.float32).contiguous()
            tvals = c_noise
        tvals = tvals.contiguous()
        bott = None
        if bottleneck is not None:
            bott = torch.empty(ctx.shape[0], 64, device=x.device)
        F = self.eps(x, coef.contiguous(), tvals, ctx, bottleneck=bott)
        if bottleneck is not None:
            bottleneck.copy_(bott[-B:])           # the conditional half (solvers_amed.py:24-25)
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

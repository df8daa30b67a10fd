"""solvers — drop-in for diff-solvers-main/solvers.py (identical to gits-main/solvers.py).

Same sampler names, argument lists, defaults, return conventions and error behaviour as the reference
(solvers.py:18-821), so `sample.py` / `fid.py` / `gits_utils.py` can import this module unchanged.  Underneath,
each step is: one native denoiser evaluation (B200Net, wgmma kernels) + ONE fused update kernel that reads the
state, the denoiser output and up to four history buffers and writes the next state and the new history entry.
No CPU fallback: tensors must be on a CUDA device.
"""
import math

import torch

from . import _cstructs as S
from .ldm_net import B200LDMNet
from .net import B200Net
from .optimal import B200OptimalDenoiser, get_denoised_opt, optimal_sampler      # noqa: F401  (diff-analyzer's solvers.py)
from .solver_utils import *                       # noqa: F401,F403  (the reference does `from solver_utils import *`)
from .solver_utils import (dpm_pp_coefs, dyn_threshold, get_schedule, solver_update, unipc_coefs)

_NATIVE_CLASSES = ('SongUNet', 'DhariwalUNet')


def _weights_fingerprint(module):
    """Cheap identity of a torch module's weights: storage address and in-place version counter of every tensor of its state_dict
    (load_state_dict / optimiser / EMA updates bump the version; re-assignment changes the address)."""
    return tuple((v.data_ptr(), v._version) for v in module.state_dict(keep_vars=True).values())


def invalidate_native(net):
    """Drop the compiled snapshot `as_native` cached on a reference module (it is re-compiled on the next call)."""
    try:
        object.__delattr__(net, '_b200_native')
    except AttributeError:
        pass


def as_native(net, precision=None):
    """The native denoiser for `net`:
      * a B200Net / B200LDMNet                      -> itself;
      * a reference EDMPrecond over SongUNet / DhariwalUNet (networks_edm.py:459-496) -> B200Net.from_reference, compiled once and
        cached on the module together with a fingerprint of its weights (a later load_state_dict / EMA update re-compiles);
      * a reference CFGPrecond over a latent-diffusion UNetModel (networks_edm.py:630-759) -> B200LDMNet.from_reference, same cache;
      * anything else (VP/VE/iDDPM preconditioners, foreign callables) -> the object unchanged: its D(x, sigma) is evaluated by
        PyTorch and consumed by the native update kernels.  Other preconditioners are NOT compiled: their c_skip / c_out / c_noise
        differ from EDM's and evaluating them as EDMPrecond would be silently wrong."""
    if isinstance(net, (B200Net, B200LDMNet)):
        return net
    if not hasattr(net, 'state_dict'):
        return net
    inner = getattr(net, 'model', None)
    kind = None
    if type(net).__name__ == 'EDMPrecond' and inner is not None and type(inner).__name__ in _NATIVE_CLASSES:
        kind = 'edm'
    elif type(net).__name__ == 'CFGPrecond' and hasattr(net, 'guidance_type'):
        unet = getattr(getattr(inner, 'model', None), 'diffusion_model', None)
        if unet is not None and type(unet).__name__ == 'UNetModel':
            kind = 'ldm'
    if kind is None:
        return net
    fp = _weights_fingerprint(net)
    cached = getattr(net, '_b200_native', None)
    if cached is not None and cached[0] == fp and (precision is None or cached[1].precision == precision):
        return cached[1]
    dev = next(net.parameters()).device
    kw = dict(device=dev if dev.type == 'cuda' else 'cuda', **({'precision': precision} if precision else {}))
    if kind == 'edm':
        nat = B200Net.from_reference(net, **kw)
    else:
        nat = B200LDMNet.from_reference(net, **kw)
    try:
        object.__setattr__(net, '_b200_native', (fp, nat))
    except Exception:
        pass
    return nat


def get_denoised(net, x, t, class_labels=None, condition=None, unconditional_condition=None):
    """Denoised output D(x; t) of the wrapped model (reference: solvers.py:9-14)."""
    net = as_native(net)
    if hasattr(net, 'guidance_type'):
        return net(x, t, condition=condition, unconditional_condition=unconditional_condition)
    return net(x, t, class_labels=class_labels)


class _Loop:
    """State shared by every sampler: schedule, trajectory storage, prologue/epilogue (reference: solvers.py:63-96)."""

    def __init__(self, net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
                 schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero):
        if latents.device.type != 'cuda':
            raise RuntimeError('diff_sampler_b200.solvers: latents must be on a CUDA device (there is no CPU fallback)')
        self.net = as_native(net)
        self.kw = dict(class_labels=class_labels, condition=condition, unconditional_condition=unconditional_condition)
        if t_steps is None:
            t_steps = get_schedule(num_steps, sigma_min, sigma_max, device=latents.device, schedule_type=schedule_type,
                                   schedule_rho=schedule_rho, net=net)
        self.t_dev = t_steps.to(device=latents.device, dtype=torch.float32).contiguous()
        self.t = [float(v) for v in self.t_dev.tolist()]          # one host read per sampler call; coefficients are host scalars
        self.n = len(self.t)
        self.latents = latents.to(torch.float32).contiguous()
        self.return_inters, self.return_eps, self.denoise_to_zero = return_inters, return_eps, denoise_to_zero
        shape = self.latents.shape
        n_traj = self.n + (1 if denoise_to_zero else 0)
        self.inters = torch.empty((n_traj,) + tuple(shape), device=latents.device) if return_inters else None
        self.eps = torch.empty((self.n - 1,) + tuple(shape), device=latents.device) if (return_inters and return_eps) else None
        self.x = self._slot(0)
        solver_update(self.x, self.latents, [self.t[0]], mode=S.DS_M_NONE)      # x_next = latents * t_steps[0]  (solvers.py:68)
        self.D = torch.empty_like(self.latents)
        self.u8, self.u8_done = None, False

    def want_uint8(self, kwargs):
        """`images_uint8=` (an extra keyword the reference's samplers swallow in **kwargs): a [B, H, W, C] uint8 tensor that receives the
        finished images as sample.py:311 computes them, written by the LAST update kernel of the run (no separate pass over the state)."""
        self.u8 = kwargs.get('images_uint8')
        return self

    def u8_at(self, i):
        """The byte image rides on the update that produces x_{N-1} (not when a final denoise-to-zero evaluation follows)."""
        if self.u8 is None or self.denoise_to_zero or i != self.n - 2:
            return None
        self.u8_done = True
        return self.u8

    def _slot(self, i):
        return self.inters[i] if self.inters is not None else torch.empty_like(self.latents)

    def next_slot(self, i):
        """Where x_{i+1} is written: the trajectory tensor if it is being recorded, else in place."""
        return self.inters[i + 1] if self.inters is not None else self.x

    def d_slot(self, i, fallback):
        """Where the step's d_cur is written (the eps trajectory doubles as history storage when recorded)."""
        return self.eps[i] if self.eps is not None else fallback

    def denoise(self, x, i=None, sigma=None, out=None):
        sig = self.t_dev[i] if sigma is None else sigma
        net = self.net
        out = self.D if out is None else out
        if isinstance(net, B200Net):
            return net(x, sig, class_labels=self.kw['class_labels'], out=out)
        if isinstance(net, B200OptimalDenoiser):
            return net(x, sig, out=out)
        if isinstance(net, B200LDMNet):
            return net(x, sig, condition=self.kw['condition'], unconditional_condition=self.kw['unconditional_condition'], out=out)
        if hasattr(net, 'guidance_type'):
            r = net(x, sig, condition=self.kw['condition'], unconditional_condition=self.kw['unconditional_condition'])
        else:
            r = net(x, sig, class_labels=self.kw['class_labels'])
        return r.to(torch.float32).contiguous()

    def finish(self):
        x = self.x
        if self.denoise_to_zero:                                     # solvers.py:87-90
            x = self.denoise(x, self.n - 1, out=(self.inters[self.n] if self.inters is not None else None))
            if self.inters is not None and x.data_ptr() != self.inters[self.n].data_ptr():
                self.inters[self.n].copy_(x)
        if self.u8 is not None and not self.u8_done:          # paths without a fused final update (denoise_to_zero, AMED variants)
            from .dist_utils import to_uint8_nhwc
            self.u8.copy_(to_uint8_nhwc(x))
        if self.return_inters:
            if self.return_eps and self.eps is not None:
                return self.inters, self.eps
            return self.inters
        return x


def _afs_div(t):
    return math.sqrt(1.0 + t * t)


# ---------------------------------------------------------------------------------------------------------------------

@torch.no_grad()
def euler_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                  sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                  return_eps=False, t_steps=None, **kwargs):
    """Euler sampler (= DDIM).  Reference: solvers.py:18-96.  Per step: x+ = x + (t+ - t) * (x - D)/t  [AFS first step:
    d = x / sqrt(1 + t^2), no network call]."""
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    t = L.t
    for i in range(L.n - 1):
        h = t[i + 1] - t[i]
        out, dm = L.next_slot(i), L.d_slot(i, None)
        if afs and i == 0:
            solver_update(out, L.x, [1.0, h], mode=S.DS_M_DIV, t=_afs_div(t[i]), out_m=dm, out_u8=L.u8_at(i))
        else:
            D = L.denoise(L.x, i)
            solver_update(out, L.x, [1.0, h], mode=S.DS_M_EPS, D=D, t=t[i], out_m=dm, out_u8=L.u8_at(i))
        L.x = out
    return L.finish()


@torch.no_grad()
def heun_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                 sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                 return_eps=False, t_steps=None, **kwargs):
    """Heun's 2nd-order sampler (EDM).  Reference: solvers.py:100-183.  Euler predictor + trapezoidal corrector, 2 NFE/step."""
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    t = L.t
    xp = torch.empty_like(L.latents)
    d_buf = torch.empty_like(L.latents)
    for i in range(L.n - 1):
        h = t[i + 1] - t[i]
        d = L.d_slot(i, d_buf)
        if afs and i == 0:
            solver_update(xp, L.x, [1.0, h], mode=S.DS_M_DIV, t=_afs_div(t[i]), out_m=d)
        else:
            D = L.denoise(L.x, i)
            solver_update(xp, L.x, [1.0, h], mode=S.DS_M_EPS, D=D, t=t[i], out_m=d)
        D2 = L.denoise(xp, i + 1)
        out = L.next_slot(i)
        # x+ = x + h*(0.5*d + 0.5*d'),  d' = (x_pred - D')/t+       (solvers.py:166-168)
        solver_update(out, L.x, [1.0, 0.5 * h, 0.5 * h], mode=S.DS_M_EPS, D=D2, xs=xp, t=t[i + 1], hist=[d], out_u8=L.u8_at(i))
        L.x = out
    return L.finish()


@torch.no_grad()
def dpm_2_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                  sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                  return_eps=False, r=0.5, t_steps=None, **kwargs):
    """DPM-Solver-2.  Reference: solvers.py:187-273.  Midpoint at t_mid = t+^r * t^(1-r)."""
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    t = L.t
    xp = torch.empty_like(L.latents)
    d_buf = torch.empty_like(L.latents)
    for i in range(L.n - 1):
        h = t[i + 1] - t[i]
        t_mid = (t[i + 1] ** r) * (t[i] ** (1 - r))
        d = L.d_slot(i, d_buf)
        if afs and i == 0:
            solver_update(xp, L.x, [1.0, t_mid - t[i]], mode=S.DS_M_DIV, t=_afs_div(t[i]), out_m=d)
        else:
            D = L.denoise(L.x, i)
            solver_update(xp, L.x, [1.0, t_mid - t[i]], mode=S.DS_M_EPS, D=D, t=t[i], out_m=d)
        D2 = L.denoise(xp, sigma=torch.tensor([t_mid], device=xp.device, dtype=torch.float32))
        out = L.next_slot(i)
        solver_update(out, L.x, [1.0, h * (1 / (2 * r)), h * (1 - 1 / (2 * r))], mode=S.DS_M_EPS, D=D2, xs=xp, t=t_mid, hist=[d], out_u8=L.u8_at(i))
        L.x = out
    return L.finish()


def _multistep(L, afs, max_order, coef_fn, afs_first_by_index=True):
    """Shared driver of the explicit linear multistep samplers (iPNDM, iPNDM_v, DEIS):
       x+ = x + sum_k c_k * d_{-k},   history = previous d's (ring of max_order-1 buffers)."""
    t = L.t
    hist = []                       # most recent first
    spare = [torch.empty_like(L.latents) for _ in range(max(max_order, 1))]
    for i in range(L.n - 1):
        order = min(max_order, i + 1)
        c = coef_fn(i, order)                                   # [c_cur, c_prev1, ...]
        d_new = L.d_slot(i, spare[i % len(spare)])
        out = L.next_slot(i)
        # AFS replaces the FIRST evaluation only.  ipndm_v / deis decide it by "history is empty" (solvers.py:445,570); with
        # max_order == 1 nothing is ever pushed, so the step index decides there (the reference raises IndexError for that case).
        first = (i == 0) if (afs_first_by_index or max_order == 1) else (len(hist) == 0)
        if afs and first:
            solver_update(out, L.x, [1.0] + c, mode=S.DS_M_DIV, t=_afs_div(t[i]), hist=hist[:order - 1], out_m=d_new, out_u8=L.u8_at(i))
        else:
            D = L.denoise(L.x, i)
            solver_update(out, L.x, [1.0] + c, mode=S.DS_M_EPS, D=D, t=t[i], hist=hist[:order - 1], out_m=d_new, out_u8=L.u8_at(i))
        L.x = out
        if max_order > 1:
            hist = ([d_new] + hist)[:max_order - 1]
    return L.finish()


@torch.no_grad()
def ipndm_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                  sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                  return_eps=False, max_order=4, t_steps=None, **kwargs):
    """Improved PNDM (Adams-Bashforth 1..4 with the classical fixed coefficients).  Reference: solvers.py:277-374.
    Note: the reference indexes an empty list when max_order == 1 (solvers.py:358-361); here max_order == 1 is plain Euler."""
    assert max_order >= 1 and max_order <= 4
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    AB = {1: [1.0], 2: [3 / 2, -1 / 2], 3: [23 / 12, -16 / 12, 5 / 12], 4: [55 / 24, -59 / 24, 37 / 24, -9 / 24]}
    return _multistep(L, afs, max_order, lambda i, order: [(L.t[i + 1] - L.t[i]) * a for a in AB[order]])


def _abv(t, i, order):
    """Variable-step Adams-Bashforth weights from the last `order` step sizes (reference: solvers.py:451-477)."""
    hn = t[i + 1] - t[i]
    if order == 1:
        return [1.0]
    h1 = t[i] - t[i - 1]
    if order == 2:
        return [(2 + hn / h1) / 2, -(hn / h1) / 2]
    h2 = t[i - 1] - t[i - 2]
    u = (1 - hn / (3 * (hn + h1)) * (hn * (hn + h1)) / (h1 * (h1 + h2))) / 2
    if order == 3:
        return [(2 + hn / h1) / 2 + u, -(hn / h1) / 2 - (1 + h1 / h2) * u, u * h1 / h2]
    h3 = t[i - 2] - t[i - 3]
    v = ((1 - hn / (3 * (hn + h1))) / 2 + (1 - hn / (2 * (hn + h1))) * hn / (6 * (hn + h1 + h2))) \
        * (hn * (hn + h1) * (hn + h1 + h2)) / (h1 * (h1 + h2) * (h1 + h2 + h3))
    g = h1 * (h1 + h2) / (h2 * (h2 + h3))
    return [(2 + hn / h1) / 2 + u + v,
            -(hn / h1) / 2 - (1 + h1 / h2) * u - (1 + h1 / h2 + g) * v,
            u * h1 / h2 + (h1 / h2 + g * (1 + h2 / h3)) * v,
            -v * g * h1 / h2]


@torch.no_grad()
def ipndm_v_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                    sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                    return_eps=False, max_order=4, t_steps=None, **kwargs):
    """Variable-step Adams-Bashforth.  Reference: solvers.py:378-499."""
    assert max_order >= 1 and max_order <= 4
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    return _multistep(L, afs, max_order, lambda i, order: [(L.t[i + 1] - L.t[i]) * a for a in _abv(L.t, i, order)],
                      afs_first_by_index=False)


@torch.no_grad()
def deis_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                 sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                 return_eps=False, max_order=4, coeff_list=None, t_steps=None, **kwargs):
    """DEIS (tAB / rhoAB) with pre-computed coefficients from solver_utils.get_deis_coeff_list.  Reference: solvers.py:503-607."""
    assert max_order >= 1 and max_order <= 4
    assert coeff_list is not None
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)

    def coefs(i, order):
        if order == 1:
            return [L.t[i + 1] - L.t[i]]                        # first step is Euler (solvers.py:575-576)
        return [float(c) for c in coeff_list[i][:order]]
    return _multistep(L, afs, max_order, coefs, afs_first_by_index=False)


@torch.no_grad()
def dpm_pp_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                   sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                   return_eps=False, max_order=3, predict_x0=True, lower_order_final=True, t_steps=None, **kwargs):
    """Multistep DPM-Solver++ (1 / 2M / 3M), data- or noise-prediction form.  Reference: solvers.py:612-713 and
    solver_utils.py:90-163.  As in the reference, `num_steps` is read for lower_order_final even when t_steps is given."""
    assert max_order >= 1 and max_order <= 3
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, return_eps, denoise_to_zero).want_uint8(kwargs)
    t = L.t
    if num_steps is None:
        num_steps = L.n
    hist, hist_t = [], []            # most recent first
    spare = [torch.empty_like(L.latents) for _ in range(4)]
    thr = torch.empty(L.latents.shape[0], device=L.latents.device)
    d_tmp = torch.empty_like(L.latents)
    for i in range(L.n - 1):
        if lower_order_final:
            order = i + 1 if i + 1 < max_order else min(max_order, num_steps - (i + 1))
        else:
            order = min(max_order, i + 1)
        ts = (hist_t[::-1] + [t[i]])[-3:]
        c = dpm_pp_coefs(ts, t[i + 1], order, predict_x0)
        m_new = spare[i % 4]
        out = L.next_slot(i)
        coef = [c[0], c[1]] + list(c[2:1 + order])
        if afs and i == 0:
            # d = x/sqrt(1+t^2); denoised = x - t*d                               (solvers.py:678-680)
            d_afs = L.d_slot(i, d_tmp)
            if predict_x0:
                solver_update(L.D, L.x, [1.0, -t[i]], mode=S.DS_M_DIV, t=_afs_div(t[i]), out_m=d_afs)
                dyn_threshold(L.D, out=thr)
                solver_update(out, L.x, coef, mode=S.DS_M_X0, D=L.D, thr=thr, hist=hist[:order - 1], out_m=m_new)
            else:
                m_new = d_afs if L.eps is not None else m_new
                solver_update(out, L.x, coef, mode=S.DS_M_DIV, t=_afs_div(t[i]), hist=hist[:order - 1], out_m=m_new)
        else:
            D = L.denoise(L.x, i)
            if predict_x0:
                dyn_threshold(D, out=thr)
                if L.eps is not None:      # GITS-style callers also want d_cur = (x - D)/t
                    solver_update(None, L.x, [0.0, 0.0], mode=S.DS_M_EPS, D=D, t=t[i], out_m=L.eps[i])
                solver_update(out, L.x, coef, mode=S.DS_M_X0, D=D, thr=thr, hist=hist[:order - 1], out_m=m_new, out_u8=L.u8_at(i))
            else:
                m_new = L.d_slot(i, m_new)
                solver_update(out, L.x, coef, mode=S.DS_M_EPS, D=D, t=t[i], hist=hist[:order - 1], out_m=m_new, out_u8=L.u8_at(i))
        L.x = out
        hist = ([m_new] + hist)[:3]
        hist_t = ([t[i]] + hist_t)[:3]
    return L.finish()


@torch.no_grad()
def unipc_sampler(net, latents, class_labels=None, condition=None, unconditional_condition=None, num_steps=None, sigma_min=0.002,
                  sigma_max=80, schedule_type='polynomial', schedule_rho=7, afs=False, denoise_to_zero=False, return_inters=False,
                  return_eps=False, max_order=3, predict_x0=True, lower_order_final=True, variant='bh2', t_steps=None, **kwargs):
    """UniPC-p predictor/corrector.  Reference: solvers.py:717-821 and solver_utils.py:174-287.  The corrector's extra
    network evaluation sits between two launches of the same fused update kernel."""
    assert max_order > 0 and max_order < 4
    L = _Loop(net, latents, class_labels, condition, unconditional_condition, num_steps, sigma_min, sigma_max, schedule_type,
              schedule_rho, t_steps, return_inters, False, denoise_to_zero).want_uint8(kwargs)
    t = L.t
    if num_steps is None:
        num_steps = L.n
    B = L.latents.shape[0]
    thr = torch.empty(B, device=L.latents.device)
    pool = [torch.empty_like(L.latents) for _ in range(5)]
    x_pred = torch.empty_like(L.latents)
    m0 = pool[0]
    if afs:
        if predict_x0:
            solver_update(L.D, L.x, [1.0, -t[0]], mode=S.DS_M_DIV, t=_afs_div(t[0]))
            dyn_threshold(L.D, out=thr)
            solver_update(None, L.x, [0.0, 0.0], mode=S.DS_M_X0, D=L.D, thr=thr, out_m=m0)
        else:
            solver_update(None, L.x, [0.0, 0.0], mode=S.DS_M_DIV, t=_afs_div(t[0]), out_m=m0)
    else:
        D = L.denoise(L.x, 0)
        if predict_x0:
            dyn_threshold(D, out=thr)
            solver_update(None, L.x, [0.0, 0.0], mode=S.DS_M_X0, D=D, thr=thr, out_m=m0)
        else:
            solver_update(None, L.x, [0.0, 0.0], mode=S.DS_M_EPS, D=D, t=t[0], out_m=m0)
    hist, hist_t = [m0], [t[0]]          # most recent first
    used = 1
    for i in range(L.n - 1):
        if i + 1 < max_order:
            order, use_corr, grow = i + 1, True, True
        else:
            order = min(max_order, num_steps - i - 1) if lower_order_final else max_order
            use_corr, grow = (i != num_steps - 2), False
        ts = hist_t[:order][::-1]
        pred, corr = unipc_coefs(ts, t[i + 1], order, variant, predict_x0, use_corr)
        hs = hist[:order]
        out = L.next_slot(i)
        target = x_pred if use_corr else out
        solver_update(target, L.x, [pred[0], 0.0] + pred[1:1 + order], mode=S.DS_M_NONE, hist=hs)
        m_t = None
        if use_corr:
            D = L.denoise(x_pred, i + 1)
            m_t = pool[used % 5]
            used += 1
            cf = [corr[0], corr[1]] + corr[2:2 + order]
            if predict_x0:
                dyn_threshold(D, out=thr)
                solver_update(out, L.x, cf, mode=S.DS_M_X0, D=D, thr=thr, hist=hs, out_m=m_t)
            else:
                solver_update(out, L.x, cf, mode=S.DS_M_EPS, D=D, xs=x_pred, t=t[i + 1], hist=hs, out_m=m_t)
        L.x = out
        # buffer bookkeeping exactly as solvers.py:797-810: while warming up the lists grow; afterwards they shift, and the last
        # step (no corrector) keeps the stale newest model entry but still records t_next.
        if grow:
            hist, hist_t = [m_t] + hist, [t[i + 1]] + hist_t
        else:
            if i < num_steps - 2:
                hist = ([m_t] + hist)[:max_order]
            else:                               # the reference shifts without storing: [a, b, c] -> [b, c, c] (solvers.py:805-810)
                hist = ([hist[0]] + hist)[:max_order]
            hist_t = ([t[i + 1]] + hist_t)[:max_order]
    return L.finish()

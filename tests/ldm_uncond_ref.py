"""CPU restatement of the unconditional latent-diffusion eps-net (LSUN-Bedroom / FFHQ LDM-VQ-f4) for the tests.

The `UNetModel` of models/ldm/configs/latent-diffusion/lsun_bedrooms-ldm-vq-4.yaml (= ffhq-ldm-vq-4.yaml) with the legacy
AttentionBlock (openaimodel.py:278-324: GroupNorm32 -> qkv 1x1 -> QKVAttentionLegacy :347-372 -> proj_out -> residual), heads of
num_head_channels = 32, no cross-attention, under CFGPrecond(guidance_type='uncond') with the linear beta schedule 0.0015 .. 0.0195.
A functional forward over a flat parameter dict, in any dtype (float64 for the parity tests); oracle/ldm_oracle.py supplies the
ResBlock, the timestep embedding and the sigma <-> t interpolation it shares with Stable Diffusion.
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ldm_oracle as LO

CONFIGS = {
    # lsun_bedrooms-ldm-vq-4.yaml:14-34: attention at downsampling factors 8, 4, 2 (32^2, 16^2, 8^2 latents)
    'ldm_vq4': dict(in_channels=3, out_channels=3, model_channels=224, attention_resolutions=(2, 4, 8), num_res_blocks=2,
                    channel_mult=(1, 2, 3, 4), num_head_channels=32, img_resolution=64),
    # same traps at a small size: widths 96 / 192 / 288 (not multiples of 64), 3- and 9-head levels (odd), a space-to-depth at 96,
    # decoder concats of 480 / 384 / 288 channels; the middle block at 8 x 8 as AMED's tap expects
    'tiny_uncond': dict(in_channels=3, out_channels=3, model_channels=96, attention_resolutions=(1, 2, 4), num_res_blocks=1,
                        channel_mult=(1, 2, 3), num_head_channels=32, img_resolution=32),
}
BETAS = (0.0015, 0.0195)


def structure(cfg):
    """Module list of UNetModel.__init__ (openaimodel.py:506-689, use_spatial_transformer=False): as ldm_oracle.structure, with
    ('qkv_attn', name, ch, heads, 32) for the legacy attention blocks."""
    mc, mult, nrb, attn, hc = cfg['model_channels'], cfg['channel_mult'], cfg['num_res_blocks'], cfg['attention_resolutions'], \
        cfg['num_head_channels']
    inp = [('input_blocks.0', [('conv', 'input_blocks.0.0', cfg['in_channels'], mc)])]
    chans = [mc]
    ch, ds, idx = mc, 1, 1
    for level, m in enumerate(mult):
        for _ in range(nrb):
            layers = [('res', f'input_blocks.{idx}.0', ch, m * mc)]
            ch = m * mc
            if ds in attn:
                layers.append(('qkv_attn', f'input_blocks.{idx}.1', ch, ch // hc, hc))
            inp.append((f'input_blocks.{idx}', layers))
            chans.append(ch)
            idx += 1
        if level != len(mult) - 1:
            inp.append((f'input_blocks.{idx}', [('down', f'input_blocks.{idx}.0', ch, ch)]))
            chans.append(ch)
            idx += 1
            ds *= 2
    mid = [('middle_block', [('res', 'middle_block.0', ch, ch), ('qkv_attn', 'middle_block.1', ch, ch // hc, hc),
                             ('res', 'middle_block.2', ch, ch)])]
    out = []
    idx = 0
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nrb + 1):
            ich = chans.pop()
            layers = [('res', f'output_blocks.{idx}.0', ch + ich, mc * m)]
            ch = mc * m
            k = 1
            if ds in attn:
                layers.append(('qkv_attn', f'output_blocks.{idx}.{k}', ch, ch // hc, hc))
                k += 1
            if level and i == nrb:
                layers.append(('up', f'output_blocks.{idx}.{k}', ch, ch))
                ds //= 2
            out.append((f'output_blocks.{idx}', layers))
            idx += 1
    return inp, mid, out, ch


def param_shapes(cfg):
    """Ordered (name -> shape) of UNetModel.state_dict() for this config (qkv / proj_out are 1-D convolutions)."""
    mc = cfg['model_channels']
    ted = mc * 4
    sh = OrderedDict()

    def conv(n, cin, cout, k, dims=2):
        sh[n + '.weight'] = (cout, cin) + (k,) * dims
        sh[n + '.bias'] = (cout,)

    def norm(n, c):
        sh[n + '.weight'] = (c,)
        sh[n + '.bias'] = (c,)

    sh['time_embed.0.weight'], sh['time_embed.0.bias'] = (ted, mc), (ted,)
    sh['time_embed.2.weight'], sh['time_embed.2.bias'] = (ted, ted), (ted,)
    inp, mid, out, ch_final = structure(cfg)
    for _, layers in inp + mid + out:
        for L in layers:
            kind, n = L[0], L[1]
            if kind == 'conv':
                conv(n, L[2], L[3], 3)
            elif kind == 'res':
                cin, cout = L[2], L[3]
                norm(n + '.in_layers.0', cin)
                conv(n + '.in_layers.2', cin, cout, 3)
                sh[n + '.emb_layers.1.weight'], sh[n + '.emb_layers.1.bias'] = (cout, ted), (cout,)
                norm(n + '.out_layers.0', cout)
                conv(n + '.out_layers.3', cout, cout, 3)
                if cin != cout:
                    conv(n + '.skip_connection', cin, cout, 1)
            elif kind == 'qkv_attn':
                c = L[2]
                norm(n + '.norm', c)
                conv(n + '.qkv', c, 3 * c, 1, dims=1)
                conv(n + '.proj_out', c, c, 1, dims=1)
            elif kind == 'down':
                conv(n + '.op', L[2], L[3], 3)
            elif kind == 'up':
                conv(n + '.conv', L[2], L[3], 3)
    norm('out.0', ch_final)
    conv('out.2', mc, cfg['out_channels'], 3)
    return sh


def make_params(name, seed=0):
    """ldm_oracle.make_params' recipe (non-zero everywhere, so proj_out and out.2, zero-initialised in the reference, take part)."""
    cfg = CONFIGS[name]
    g = torch.Generator().manual_seed(seed + 777)
    P = OrderedDict()
    for k, shp in param_shapes(cfg).items():
        if len(shp) == 1:
            v = (torch.rand(shp, generator=g) * 2 - 1) * 0.1
            P[k] = v + 1.0 if k.endswith('.weight') else v
        else:
            fan_in = int(np.prod(shp[1:]))
            P[k] = (torch.rand(shp, generator=g) * 2 - 1) * math.sqrt(3.0 / fan_in)
    return P, cfg


def legacy_attention(qkv, heads):
    """QKVAttentionLegacy.forward (openaimodel.py:361-372): qkv [N, heads*3*d, T] -> [N, heads*d, T]."""
    bs, width, length = qkv.shape
    ch = width // (3 * heads)
    q, k, v = qkv.reshape(bs * heads, ch * 3, length).split(ch, dim=1)
    scale = 1 / math.sqrt(math.sqrt(ch))
    w = torch.einsum('bct,bcs->bts', q * scale, k * scale)
    w = torch.softmax(w, dim=-1)
    return torch.einsum('bts,bcs->bct', w, v).reshape(bs, -1, length)


def _attn_block(P, n, x, heads):
    """AttentionBlock._forward (openaimodel.py:310-319)."""
    b, c, h, w = x.shape
    xf = x.reshape(b, c, -1)
    qkv = F.conv1d(F.group_norm(xf, 32, P[n + '.norm.weight'], P[n + '.norm.bias'], 1e-5), P[n + '.qkv.weight'], P[n + '.qkv.bias'])
    hh = F.conv1d(legacy_attention(qkv, heads), P[n + '.proj_out.weight'], P[n + '.proj_out.bias'])
    return (xf + hh).reshape(b, c, h, w)


def unet_forward(P, cfg, x, timesteps, taps=None):
    """openaimodel.py:710-741 UNetModel.forward without context; taps['middle_block'] = the middle block's output."""
    inp, mid, out, _ = structure(cfg)
    temb = LO.timestep_embedding(timesteps.detach().cpu(), cfg['model_channels']).to(device=x.device, dtype=x.dtype)
    emb = F.linear(temb, P['time_embed.0.weight'], P['time_embed.0.bias'])
    emb = F.linear(F.silu(emb), P['time_embed.2.weight'], P['time_embed.2.bias'])

    def run(layers, h):
        for L in layers:
            kind, n = L[0], L[1]
            if kind == 'conv':
                h = F.conv2d(h, P[n + '.weight'], P[n + '.bias'], padding=1)
            elif kind == 'res':
                h = LO._res(P, n, h, emb)
            elif kind == 'qkv_attn':
                h = _attn_block(P, n, h, L[3])
            elif kind == 'down':
                h = F.conv2d(h, P[n + '.op.weight'], P[n + '.op.bias'], stride=2, padding=1)
            elif kind == 'up':
                h = F.conv2d(F.interpolate(h, scale_factor=2, mode='nearest'), P[n + '.conv.weight'], P[n + '.conv.bias'], padding=1)
        return h
    hs = []
    h = x
    for _, layers in inp:
        h = run(layers, h)
        hs.append(h)
    h = run(mid[0][1], h)
    if taps is not None:
        taps['middle_block'] = h
    for _, layers in out:
        h = run(layers, torch.cat([h, hs.pop()], dim=1))
    return F.conv2d(F.silu(F.group_norm(h, 32, P['out.0.weight'], P['out.0.bias'], 1e-5)), P['out.2.weight'], P['out.2.bias'], padding=1)


class OracleUncondNet(LO.OracleCFGNet):
    """CFGPrecond(guidance_type='uncond') (networks_edm.py:670-692) over the functional eps-net: D = x - sigma * eps(c_in x, c_noise).
    dtype: the eps-net's arithmetic (float64 for parity); the sigma <-> t mapping stays float32, as in the reference."""

    def __init__(self, P, cfg, dtype=torch.float64, epsilon_t=1e-3):
        self.P = OrderedDict((k, v.to(dtype)) for k, v in P.items())
        self.cfg, self.dtype = cfg, dtype
        self.img_resolution, self.img_channels, self.label_dim = cfg['img_resolution'], cfg['in_channels'], 0
        self.guidance_rate, self.guidance_type = 1.0, 'uncond'
        log_alphas = 0.5 * torch.log(LO.make_alphas_cumprod(*BETAS))
        self.M = len(log_alphas)
        self.t_array = torch.linspace(0., 1., self.M + 1)[1:].reshape((1, -1))
        self.log_alpha_array = log_alphas.reshape((1, -1))
        self.sigma_min = float(self.sigma(epsilon_t))
        self.sigma_max = float(self.sigma(1))
        self.taps = None

    def __call__(self, x, sigma, condition=None, unconditional_condition=None, **_):
        """Runs on x's device (the schedule arithmetic on the CPU)."""
        sigma = torch.as_tensor(sigma).detach().cpu().to(torch.float32).reshape(-1,)
        c_in = 1 / (sigma ** 2 + 1).sqrt()
        c_noise = self.M * self.sigma_inv(sigma) - 1.
        if c_noise.numel() == 1:
            c_noise = c_noise.expand(x.shape[0])
        if next(iter(self.P.values())).device != x.device:
            self.P = OrderedDict((k, v.to(x.device)) for k, v in self.P.items())
        dt = lambda t: t.to(device=x.device, dtype=self.dtype)
        xd = dt(x)
        eps = unet_forward(self.P, self.cfg, dt(c_in).reshape(-1, 1, 1, 1) * xd, dt(c_noise), taps=self.taps)
        return xd - dt(sigma).reshape(-1, 1, 1, 1) * eps

"""ORACLE — test infrastructure, not product code (see oracle/edm_oracle.py header).

float64 restatement (CPU, or a GPU for the full-size net) of the Consistency-Models denoiser: CMPrecond (models/networks_edm.py:504-549) around the CM UNetModel
(models/cm/unet.py:505-772) with additive time conditioning (use_scale_shift_norm=False), ResBlock up/down sampling
(resblock_updown=True) and the flash attention layout of QKVFlashAttention (unet.py:331-374).  Written over the reference's own
state-dict names; the block structure comes from the loader settings (models/cm/cm_model_loader.py).
Pinned against the real reference by tests/golden/ref_cm.npz (oracle/gen_cm_golden.py).
"""
import math

import torch
import torch.nn.functional as F


def _mult(s):
    cm = s.get('channel_mult', '')
    if isinstance(cm, (tuple, list)):
        return tuple(cm)
    if cm == '':
        return {512: (0.5, 1, 1, 2, 2, 4, 4), 256: (1, 1, 2, 2, 4, 4), 128: (1, 1, 2, 3, 4), 64: (1, 2, 3, 4)}[s['image_size']]
    return tuple(int(m) for m in cm.split(','))


def timestep_embedding(t, dim, max_period=10000):
    """nn.py:119-138: [cos | sin] of t * exp(-ln(max_period) i / half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    a = t.double()[:, None] * freqs[None]
    return torch.cat([torch.cos(a), torch.sin(a)], dim=-1)


class CMOracle:
    """D(x, sigma) of CMPrecond(UNetModel(setting)) in float64.  sd: UNetModel.state_dict() (no prefix).
    `taps`: set to a dict to record the middle_block output under 'middle_block' (AMED's read-out, solvers_amed.py:11-14)."""

    def __init__(self, sd, setting, sigma_data=0.5, device='cpu'):
        self.device = torch.device(device)       # float64 on a GPU makes the full-size 256x256 net practical to evaluate
        self.W = {k: v.detach().to(self.device, torch.float64) for k, v in sd.items()}
        self.s = dict(setting)
        self.sigma_data = sigma_data
        self.img_resolution = self.s['image_size']
        self.img_channels = 3
        self.label_dim = 0
        self.sigma_min, self.sigma_max = 0.002, 80.0
        self.taps = None
        mc = self.s['num_channels']
        self.heads_width = self.s['num_head_channels']
        self.attn_ds = {self.s['image_size'] // int(r) for r in self.s['attention_resolutions'].split(',')}
        self.mc, self.mult, self.nb = mc, _mult(self.s), self.s['num_res_blocks']

    def round_sigma(self, sigma):
        return torch.as_tensor(sigma)

    # ---- layers --------------------------------------------------------------------------------------------------
    def _gn(self, n, x):                              # GroupNorm32(32, C), eps 1e-5 (nn.py:19-21, :109-116)
        return F.group_norm(x, 32, self.W[n + '.weight'], self.W[n + '.bias'], eps=1e-5)

    def _conv(self, n, x):
        w = self.W[n + '.weight']
        if w.dim() == 3:                              # conv1d 1x1 over the flattened positions
            w = w[..., None]
        return F.conv2d(x, w, self.W[n + '.bias'], padding=w.shape[-1] // 2)

    def _res(self, n, x, emb, up=False, down=False):
        """ResBlock._forward (unet.py:236-256), use_scale_shift_norm=False."""
        h = F.silu(self._gn(n + '.in_layers.0', x))
        if up:
            h, x = F.interpolate(h, scale_factor=2, mode='nearest'), F.interpolate(x, scale_factor=2, mode='nearest')
        elif down:
            h, x = F.avg_pool2d(h, 2), F.avg_pool2d(x, 2)
        h = self._conv(n + '.in_layers.2', h)
        e = F.linear(F.silu(emb), self.W[n + '.emb_layers.1.weight'], self.W[n + '.emb_layers.1.bias'])
        h = h + e[:, :, None, None]
        h = self._conv(n + '.out_layers.3', F.silu(self._gn(n + '.out_layers.0', h)))
        skip = self._conv(n + '.skip_connection', x) if (n + '.skip_connection.weight') in self.W else x
        return skip + h

    def _attn(self, n, x):
        """AttentionBlock._forward (unet.py:316-328) with QKVFlashAttention (:364-374): qkv rows are [q|k|v][head][d], scale 1/sqrt(d)."""
        B, C, H, Wd = x.shape
        L = H * Wd
        nh = C // self.heads_width
        d = C // nh
        qkv = self._conv(n + '.qkv', self._gn(n + '.norm', x)).reshape(B, 3, nh, d, L)
        q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]                  # [B, nh, d, L]
        p = torch.softmax(torch.einsum('bhdq,bhdk->bhqk', q, k) / math.sqrt(d), dim=-1)
        o = torch.einsum('bhqk,bhdk->bhdq', p, v).reshape(B, C, H, Wd)
        return x + self._conv(n + '.proj_out', o)

    # ---- UNetModel.forward (unet.py:743-772) ------------------------------------------------------------------------
    def unet(self, x, t):
        emb = timestep_embedding(t, self.mc)
        emb = F.linear(emb, self.W['time_embed.0.weight'], self.W['time_embed.0.bias'])
        emb = F.linear(F.silu(emb), self.W['time_embed.2.weight'], self.W['time_embed.2.bias'])
        hs = []
        h = self._conv('input_blocks.0.0', x)
        hs.append(h)
        i, ds = 1, 1
        for level in range(len(self.mult)):
            for _ in range(self.nb):
                h = self._res(f'input_blocks.{i}.0', h, emb)
                if ds in self.attn_ds:
                    h = self._attn(f'input_blocks.{i}.1', h)
                hs.append(h)
                i += 1
            if level != len(self.mult) - 1:
                h = self._res(f'input_blocks.{i}.0', h, emb, down=True)
                hs.append(h)
                i += 1
                ds *= 2
        h = self._res('middle_block.0', h, emb)
        h = self._attn('middle_block.1', h)
        h = self._res('middle_block.2', h, emb)
        if self.taps is not None:
            self.taps['middle_block'] = h.float()          # what the native tap returns, and what the AMED predictor reads
        i = 0
        for level in reversed(range(len(self.mult))):
            for j in range(self.nb + 1):
                h = torch.cat([h, hs.pop()], dim=1)
                h = self._res(f'output_blocks.{i}.0', h, emb)
                k = 1
                if ds in self.attn_ds:
                    h = self._attn(f'output_blocks.{i}.1', h)
                    k = 2
                if level and j == self.nb:
                    h = self._res(f'output_blocks.{i}.{k}', h, emb, up=True)
                    ds //= 2
                i += 1
        return self._conv('out.2', F.silu(self._gn('out.0', h)))

    @torch.no_grad()
    def __call__(self, x, sigma, class_labels=None, **_):
        """CMPrecond.forward (networks_edm.py:533-549)."""
        home = x.device
        x = x.to(self.device, torch.float64)
        B = x.shape[0]
        sigma = torch.as_tensor(sigma).to(self.device, torch.float64).reshape(-1)
        if sigma.numel() == 1:
            sigma = sigma.repeat(B)
        sd = self.sigma_data
        c_skip = (sd ** 2 / (sigma ** 2 + sd ** 2)).reshape(-1, 1, 1, 1)
        c_out = (sigma * sd / (sigma ** 2 + sd ** 2).sqrt()).reshape(-1, 1, 1, 1)
        c_in = (1 / (sd ** 2 + sigma ** 2).sqrt()).reshape(-1, 1, 1, 1)
        F_x = self.unet(c_in * x, 1000 * sigma.log() / 4)
        return (c_skip * x + c_out * F_x).float().to(home)

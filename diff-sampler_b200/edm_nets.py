"""Host-side description of the EDM denoisers this engine runs: parameter dictionaries (reference
state_dict naming) and the block structure derived from them.

Reference: diff-solvers-main/models/networks_edm.py — SongUNet :220-355, DhariwalUNet :363-453,
UNetBlock :125-179, EDMPrecond :459-496; architecture configs from sfd-main/training/training_loop.py:62-76.
"""
import math
import re
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import List, Optional

import torch

NET_CONFIGS = {
    'cifar10': dict(kind='song', img_resolution=32, img_channels=3, label_dim=0, augment_dim=9, model_channels=128,
                    channel_mult=(2, 2, 2), num_blocks=4, attn_resolutions=(16,)),
    'ffhq': dict(kind='song', img_resolution=64, img_channels=3, label_dim=0, augment_dim=9, model_channels=128,
                 channel_mult=(1, 2, 2, 2), num_blocks=4, attn_resolutions=(16,)),
    'afhqv2': dict(kind='song', img_resolution=64, img_channels=3, label_dim=0, augment_dim=9, model_channels=128,
                   channel_mult=(1, 2, 2, 2), num_blocks=4, attn_resolutions=(16,)),
    'imagenet64': dict(kind='adm', img_resolution=64, img_channels=3, label_dim=1000, augment_dim=0, model_channels=192,
                       channel_mult=(1, 2, 3, 4), num_blocks=3, attn_resolutions=(32, 16, 8)),
    'tiny_song': dict(kind='song', img_resolution=16, img_channels=3, label_dim=0, augment_dim=9, model_channels=64,
                      channel_mult=(1, 2), num_blocks=1, attn_resolutions=(16,)),
    'tiny_song4': dict(kind='song', img_resolution=16, img_channels=3, label_dim=0, augment_dim=9, model_channels=64,
                       channel_mult=(1, 1), num_blocks=4, attn_resolutions=(8,)),
    'tiny_adm': dict(kind='adm', img_resolution=16, img_channels=3, label_dim=10, augment_dim=0, model_channels=64,
                     channel_mult=(1, 2), num_blocks=1, attn_resolutions=(16, 8)),
}


# ---------------------------------------------------------------------------------------------------------------------
# random initialisation (same draw order and distributions as the reference constructors, so a seed gives the same net)

def _draw(shape, mode, fan_in, fan_out):
    if mode == 'xavier_uniform':
        return math.sqrt(6 / (fan_in + fan_out)) * (torch.rand(*shape) * 2 - 1)
    if mode == 'kaiming_uniform':
        return math.sqrt(3 / fan_in) * (torch.rand(*shape) * 2 - 1)
    if mode == 'kaiming_normal':
        return math.sqrt(1 / fan_in) * torch.randn(*shape)
    raise ValueError(mode)


class _Init:
    def __init__(self):
        self.p = OrderedDict()

    def dense(self, name, fin, fout, bias=True, mode='kaiming_normal', w=1.0, b=0.0):
        self.p[name + '.weight'] = _draw([fout, fin], mode, fin, fout) * w
        if bias:
            self.p[name + '.bias'] = _draw([fout], mode, fin, fout) * b

    def conv(self, name, cin, cout, k, mode='kaiming_normal', w=1.0, b=0.0):
        if k == 0:
            return
        self.p[name + '.weight'] = _draw([cout, cin, k, k], mode, cin * k * k, cout * k * k) * w
        self.p[name + '.bias'] = _draw([cout], mode, cin * k * k, cout * k * k) * b

    def norm(self, name, c):
        self.p[name + '.weight'] = torch.ones(c)
        self.p[name + '.bias'] = torch.zeros(c)

    def block(self, name, cin, cout, emb, kind, up=False, down=False, attention=False):
        if kind == 'song':
            ini, zero, att = dict(mode='xavier_uniform'), dict(mode='xavier_uniform', w=1e-5), dict(mode='xavier_uniform', w=math.sqrt(0.2))
            adaptive, proj = False, True
        else:
            ini = dict(mode='kaiming_uniform', w=math.sqrt(1 / 3), b=math.sqrt(1 / 3))
            zero, att = dict(mode='kaiming_uniform', w=0.0, b=0.0), None
            adaptive, proj = True, False
        self.norm(name + '.norm0', cin)
        self.conv(name + '.conv0', cin, cout, 3, **ini)
        self.dense(name + '.affine', emb, cout * (2 if adaptive else 1), **ini)
        self.norm(name + '.norm1', cout)
        self.conv(name + '.conv1', cout, cout, 3, **zero)
        if cout != cin or up or down:
            self.conv(name + '.skip', cin, cout, 1 if (proj or cout != cin) else 0, **ini)
        if attention:
            self.norm(name + '.norm2', cout)
            self.conv(name + '.qkv', cout, cout * 3, 1, **(att or ini))
            self.conv(name + '.proj', cout, cout, 1, **zero)


def init_params(config, seed=0):
    """Random-init parameter dict (keys as EDMPrecond.state_dict(): 'model.enc.32x32_conv.weight', ...)."""
    cfg = dict(NET_CONFIGS[config]) if isinstance(config, str) else dict(config)
    kind, R, cimg = cfg['kind'], cfg['img_resolution'], cfg['img_channels']
    mc, mult, nb, attn = cfg['model_channels'], cfg['channel_mult'], cfg['num_blocks'], cfg['attn_resolutions']
    label_dim, aug = cfg.get('label_dim', 0), cfg.get('augment_dim', 0)
    emb = mc * 4
    torch.manual_seed(seed)
    I = _Init()
    if kind == 'song':
        ini = dict(mode='xavier_uniform')
        if label_dim:
            I.dense('map_label', label_dim, mc, **ini)
        if aug:
            I.dense('map_augment', aug, mc, bias=False, **ini)
        I.dense('map_layer0', mc, emb, **ini)
        I.dense('map_layer1', emb, emb, **ini)
    else:
        ini = dict(mode='kaiming_uniform', w=math.sqrt(1 / 3), b=math.sqrt(1 / 3))
        if aug:
            I.dense('map_augment', aug, mc, bias=False, mode='kaiming_uniform', w=0.0, b=0.0)
        I.dense('map_layer0', mc, emb, **ini)
        I.dense('map_layer1', emb, emb, **ini)
        if label_dim:
            I.dense('map_label', label_dim, emb, bias=False, mode='kaiming_normal', w=math.sqrt(label_dim))
    cout = cimg
    skips = []
    for level, m in enumerate(mult):
        res = R >> level
        if level == 0:
            cin, cout = cout, (mc if kind == 'song' else mc * m)
            I.conv(f'enc.{res}x{res}_conv', cin, cout, 3, **ini)
        else:
            I.block(f'enc.{res}x{res}_down', cout, cout, emb, kind, down=True)
        skips.append(cout)
        for idx in range(nb):
            cin, cout = cout, mc * m
            I.block(f'enc.{res}x{res}_block{idx}', cin, cout, emb, kind, attention=(res in attn))
            skips.append(cout)
    for level, m in reversed(list(enumerate(mult))):
        res = R >> level
        if level == len(mult) - 1:
            I.block(f'dec.{res}x{res}_in0', cout, cout, emb, kind, attention=True)
            I.block(f'dec.{res}x{res}_in1', cout, cout, emb, kind)
        else:
            I.block(f'dec.{res}x{res}_up', cout, cout, emb, kind, up=True)
        for idx in range(nb + 1):
            cin = cout + skips.pop()
            cout = mc * m
            att = (idx == nb and res in attn) if kind == 'song' else (res in attn)
            I.block(f'dec.{res}x{res}_block{idx}', cin, cout, emb, kind, attention=att)
        if kind == 'song' and level == 0:
            I.norm(f'dec.{res}x{res}_aux_norm', cout)
            I.conv(f'dec.{res}x{res}_aux_conv', cout, cimg, 3, mode='xavier_uniform', w=1e-5)
    if kind == 'adm':
        I.norm('out_norm', cout)
        I.conv('out_conv', cout, cimg, 3, mode='kaiming_uniform', w=0.0, b=0.0)
    return OrderedDict(('model.' + k, v) for k, v in I.p.items()), cfg


def dezero_(params, kind, seed=0):
    """Give the init_zero layers O(1) weights so that |F_x| = O(1) (the meaningful parity/benchmark weight set for
    random-init nets; SURVEY.md section 7 hard part 1).  SongUNet: x1e5 (draws were scaled by 1e-5); ADM: re-drawn."""
    g = torch.Generator().manual_seed(seed + 12345)
    for k in list(params.keys()):
        base = k.rsplit('.', 1)[0]
        leaf = base.rsplit('.', 1)[-1]
        if leaf in ('conv1', 'proj') or base.endswith('aux_conv') or base.endswith('out_conv'):
            if kind == 'song':
                params[k] = params[k] * 1e5
            elif k.endswith('.weight'):
                fan_in = params[k][0].numel()
                params[k] = math.sqrt(1 / fan_in) * (torch.rand(params[k].shape, generator=g) * 2 - 1)
    return params


# ---------------------------------------------------------------------------------------------------------------------
# structure, derived from parameter names and shapes (works for our own init and for a reference net's state_dict)

@dataclass
class BlockSpec:
    name: str
    cin: int
    cout: int
    res_in: int
    res_out: int
    up: bool
    down: bool
    heads: int
    skip: str                # 'identity' | 'conv' | 'resample'
    adaptive_scale: bool
    skip_scale: float
    eps: float
    concat: int = 0          # channels taken from the skip stack (virtual concat), 0 = none
    aff_off: int = 0         # column offset of this block's affine output in the fused affine matrix
    aff_width: int = 0


@dataclass
class NetSpec:
    kind: str
    img_resolution: int
    img_channels: int
    label_dim: int
    noise_channels: int
    emb_channels: int
    stem: str
    stem_cout: int
    enc: List[BlockSpec] = field(default_factory=list)
    dec: List[BlockSpec] = field(default_factory=list)
    head_norm: str = ''
    head_conv: str = ''
    head_eps: float = 1e-5
    aff_total: int = 0
    sigma_data: float = 0.5
    sigma_min: float = 0.002
    sigma_max: float = 80.0
    prefix: str = 'model.'
    bottleneck_block: Optional[str] = None
    noise_scale: float = 1.0         # the embedding reads noise_scale * ln(sigma) / 4 (1: EDM, 1000: Consistency Models' CMPrecond)


def spec_from_params(params, img_resolution, img_channels, label_dim, prefix='model.'):
    keys = [k[len(prefix):] for k in params.keys() if k.startswith(prefix)]
    kind = 'adm' if 'out_norm.weight' in keys else 'song'
    P = lambda k: params[prefix + k]
    emb = P('map_layer1.weight').shape[0]
    noise = P('map_layer0.weight').shape[1]
    order = []
    for k in keys:
        m = re.match(r'(enc|dec)\.(\d+)x\d+_([a-z0-9_]+?)\.', k)
        if m:
            nm = k.split('.')[0] + '.' + k.split('.')[1]
            if nm not in order:
                order.append(nm)
    stem = order[0]
    assert stem.endswith('_conv'), stem
    spec = NetSpec(kind=kind, img_resolution=img_resolution, img_channels=img_channels, label_dim=label_dim, noise_channels=noise,
                   emb_channels=emb, stem=stem, stem_cout=P(stem + '.weight').shape[0])
    skip_stack = [spec.stem_cout]
    cur_c, cur_res = spec.stem_cout, img_resolution
    aff = 0
    for nm in order[1:]:
        part, tail = nm.split('.')
        res = int(tail.split('x')[0])
        role = tail.split('_', 1)[1]
        if role in ('aux_norm', 'aux_conv'):
            if role == 'aux_norm':
                spec.head_norm, spec.head_eps = nm, 1e-6
            else:
                spec.head_conv = nm
            continue
        w0 = P(nm + '.conv0.weight')
        cin, cout = w0.shape[1], w0.shape[0]
        up, down = role == 'up', role == 'down'
        res_in = res // 2 if up else (res * 2 if down else res)
        heads = 0
        if (nm + '.qkv.weight') in keys:
            heads = 1 if kind == 'song' else cout // 64
        if (nm + '.skip.weight') in keys:
            skip = 'conv'
        elif up or down:
            skip = 'resample'
        else:
            assert cin == cout
            skip = 'identity'
        adaptive = kind == 'adm'
        b = BlockSpec(name=nm, cin=cin, cout=cout, res_in=res_in, res_out=res, up=up, down=down, heads=heads, skip=skip,
                      adaptive_scale=adaptive, skip_scale=(math.sqrt(0.5) if kind == 'song' else 1.0),
                      eps=(1e-6 if kind == 'song' else 1e-5), aff_off=aff, aff_width=P(nm + '.affine.weight').shape[0])
        aff += b.aff_width
        if part == 'enc':
            assert cin == cur_c and res_in == cur_res, (nm, cin, cur_c, res_in, cur_res)
            spec.enc.append(b)
            skip_stack.append(cout)
        else:
            if cin != cur_c:
                b.concat = skip_stack.pop()
                assert cur_c + b.concat == cin, (nm, cur_c, b.concat, cin)
            spec.dec.append(b)
        cur_c, cur_res = cout, res
    if kind == 'adm':
        spec.head_norm, spec.head_conv, spec.head_eps = 'out_norm', 'out_conv', 1e-5
    spec.aff_total = aff
    # AMED reads the encoder bottleneck: '8x8_block2' for class-conditional nets, '8x8_block3' otherwise (solvers_amed.py:16)
    want = 'enc.8x8_block2' if label_dim else 'enc.8x8_block3'
    names = [b.name for b in spec.enc]
    spec.bottleneck_block = want if want in names else (names[-1] if names else None)
    return spec

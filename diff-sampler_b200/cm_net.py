"""Host-side importer for the Consistency-Models LSUN-256 denoisers (lsun_bedroom, lsun_cat): the EDM-trained pixel-space
U-Nets that diff-solvers-main/sample.py loads with models/cm/cm_model_loader.py:load_cm_model and wraps in CMPrecond.

The CM `UNetModel` (models/cm/unet.py:505-772) is the ADM topology DhariwalUNet lowers, with additive (not scale-shift) time
conditioning, so it runs through plan.compile_plan unchanged once its state dict is renamed to the EDM block order:

  input_blocks.0.0                        -> enc.{R}x{R}_conv
  input_blocks.i.0 (ResBlock [+ .1 Attn]) -> enc.{r}x{r}_block{j}   /  (ResBlock down=True) -> enc.{r}x{r}_down
  middle_block.0 + .1 (Attn), .2          -> dec.{r}x{r}_in0, dec.{r}x{r}_in1
  output_blocks.i.0 [+ .1 Attn]           -> dec.{r}x{r}_block{j};  the trailing ResBlock(up=True) -> dec.{2r}x{2r}_up
  time_embed.0 / .2, out.0 / .2           -> map_layer0 / map_layer1, out_norm / out_conv

Inside a ResBlock: in_layers.0 / .2 -> norm0 / conv0, emb_layers.1 -> affine, out_layers.0 / .3 -> norm1 / conv1,
skip_connection -> skip; an AttentionBlock folds into the block before it: norm -> norm2, qkv -> qkv (rows permuted, see
qkv_cm_to_edm), proj_out -> proj.  Where the ResBlocks resample cannot be read from the state dict (Downsample / Upsample
without a conv have no parameters), so the structure comes from the loader's settings (cm_model_loader.py:95-115).
"""
import math
from collections import OrderedDict

import torch

from .edm_nets import BlockSpec, NetSpec


def lsun_setting():
    """The settings load_cm_model uses for every non-ImageNet checkpoint (cm_model_loader.py:95-115)."""
    return dict(image_size=256, num_channels=256, num_res_blocks=2, num_heads=4, num_heads_upsample=-1, num_head_channels=64,
                attention_resolutions='32,16,8', channel_mult='', dropout=0.1, class_cond=False, use_checkpoint=False,
                use_scale_shift_norm=False, resblock_updown=True, use_fp16=True, use_new_attention_order=False, learn_sigma=False)


# CMPrecond feeds 1000 * ln(sigma) / 4 to the U-Net's timestep embedding (networks_edm.py:539-540)
CM_NOISE_SCALE = 1000.0


def _channel_mult(setting):
    cm = setting.get('channel_mult', '')
    if isinstance(cm, (tuple, list)):
        return tuple(cm)
    if cm == '':
        defaults = {512: (0.5, 1, 1, 2, 2, 4, 4), 256: (1, 1, 2, 2, 4, 4), 128: (1, 1, 2, 3, 4), 64: (1, 2, 3, 4)}
        if setting['image_size'] not in defaults:
            raise ValueError(f"image_size={setting['image_size']}: no default channel_mult")
        return defaults[setting['image_size']]
    return tuple(int(m) for m in cm.split(','))


def _attention_ds(setting):
    """Downsampling factors that carry attention (create_model turns resolutions into image_size // res)."""
    ar = setting.get('attention_resolutions', '16')
    res = [int(r) for r in ar.split(',')] if isinstance(ar, str) else [int(r) for r in ar]
    return {setting['image_size'] // r for r in res}


def check_setting(setting):
    """Reject the configurations this lowering does not cover, naming the field."""
    s = setting
    if s.get('use_scale_shift_norm'):
        raise ValueError('use_scale_shift_norm=True (FiLM conditioning) is not lowered for CM nets')
    if s.get('class_cond'):
        raise ValueError('class_cond=True is not lowered for CM nets')
    if s.get('learn_sigma'):
        raise ValueError('learn_sigma=True (6 output channels) is not lowered for CM nets')
    if not s.get('resblock_updown'):
        raise ValueError('resblock_updown=False (conv / pooling resamplers) is not lowered for CM nets')
    mc, mult = s['num_channels'], _channel_mult(s)
    widths = [int(m * mc) for m in mult]
    if min(widths) < 128:
        # GroupNorm32 always uses 32 groups; the plan uses min(32, C // 4) groups, which agrees from 128 channels on
        raise ValueError(f'num_channels={mc}, channel_mult={mult}: widths below 128 channels are not lowered for CM nets')
    ads = _attention_ds(s)
    for level, w in enumerate(widths):
        if (1 << level) in ads or level == len(widths) - 1:          # the middle block always attends
            hc = s.get('num_head_channels', -1)
            width = hc if hc != -1 else w // s.get('num_heads', 1)
            if width != 64 or w % 64:
                raise ValueError(f'num_head_channels={hc} (num_heads={s.get("num_heads")}): attention heads must be 64 wide')


def structure(setting=None):
    """NetSpec of the CM UNetModel built from `setting` (default lsun_setting()), plus the CM module path of every block:
    {edm block name: (resblock path, attention path or None)}, stem and head paths included under their EDM names."""
    s = dict(lsun_setting() if setting is None else setting)
    check_setting(s)
    R, mc = s['image_size'], s['num_channels']
    mult, nb, ads = _channel_mult(s), s['num_res_blocks'], _attention_ds(s)
    emb = 4 * mc
    ch = int(mult[0] * mc)
    spec = NetSpec(kind='cm', img_resolution=R, img_channels=3, label_dim=0, noise_channels=mc, emb_channels=emb,
                   stem=f'enc.{R}x{R}_conv', stem_cout=ch, head_norm='out_norm', head_conv='out_conv', head_eps=1e-5)
    spec.noise_scale = CM_NOISE_SCALE
    paths = OrderedDict([(spec.stem, ('input_blocks.0.0', None))])
    aff = 0

    def block(part, name, cm_res, cm_attn, cin, cout, res_in, res_out, up=False, down=False, heads=0, concat=0):
        nonlocal aff
        skip = 'conv' if cin != cout else ('resample' if (up or down) else 'identity')
        if concat and skip == 'identity':
            raise ValueError(f'{name}: a concatenating block with an identity skip is not lowered')
        b = BlockSpec(name=name, cin=cin, cout=cout, res_in=res_in, res_out=res_out, up=up, down=down, heads=heads, skip=skip,
                      adaptive_scale=False, skip_scale=1.0, eps=1e-5, concat=concat, aff_off=aff, aff_width=cout)
        aff += cout
        (spec.enc if part == 'enc' else spec.dec).append(b)
        paths[name] = (cm_res, cm_attn)

    chans = [ch]                     # input_block_chans of the reference constructor
    i, ds = 1, 1
    for level, m in enumerate(mult):
        r = R // ds
        for j in range(nb):
            cout = int(m * mc)
            att = ds in ads
            block('enc', f'enc.{r}x{r}_block{j}', f'input_blocks.{i}.0', f'input_blocks.{i}.1' if att else None, ch, cout, r, r,
                  heads=cout // 64 if att else 0)
            ch = cout
            chans.append(ch)
            i += 1
        if level != len(mult) - 1:
            block('enc', f'enc.{r // 2}x{r // 2}_down', f'input_blocks.{i}.0', None, ch, ch, r, r // 2, down=True)
            chans.append(ch)
            i += 1
            ds *= 2
    r = R // ds
    block('dec', f'dec.{r}x{r}_in0', 'middle_block.0', 'middle_block.1', ch, ch, r, r, heads=ch // 64)
    block('dec', f'dec.{r}x{r}_in1', 'middle_block.2', None, ch, ch, r, r)
    spec.bottleneck_block = f'dec.{r}x{r}_in1'           # the middle_block output, AMED's tap for 256-pixel nets (solvers_amed.py:11-14)
    i = 0
    for level, m in reversed(list(enumerate(mult))):
        r = R // ds
        for j in range(nb + 1):
            ich = chans.pop()
            cout = int(m * mc)
            att = ds in ads
            block('dec', f'dec.{r}x{r}_block{j}', f'output_blocks.{i}.0', f'output_blocks.{i}.1' if att else None, ch + ich, cout,
                  r, r, heads=cout // 64 if att else 0, concat=ich)
            ch = cout
            if level and j == nb:
                block('dec', f'dec.{2 * r}x{2 * r}_up', f'output_blocks.{i}.{2 if att else 1}', None, ch, ch, r, 2 * r, up=True)
                ds //= 2
            i += 1
    paths['out_norm'] = ('out.0', None)
    paths['out_conv'] = ('out.2', None)
    spec.aff_total = aff
    return spec, paths


def qkv_cm_to_edm(w, heads):
    """Rows of the CM qkv conv ([q|k|v][head][d]: QKVFlashAttention's `b (three h d) s`, unet.py:365-366) in the EDM order
    [head][d][q|k|v] that plan._qkv_split reads (networks_edm.py:174)."""
    c3 = w.shape[0]
    d = c3 // 3 // heads
    return w.reshape(3, heads, d, *w.shape[1:]).movedim(0, 2).reshape(c3, *w.shape[1:])


def convert(state_dict, setting=None, prefix=''):
    """(NetSpec, EDM-named float32 parameter dict with the 'model.' prefix plan.pack_weights reads) from a CM UNetModel state
    dict (keys under `prefix`: '' for the released checkpoint, 'model.' for CMPrecond.state_dict())."""
    spec, paths = structure(setting)
    sd = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
    used = set()
    out = OrderedDict()

    def take(src, dst, shape=None):
        for leaf in ('weight', 'bias'):
            k = f'{src}.{leaf}'
            if k not in sd:
                raise KeyError(f'CM state dict has no {prefix}{k} (needed for {dst})')
            t = sd[k].detach().to(torch.float32).cpu()           # convert_to_fp16 leaves the torso in half precision
            if leaf == 'weight' and shape is not None:
                t = shape(t)
            out[f'model.{dst}.{leaf}'] = t
            used.add(k)

    def conv1x1(t):                  # [Cout, Cin, 1, 1] (conv_nd(2, ...), unet.py:290, :304), or [Cout, Cin, 1] from a conv1d build
        return t.reshape(t.shape[0], t.shape[1], 1, 1)

    take('time_embed.0', 'map_layer0')
    take('time_embed.2', 'map_layer1')
    take(paths[spec.stem][0], spec.stem)
    for b in spec.enc + spec.dec:
        res, attn = paths[b.name]
        n = b.name
        take(f'{res}.in_layers.0', n + '.norm0')
        take(f'{res}.in_layers.2', n + '.conv0')
        take(f'{res}.emb_layers.1', n + '.affine')
        take(f'{res}.out_layers.0', n + '.norm1')
        take(f'{res}.out_layers.3', n + '.conv1')
        if b.skip == 'conv':
            take(f'{res}.skip_connection', n + '.skip')
        if attn:
            take(f'{attn}.norm', n + '.norm2')
            take(f'{attn}.qkv', n + '.qkv', lambda t: conv1x1(qkv_cm_to_edm(t, b.heads)))
            out[f'model.{n}.qkv.bias'] = qkv_cm_to_edm(out[f'model.{n}.qkv.bias'], b.heads)
            take(f'{attn}.proj_out', n + '.proj', conv1x1)
    take('out.0', 'out_norm')
    take('out.2', 'out_conv')
    for b in spec.enc + spec.dec:                                 # shapes must agree with the structure the settings describe
        w0 = out[f'model.{b.name}.conv0.weight']
        if tuple(w0.shape[:2]) != (b.cout, b.cin):
            raise ValueError(f'{paths[b.name][0]}: conv of shape {tuple(w0.shape)} does not match the settings ({b.cin} -> {b.cout})')
        if out[f'model.{b.name}.affine.weight'].shape != (b.cout, spec.emb_channels):
            raise ValueError(f'{paths[b.name][0]}.emb_layers.1: expected an additive {b.cout}-wide embedding projection')
    extra = sorted(k for k in sd if k not in used)
    if extra:
        raise ValueError(f'CM state dict has parameters the settings do not describe: {extra[:4]}')
    return spec, out


# ---------------------------------------------------------------------------------------------------------------------
# random weights with the real key names and shapes (tests, tools/cm_probe.py)

def init_state_dict(setting=None, seed=0, dezero=True):
    """A UNetModel-layout state dict for `setting` with PyTorch-default-like uniform draws.  dezero=True gives the zero_module
    layers (out_layers.3, proj_out, out.2) O(1) weights so the parity checks see every path."""
    spec, paths = structure(setting)
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()

    def lin(name, fin, fout, k=None, zero=False):
        shape = [fout, fin] + ([k, k] if k else [])
        fan = fin * (k * k if k else 1)
        bound = 0.0 if zero and not dezero else 1.0 / math.sqrt(fan)
        sd[name + '.weight'] = (torch.rand(shape, generator=g) * 2 - 1) * bound
        sd[name + '.bias'] = (torch.rand([fout], generator=g) * 2 - 1) * (1.0 / math.sqrt(fan))

    def gn(name, c):
        sd[name + '.weight'] = 1 + 0.1 * torch.randn(c, generator=g)
        sd[name + '.bias'] = 0.1 * torch.randn(c, generator=g)

    mc, emb = spec.noise_channels, spec.emb_channels
    lin('time_embed.0', mc, emb)
    lin('time_embed.2', emb, emb)
    lin(paths[spec.stem][0], 3, spec.stem_cout, 3)
    for b in spec.enc + spec.dec:
        res, attn = paths[b.name]
        gn(f'{res}.in_layers.0', b.cin)
        lin(f'{res}.in_layers.2', b.cin, b.cout, 3)
        lin(f'{res}.emb_layers.1', emb, b.cout)
        gn(f'{res}.out_layers.0', b.cout)
        lin(f'{res}.out_layers.3', b.cout, b.cout, 3, zero=True)
        if b.skip == 'conv':
            lin(f'{res}.skip_connection', b.cin, b.cout, 1)
        if attn:
            gn(f'{attn}.norm', b.cout)
            lin(f'{attn}.qkv', b.cout, 3 * b.cout, 1)
            lin(f'{attn}.proj_out', b.cout, b.cout, 1, zero=True)
    gn('out.0', spec.stem_cout)
    lin('out.2', spec.stem_cout, 3, 3, zero=True)
    return sd


TINY_SETTING = dict(lsun_setting(), image_size=32, num_channels=64, num_res_blocks=1, channel_mult='2,2,2', attention_resolutions='16,8')

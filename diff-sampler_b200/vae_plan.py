"""Plan compiler for the latent-diffusion first-stage DECODER (SURVEY section 8(f)3: what `decode_first_stage` runs after sampling,
sample.py:299).  OPT-IN and not yet run on hardware (tests/test_gpu_parity.py::test_vae_decoder_parity is gated).

Reference being lowered (paths under models/ldm/): models/diffusion/ddpm.py:714 (z / scale_factor), models/autoencoder.py
`AutoencoderKL.decode` (post_quant_conv 1x1 then the decoder), modules/diffusionmodules/model.py:462-569 `Decoder.forward`,
:82-141 `ResnetBlock` (temb=None), :150-203 `AttnBlock` (one head over all channels), :42-57 `Upsample` (nearest x2 + conv3x3).

Same op set and executor as the denoisers (plan.py / ldm_plan.py): GroupNorm(32, eps 1e-6) statistics + apply(+swish) kernels, the
wgmma GEMM kernel for every convolution (1x1 skip `nin_shortcut` appended along K) and for the QK^T / PV products of the single
wide-head attention, the row softmax.  New for this net: image rows wider than one 128-pixel M tile (256- and 512-wide levels) --
`gemm_desc.conv_gemm` then tiles them as 128-pixel row segments.
io slots: X = latents [B, z_ch, R, R] (NCHW fp32), LABELS = coef [1][4] with 1/scale_factor in slot 2, D = images [B, out_ch, sR, sR].

VQ first stages (`VQModelInterface.decode`, autoencoder.py:274-282, e.g. the VQ-f4 of the LSUN-Bedroom / FFHQ LDMs) differ only in
front: the state dict also holds `quantize.embedding.weight` [n_embed, embed_dim], and unless the caller passes force_not_quantize the
input op snaps every latent pixel to its nearest codebook row (VectorQuantizer2 inference: argmin of the squared L2 distance, then that
row) while it writes post_quant_conv's operand planes (csrc/elementwise.cu vq_prep_input_kernel).
"""
from collections import OrderedDict

import torch

from . import _cstructs as S
from . import gemm_desc as G
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob, io


def vae_structure(params):
    """Execution-ordered module list from `first_stage_model.state_dict()` names / shapes (decoder.*, post_quant_conv.* and, for a VQ
    first stage, quantize.embedding.weight):
    [('conv', name, cin, cout) | ('res', name, cin, cout) | ('attn', name, c) | ('up', name, c)], meta (+ n_embed for a VQ first stage)."""
    def shp(k):
        return tuple(params[k].shape)
    P = params
    assert 'decoder.conv_in.weight' in P and 'post_quant_conv.weight' in P, 'not an AutoencoderKL / VQModel decoder state_dict'
    block_in = shp('decoder.conv_in.weight')[0]
    mods = [('conv', 'decoder.conv_in', shp('decoder.conv_in.weight')[1], block_in)]
    for n in ('decoder.mid.block_1', 'decoder.mid.attn_1', 'decoder.mid.block_2'):
        if n + '.conv1.weight' in P:
            mods.append(('res', n, shp(n + '.conv1.weight')[1], shp(n + '.conv1.weight')[0]))
        elif n + '.q.weight' in P:
            mods.append(('attn', n, shp(n + '.q.weight')[0]))
    levels = sorted({int(k.split('.')[2]) for k in P if k.startswith('decoder.up.')})
    for lvl in reversed(levels):
        i = 0
        while f'decoder.up.{lvl}.block.{i}.conv1.weight' in P:
            n = f'decoder.up.{lvl}.block.{i}'
            mods.append(('res', n, shp(n + '.conv1.weight')[1], shp(n + '.conv1.weight')[0]))
            assert f'decoder.up.{lvl}.attn.{i}.q.weight' not in P, 'attention inside the up levels is not lowered (SD-v1: attn_resolutions = [])'
            i += 1
        if f'decoder.up.{lvl}.upsample.conv.weight' in P:
            mods.append(('up', f'decoder.up.{lvl}.upsample', shp(f'decoder.up.{lvl}.upsample.conv.weight')[0]))
    c_end = shp('decoder.norm_out.weight')[0]
    meta = dict(z_channels=shp('post_quant_conv.weight')[0], embed_dim=shp('post_quant_conv.weight')[1], out_ch=shp('decoder.conv_out.weight')[0],
                c_end=c_end, upscale=2 ** sum(1 for m in mods if m[0] == 'up'))
    for m in mods:
        for c in m[2:]:
            assert m[0] == 'conv' or c % 64 == 0, f'{m[1]}: channel counts must be multiples of 64, got {c}'
    if 'quantize.embedding.weight' in P:                          # VQModelInterface: latents are snapped to a codebook row first
        n_embed, e_dim = shp('quantize.embedding.weight')
        if e_dim != meta['embed_dim'] or e_dim > 8:
            raise ValueError(f'quantize.embedding.weight {(n_embed, e_dim)}: the codebook must have embed_dim = '
                             f'{meta["embed_dim"]} <= 8 columns')
        meta['n_embed'] = n_embed
    return mods, meta


def pack_vae_weights(mods, meta, params):
    P = lambda k: params[k].detach().float().cpu()
    wb = WeightBlob()

    wb.add_gemm('post_quant_conv', P('post_quant_conv.weight'), bias=P('post_quant_conv.bias'))
    for m in mods:
        n = m[1]
        if m[0] == 'conv':
            wb.add_gemm(n, P(n + '.weight'), bias=P(n + '.bias'))
        elif m[0] == 'res':
            assert (n + '.conv_shortcut.weight') not in params, '3x3 conv_shortcut is not lowered (SD-v1 uses nin_shortcut)'
            skip = n + '.nin_shortcut' if (n + '.nin_shortcut.weight') in params else None
            wb.add_res_block(n, P, n + '.norm1', n + '.conv1', n + '.norm2', n + '.conv2', skip)
        elif m[0] == 'attn':
            c = m[2]
            wq, wk, wv = (P(f'{n}.{t}.weight').reshape(c, c) for t in 'qkv')
            wb.add_attn_block(n, P, n + '.norm', (torch.cat([wq, wk]), torch.cat([P(n + '.q.bias'), P(n + '.k.bias')])),
                              (wv, P(n + '.v.bias')), (P(n + '.proj_out.weight'), P(n + '.proj_out.bias')))
        elif m[0] == 'up':
            wb.add_gemm(n, P(n + '.conv.weight'), bias=P(n + '.conv.bias'))
    wb.add_norm('norm_out', P, 'decoder.norm_out')
    wb.add_gemm('conv_out', P('decoder.conv_out.weight'), bias=P('decoder.conv_out.bias'))
    if 'n_embed' in meta:
        wb.add('quantize:e', P('quantize.embedding.weight'))          # fp32 [n_embed][embed_dim]
    return wb


def compile_vae_plan(mods, meta, wb, B, R, npass=3, quantize=False, debug_indices=False):
    """Lower the decoder for B latents of resolution R x R.  quantize (VQ first stages only): snap each latent pixel to its nearest
    codebook row before post_quant_conv, as VQModelInterface.decode does unless force_not_quantize; debug_indices then also keeps the
    chosen rows in the int32 arena buffer 'vq_idx' [B][R * R]."""
    if quantize and 'n_embed' not in meta:
        raise ValueError('quantize: this first stage has no codebook (not a VQModelInterface)')
    pb = PlanBuilder(wb, B, npass)
    emit, W = pb.emit, wb.ref
    pb.stats()

    # ---- z / scale_factor (-> nearest codebook row) -> fp16 planes (channels zero-padded to 64) -> post_quant_conv (1x1) -> conv_in ------
    HW = R * R
    pb.need('in_planes', NPL * B * HW * 64 * H2)
    vq = {}
    if quantize:
        vq = dict(codebook=W('quantize:e'), n_embed=meta['n_embed'])
    emit(lambda R_: S.PrepInputDesc(x=io(S.DS_IO_X), coef=io(S.DS_IO_LABELS), coef_stride=0, B=B, C=meta['embed_dim'], HW=HW, nplanes=NPL,
                                    x_batch=B, out=R_('in_planes'), idx=R_('vq_idx') if quantize and debug_indices else 0, **vq))
    # dedicated buffer: only z_channels of its 64 columns are ever written, the rest stay at the arena's initial zeros
    pb.need('pq_planes', NPL * B * HW * 64 * H2)
    emit(lambda R_: G.conv_gemm(R_('in_planes'), B, R, R, 64, W('post_quant_conv:w'), meta['z_channels'], taps=1, npass=npass,
                                out_h16=R_('pq_planes'), ldo=64, bias=W('post_quant_conv:b'))[0])
    cur, cur_c, H = None, None, R
    for m in mods:
        pb.tag += 1
        out = 'h:' + m[1]
        if m[0] == 'conv':
            cur, cur_c = pb.need(out, B * HW * m[3] * F4), m[3]
            emit(lambda R_, m=m, cur=cur: G.conv_gemm(R_('pq_planes'), B, R, R, 64, W(m[1] + ':w'), m[3], taps=9, npass=npass, out_f32=R_(cur),
                                                      bias=W(m[1] + ':b'))[0])
        elif m[0] == 'res':
            _, n, cin, cout = m
            pb.res_block(n, [(cur, cin)], H, cout, out, eps=1e-6, skip='conv' if cin != cout else 'identity')
            cur, cur_c = pb.need(out, B * H * H * cout * F4), cout
        elif m[0] == 'attn':
            assert H * H % 64 == 0, 'attention needs a multiple of 64 positions (K extent of the PV product)'
            for name in ('qk', 'vt', 'S', 'P'):       # this plan's arena keeps 'o' after the unfused attention's scores
                pb.need(name, 0)
            pb.attn_block(m[1], cur, cur_c, H, out, eps=1e-6, heads=1, d=cur_c, scale=float(cur_c) ** -0.5, fused=False)
            cur = out
        elif m[0] == 'up':
            pb.upsample_conv(m[1], cur, cur_c, H, m[2], out)
            cur, H = out, 2 * H
    # ---- norm_out + swish + conv_out -> images, NCHW fp32 ----------------------------------------------------------------------------
    pb.tag += 1
    pb.head_conv(cur, cur_c, H, 'norm_out', 1e-6, 'conv_out', meta['out_ch'], nchw_out=(meta['out_ch'], io(S.DS_IO_D)))
    assert H == R * meta['upscale']
    if quantize and debug_indices:
        pb.need('vq_idx', B * HW * 4)                             # last: the other buffers keep the offsets of the plain plan
    return pb.finish(B=B, R=R, out_res=H, npass=npass, **({'quantize': True} if quantize else {}))

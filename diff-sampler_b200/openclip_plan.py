"""Plan compilers of the CLIP score: open_clip's ViT-g-14 (`laion2b_s34b_b88k`) image and text towers as clip_score.py runs them
(diff-solvers-main/clip_score.py:59-89), from weights in open_clip's state-dict layout.  DESIGN.md 4.11.

Image tower, B uint8 images [B][3][H][W] (io X, element strides `strides`) -> io D [B][E] fp32, L2-normalised:
  * ds_clip_input: Pillow's bicubic resize of the shorter side to S, the S x S centre crop, ToTensor and Normalize (open_clip's
    transform, clip_score.py:59 `preprocess`, :81), bit-exact, from the resample tables of `bicubic_tables` (io CTX);
  * the 14 x 14 / stride 14 patch convolution is ds_im2col (K = 588 -> 640) and ONE batched rows GEMM whose epilogue adds the
    positional rows 1..256 (the residual operand, the same for every sample) and writes rows 1..256 of each sample's 257;
  * row 0 of each sample, class_embedding + positional row 0, is one gather of that precomputed weight row; ln_pre;
  * 40 pre-LN blocks (clip_plan.transformer_layer, exact GELU, 16 heads of 88 on attn_wide_kernel);
  * ln_post of token 0, @ proj, L2-normalised (clip_plan.pooled_head).
Text tower, B prompts of open_clip token ids [B][77] int32 (io X) -> io D [B][E]: clip_plan.compile_clip_plan with exact GELU and the
pooled head (ln_final of the row at argmax(ids), @ text_projection).
Pure host logic: no GPU needed to compile a plan."""
import math

import torch

from . import _cstructs as S
from . import gemm_desc as G
from .clip_plan import compile_clip_plan, layernorm, pooled_head, reserve_layer_buffers, transformer_layer
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob, io

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)         # open_clip.constants OPENAI_DATASET_MEAN / _STD (ViT-g-14's transform)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
PRECISION_BITS = 22                                      # Pillow's 8-bit resample passes: 32 - 8 - 2 fraction bits


def openclip_config(sd, vision_head_width=88, text_head_width=64):
    """Dimensions from an open_clip CLIP state dict.  The head counts are not in it: ViT-g-14's towers have 88-wide (image) and
    64-wide (text) heads."""
    v = 'visual.'
    n_v = 1 + max(int(k.split('.')[3]) for k in sd if k.startswith(v + 'transformer.resblocks.'))
    n_t = 1 + max(int(k.split('.')[2]) for k in sd if k.startswith('transformer.resblocks.'))
    wv, P = sd[v + 'conv1.weight'].shape[0], sd[v + 'conv1.weight'].shape[2]
    grid = math.isqrt(sd[v + 'positional_embedding'].shape[0] - 1)
    wt = sd['token_embedding.weight'].shape[1]
    return dict(image_size=grid * P, patch_size=P, vision_width=wv, vision_layers=n_v, vision_heads=wv // vision_head_width,
                vision_mlp=sd[v + 'transformer.resblocks.0.mlp.c_fc.weight'].shape[0], embed_dim=sd[v + 'proj'].shape[1],
                vocab_size=sd['token_embedding.weight'].shape[0], context_length=sd['positional_embedding'].shape[0], text_width=wt,
                text_layers=n_t, text_heads=wt // text_head_width, text_mlp=sd['transformer.resblocks.0.mlp.c_fc.weight'].shape[0])


def text_config(cfg):
    """The clip_plan config of the text tower."""
    return dict(vocab_size=cfg['vocab_size'], hidden_size=cfg['text_width'], max_position_embeddings=cfg['context_length'],
                num_hidden_layers=cfg['text_layers'], intermediate_size=cfg['text_mlp'], num_attention_heads=cfg['text_heads'])


def _add_blocks(wb, P, src, dst, n):
    """open_clip ResidualAttentionBlocks `src`.<i> as the weights clip_plan.transformer_layer reads under `dst`l<i>."""
    for i in range(n):
        s, d = f'{src}.{i}.', f'{dst}l{i}.'
        w, b = P(s + 'attn.in_proj_weight'), P(s + 'attn.in_proj_bias')
        H = w.shape[1]
        wb.add_gemm(d + 'qk', w[:2 * H], bias=b[:2 * H])
        wb.add(d + 'v:w', G.split_planes(w[2 * H:]))
        wb.add(d + 'v:b', b[2 * H:])
        wb.add_gemm(d + 'out', P(s + 'attn.out_proj.weight'), bias=P(s + 'attn.out_proj.bias'))
        wb.add_gemm(d + 'fc1', P(s + 'mlp.c_fc.weight'), bias=P(s + 'mlp.c_fc.bias'))
        wb.add_gemm(d + 'fc2', P(s + 'mlp.c_proj.weight'), bias=P(s + 'mlp.c_proj.bias'))
        wb.add_norm(d + 'layer_norm1', P, s + 'ln_1')
        wb.add_norm(d + 'layer_norm2', P, s + 'ln_2')


def pack_openclip_weights(sd, cfg):
    """One weight blob for both towers: the image tower under 'v.', the text tower under 't.'.  `proj` and `text_projection` are
    applied as x @ P, so their transposes are the GEMM weights."""
    P = lambda k: sd[k].detach().float().cpu()
    wb = WeightBlob()
    conv = P('visual.conv1.weight')                                              # [W][3][P][P] -> [W][(kh, kw, c)], im2col's order
    wb.add_gemm('v.conv1', conv.permute(0, 2, 3, 1).reshape(conv.shape[0], -1))
    pos = P('visual.positional_embedding')
    wb.add('v.cls', P('visual.class_embedding') + pos[0])
    wb.add('v.pos', pos)
    wb.add_norm('v.ln_pre', P, 'visual.ln_pre')
    _add_blocks(wb, P, 'visual.transformer.resblocks', 'v.', cfg['vision_layers'])
    wb.add_norm('v.final', P, 'visual.ln_post')
    wb.add_gemm('v.proj', P('visual.proj').t().contiguous())
    wb.add('t.tok', P('token_embedding.weight'))
    wb.add('t.pos', P('positional_embedding'))
    _add_blocks(wb, P, 'transformer.resblocks', 't.', cfg['text_layers'])
    wb.add_norm('t.final', P, 'ln_final')
    wb.add_gemm('t.proj', P('text_projection').t().contiguous())
    return wb


# ---------------------------------------------------------------------------------------------------------------------------- input
def _bicubic(x):
    """Pillow's bicubic_filter (a = -0.5), in the order of its double operations."""
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def pil_bicubic_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc (libImaging/Resample.c) for the bicubic filter over the whole input:
    ([first source index], [tap count], [[22-bit fixed-point weights]]) per output index, and ksize (taps per row of the table).
    Python floats are IEEE doubles and these operations are evaluated one at a time, as the C code does."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    x0, n, kk = [], [], []
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        k = [int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS)) for w in k]
        x0.append(xmin)
        n.append(xmax)
        kk.append(k)
    return x0, n, kk, ksize


def resize_geometry(H, W, S):
    """torchvision Resize(S) of an H x W image (shorter side to S, longer side int(S * long / short)) and CenterCrop(S)'s offsets
    (int(round((size - S) / 2)), Python's round): (Rh, Rw, top, left)."""
    short, long_ = (W, H) if W <= H else (H, W)
    new_long = int(S * long_ / short)
    Rw, Rh = (S, new_long) if W <= H else (new_long, S)
    return Rh, Rw, int(round((Rh - S) / 2.0)), int(round((Rw - S) / 2.0))


def bicubic_tables(H, W, S):
    """The ds_clip_input tables of H x W inputs: int32 [y0 | ny | x0 | nx | wy [S][ky] | wx [S][kx]] indexed by crop row / column,
    and (ky, kx)."""
    Rh, Rw, top, left = resize_geometry(H, W, S)
    parts, ks = [], []
    for size, rsize, off in ((H, Rh, top), (W, Rw, left)):
        x0, n, kk, ksize = pil_bicubic_coeffs(size, rsize)
        w = torch.zeros(S, ksize, dtype=torch.int32)
        for i in range(S):
            w[i, :n[off + i]] = torch.tensor(kk[off + i], dtype=torch.int32)
        parts.append((torch.tensor(x0[off:off + S], dtype=torch.int32), torch.tensor(n[off:off + S], dtype=torch.int32), w))
        ks.append(ksize)
    (y0, ny, wy), (x0, nx, wx) = parts
    return torch.cat([y0, ny, x0, nx, wy.reshape(-1), wx.reshape(-1)]), ks[0], ks[1]


def table_taps(H, W, S):
    """(ky, kx) of bicubic_tables(H, W, S), from the sizes alone."""
    Rh, Rw, _, _ = resize_geometry(H, W, S)
    return tuple(int(math.ceil(2.0 * max(float(n) / r, 1.0))) * 2 + 1 for n, r in ((H, Rh), (W, Rw)))


# ---------------------------------------------------------------------------------------------------------------------------- plans
def compile_image_plan(cfg, wb, B, H, W, npass=3, strides=None, eps=1e-5):
    """Image embeddings of B uint8 images [B][3][H][W] (io X; element strides `strides` = (sn, sc, sy, sx), default contiguous NCHW;
    the bicubic_tables(H, W, S) in io CTX) into io D [B][E] fp32, L2-normalised."""
    sn, sc, sy, sx = strides or (3 * H * W, H * W, W, 1)
    Sz, P, Wd, I = cfg['image_size'], cfg['patch_size'], cfg['vision_width'], cfg['vision_mlp']
    nh = cfg['vision_heads']
    hd = Wd // nh
    g = Sz // P
    L = g * g + 1
    M = B * L
    K64 = -(-(P * P * 3) // 64) * 64
    keys_pitch = -(-L // 8) * 8
    ky, kx = table_taps(H, W, Sz)
    pb = PlanBuilder(wb, B, npass, tag=None)
    Wt = wb.ref
    reserve_layer_buffers(pb, M, Wd, I, keys_pitch)
    pb.need('img', B * Sz * Sz * 3 * F4)
    pb.need('cols', NPL * B * g * g * K64 * H2)

    pb.emit(lambda R: S.ClipInputDesc(src=io(S.DS_IO_X), tab=io(S.DS_IO_CTX), out=R('img'), sn=sn, sc=sc, sy=sy, sx=sx, B=B, H=H, W=W,
                                      S=Sz, ky=ky, kx=kx, mean=OPENAI_MEAN, std=OPENAI_STD))
    pb.emit(lambda R: S.Im2colDesc(src=R('img'), out=R('cols'), B=B, H=Sz, W=Sz, C=3, src_pitch=3, src_c0=0, kh=P, kw=P, sh=P, sw=P,
                                   ph=0, pw=0, K64=K64, nplanes=NPL))
    # [CLS; patches] + pos: the patch rows of sample z are rows 1 .. L-1 of its block, positional rows 1 .. L-1 the residual operand
    pb.emit(lambda R: G.rows_gemm(R('cols'), g * g, K64, B, Wt('v.conv1:w'), G.padded_rows(Wd), K64, 1, K64, num_z=B, nh=1, a_n_per_zb=1,
                                  m_valid=g * g, n_valid=Wd, npass=npass, out_f32=R('h1', 4 * Wd), o_zb=L * Wd, ldo=Wd,
                                  residual=Wt('v.pos', 4 * Wd), ldr=Wd)[0])
    pb.emit(lambda R: S.ClipHeadDesc(src=Wt('v.cls'), out=R('h1'), src_stride=0, out_stride=L * Wd, B=B, C=Wd, T=1, row=0,
                                     mode=S.DS_CLIP_GATHER))
    layernorm(pb, 'h1', 'v.ln_pre', 'h0', M, Wd, eps, fmt=2)
    for i in range(cfg['vision_layers']):
        transformer_layer(pb, f'v.l{i}', M, L, Wd, I, nh, hd, keys_pitch, eps, causal=0, act='gelu')
    pooled_head(pb, 'h0', L * Wd, Wd, 'v.final', 'v.proj', cfg['embed_dim'], eps)
    return pb.finish(B=B, H=H, W=W, npass=npass, strides=(sn, sc, sy, sx))


def compile_text_plan(cfg, wb, B, T, npass=3, eps=1e-5):
    """Text embeddings of B prompts of T open_clip token ids (io X, int32) into io D [B][E] fp32, L2-normalised."""
    return compile_clip_plan(text_config(cfg), wb, B, T, eps=eps, npass=npass, act='gelu', prefix='t.', proj_dim=cfg['embed_dim'])

"""Plan compiler for the latent-diffusion eps-net (Stable Diffusion v1.x `UNetModel`, BASELINE config 5).

Reference being lowered: models/ldm/modules/diffusionmodules/openaimodel.py:710-741 (UNetModel.forward), ResBlock :255-275,
Downsample :134-160, Upsample :91-119; models/ldm/modules/attention.py SpatialTransformer :250-261, BasicTransformerBlock :211-215,
CrossAttention :170-193, GEGLU :42-44; util.py:151-171 (timestep_embedding).  Same op set and executor as the EDM nets (plan.py):
every contraction is the wgmma GEMM kernel; LayerNorm / GEGLU / softmax / GroupNorm are the HBM-bound companions.

The unconditional LSUN-Bedroom / FFHQ LDM-VQ-f4 eps-nets (models/ldm/configs/latent-diffusion/lsun_bedrooms-ldm-vq-4.yaml) use the
same UNetModel with the legacy AttentionBlock (openaimodel.py:278-324, QKVAttentionLegacy :347-372) instead of the SpatialTransformer:
GroupNorm -> qkv 1x1 -> softmax attention over 32-wide heads -> proj_out -> residual, and have no cross-attention.  Their level widths
(224, 672) and concat widths (1568, 1120) are not multiples of 64: the GEMMs zero-fill the last 64-channel K block (gemm_desc.conv_gemm).

Layout notes specific to this net:
  * head dims 40 / 80 / 160 are zero-padded to 64 / 128 / 192 inside the packed q/k/v/out weights (K blocks are 64 wide);
  * the 77 context tokens are not padded in memory: K extents / key counts that are not multiples of 64 are zero-filled by TMA;
  * the stride-2 Downsample conv runs on a space-to-depth repack (gn_apply resample=3) with a per-tap (shift, phase) table;
  * classifier-free guidance evaluates the batch [uncond | cond] = 2B samples in one pass; eps is written NCHW.
"""
import math
import re
from collections import OrderedDict

import torch

from . import _cstructs as S
from . import gemm_desc as G
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob, io

CTX_TOKENS_PITCH = 128        # P / V^T row pitch for the 77 context tokens (multiple of 8 elements for TMA strides)


def dpad(d):
    return -(-d // 64) * 64


def ldm_structure(params, num_heads, num_head_channels=-1):
    """Block structure from UNetModel.state_dict() names/shapes:
    [(block_name, [('conv'|'res'|'attn'|'qkv_attn'|'down'|'up', module_name, ...)])] for input / middle / output blocks.
    Heads per attention layer: ch // num_head_channels when num_head_channels > 0 (openaimodel.py:540-544), else num_heads."""
    names = list(params.keys())
    mods = OrderedDict()
    for k in names:
        m = re.match(r'((?:input_blocks|output_blocks)\.\d+\.\d+|middle_block\.\d+)\.', k)
        if m:
            mods.setdefault(m.group(1), []).append(k)

    def kind_of(mod, keys):
        if any('.in_layers.' in k for k in keys):
            w = params[mod + '.in_layers.2.weight']
            return ('res', mod, w.shape[1], w.shape[0])
        if any('.transformer_blocks.' in k for k in keys):
            ch = params[mod + '.norm.weight'].shape[0]
            inner = params[mod + '.proj_in.weight'].shape[0]
            return ('attn', mod, ch, num_heads, inner // num_heads)
        if (mod + '.qkv.weight') in params:           # legacy AttentionBlock
            ch = params[mod + '.norm.weight'].shape[0]
            heads = ch // num_head_channels if num_head_channels > 0 else num_heads
            return ('qkv_attn', mod, ch, heads, ch // heads)
        if (mod + '.op.weight') in params:
            w = params[mod + '.op.weight']
            return ('down', mod, w.shape[1], w.shape[0])
        if (mod + '.conv.weight') in params:
            w = params[mod + '.conv.weight']
            return ('up', mod, w.shape[1], w.shape[0])
        w = params[mod + '.weight']
        return ('conv', mod, w.shape[1], w.shape[0])

    def block_key(mod):
        parts = mod.split('.')
        return parts[0] if parts[0] == 'middle_block' else parts[0] + '.' + parts[1]
    blocks = OrderedDict()
    for mod, keys in mods.items():
        blocks.setdefault(block_key(mod), []).append(kind_of(mod, keys))
    inp = [(b, l) for b, l in blocks.items() if b.startswith('input_blocks')]
    mid = [(b, l) for b, l in blocks.items() if b.startswith('middle_block')]
    out = [(b, l) for b, l in blocks.items() if b.startswith('output_blocks')]
    inp.sort(key=lambda t: int(t[0].split('.')[1]))
    out.sort(key=lambda t: int(t[0].split('.')[1]))
    return dict(inp=inp, mid=mid, out=out, model_channels=params['time_embed.0.weight'].shape[1], ted=params['time_embed.0.weight'].shape[0],
                in_channels=params['input_blocks.0.0.weight'].shape[1], out_channels=params['out.2.weight'].shape[0], num_heads=num_heads)


def _pad_heads_rows(w, heads, dh):
    """[heads*dh, K] -> [heads*dpad, K] with zero rows."""
    dp = dpad(dh)
    out = torch.zeros(heads * dp, w.shape[1])
    out.view(heads, dp, -1)[:, :dh] = w.reshape(heads, dh, -1)
    return out


def _pad_heads_cols(w, heads, dh):
    """[N, heads*dh] -> [N, heads*dpad] with zero columns."""
    dp = dpad(dh)
    out = torch.zeros(w.shape[0], heads * dp)
    out.view(w.shape[0], heads, dp)[:, :, :dh] = w.reshape(w.shape[0], heads, dh)
    return out


def _legacy_qkv_split(w, b, heads, pairs):
    """The legacy AttentionBlock's qkv rows, ordered [head][q|k|v][d] (QKVAttentionLegacy, openaimodel.py:361-363), as
    [q heads | k heads] rows and separate v rows, each head in a slot of 32 rows (pairs: the head count rounded up to even, the extra
    head all zeros) or of 64 rows (the zero-padded layout of the 64-wide attention kernel).  Returns (w_qk, b_qk, w_v, b_v)."""
    c3 = w.shape[0]
    d = c3 // 3 // heads
    dp = 32 if pairs else dpad(d)
    hs = heads + heads % 2 if pairs else heads
    w3 = w.reshape(heads, 3, d, -1)
    b3 = b.reshape(heads, 3, d)

    def slots(x):
        out = torch.zeros((hs, dp) + tuple(x.shape[2:]), dtype=x.dtype)
        out[:heads, :d] = x
        return out.reshape((hs * dp,) + tuple(x.shape[2:]))
    wq, wk, wv = (slots(w3[:, i]) for i in range(3))
    bq, bk, bv = (slots(b3[:, i]) for i in range(3))
    return torch.cat([wq, wk]), torch.cat([bq, bk]), wv, bv


def _legacy_proj_cols(w, heads, pairs):
    """proj_out weight [C, heads*d] -> [C, slots*dp]: zero columns for the padding rows / head of _legacy_qkv_split."""
    d = w.shape[1] // heads
    dp = 32 if pairs else dpad(d)
    hs = heads + heads % 2 if pairs else heads
    out = torch.zeros(w.shape[0], hs, dp, dtype=w.dtype)
    out[:, :heads, :d] = w.reshape(w.shape[0], heads, d)
    return out.reshape(w.shape[0], hs * dp)


def pack_ldm_weights(st, params, f8=False, f8_linear=False, head_pairs=True):
    """f8=True: the ResBlock convolutions (in_layers.2, out_layers.3 + skip_connection) are packed for the f8 GEMM mode (csrc/ops.h).
    f8_linear=True (opt-in, needs f8): also the transformer linears whose A operand has a single consumer -- proj_in, attn2.to_q, the
    GEGLU feed-forward pair and proj_out (75 % of the transformer's linear FLOPs).
    head_pairs: the legacy attention's 32-wide heads run two per CTA (attn_pair_kernel); False pads each head to 64 (attn_kernel),
    kept as a comparator.  info['f8_shift'] is the blob's own record of the f8-packed GEMMs (WeightBlob.f8_shift)."""
    assert f8 or not f8_linear
    P = lambda k: params[k].detach().float().cpu()
    wb = WeightBlob()
    info = dict(res=[], ctx_dim=None, head_pairs=bool(head_pairs), f8_shift=wb.f8_shift)
    for k in ('time_embed.0', 'time_embed.2'):
        wb.add(k + ':w', P(k + '.weight'))
        wb.add(k + ':b', P(k + '.bias'))
    aff_w, aff_b = [], []
    aff_off = 0
    for _, layers in st['inp'] + st['mid'] + st['out']:
        for L in layers:
            kind, n = L[0], L[1]
            if kind == 'conv':
                wb.add_gemm(n, P(n + '.weight'), bias=P(n + '.bias'))
            elif kind == 'res':
                skip = n + '.skip_connection' if (n + '.skip_connection.weight') in params else None
                wb.add_res_block(n, P, n + '.in_layers.0', n + '.in_layers.2', n + '.out_layers.0', n + '.out_layers.3', skip, f8=f8)
                aff_w.append(P(n + '.emb_layers.1.weight'))
                aff_b.append(P(n + '.emb_layers.1.bias'))
                info['res'].append((n, aff_off))
                aff_off += aff_w[-1].shape[0]
            elif kind == 'attn':
                _, _, ch, heads, dh = L
                t = n + '.transformer_blocks.0'
                wb.add_norm(n + '.norm', P)
                wb.add_gemm(n + '.proj_in', P(n + '.proj_in.weight').reshape(heads * dh, ch), bias=P(n + '.proj_in.bias'), f8=f8_linear)
                for k in (1, 2, 3):
                    wb.add_norm(f'{t}.norm{k}', P)
                # self-attention: [q | k] rows for one GEMM, v as the M operand of the V^T GEMM
                wq, wk, wv = (_pad_heads_rows(P(f'{t}.attn1.to_{x}.weight'), heads, dh) for x in 'qkv')
                wb.add_gemm(t + '.attn1.qk', torch.cat([wq, wk]))
                wb.add(t + '.attn1.v:w', G.split_planes(wv))
                wb.add_gemm(t + '.attn1.out', _pad_heads_cols(P(t + '.attn1.to_out.0.weight'), heads, dh), bias=P(t + '.attn1.to_out.0.bias'))
                # cross-attention
                wb.add_gemm(t + '.attn2.q', _pad_heads_rows(P(t + '.attn2.to_q.weight'), heads, dh), f8=f8_linear)
                wb.add_gemm(t + '.attn2.k', _pad_heads_rows(P(t + '.attn2.to_k.weight'), heads, dh))
                wb.add(t + '.attn2.v:w', G.split_planes(_pad_heads_rows(P(t + '.attn2.to_v.weight'), heads, dh)))
                wb.add_gemm(t + '.attn2.out', _pad_heads_cols(P(t + '.attn2.to_out.0.weight'), heads, dh), bias=P(t + '.attn2.to_out.0.bias'))
                info['ctx_dim'] = P(t + '.attn2.to_k.weight').shape[1]
                wb.add_gemm(t + '.ff1', P(t + '.ff.net.0.proj.weight'), bias=P(t + '.ff.net.0.proj.bias'), f8=f8_linear)
                wb.add_gemm(t + '.ff2', P(t + '.ff.net.2.weight'), bias=P(t + '.ff.net.2.bias'), f8=f8_linear)
                wb.add_gemm(n + '.proj_out', P(n + '.proj_out.weight').reshape(ch, heads * dh), bias=P(n + '.proj_out.bias'), f8=f8_linear)
            elif kind == 'qkv_attn':
                _, _, ch, heads, dh = L
                wqk, bqk, wv, bv = _legacy_qkv_split(P(n + '.qkv.weight').reshape(3 * ch, ch), P(n + '.qkv.bias'), heads, head_pairs)
                wproj = _legacy_proj_cols(P(n + '.proj_out.weight').reshape(ch, ch), heads, head_pairs)
                wb.add_attn_block(n, P, n + '.norm', (wqk, bqk), (wv, bv), (wproj, P(n + '.proj_out.bias')))
            elif kind == 'down':
                wb.add_gemm(n, P(n + '.op.weight'), bias=P(n + '.op.bias'))
            elif kind == 'up':
                wb.add_gemm(n, P(n + '.conv.weight'), bias=P(n + '.conv.bias'), f8=f8)
    wb.add('affine:w', torch.cat(aff_w, dim=0))
    wb.add('affine:b', torch.cat(aff_b, dim=0))
    info['aff_total'] = aff_off
    wb.add_norm('out.0', P)
    wb.add_gemm('out.2', P('out.2.weight'), bias=P('out.2.bias'))
    return wb, info


def compile_ldm_plan(st, wb, info, B, Bt, nT, R, npass=3, ctx_tokens=77, flash_attn=True, f8=False, f8_linear=False):
    """Lower the eps-net for Bt samples (Bt = B, or 2B under classifier-free guidance) at latent resolution R.
    nT in {1, Bt}: number of timestep values.  io: X = x [B,C,R,R], SIGMA = timesteps [nT], LABELS = coef [B|1][4] (c_in in slot 2),
    CTX = context [Bt, 77, ctx_dim] (nets with cross-attention only), D = eps [Bt,C,R,R] (NCHW), BOTTLENECK = channel-mean of the
    middle block [Bt, 64]."""
    assert nT in (1, Bt)
    assert not f8 or (npass == 3 and wb.f8_shift)
    assert f8 or not f8_linear
    fmt_lin = 1 if f8_linear else 0
    pb = PlanBuilder(wb, Bt, npass, f8=f8)
    emit, W = pb.emit, wb.ref
    mc, ted = st['model_channels'], st['ted']
    cd = info['ctx_dim']
    T = ctx_tokens
    TP = CTX_TOKENS_PITCH
    pb.stats()
    # ---------------- timestep embedding (util.py:151-171, openaimodel.py:723-724) + all emb_layers in one launch -------------
    pb.need('emb0', nT * mc * F4)
    pb.need('e1', nT * ted * F4)
    pb.need('e2', nT * ted * F4)
    pb.need('aff', nT * info['aff_total'] * F4)
    emit(lambda R_: S.PosembDesc(sigma=io(S.DS_IO_SIGMA), nsig=nT, num_channels=mc, endpoint=0, swap_sincos=0, sigma_data=0.5, mode=1,
                                 coef=0, emb=R_('emb0')))
    emit(lambda R_: S.LinearDesc(in_=R_('emb0'), in_stride=mc if nT > 1 else 0, W=W('time_embed.0:w'), b=W('time_embed.0:b'), out=R_('e1'),
                                 n_rows=nT, in_f=mc, out_f=ted, act=1, in_scale=1.0))
    # every consumer applies SiLU first (ResBlock.emb_layers = SiLU -> Linear, openaimodel.py:205-211): store silu(emb)
    emit(lambda R_: S.LinearDesc(in_=R_('e1'), in_stride=ted if nT > 1 else 0, W=W('time_embed.2:w'), b=W('time_embed.2:b'), out=R_('e2'),
                                 n_rows=nT, in_f=ted, out_f=ted, act=1, in_scale=1.0))
    emit(lambda R_: S.LinearDesc(in_=R_('e2'), in_stride=ted if nT > 1 else 0, W=W('affine:w'), b=W('affine:b'), out=R_('aff'), n_rows=nT,
                                 in_f=ted, out_f=info['aff_total'], act=0, in_scale=1.0))
    aff_stride = info['aff_total'] if nT > 1 else 0
    aff_off = dict(info['res'])
    # ---------------- context tokens -> fp16 planes (once per forward, shared by every cross-attention) ------------------------
    if cd is not None:
        pb.need('ctx', NPL * Bt * T * cd * H2)
        pb.to_planes(io(S.DS_IO_CTX), cd, T, 1, Bt, 'ctx')

    def lower_transformer(L, src, H):
        """SpatialTransformer with one BasicTransformerBlock (attention.py:250-261, :211-215)."""
        _, n, ch, heads, dh = L
        t = n + '.transformer_blocks.0'
        inner, dp = heads * dh, dpad(dh)
        hp = heads * dp
        Lq = H * H
        M = Bt * Lq
        pb.need('act', NPL * M * max(ch, inner) * H2)
        pb.group_norm([(src, ch)], H, n + '.norm', 1e-6, 'act', silu=0, fmt=fmt_lin)
        for nm in ('t0', 't1', 't2', 't3'):
            pb.need(nm, M * inner * F4)
        emit(lambda R_: G.conv_gemm(R_('act'), Bt, H, H, ch, W(n + '.proj_in:w'), inner, taps=1, npass=npass, out_f32=R_('t0'),
                                    bias=W(n + '.proj_in:b'), **pb.f8_args(n + '.proj_in'))[0])
        pb.need('ln', NPL * M * inner * H2)
        pb.need('qk', NPL * M * 2 * hp * H2)
        pb.need('vt', NPL * Bt * hp * max(Lq, TP) * H2)
        # fused QK^T -> softmax -> PV (attention.cu): at 64x64 latents the 4096 x 4096 score matrix per head never reaches HBM
        fused = flash_attn and dp == 64

        def ln(k, srcbuf, fmt=0):
            emit(lambda R_: S.LayernormDesc(src=R_(srcbuf), gamma=W(f'{t}.norm{k}:g'), beta=W(f'{t}.norm{k}:b'), out=R_('ln'), rows=M, C=inner,
                                            nplanes=NPL, eps=1e-5, fmt=fmt))
        # ---- self-attention (attn1): x = attn1(norm1(x)) + x
        ln(1, 't0')
        emit(lambda R_: G.conv_gemm(R_('ln'), Bt, H, H, inner, W(t + '.attn1.qk:w'), 2 * hp, taps=1, npass=npass, out_h16=R_('qk'))[0])
        pb.vt_gemm(t + '.attn1.v:w', 'ln', inner, hp, Lq, Lq)
        pb.attention(fused, 'qk', 'qk', 'o', heads, Lq, Lq, dp, dh ** -0.5, Lq)
        pb.need('o', NPL * M * hp * H2)
        emit(lambda R_: G.conv_gemm(R_('o'), Bt, H, H, hp, W(t + '.attn1.out:w'), inner, taps=1, npass=npass, out_f32=R_('t1'),
                                    bias=W(t + '.attn1.out:b'), residual=R_('t0'), ldr=inner)[0])
        # ---- cross-attention (attn2): x = attn2(norm2(x), context) + x
        ln(2, 't1', fmt=fmt_lin)           # single consumer: the to_q GEMM below
        pb.need('q2', NPL * M * hp * H2)
        pb.need('k2', NPL * Bt * T * hp * H2)
        emit(lambda R_: G.conv_gemm(R_('ln'), Bt, H, H, inner, W(t + '.attn2.q:w'), hp, taps=1, npass=npass, out_h16=R_('q2'),
                                    **pb.f8_args(t + '.attn2.q'))[0])
        emit(lambda R_: G.rows_gemm(R_('ctx'), Bt * T, cd, 1, W(t + '.attn2.k:w'), G.padded_rows(hp), cd, 1, cd, num_z=1, nh=1, m_valid=Bt * T,
                                    n_valid=hp, npass=npass, out_h16=R_('k2'), ldo=hp, o_plane=Bt * T * hp)[0])
        pb.vt_gemm(t + '.attn2.v:w', 'ctx', cd, hp, T, TP)
        pb.attention(fused, 'q2', 'k2', 'o', heads, Lq, T, dp, dh ** -0.5, TP, s_pitch=80)
        emit(lambda R_: G.conv_gemm(R_('o'), Bt, H, H, hp, W(t + '.attn2.out:w'), inner, taps=1, npass=npass, out_f32=R_('t2'),
                                    bias=W(t + '.attn2.out:b'), residual=R_('t1'), ldr=inner)[0])
        # ---- GEGLU feed-forward: x = ff(norm3(x)) + x
        ln(3, 't2', fmt=fmt_lin)
        pb.need('ff', M * 8 * inner * F4)
        pb.need('gg', NPL * M * 4 * inner * H2)
        emit(lambda R_: G.conv_gemm(R_('ln'), Bt, H, H, inner, W(t + '.ff1:w'), 8 * inner, taps=1, npass=npass, out_f32=R_('ff'),
                                    bias=W(t + '.ff1:b'), **pb.f8_args(t + '.ff1'))[0])
        emit(lambda R_: S.GegluDesc(src=R_('ff'), out=R_('gg'), rows=M, I=4 * inner, nplanes=NPL, fmt=fmt_lin))
        emit(lambda R_: G.conv_gemm(R_('gg'), Bt, H, H, 4 * inner, W(t + '.ff2:w'), inner, taps=1, npass=npass, out_f32=R_('t3'),
                                    bias=W(t + '.ff2:b'), residual=R_('t2'), ldr=inner, **pb.f8_args(t + '.ff2'))[0])
        # ---- proj_out + outer residual
        pb.to_planes('t3', inner, H, H, Bt, 'ln', fmt=fmt_lin)
        out = pb.need('h:' + n, M * ch * F4)
        emit(lambda R_: G.conv_gemm(R_('ln'), Bt, H, H, inner, W(n + '.proj_out:w'), ch, taps=1, npass=npass, out_f32=R_(out),
                                    bias=W(n + '.proj_out:b'), residual=R_(src), ldr=ch, **pb.f8_args(n + '.proj_out'))[0])
        return out, ch

    def lower_down(L, src, H):
        _, n, cin, cout = L
        Ho = H // 2
        cpad = dpad(cin)            # each space-to-depth phase starts on a 64-channel K block of the GEMM
        pb.need('s2d', NPL * Bt * H * H * cpad * H2)
        pb.to_planes(src, cin, H, H, Bt, 's2d', resample=3, phase_pitch=cpad if cpad != cin else 0)
        out = pb.need('h:' + n, Bt * Ho * Ho * cout * F4)
        emit(lambda R_: G.conv_gemm(R_('s2d'), Bt, Ho, Ho, cin, W(n + ':w'), cout, taps=9, npass=npass, out_f32=R_(out), bias=W(n + ':b'),
                                    s2d=True)[0])
        return out, cout, Ho

    def lower(L, parts, H):
        """One module of a block over `parts` (the input, and for the first ResBlock of an output block the skip) at H x H:
        (output buffer, channels, output resolution)."""
        pb.tag += 1
        kind, n = L[0], L[1]
        out = 'h:' + n
        src = parts[0][0]
        if kind == 'res':
            _, _, cin, cout = L
            pb.res_block(n, parts, H, cout, out, eps=1e-5, skip='conv' if cin != cout else 'identity',
                         emb=('aff', aff_off[n] * F4), emb_stride=aff_stride)
            pb.need(out, Bt * H * H * cout * F4)
            return out, cout, H
        if kind == 'qkv_attn':
            _, _, ch, heads, dh = L
            pairs = info['head_pairs']
            nh, dp = (heads + heads % 2, 32) if pairs else (heads, dpad(dh))
            pb.attn_block(n, src, ch, H, out, eps=1e-5, heads=nh, d=dp, scale=dh ** -0.5, fused=flash_attn or pairs, pairs=pairs)
            return out, ch, H
        if kind == 'down':
            return lower_down(L, src, H)
        if kind == 'up':
            pb.upsample_conv(n, src, L[2], H, L[3], out)
            return out, L[3], 2 * H
        return lower_transformer(L, src, H) + (H,)

    # ---------------- input conv --------------------------------------------------------------------------------------------
    cimg = st['in_channels']
    pb.need('in_planes', NPL * Bt * R * R * 64 * H2)
    emit(lambda R_: S.PrepInputDesc(x=io(S.DS_IO_X), coef=io(S.DS_IO_LABELS), coef_stride=4 if B > 1 and nT > 1 else 0, B=Bt, C=cimg,
                                    HW=R * R, nplanes=NPL, x_batch=B, out=R_('in_planes')))
    first = st['inp'][0][1][0]
    h = pb.need('h:' + first[1], Bt * R * R * first[3] * F4)
    emit(lambda R_: G.conv_gemm(R_('in_planes'), Bt, R, R, 64, W(first[1] + ':w'), first[3], taps=9, npass=npass, out_f32=R_(h),
                                bias=W(first[1] + ':b'))[0])
    cur, cur_c, H = h, first[3], R
    hs = [(cur, cur_c)]
    for _, layers in st['inp'][1:]:
        for L in layers:
            cur, cur_c, H = lower(L, [(cur, cur_c)], H)
        hs.append((cur, cur_c))
    for L in st['mid'][0][1]:
        cur, cur_c, H = lower(L, [(cur, cur_c)], H)
    mid_out, mid_c, mid_H = cur, cur_c, H
    emit(lambda R_: S.ChanmeanDesc(src=R_(mid_out), out=io(S.DS_IO_BOTTLENECK), rows=Bt * mid_H * mid_H, C=mid_c))
    for _, layers in st['out']:
        sk = hs.pop()
        for i, L in enumerate(layers):
            cur, cur_c, H = lower(L, [(cur, cur_c)] + ([sk] if i == 0 else []), H)
    # ---------------- out: GN + SiLU + conv3x3 -> eps (NCHW) -----------------------------------------------------------------
    assert H == R
    pb.tag += 1
    pb.head_conv(cur, cur_c, H, 'out.0', 1e-5, 'out.2', st['out_channels'], nchw_out=(st['out_channels'], io(S.DS_IO_D)))
    return pb.finish(B=B, Bt=Bt, nT=nT, npass=npass, ctx_tokens=ctx_tokens)

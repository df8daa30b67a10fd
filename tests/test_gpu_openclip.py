"""CLIP score on the H100: the wide-head attention kernel, the image input kernel (bit for bit), exact GELU and the pooled heads against
float64 / the CPU restatement; both towers against the float64 oracle at a small config and at ViT-g-14 dimensions; chunking, CUDA-graph
replay and the end-to-end score."""
import functools

import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import _lib
from diff_sampler_b200 import openclip_plan as OP
from diff_sampler_b200.fid_stats import ScoreStats
from diff_sampler_b200.openclip_net import B200OpenCLIP, score_embeddings
from oracle import openclip_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _split(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def _planes(x):
    """fp32 [..] -> fp16 planes [2][..] on the device, and the float64 value they hold."""
    hi, lo = _split(x)
    return torch.stack([hi, lo]).to(DEV), hi.double() + lo.double()


@pytest.mark.parametrize('nh,hd,L,Lk', [(16, 88, 257, 257), (4, 72, 257, 257), (4, 80, 257, 257), (4, 128, 257, 257),
                                        (16, 88, 100, 190), (3, 96, 300, 77)])
def test_wide_attention_against_float64(nh, hd, L, Lk):
    B, C = 2, nh * hd
    g = torch.Generator().manual_seed(hd + L)
    qk_pitch = 2 * C
    q = torch.randn(B, L, qk_pitch, generator=g)
    k = torch.randn(B, Lk, qk_pitch, generator=g)
    vp = -(-Lk // 8) * 8
    vt = torch.randn(B, C, vp, generator=g)
    qd, q64 = _planes(q)
    kd, k64 = _planes(k)
    vd, v64 = _planes(vt)
    out = torch.zeros(2, B, L, C, dtype=torch.float16, device=DEV)
    scale = hd ** -0.5
    d = S.AttnDesc(q=qd.data_ptr(), k=kd.data_ptr(), vt=vd.data_ptr(), out=out.data_ptr(), B=B, nh=nh, L=L, Lk=Lk, q_pitch=qk_pitch,
                   q_c0=0, k_pitch=qk_pitch, k_c0=C, vt_pitch=vp, o_pitch=C, nplanes=2, scale=scale, causal=0, pad0=hd)
    _lib.op_launch(d)
    torch.cuda.synchronize()
    got = out[0].double().cpu() + out[1].double().cpu()
    want = torch.zeros(B, L, C, dtype=torch.float64)
    for h in range(nh):
        qs, ks = q64[:, :, h * hd:(h + 1) * hd], k64[:, :, C + h * hd:C + (h + 1) * hd]
        p = torch.softmax(scale * qs @ ks.transpose(1, 2), dim=2)
        want[:, :, h * hd:(h + 1) * hd] = p @ v64[:, h * hd:(h + 1) * hd, :Lk].transpose(1, 2)
    err = ((got - want).abs().max() / want.abs().max()).item()
    print(f'wide attention nh {nh} hd {hd} L {L} Lk {Lk}: {err:.2e} of max |O|')
    assert err < 2e-5


# ------------------------------------------------------------------------------------------ the wide kernel at its edges
WIDE_HDS = list(range(72, 129, 8))            # every width attn_check accepts: the second 64-channel box holds 8 .. 64 channels
WIDE_LKS = [1, 63, 64, 65, 128, 129, 257, 730, 1025]
WIDE_LS = [1, 127, 128, 129, 257]
GUARD = 4096                                  # fp16 elements of NaN before and after every buffer


def _guarded(n):
    """A NaN-filled fp16 buffer with GUARD elements on both sides, and its inner n elements."""
    buf = torch.full((2 * GUARD + n,), float('nan'), dtype=torch.float16, device=DEV)
    return buf, buf[GUARD:GUARD + n]


def _wide_case(nh, hd, L, Lk, B=2, layout='qk', v_mean=0.0, late=False, seed=0):
    """attn_wide_kernel against float64 softmax attention on the same fp16 hi + lo operands.  Every byte the kernel must not read or
    write is NaN: the Q / K channels outside the heads' window of each row, the V^T columns Lk .. vt_pitch, the output channels
    nh hd .. o_pitch, and a guard before and after each buffer.  A read of any of them would make an output NaN; the output
    sentinels must still be NaN afterwards, the inputs bit for bit unchanged.  Returns the error / max |O|.

    layout 'qk': the plan's [q | k] rows (L == Lk, q_pitch = k_pitch = 2 C, k_c0 = C, vt_pitch = Lk rounded up to 8, o_pitch = C);
    'sep': Q and K in buffers of their own with q_c0 = 16, k_c0 = 40, pitches C + 40 and C + 48, 8 spare V^T columns, o_pitch C + 16.
    late: every third query row gets its maximum logit, about 30 above the rest, from the last key alone, so the last key block
    rescales O (alpha ~ e^-30) after all the others have been accumulated."""
    C, scale = nh * hd, hd ** -0.5
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, L, nh, hd, generator=g, device=DEV)
    k = torch.randn(B, Lk, nh, hd, generator=g, device=DEV)
    v = torch.randn(B, Lk, nh, hd, generator=g, device=DEV) + v_mean
    if late:
        u = torch.randn(nh, hd, generator=g, device=DEV)
        u /= u.norm(dim=1, keepdim=True)
        q[:, ::3] = 3 * u
        k[:, Lk - 1] = 10 / scale * u                                    # logit scale * 3 * 10 / scale = 30
    if layout == 'qk':
        assert L == Lk
        q_c0, k_c0, qp, kp, vp, op = 0, C, 2 * C, 2 * C, -(-Lk // 8) * 8, C
    else:
        q_c0, k_c0, qp, kp, vp, op = 16, 40, C + 40, C + 48, -(-Lk // 8) * 8 + 8, C + 16

    def operand(rows, pitch, c0, x):                                      # fp32 [B][rows][pitch], NaN outside the heads
        t = torch.full((B, rows, pitch), float('nan'), device=DEV)
        t[:, :, c0:c0 + C] = x.reshape(B, rows, C)
        return t
    qf = operand(L, qp, q_c0, q)
    kf = operand(Lk, kp, k_c0, k)
    if layout == 'qk':
        qf[:, :, k_c0:k_c0 + C] = kf[:, :, k_c0:k_c0 + C]
        kf = None
    vf = torch.full((B, C, vp), float('nan'), device=DEV)
    vf[:, :, :Lk] = v.permute(0, 2, 3, 1).reshape(B, C, Lk)
    bufs = []

    def place(x):                                                         # fp16 planes [2][..] inside a guarded buffer
        hi, lo = _split(x)
        buf, inner = _guarded(2 * x.numel())
        inner.view(2, -1).copy_(torch.stack([hi, lo]).reshape(2, -1))
        bufs.append((buf, buf.clone()))
        return inner, hi.double() + lo.double()
    qd, q64 = place(qf)
    kd, k64 = place(kf) if kf is not None else (qd, q64)
    vd, v64 = place(vf)
    obuf, od = _guarded(2 * B * L * op)
    _lib.op_launch(S.AttnDesc(q=qd.data_ptr(), k=kd.data_ptr(), vt=vd.data_ptr(), out=od.data_ptr(), B=B, nh=nh, L=L, Lk=Lk, q_pitch=qp,
                              q_c0=q_c0, k_pitch=kp, k_c0=k_c0, vt_pitch=vp, o_pitch=op, nplanes=2, scale=scale, causal=0, pad0=hd))
    torch.cuda.synchronize()
    for buf, before in bufs:
        assert torch.equal(buf.view(torch.int16), before.view(torch.int16)), 'an input buffer changed'
    out = od.view(2, B, L, op)
    assert torch.isfinite(out[..., :C]).all(), 'non-finite output: a NaN sentinel was read, or a row was left unwritten'
    assert torch.isnan(out[..., C:]).all() and torch.isnan(obuf[:GUARD]).all() and torch.isnan(obuf[GUARD + od.numel():]).all(), \
        'a store outside the output rows'
    got = (out[0].double() + out[1].double())[..., :C].reshape(B, L, nh, hd).transpose(1, 2)
    qs = q64[:, :, q_c0:q_c0 + C].reshape(B, L, nh, hd).transpose(1, 2)
    ks = k64[:, :, k_c0:k_c0 + C].reshape(B, Lk, nh, hd).transpose(1, 2)
    vs = v64[:, :, :Lk].reshape(B, nh, hd, Lk).transpose(2, 3)
    s = scale * qs @ ks.transpose(2, 3)
    want = torch.softmax(s, dim=3) @ vs
    if late:                                                              # the construction did what it claims
        top = s[:, :, ::3].topk(2, dim=3)
        assert (top.indices[..., 0] == Lk - 1).all() and (top.values[..., 0] - top.values[..., 1]).min() > 25
    err = ((got - want).abs().max() / want.abs().max()).item()
    print(f'wide attention hd {hd:3d} L {L:4d} Lk {Lk:4d} nh {nh} B {B} {layout}{f" v_mean {v_mean}" if v_mean else ""}'
          f'{" late max" if late else ""}: {err:.2e} of max |O|')
    return err


# Error / max |O| measured on an H100 80GB HBM3 (700 W power limit), worst over the head widths: 3.6e-6 up to 257 keys, 7.0e-6 at 730
# and 8.9e-6 at 1025 keys with values of mean 1; 3.0e-6 with the late maximum, 3.0e-6 over 3072 CTAs.  O accumulates inside the wgmma
# across all key blocks, so the error grows about linearly with the key count; at that rate it would reach this bound near 2300 keys.
WIDE_TOL = 2e-5


@pytest.mark.parametrize('Lk', WIDE_LKS)
@pytest.mark.parametrize('hd', WIDE_HDS)
def test_wide_attention_widths_and_key_counts(hd, Lk):
    """Self-attention in the plan's layout at every accepted head width and at key counts of one key, a partial block, an exact
    block, one key into the next block, and the two plan sizes (257, 730 tokens) and one past them; values of mean 1 at 730 and
    1025 keys, where O's error grows with the key count."""
    assert _wide_case(4, hd, Lk, Lk, v_mean=1.0 if Lk >= 730 else 0.0, seed=hd + Lk) < WIDE_TOL


@pytest.mark.parametrize('Lk', [1, 65, 730])
@pytest.mark.parametrize('L', WIDE_LS)
def test_wide_attention_cross_shapes_and_pitches(L, Lk):
    """Cross-attention (L != Lk apart from 1 x 1) over separate Q and K buffers with channel offsets, unequal pitches, spare V^T
    columns and an output pitch wider than the heads; the head width cycles through the accepted widths."""
    hd = WIDE_HDS[(WIDE_LS.index(L) * 3 + [1, 65, 730].index(Lk)) % len(WIDE_HDS)]
    assert _wide_case(3, hd, L, Lk, B=3, layout='sep', v_mean=0.5, seed=L + Lk) < WIDE_TOL


@pytest.mark.parametrize('hd,L,Lk,layout', [(72, 129, 129, 'qk'), (88, 257, 257, 'qk'), (80, 730, 730, 'qk'), (128, 1025, 1025, 'qk'),
                                             (104, 300, 1025, 'sep'), (120, 129, 730, 'sep')])
def test_wide_attention_late_maximum(hd, L, Lk, layout):
    """Rows whose maximum logit first appears in the last, partial key block, about 30 above all the others."""
    assert _wide_case(4, hd, L, Lk, layout=layout, v_mean=1.0, late=True, seed=hd) < WIDE_TOL


def test_wide_attention_many_waves():
    """Batch 64 x 16 heads of 88 x 3 query tiles: 3072 CTAs (the max_batch chunk of ViT-g-14), many waves over the SMs."""
    assert _wide_case(16, 88, 257, 257, B=64, seed=1) < WIDE_TOL


@pytest.mark.parametrize('H,W', [(512, 512), (256, 256), (64, 64), (512, 768), (768, 512), (224, 300)])
@pytest.mark.parametrize('nhwc', [False, True])
def test_image_input_is_bit_identical_to_the_restatement(H, W, nhwc):
    B, Sz = 3, 224
    u8 = torch.randint(0, 256, (B, 3, H, W), generator=torch.Generator().manual_seed(H + W), dtype=torch.uint8)
    x = (u8.permute(0, 2, 3, 1).contiguous().to(DEV).permute(0, 3, 1, 2)) if nhwc else u8.to(DEV)
    tab, ky, kx = OP.bicubic_tables(H, W, Sz)
    tab = tab.to(DEV)
    out = torch.empty(B, Sz, Sz, 3, device=DEV)
    sn, sc, sy, sx = x.stride()
    _lib.op_launch(S.ClipInputDesc(src=x.data_ptr(), tab=tab.data_ptr(), out=out.data_ptr(), sn=sn, sc=sc, sy=sy, sx=sx, B=B, H=H, W=W, S=Sz,
                                   ky=ky, kx=kx, mean=OP.OPENAI_MEAN, std=OP.OPENAI_STD))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu().permute(0, 3, 1, 2), O.preprocess(u8, Sz))


def test_gelu_and_pooled_heads_against_float64():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 256, generator=g) * 3
    xd = x.to(DEV)
    out = torch.zeros(2, 300, 256, dtype=torch.float16, device=DEV)
    _lib.op_launch(S.GegluDesc(src=xd.data_ptr(), out=out.data_ptr(), rows=300, I=256, nplanes=2, fmt=0, mode=2))
    want = torch.nn.functional.gelu(x.double())
    got = out[0].double().cpu() + out[1].double().cpu()
    assert (got - want).abs().max() < 1e-6 * want.abs().max()

    B, T, C = 5, 77, 96
    src = torch.randn(B, T, C, generator=g).to(DEV)
    ids = O.make_ids(B, T, 1000, seed=1).to(DEV)
    pooled = torch.zeros(B, C, device=DEV)
    _lib.op_launch(S.ClipHeadDesc(src=src.data_ptr(), ids=ids.data_ptr(), out=pooled.data_ptr(), src_stride=T * C, out_stride=C, B=B, C=C,
                                  T=T, mode=S.DS_CLIP_GATHER))
    assert torch.equal(pooled, src[torch.arange(B, device=DEV), ids.long().argmax(-1)])
    _lib.op_launch(S.ClipHeadDesc(src=src.data_ptr(), out=pooled.data_ptr(), src_stride=T * C, out_stride=C, B=B, C=C, T=T, row=0,
                                  mode=S.DS_CLIP_GATHER))
    assert torch.equal(pooled, src[:, 0])
    nrm = torch.zeros(B, C, device=DEV)
    _lib.op_launch(S.ClipHeadDesc(src=pooled.data_ptr(), out=nrm.data_ptr(), B=B, C=C, mode=S.DS_CLIP_L2NORM))
    p64 = pooled.double().cpu()
    assert (nrm.double().cpu() - p64 / p64.norm(dim=1, keepdim=True)).abs().max() < 1e-7
    other = torch.randn(B, C, generator=g).to(DEV)
    s = score_embeddings(pooled, other)
    assert (s.double().cpu() - 100 * (p64 * other.double().cpu()).sum(1)).abs().max() < 1e-4


def _check(clip, sd, cfg, u8, ids, tol_e, tol_s, label):
    ei, et = clip.encode_image(u8.to(DEV)), clip.encode_text(ids.to(DEV))
    dev_sd = {k: v.to(DEV, torch.float64) for k, v in sd.items()}
    wi = O.normalize(O.image_features(dev_sd, O.preprocess(u8, cfg['image_size']), cfg['vision_heads'])).cpu()
    wt = O.normalize(O.text_features(dev_sd, ids, cfg['text_heads'])).cpu()
    err_i = ((ei.double().cpu() - wi).abs().max() / wi.abs().max()).item()
    err_t = ((et.double().cpu() - wt).abs().max() / wt.abs().max()).item()
    s = score_embeddings(ei, et).double().cpu()
    err_s = (s - 100 * (wi * wt).sum(1)).abs().max().item()
    print(f'{label}: image {err_i:.2e}, text {err_t:.2e} of max |e|; score {err_s:.2e}')
    assert err_i < tol_e and err_t < tol_e and err_s < tol_s
    return ei, et


# (embedding error / max |e|, score error).  Measured on an H100 80GB HBM3: fp16x3 at most 8.3e-6 and 2.0e-5, fp16 at most 8.6e-4 and
# 8.3e-3 (ViT-g-14 dimensions and the small config); the fp16 bounds keep about 6x of that.
SMALL_TOL = {'fp16x3': (2e-4, 1e-2), 'fp16': (5e-3, 5e-2)}


@pytest.mark.parametrize('precision', ['fp16x3', 'fp16'])
def test_small_towers_against_the_oracle(precision):
    cfg = dict(O.SMALL)
    sd = O.make_weights(cfg, seed=3)
    clip = B200OpenCLIP(sd, precision=precision, vision_head_width=88, text_head_width=64, cuda_graph=False)
    u8 = torch.randint(0, 256, (4, 3, 96, 120), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    _check(clip, sd, cfg, u8, O.make_ids(4, 77, cfg['vocab_size'], seed=4), *SMALL_TOL[precision], f'small {precision}')


@functools.lru_cache(maxsize=1)
def _vit_g_14_weights():
    return O.make_weights(O.VIT_G_14, seed=7)


@pytest.mark.parametrize('precision', ['fp16x3', 'fp16'])
def test_vit_g_14_towers_against_the_oracle(precision):
    """ViT-g-14 dimensions (40 + 24 layers, 16 heads of 88 / 64), random weights, B = 2."""
    cfg = dict(O.VIT_G_14)
    sd = _vit_g_14_weights()
    clip = B200OpenCLIP(sd, precision=precision)
    u8 = torch.randint(0, 256, (2, 3, 512, 512), generator=torch.Generator().manual_seed(8), dtype=torch.uint8)
    _check(clip, sd, cfg, u8, O.make_ids(2, 77, cfg['vocab_size'], seed=8), *SMALL_TOL[precision], f'ViT-g-14 {precision}')


def test_chunks_and_graph_replay_are_bitwise_equal_to_one_eager_batch():
    cfg = dict(O.SMALL)
    sd = O.make_weights(cfg, seed=3)
    u8 = torch.randint(0, 256, (7, 64, 80, 3), generator=torch.Generator().manual_seed(9), dtype=torch.uint8).to(DEV)
    x = u8.permute(0, 3, 1, 2)                                            # the samplers' NHWC output, no copy
    ids = O.make_ids(7, 77, cfg['vocab_size'], seed=9).to(DEV)
    eager = B200OpenCLIP(sd, max_batch=64, cuda_graph=False)
    chunked = B200OpenCLIP(sd, max_batch=3, cuda_graph=True)
    ei, et = eager.encode_image(x), eager.encode_text(ids)
    for _ in range(2):                                                    # capture, then replay
        assert torch.equal(chunked.encode_image(x), ei)
        assert torch.equal(chunked.encode_text(ids), et)
    assert torch.equal(eager.score(x, ids), score_embeddings(ei, et))


def test_end_to_end_mean_score_against_the_oracle():
    cfg = dict(O.SMALL)
    sd = O.make_weights(cfg, seed=11)
    clip = B200OpenCLIP(sd)
    stats = ScoreStats()
    want = []
    for b in range(3):
        u8 = torch.randint(0, 256, (5, 3, 128, 96), generator=torch.Generator().manual_seed(20 + b), dtype=torch.uint8)
        ids = O.make_ids(5, 77, cfg['vocab_size'], seed=20 + b)
        stats.append(clip.score(u8.to(DEV), ids.to(DEV)))
        want.append(O.scores(sd, u8, ids, cfg['vision_heads'], cfg['text_heads'], cfg['image_size']))
    want = torch.cat(want).mean().item()
    got = stats.reduce().mean()
    print(f'mean score {got:.6f} vs oracle {want:.6f}')
    assert abs(got - want) < 1e-3

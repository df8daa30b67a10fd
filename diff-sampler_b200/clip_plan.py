"""Plan compiler for the CLIP text encoder behind `get_learned_conditioning` (SURVEY section 8(f)3).

Reference being lowered: diff-solvers-main/sample.py:286-289 -> models/ldm/models/diffusion/ddpm.py get_learned_conditioning ->
models/ldm/modules/encoders/modules.py:137-159 (`FrozenCLIPEmbedder.forward`: tokenizer -> `CLIPTextModel(input_ids).last_hidden_state`).
The arithmetic is Hugging Face transformers' CLIP text tower (modeling_clip.py: CLIPTextEmbeddings, CLIPEncoderLayer, CLIPAttention with
a causal mask, CLIPMLP with quick_gelu, final_layer_norm); oracle/clip_oracle.py restates it and is pinned to transformers' own module.

Same executor and op set as the denoisers: every linear is the wgmma GEMM kernel (fp16x3 split operands, fp32 accumulation), the
12-head causal attention is the fused attention kernel (csrc/attention.cu, causal=1), LayerNorm / quick-GELU / the embedding gather are
the HBM-bound companions.  Rows are the B x 77 tokens (77 is not a multiple of the 128-row tile: TMA zero-fills the ragged tiles and
the epilogue masks them).  The tokenizer is caller-side (vocabulary files): the plan starts at int32 token ids.

io: X = token ids int32 [B, T]; D = last_hidden_state fp32 [B, T, H].
"""
import torch

from . import _cstructs as S
from . import gemm_desc as G
from .plan import F4, H2, NPL, PlanBuilder, WeightBlob, io

KEYS_PITCH = 128              # V^T row pitch (keys per row; a multiple of 8 elements for the TMA strides)


def clip_config(params):
    """Dimensions from CLIPTextModel.state_dict() shapes (the head count is not in the state_dict: 64-wide heads as in every CLIP text
    tower the reference loads; callers with another head width pass num_heads)."""
    tok = params['text_model.embeddings.token_embedding.weight']
    pos = params['text_model.embeddings.position_embedding.weight']
    n_layers = 1 + max(int(k.split('.')[3]) for k in params if k.startswith('text_model.encoder.layers.'))
    return dict(vocab_size=tok.shape[0], hidden_size=tok.shape[1], max_position_embeddings=pos.shape[0], num_hidden_layers=n_layers,
                intermediate_size=params['text_model.encoder.layers.0.mlp.fc1.weight'].shape[0])


def pack_clip_weights(params, cfg):
    P = lambda k: params[k].detach().float().cpu()
    wb = WeightBlob()
    H = cfg['hidden_size']
    assert H % 64 == 0 and cfg['intermediate_size'] % 64 == 0

    wb.add('tok', P('text_model.embeddings.token_embedding.weight'))
    wb.add('pos', P('text_model.embeddings.position_embedding.weight'))
    for i in range(cfg['num_hidden_layers']):
        p = f'text_model.encoder.layers.{i}.'
        a = p + 'self_attn.'
        wb.add_gemm(f'l{i}.qk', torch.cat([P(a + 'q_proj.weight'), P(a + 'k_proj.weight')]),
                    bias=torch.cat([P(a + 'q_proj.bias'), P(a + 'k_proj.bias')]))
        wb.add(f'l{i}.v:w', G.split_planes(P(a + 'v_proj.weight')))          # A operand of the V^T product: rows unpadded
        wb.add(f'l{i}.v:b', P(a + 'v_proj.bias'))
        wb.add_gemm(f'l{i}.out', P(a + 'out_proj.weight'), bias=P(a + 'out_proj.bias'))
        wb.add_gemm(f'l{i}.fc1', P(p + 'mlp.fc1.weight'), bias=P(p + 'mlp.fc1.bias'))
        wb.add_gemm(f'l{i}.fc2', P(p + 'mlp.fc2.weight'), bias=P(p + 'mlp.fc2.bias'))
        for k in ('layer_norm1', 'layer_norm2'):
            wb.add_norm(f'l{i}.{k}', P, p + k)
    wb.add_norm('final', P, 'text_model.final_layer_norm')
    return wb


ACTS = {'quick_gelu': 1, 'gelu': 2}      # ds_geglu_desc.mode of the MLP activation: CLIPTextModel's quick-GELU, open_clip's exact GELU


def reserve_layer_buffers(pb, M, H, I, keys_pitch):
    """The arena scratch of transformer_layer for M = B x T token rows of width H and MLP width I (call before the first layer; the
    text plan's arena order is h0, h1, ln, qk, vt, o, ff, gg)."""
    B = pb.B
    pb.need('h0', M * H * F4)
    pb.need('h1', M * H * F4)
    pb.need('ln', NPL * M * H * H2)
    pb.need('qk', NPL * M * 2 * H * H2)
    pb.need('vt', NPL * B * H * keys_pitch * H2)
    pb.need('o', NPL * M * H * H2)
    pb.need('ff', M * I * F4)
    pb.need('gg', NPL * M * I * H2)


def layernorm(pb, src, key, out, rows, C, eps, fmt=0):
    """LayerNorm of the fp32 rows `src` with the gain / bias `key`:g / `key`:b into `out` (an arena name or a reference): fp16 planes, or
    fp32 with fmt=2."""
    W = pb.wb.ref
    pb.emit(lambda R: S.LayernormDesc(src=R(src), gamma=W(key + ':g'), beta=W(key + ':b'), out=R(out) if isinstance(out, str) else out,
                                      rows=rows, C=C, nplanes=NPL, eps=eps, fmt=fmt))


def linear(pb, a, M, K, key, N, bias=True, **kw):
    """[M][K] activation planes `a` x packed weight `key`:w [N][K] (+ bias `key`:b) through the batched-rows GEMM form; keyword values
    that are callables are resolved against the arena."""
    W = pb.wb.ref
    pb.emit(lambda R: G.rows_gemm(R(a), M, K, 1, W(key + ':w'), G.padded_rows(N), K, 1, K, num_z=1, nh=1, m_valid=M, n_valid=N,
                                  npass=pb.npass, bias_n=W(key + ':b') if bias else 0, ldo=N,
                                  **{k: (v(R) if callable(v) else v) for k, v in kw.items()})[0])


def transformer_layer(pb, key, M, T, H, I, nh, hd, keys_pitch, eps, causal, act):
    """One pre-LN residual attention block over the stream 'h0' [M = B x T][H] fp32 (CLIPEncoderLayer; open_clip
    ResidualAttentionBlock), back into 'h0':
        h1 = h0 + out(attention(LN1(h0)))        [q | k] one GEMM, V^T one GEMM, fused attention with nh heads of width hd
        h0 = h1 + fc2(act(fc1(LN2(h1))))         act: 'quick_gelu' or 'gelu' (exact erf)
    Weights under `key`: .qk (q rows then k rows), .v:w / .v:b, .out, .fc1, .fc2, .layer_norm1, .layer_norm2."""
    layernorm(pb, 'h0', key + '.layer_norm1', 'ln', M, H, eps)
    linear(pb, 'ln', M, H, key + '.qk', 2 * H, out_h16=lambda R: R('qk'), o_plane=M * 2 * H)
    pb.vt_gemm(key + '.v:w', 'ln', H, H, T, keys_pitch, bias=key + '.v:b')
    pb.attention(True, 'qk', 'qk', 'o', nh, T, T, hd, hd ** -0.5, keys_pitch, causal=causal)
    linear(pb, 'o', M, H, key + '.out', H, out_f32=lambda R: R('h1'), residual=lambda R: R('h0'), ldr=H)
    layernorm(pb, 'h1', key + '.layer_norm2', 'ln', M, H, eps)
    linear(pb, 'ln', M, H, key + '.fc1', I, out_f32=lambda R: R('ff'))
    pb.emit(lambda R: S.GegluDesc(src=R('ff'), out=R('gg'), rows=M, I=I, nplanes=NPL, fmt=0, mode=ACTS[act]))
    linear(pb, 'gg', M, I, key + '.fc2', H, out_f32=lambda R: R('h0'), residual=lambda R: R('h1'), ldr=H)


def pooled_head(pb, src, src_stride, C, norm, proj, E, eps, ids=None, row=0):
    """One row per sample of the fp32 stream `src` (sample n at n * src_stride floats: the row argmax(ids[n]) of the token ids `ids`, or
    `row`) -> LayerNorm `norm` -> @ the projection `proj`:w [E][C] (no bias) -> L2-normalised into io D [B][E] fp32."""
    B = pb.B
    pb.need('pool', B * C * F4)
    pb.need('pool16', NPL * B * C * H2)
    pb.need('emb', B * E * F4)
    pb.emit(lambda R: S.ClipHeadDesc(src=R(src), ids=ids or 0, out=R('pool'), src_stride=src_stride, out_stride=C, B=B, C=C,
                                     T=src_stride // C, row=row, mode=S.DS_CLIP_GATHER))
    layernorm(pb, 'pool', norm, 'pool16', B, C, eps)
    linear(pb, 'pool16', B, C, proj, E, bias=False, out_f32=lambda R: R('emb'))
    pb.emit(lambda R: S.ClipHeadDesc(src=R('emb'), out=io(S.DS_IO_D), B=B, C=E, mode=S.DS_CLIP_L2NORM))


def compile_clip_plan(cfg, wb, B, T, num_heads=None, eps=1e-5, npass=3, act='quick_gelu', prefix='', proj_dim=None):
    """Lower the text encoder for B prompts of T tokens (T <= max_position_embeddings).  Weights under `prefix` (tok, pos, l<i>.*,
    final).  proj_dim=None: last_hidden_state into io D; else the pooled text embedding of open_clip's encode_text, L2-normalised: the
    final LayerNorm of the row at argmax(ids) @ `prefix`proj [proj_dim][H] into io D [B][proj_dim]."""
    H, I = cfg['hidden_size'], cfg['intermediate_size']
    nh = num_heads or cfg.get('num_attention_heads') or H // 64
    if H != nh * 64:
        raise ValueError(f'the attention kernel has 64-wide heads; hidden_size {H} with {nh} heads is not supported')
    if T > cfg['max_position_embeddings'] or T > KEYS_PITCH:
        raise ValueError(f'{T} tokens exceed the position table ({cfg["max_position_embeddings"]})')
    M = B * T
    pb = PlanBuilder(wb, B, npass, tag=None)           # each op tagged with its index
    W = wb.ref
    reserve_layer_buffers(pb, M, H, I, KEYS_PITCH)
    pb.emit(lambda R_: S.EmbedDesc(ids=io(S.DS_IO_X), tok=W(prefix + 'tok'), pos=W(prefix + 'pos'), out=R_('h0'), rows=M, T=T, C=H,
                                   vocab=cfg['vocab_size']))
    for i in range(cfg['num_hidden_layers']):
        transformer_layer(pb, f'{prefix}l{i}', M, T, H, I, nh, 64, KEYS_PITCH, eps, causal=1, act=act)
    if proj_dim is None:
        layernorm(pb, 'h0', prefix + 'final', io(S.DS_IO_D), M, H, eps, fmt=2)
    else:
        pooled_head(pb, 'h0', T * H, H, prefix + 'final', prefix + 'proj', proj_dim, eps, ids=io(S.DS_IO_X))
    return pb.finish(B=B, T=T, npass=npass)

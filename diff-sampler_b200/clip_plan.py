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


def compile_clip_plan(cfg, wb, B, T, num_heads=None, eps=1e-5, npass=3):
    """Lower the text encoder for B prompts of T tokens (T <= max_position_embeddings)."""
    H, I = cfg['hidden_size'], cfg['intermediate_size']
    nh = num_heads or cfg.get('num_attention_heads') or H // 64
    if H != nh * 64:
        raise ValueError(f'the attention kernel has 64-wide heads; hidden_size {H} with {nh} heads is not supported')
    if T > cfg['max_position_embeddings'] or T > KEYS_PITCH:
        raise ValueError(f'{T} tokens exceed the position table ({cfg["max_position_embeddings"]})')
    M = B * T
    pb = PlanBuilder(wb, B, npass, tag=None)           # each op tagged with its index
    emit, W = pb.emit, wb.ref
    pb.need('h0', M * H * F4)
    pb.need('h1', M * H * F4)
    pb.need('ln', NPL * M * H * H2)
    pb.need('qk', NPL * M * 2 * H * H2)
    pb.need('vt', NPL * B * H * KEYS_PITCH * H2)
    pb.need('o', NPL * M * H * H2)
    pb.need('ff', M * I * F4)
    pb.need('gg', NPL * M * I * H2)

    def layernorm(src, g, b, out, fmt=0):
        emit(lambda R_: S.LayernormDesc(src=R_(src), gamma=W(g), beta=W(b), out=out(R_), rows=M, C=H, nplanes=NPL, eps=eps, fmt=fmt))

    def linear(a, K, key, N, **kw):
        """[M][K] activation planes x packed weight [N][K] (+ bias[N]) through the batched-rows GEMM form."""
        emit(lambda R_: G.rows_gemm(R_(a), M, K, 1, W(key + ':w'), G.padded_rows(N), K, 1, K, num_z=1, nh=1, m_valid=M, n_valid=N, npass=npass,
                                    bias_n=W(key + ':b'), ldo=N, **{k: (v(R_) if callable(v) else v) for k, v in kw.items()})[0])

    emit(lambda R_: S.EmbedDesc(ids=io(S.DS_IO_X), tok=W('tok'), pos=W('pos'), out=R_('h0'), rows=M, T=T, C=H, vocab=cfg['vocab_size']))
    for i in range(cfg['num_hidden_layers']):
        L = f'l{i}'
        # ---- h1 = h0 + out_proj(causal_attention(LN1(h0)))
        layernorm('h0', L + '.layer_norm1:g', L + '.layer_norm1:b', lambda R_: R_('ln'))
        linear('ln', H, L + '.qk', 2 * H, out_h16=lambda R_: R_('qk'), o_plane=M * 2 * H)
        pb.vt_gemm(L + '.v:w', 'ln', H, H, T, KEYS_PITCH, bias=L + '.v:b')
        pb.attention(True, 'qk', 'qk', 'o', nh, T, T, 64, 64 ** -0.5, KEYS_PITCH, causal=1)
        linear('o', H, L + '.out', H, out_f32=lambda R_: R_('h1'), residual=lambda R_: R_('h0'), ldr=H)
        # ---- h0 = h1 + fc2(quick_gelu(fc1(LN2(h1))))
        layernorm('h1', L + '.layer_norm2:g', L + '.layer_norm2:b', lambda R_: R_('ln'))
        linear('ln', H, L + '.fc1', I, out_f32=lambda R_: R_('ff'))
        emit(lambda R_: S.GegluDesc(src=R_('ff'), out=R_('gg'), rows=M, I=I, nplanes=NPL, fmt=0, mode=1))
        linear('gg', I, L + '.fc2', H, out_f32=lambda R_: R_('h0'), residual=lambda R_: R_('h1'), ldr=H)
    layernorm('h0', 'final:g', 'final:b', lambda R_: io(S.DS_IO_D), fmt=2)

    return pb.finish(B=B, T=T, npass=npass)

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
from .plan import Plan, WeightBlob, _Arena

F4, H2 = 4, 2
KEYS_PITCH = 128              # V^T row pitch (keys per row; a multiple of 8 elements for the TMA strides)


def prows(n):
    bn, tiles = G.pick_bn(n)
    return bn * tiles


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

    def lin(key, w, b):
        wb.add(key + ':w', G.pack_conv_weight(w.reshape(w.shape[0], w.shape[1], 1, 1)))
        wb.add(key + ':b', b)

    wb.add('tok', P('text_model.embeddings.token_embedding.weight'))
    wb.add('pos', P('text_model.embeddings.position_embedding.weight'))
    for i in range(cfg['num_hidden_layers']):
        p = f'text_model.encoder.layers.{i}.'
        a = p + 'self_attn.'
        lin(f'l{i}.qk', torch.cat([P(a + 'q_proj.weight'), P(a + 'k_proj.weight')]), torch.cat([P(a + 'q_proj.bias'), P(a + 'k_proj.bias')]))
        wb.add(f'l{i}.v:w', G.split_planes(P(a + 'v_proj.weight')))          # A operand of the V^T product: rows unpadded
        wb.add(f'l{i}.v:b', P(a + 'v_proj.bias'))
        lin(f'l{i}.out', P(a + 'out_proj.weight'), P(a + 'out_proj.bias'))
        lin(f'l{i}.fc1', P(p + 'mlp.fc1.weight'), P(p + 'mlp.fc1.bias'))
        lin(f'l{i}.fc2', P(p + 'mlp.fc2.weight'), P(p + 'mlp.fc2.bias'))
        for k in ('layer_norm1', 'layer_norm2'):
            wb.add(f'l{i}.{k}:g', P(p + k + '.weight'))
            wb.add(f'l{i}.{k}:b', P(p + k + '.bias'))
    wb.add('final:g', P('text_model.final_layer_norm.weight'))
    wb.add('final:b', P('text_model.final_layer_norm.bias'))
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
    npl = 2
    A = _Arena()
    ops = []
    emit = ops.append
    io = lambda slot: S.ref(S.SPACE_IO, slot)
    W = wb.ref
    A.need('h0', M * H * F4)
    A.need('h1', M * H * F4)
    A.need('ln', npl * M * H * H2)
    A.need('qk', npl * M * 2 * H * H2)
    A.need('vt', npl * B * H * KEYS_PITCH * H2)
    A.need('o', npl * M * H * H2)
    A.need('ff', M * I * F4)
    A.need('gg', npl * M * I * H2)

    def layernorm(src, g, b, out, fmt=0):
        emit(lambda R_: S.LayernormDesc(src=R_(src), gamma=W(g), beta=W(b), out=out(R_), rows=M, C=H, nplanes=npl, eps=eps, fmt=fmt))

    def linear(a, K, key, N, **kw):
        """[M][K] activation planes x packed weight [N][K] (+ bias[N]) through the batched-rows GEMM form."""
        emit(lambda R_: G.rows_gemm(R_(a), M, K, 1, W(key + ':w'), prows(N), K, 1, K, num_z=1, nh=1, m_valid=M, n_valid=N, npass=npass,
                                    bias_n=W(key + ':b'), ldo=N, **{k: (v(R_) if callable(v) else v) for k, v in kw.items()})[0])

    emit(lambda R_: S.EmbedDesc(ids=io(S.DS_IO_X), tok=W('tok'), pos=W('pos'), out=R_('h0'), rows=M, T=T, C=H, vocab=cfg['vocab_size']))
    for i in range(cfg['num_hidden_layers']):
        L = f'l{i}'
        # ---- h1 = h0 + out_proj(causal_attention(LN1(h0)))
        layernorm('h0', L + '.layer_norm1:g', L + '.layer_norm1:b', lambda R_: R_('ln'))
        linear('ln', H, L + '.qk', 2 * H, out_h16=lambda R_: R_('qk'), o_plane=M * 2 * H)
        # V^T[b][c][key] = sum_k Wv[c][k] LN[b][key][k] + bv[c]: written transposed, the layout the P.V product reads
        emit(lambda R_, L=L: G.rows_gemm(W(L + '.v:w'), H, H, 1, R_('ln'), T, H, B, H, num_z=B, nh=1, m_valid=H, n_valid=T, npass=npass,
                                         b_z_per_zb=1, bias_m=W(L + '.v:b'), out_h16=R_('vt'), o_zb=H * KEYS_PITCH, ldo=KEYS_PITCH,
                                         o_plane=B * H * KEYS_PITCH)[0])
        emit(lambda R_: S.AttnDesc(q=R_('qk'), k=R_('qk'), vt=R_('vt'), out=R_('o'), B=B, nh=nh, L=T, Lk=T, q_pitch=2 * H, q_c0=0, k_pitch=2 * H,
                                   k_c0=H, vt_pitch=KEYS_PITCH, o_pitch=H, nplanes=npl, scale=64 ** -0.5, causal=1))
        linear('o', H, L + '.out', H, out_f32=lambda R_: R_('h1'), residual=lambda R_: R_('h0'), ldr=H)
        # ---- h0 = h1 + fc2(quick_gelu(fc1(LN2(h1))))
        layernorm('h1', L + '.layer_norm2:g', L + '.layer_norm2:b', lambda R_: R_('ln'))
        linear('ln', H, L + '.fc1', I, out_f32=lambda R_: R_('ff'))
        emit(lambda R_: S.GegluDesc(src=R_('ff'), out=R_('gg'), rows=M, I=I, nplanes=npl, fmt=0, mode=1))
        linear('gg', I, L + '.fc2', H, out_f32=lambda R_: R_('h0'), residual=lambda R_: R_('h1'), ldr=H)
    layernorm('h0', 'final:g', 'final:b', lambda R_: io(S.DS_IO_D), fmt=2)

    total = A.finalize()
    arr = (S.PlanOp * len(ops))()
    for i, builder in enumerate(ops):
        desc = builder(A.ref)
        arr[i].type = S.OP_TYPE_OF[type(desc)]
        arr[i].tag = i
        setattr(arr[i].u, S.UNION_FIELD[arr[i].type], desc)
    meta = dict(B=B, T=T, npass=npass, n_ops=len(ops), n_gemm=sum(1 for i in range(len(ops)) if arr[i].type == S.DS_OP_GEMM))
    return Plan(arr, len(ops), total, dict(A.offsets), meta)

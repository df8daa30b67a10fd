"""Float64 restatement of the CLIP score of diff-solvers-main/clip_score.py (also amed-solver-main, gits-main, sfd-main): open_clip's
ViT-g-14 image and text towers, its image transform, and the score.  Pinned to transformers' CLIPModel (tests/test_openclip_host.py)
and to Pillow + torchvision for the transform.

  clip_score.py:59    model, _, preprocess = open_clip.create_model_and_transforms('ViT-g-14', pretrained='laion2b_s34b_b88k')
  clip_score.py:81    preprocess(to_pil(img)): Resize(224, BICUBIC) -> CenterCrop(224) -> ToTensor -> Normalize(OPENAI mean / std)
  clip_score.py:84-86 encode_image / encode_text, each divided by its norm
  clip_score.py:89    100 * (image_features * text_features).sum(-1), summed and divided by N (:90, :93)

Weights in open_clip's state-dict layout (visual.*, transformer.*, token_embedding, positional_embedding, ln_final, text_projection).
"""
import numpy as np
import torch

from diff_sampler_b200.openclip_plan import OPENAI_MEAN, OPENAI_STD, PRECISION_BITS, pil_bicubic_coeffs, resize_geometry


# ------------------------------------------------------------------------------------------------------------------ preprocessing
def _clip8(v):
    return np.where(v >= (1 << PRECISION_BITS << 8), 255, np.where(v <= 0, 0, v >> PRECISION_BITS))


def _pass(x, size, axis):
    """One Pillow 8-bit resample pass of the uint8 array x along `axis` to `size` samples (ImagingResampleHorizontal_8bpc /
    ImagingResampleVertical_8bpc): int32 sums from 2^21, clip8."""
    x0, n, kk, _ = pil_bicubic_coeffs(x.shape[axis], size)
    xm = np.moveaxis(x.astype(np.int64), axis, -1)
    out = np.empty(xm.shape[:-1] + (size,), dtype=np.int64)
    for i in range(size):
        k = np.asarray(kk[i], dtype=np.int64)
        out[..., i] = _clip8((1 << (PRECISION_BITS - 1)) + (xm[..., x0[i]:x0[i] + n[i]] * k).sum(-1))
    return np.moveaxis(out, -1, axis)


def preprocess(images, S=224):
    """uint8 [B, 3, H, W] -> the fp32 [B, 3, S, S] tensor open_clip's transform makes of to_pil(image): Pillow's bicubic resize
    (horizontal pass, then vertical; Image.resize skips a pass whose size does not change, which is the identity here), the centre
    crop, x / 255 and (x - mean) / std in fp32."""
    x = images.cpu().numpy()
    H, W = x.shape[2:]
    Rh, Rw, top, left = resize_geometry(H, W, S)
    if Rw != W:
        x = _pass(x, Rw, 3)
    if Rh != H:
        x = _pass(x, Rh, 2)
    x = torch.from_numpy(np.ascontiguousarray(x[:, :, top:top + S, left:left + S]).astype(np.uint8))
    v = x.float().div(255)
    return v.sub(torch.tensor(OPENAI_MEAN, dtype=torch.float32)[:, None, None]).div(torch.tensor(OPENAI_STD, dtype=torch.float32)[:, None, None])


# ------------------------------------------------------------------------------------------------------------------ towers
def _ln(x, sd, k, eps):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], sd[k + '.weight'].double(), sd[k + '.bias'].double(), eps)


def _block(x, sd, p, heads, eps, causal):
    """open_clip ResidualAttentionBlock: x + attn(ln_1(x)); x + mlp(ln_2(x)), exact GELU, scale head_dim^-1/2."""
    B, L, H = x.shape
    hd = H // heads
    h = _ln(x, sd, p + 'ln_1', eps)
    qkv = h @ sd[p + 'attn.in_proj_weight'].double().T + sd[p + 'attn.in_proj_bias'].double()
    q, k, v = (t.reshape(B, L, heads, hd).transpose(1, 2) for t in qkv.split(H, dim=-1))
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s + torch.full((L, L), float('-inf'), dtype=torch.float64, device=s.device).triu(1)
    o = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B, L, H)
    x = x + o @ sd[p + 'attn.out_proj.weight'].double().T + sd[p + 'attn.out_proj.bias'].double()
    h = _ln(x, sd, p + 'ln_2', eps)
    h = torch.nn.functional.gelu(h @ sd[p + 'mlp.c_fc.weight'].double().T + sd[p + 'mlp.c_fc.bias'].double())
    return x + h @ sd[p + 'mlp.c_proj.weight'].double().T + sd[p + 'mlp.c_proj.bias'].double()


def _layers(sd, prefix):
    return 1 + max(int(k[len(prefix):].split('.')[0]) for k in sd if k.startswith(prefix))


def image_features(sd, x, heads, eps=1e-5):
    """open_clip VisionTransformer.forward on the preprocessed fp32 [B, 3, S, S]: conv1 (no bias) -> [class; patches] + pos -> ln_pre
    -> blocks -> ln_post(token 0) @ proj.  float64 [B, E], not normalised."""
    w = sd['visual.conv1.weight'].double()
    P = w.shape[2]
    t = torch.nn.functional.conv2d(x.to(w.device, torch.float64), w, stride=P).flatten(2).transpose(1, 2)
    cls = sd['visual.class_embedding'].double().expand(t.shape[0], 1, -1)
    t = torch.cat([cls, t], dim=1) + sd['visual.positional_embedding'].double()
    t = _ln(t, sd, 'visual.ln_pre', eps)
    for i in range(_layers(sd, 'visual.transformer.resblocks.')):
        t = _block(t, sd, f'visual.transformer.resblocks.{i}.', heads, eps, causal=False)
    return _ln(t[:, 0], sd, 'visual.ln_post', eps) @ sd['visual.proj'].double()


def text_features(sd, ids, heads, eps=1e-5):
    """open_clip CLIP.encode_text on token ids [B, T]: token + positional embedding -> causal blocks -> ln_final -> the row at
    argmax(ids) (the EOT token) @ text_projection.  float64 [B, E], not normalised."""
    ids = ids.long().to(sd['token_embedding.weight'].device)
    T = ids.shape[1]
    x = sd['token_embedding.weight'].double()[ids] + sd['positional_embedding'].double()[:T]
    for i in range(_layers(sd, 'transformer.resblocks.')):
        x = _block(x, sd, f'transformer.resblocks.{i}.', heads, eps, causal=True)
    x = _ln(x, sd, 'ln_final', eps)
    return x[torch.arange(x.shape[0], device=x.device), ids.argmax(dim=-1)] @ sd['text_projection'].double()


def normalize(e):
    return e / e.norm(dim=-1, keepdim=True)


def scores(sd, images_u8, ids, vision_heads, text_heads, S=224, eps=1e-5):
    """Per-image clip_score.py score 100 <e_img, e_txt> (float64 [B]) of uint8 images [B, 3, H, W] paired with token ids [B, T]."""
    ei = normalize(image_features(sd, preprocess(images_u8, S), vision_heads, eps))
    et = normalize(text_features(sd, ids, text_heads, eps))
    return 100 * (ei * et).sum(-1)


def make_weights(cfg, seed=0):
    """Seeded open_clip-layout weights of the config keys openclip_plan.openclip_config returns (plus the head widths), scaled so
    that activations stay O(1) through the blocks."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, std=0.02: torch.randn(*s, generator=g) * std
    sd = {}
    Wv, Wt, E, P, S = cfg['vision_width'], cfg['text_width'], cfg['embed_dim'], cfg['patch_size'], cfg['image_size']
    L = (S // P) ** 2 + 1
    sd['visual.conv1.weight'] = r(Wv, 3, P, P, std=(3 * P * P) ** -0.5)
    sd['visual.class_embedding'] = r(Wv, std=0.5)
    sd['visual.positional_embedding'] = r(L, Wv, std=0.5)
    sd['visual.proj'] = r(Wv, E, std=Wv ** -0.5)
    sd['token_embedding.weight'] = r(cfg['vocab_size'], Wt, std=0.5)
    sd['positional_embedding'] = r(cfg['context_length'], Wt, std=0.2)
    sd['text_projection'] = r(Wt, E, std=Wt ** -0.5)
    for pre, W_, I, n in (('visual.transformer.resblocks.', Wv, cfg['vision_mlp'], cfg['vision_layers']),
                          ('transformer.resblocks.', Wt, cfg['text_mlp'], cfg['text_layers'])):
        for i in range(n):
            p = f'{pre}{i}.'
            sd[p + 'attn.in_proj_weight'] = r(3 * W_, W_, std=W_ ** -0.5)
            sd[p + 'attn.in_proj_bias'] = r(3 * W_)
            sd[p + 'attn.out_proj.weight'] = r(W_, W_, std=0.5 * W_ ** -0.5)
            sd[p + 'attn.out_proj.bias'] = r(W_)
            sd[p + 'mlp.c_fc.weight'] = r(I, W_, std=W_ ** -0.5)
            sd[p + 'mlp.c_fc.bias'] = r(I)
            sd[p + 'mlp.c_proj.weight'] = r(W_, I, std=0.5 * I ** -0.5)
            sd[p + 'mlp.c_proj.bias'] = r(W_)
            for k in ('ln_1', 'ln_2'):
                sd[p + k + '.weight'] = 1 + r(W_, std=0.1)
                sd[p + k + '.bias'] = r(W_, std=0.1)
    for k, W_ in (('visual.ln_pre', Wv), ('visual.ln_post', Wv), ('ln_final', Wt)):
        sd[k + '.weight'] = 1 + r(W_, std=0.1)
        sd[k + '.bias'] = r(W_, std=0.1)
    return sd


def make_ids(B, T, vocab, seed=0, lengths=None):
    """Seeded open_clip-style token ids [B, T] int32: SOT, random tokens below the special ids, EOT, zero padding.  The random tokens
    are drawn below vocab - 2 so that EOT (vocab - 1, as 49407 in the 49408-token vocabulary) is the row maximum."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(B, T, dtype=torch.int32)
    for b in range(B):
        n = lengths[b] if lengths else int(torch.randint(3, T - 1, (1,), generator=g))
        ids[b, 0] = vocab - 2
        ids[b, 1:n] = torch.randint(1, vocab - 2, (n - 1,), generator=g, dtype=torch.int32)
        ids[b, n] = vocab - 1
    return ids


# ViT-g-14 (open_clip's model config) and a small config of the same structure for the float64 plan-interpreter and GPU tests
VIT_G_14 = dict(image_size=224, patch_size=14, vision_width=1408, vision_layers=40, vision_heads=16, vision_mlp=6144, embed_dim=1024,
                vocab_size=49408, context_length=77, text_width=1024, text_layers=24, text_heads=16, text_mlp=4096)
SMALL = dict(image_size=56, patch_size=14, vision_width=704, vision_layers=2, vision_heads=8, vision_mlp=2816, embed_dim=128,
             vocab_size=1000, context_length=77, text_width=128, text_layers=2, text_heads=2, text_mlp=512)

"""B200OpenCLIP — the CLIP score of clip_score.py (diff-solvers-main/clip_score.py:59-93), native: open_clip's ViT-g-14
(`laion2b_s34b_b88k`) image and text towers and the per-image score 100 * <e_img, e_txt> of L2-normalised embeddings.  See
openclip_plan.py, DESIGN.md 4.11.

    clip = B200OpenCLIP(state_dict)                        # open_clip layout (visual.conv1.weight, ..., text_projection)
    clip = B200OpenCLIP.from_open_clip(model)              # or an open_clip CLIP module / a transformers CLIPModel:
    clip = B200OpenCLIP.from_transformers(clip_model)
    s = clip.score(images_u8, token_ids)                   # [B, 3, H, W] uint8 on the GPU, [B, 77] open_clip token ids -> [B] fp32
    stats = fid_stats.ScoreStats().append(s)               # running mean over batches and ranks

The images are the dataset's uint8 tensors (the NHWC view of the samplers' output needs no copy); the preprocessing open_clip runs
on PIL images on the host runs on the GPU, bit-exact.  Tokenisation stays with the caller (vocabulary files): pass token ids, or
give the constructor a `tokenizer` callable (list of str -> [B, 77] ids, e.g. open_clip.get_tokenizer('ViT-g-14')) and pass strings.
"""
import torch

from . import _cstructs as S
from . import _lib
from . import openclip_plan
from .inception_net import _dense
from .net import PRECISIONS, default_cuda_graph


class B200OpenCLIP:
    def __init__(self, state_dict, precision='fp16x3', max_batch=64, tokenizer=None, vision_head_width=88, text_head_width=64, eps=1e-5,
                 device='cuda', cuda_graph=None):
        """state_dict: open_clip CLIP layout (logit_scale and attn_mask, if present, are not read).  Batches larger than `max_batch` run
        in chunks of at most that many images or prompts."""
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200OpenCLIP needs a CUDA device (no CPU fallback)')
        if precision not in ('fp16x3', 'fp16'):
            raise ValueError(f'precision {precision!r}: the CLIP towers run fp16x3 or fp16')
        if max_batch < 1:
            raise ValueError(f'max_batch must be positive, got {max_batch}')
        self.lib = _lib.load()
        self.cfg = openclip_plan.openclip_config(state_dict, vision_head_width, text_head_width)
        hd = self.cfg['vision_width'] // self.cfg['vision_heads']
        if self.cfg['vision_heads'] * hd != self.cfg['vision_width'] or not (hd in (32, 64) or (72 <= hd <= 128 and hd % 8 == 0)):
            raise ValueError(f'image tower width {self.cfg["vision_width"]} with {vision_head_width}-wide heads is not supported')
        self.precision, self.npass, self.max_batch, self.eps = precision, PRECISIONS[precision], int(max_batch), float(eps)
        self.tokenizer = tokenizer
        self.cuda_graph = default_cuda_graph() if cuda_graph is None else bool(cuda_graph)
        self.wb = openclip_plan.pack_openclip_weights(state_dict, self.cfg)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self.tables = {}
        self.total_launches = 0

    @classmethod
    def from_open_clip(cls, model, **kw):
        """An open_clip `CLIP` module (open_clip.create_model_and_transforms('ViT-g-14', ...)[0]): its state dict."""
        return cls(model.state_dict(), **kw)

    @classmethod
    def from_transformers(cls, clip_model, **kw):
        """A transformers `CLIPModel` with exact GELU (hidden_act 'gelu') and the argmax text pooling (eos_token_id 2), mapped to
        open_clip's layout: the q / k / v projections concatenated as in_proj, the projections transposed."""
        conf = clip_model.config
        for c in (conf.vision_config, conf.text_config):
            if c.hidden_act != 'gelu':
                raise ValueError(f'unsupported CLIP activation {c.hidden_act!r} (the open_clip towers use exact GELU)')
        kw.setdefault('vision_head_width', conf.vision_config.hidden_size // conf.vision_config.num_attention_heads)
        kw.setdefault('text_head_width', conf.text_config.hidden_size // conf.text_config.num_attention_heads)
        kw.setdefault('eps', float(conf.vision_config.layer_norm_eps))
        return cls(openclip_state_dict_from_transformers(clip_model.state_dict()), **kw)

    # ---- plans
    def _image_plan(self, B, H, W, strides):
        tab_bytes = 4 * self._tables(H, W)[0].numel()
        return self.native.get(('image', B, H, W, strides),
                               lambda: openclip_plan.compile_image_plan(self.cfg, self.wb, B, H, W, self.npass, strides, self.eps),
                               (lambda pl: (B * 3 * H * W, B * self.cfg['embed_dim'] * 4, 0, 0, 0, tab_bytes)) if self.cuda_graph else None)

    def _text_plan(self, B, T):
        return self.native.get(('text', B, T), lambda: openclip_plan.compile_text_plan(self.cfg, self.wb, B, T, self.npass, self.eps),
                               (lambda pl: (B * T * 4, B * self.cfg['embed_dim'] * 4, 0, 0, 0, 0)) if self.cuda_graph else None)

    def _tables(self, H, W):
        """The resample tables of H x W inputs on the device (computed once per input size)."""
        if (H, W) not in self.tables:
            tab, ky, kx = openclip_plan.bicubic_tables(H, W, self.cfg['image_size'])
            self.tables[(H, W)] = (tab.to(self.device), ky, kx)
        return self.tables[(H, W)]

    # ---- public
    def encode_image(self, images):
        """images: uint8 [B, 3, H, W] on the device, any layout whose elements fill one dense block (contiguous NCHW, or the
        permute(0, 3, 1, 2) view of NHWC samples) -> L2-normalised image embeddings [B, E] fp32."""
        if images.device.type != 'cuda':
            raise _lib.DsError('B200OpenCLIP: images must live on the CUDA device (no CPU fallback)')
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f'expected uint8 images [B, 3, H, W], got {images.dtype} {tuple(images.shape)}')
        B, _, H, W = images.shape
        if not _dense(images):
            images = images.contiguous()
        out = torch.empty(B, self.cfg['embed_dim'], dtype=torch.float32, device=images.device)
        stream = torch.cuda.current_stream(images.device).cuda_stream
        strides = tuple(int(s) for s in images.stride())
        tab = self._tables(H, W)[0]
        for b0 in range(0, B, self.max_batch):
            n = min(self.max_batch, B - b0)
            h, _ = self._image_plan(n, H, W, strides)
            io = (images.data_ptr() + b0 * strides[0], out[b0].data_ptr(), None, None, None, tab.data_ptr())
            self.total_launches += self.native.run(h, io, stream)
        return out

    def encode_text(self, tokens):
        """tokens: open_clip token ids [B, T] (T <= context length; SOT 49406, EOT 49407, padding 0) on the device, or strings when
        the constructor was given a tokenizer -> L2-normalised text embeddings [B, E] fp32."""
        if isinstance(tokens, (str, list, tuple)):
            if self.tokenizer is None:
                raise _lib.DsError('B200OpenCLIP.encode_text: pass token ids, or give the constructor a tokenizer')
            tokens = self.tokenizer([tokens] if isinstance(tokens, str) else list(tokens)).to(self.device)
        if tokens.device.type != 'cuda':
            raise _lib.DsError('B200OpenCLIP: token ids must live on the CUDA device (no CPU fallback)')
        if tokens.dim() != 2:
            raise ValueError(f'expected token ids [B, T], got {tuple(tokens.shape)}')
        ids = tokens.to(torch.int32).contiguous()
        B, T = ids.shape
        out = torch.empty(B, self.cfg['embed_dim'], dtype=torch.float32, device=ids.device)
        stream = torch.cuda.current_stream(ids.device).cuda_stream
        for b0 in range(0, B, self.max_batch):
            n = min(self.max_batch, B - b0)
            h, _ = self._text_plan(n, T)
            self.total_launches += self.native.run(h, (ids[b0].data_ptr(), out[b0].data_ptr(), None, None, None, None), stream)
        return out

    def score(self, images, tokens):
        """Per-image CLIP score 100 * <e_img[i], e_txt[i]> (clip_score.py:84-89; no clamp at 0): image i with prompt i -> [B] fp32."""
        ei, et = self.encode_image(images), self.encode_text(tokens)
        if ei.shape[0] != et.shape[0]:
            raise ValueError(f'{ei.shape[0]} images but {et.shape[0]} prompts')
        return score_embeddings(ei, et)


def score_embeddings(e_img, e_txt, scale=100.0):
    """scale * <e_img[i], e_txt[i]> per row of two [B, E] fp32 device tensors, on the GPU (ds_clip_head, SCORE)."""
    e_img, e_txt = e_img.contiguous(), e_txt.contiguous()
    B, E = e_img.shape
    out = torch.empty(B, dtype=torch.float32, device=e_img.device)
    d = S.ClipHeadDesc(src=e_img.data_ptr(), src2=e_txt.data_ptr(), out=out.data_ptr(), B=B, C=E, mode=S.DS_CLIP_SCORE, scale=scale)
    _lib.op_launch(d, torch.cuda.current_stream(e_img.device).cuda_stream)
    return out


def openclip_state_dict_from_transformers(hf):
    """A transformers CLIPModel state dict in open_clip's CLIP layout (the names B200OpenCLIP reads)."""
    sd = {}
    v, t = 'vision_model.', 'text_model.'
    sd['visual.conv1.weight'] = hf[v + 'embeddings.patch_embedding.weight']
    sd['visual.class_embedding'] = hf[v + 'embeddings.class_embedding']
    sd['visual.positional_embedding'] = hf[v + 'embeddings.position_embedding.weight']
    for a, b in (('ln_pre', 'pre_layrnorm'), ('ln_post', 'post_layernorm')):
        sd[f'visual.{a}.weight'], sd[f'visual.{a}.bias'] = hf[v + b + '.weight'], hf[v + b + '.bias']
    sd['visual.proj'] = hf['visual_projection.weight'].t()
    sd['token_embedding.weight'] = hf[t + 'embeddings.token_embedding.weight']
    sd['positional_embedding'] = hf[t + 'embeddings.position_embedding.weight']
    sd['ln_final.weight'], sd['ln_final.bias'] = hf[t + 'final_layer_norm.weight'], hf[t + 'final_layer_norm.bias']
    sd['text_projection'] = hf['text_projection.weight'].t()
    for src, dst in ((v + 'encoder.layers.', 'visual.transformer.resblocks.'), (t + 'encoder.layers.', 'transformer.resblocks.')):
        n = 1 + max(int(k[len(src):].split('.')[0]) for k in hf if k.startswith(src))
        for i in range(n):
            s, d = f'{src}{i}.', f'{dst}{i}.'
            a = s + 'self_attn.'
            sd[d + 'attn.in_proj_weight'] = torch.cat([hf[a + f'{x}_proj.weight'] for x in 'qkv'])
            sd[d + 'attn.in_proj_bias'] = torch.cat([hf[a + f'{x}_proj.bias'] for x in 'qkv'])
            sd[d + 'attn.out_proj.weight'], sd[d + 'attn.out_proj.bias'] = hf[a + 'out_proj.weight'], hf[a + 'out_proj.bias']
            for x, y in (('ln_1', 'layer_norm1'), ('ln_2', 'layer_norm2'), ('mlp.c_fc', 'mlp.fc1'), ('mlp.c_proj', 'mlp.fc2')):
                sd[d + x + '.weight'], sd[d + x + '.bias'] = hf[s + y + '.weight'], hf[s + y + '.bias']
    return sd

"""B200CLIPTextEncoder — native text encoder of `get_learned_conditioning` (diff-solvers-main/sample.py:286-289;
models/ldm/modules/encoders/modules.py:137-159 `FrozenCLIPEmbedder`): token ids -> CLIPTextModel.last_hidden_state [B, 77, 768], the
`context` / `uc` tensors the CFG denoiser consumes.  SURVEY section 8(f)3.

    enc = B200CLIPTextEncoder.from_reference(net.model.cond_stage_model)       # the reference's FrozenCLIPEmbedder
    c = enc.encode(["a photo of an astronaut riding a horse"] * B)            # = net.model.get_learned_conditioning(prompts)
    c = enc(tokens)                                                           # from token ids (int tensor [B, 77])

Tokenisation stays with the reference's own `CLIPTokenizer` object (a vocabulary lookup on the host); everything after it runs as one
plan on the GPU (clip_plan.py).  No CPU fallback.
"""
from collections import OrderedDict

import torch

from . import _lib
from . import clip_plan


class B200CLIPTextEncoder:
    def __init__(self, params, num_heads=None, eps=1e-5, tokenizer=None, max_length=77, device='cuda'):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _lib.DsError('B200CLIPTextEncoder needs a CUDA device (no CPU fallback)')
        self.lib = _lib.load()
        self.cfg = clip_plan.clip_config(params)
        self.num_heads = num_heads
        self.eps = float(eps)
        self.tokenizer = tokenizer
        self.max_length = int(max_length)
        self.wb = clip_plan.pack_clip_weights(params, self.cfg)
        self.native = _lib.NativePlans(self.wb.bytes(), self.device)
        self.total_launches = 0

    @classmethod
    def from_reference(cls, module, **kw):
        """`module`: the reference's FrozenCLIPEmbedder (has `.transformer` = CLIPTextModel, `.tokenizer`, `.max_length`; modules.py:139-146),
        or a transformers CLIPTextModel itself."""
        tm = getattr(module, 'transformer', module)
        sd = OrderedDict((k, v) for k, v in tm.state_dict().items() if k.startswith('text_model.') and 'position_ids' not in k)
        conf = getattr(tm, 'config', None)
        if conf is not None:
            if getattr(conf, 'hidden_act', 'quick_gelu') != 'quick_gelu':
                raise ValueError(f'unsupported CLIP activation {conf.hidden_act!r} (the lowered MLP is quick_gelu)')
            kw.setdefault('num_heads', int(conf.num_attention_heads))
            kw.setdefault('eps', float(conf.layer_norm_eps))
        kw.setdefault('tokenizer', getattr(module, 'tokenizer', None))
        kw.setdefault('max_length', int(getattr(module, 'max_length', 77)))
        return cls(sd, **kw)

    def _plan(self, B, T):
        return self.native.get((B, T), lambda: clip_plan.compile_clip_plan(self.cfg, self.wb, B, T, num_heads=self.num_heads, eps=self.eps))

    def __call__(self, tokens, out=None):
        """tokens: integer tensor [B, T] on the CUDA device -> last_hidden_state [B, T, hidden] fp32.  A str / list of str is tokenised
        first, as FrozenCLIPEmbedder.forward(text) does."""
        if isinstance(tokens, (str, list, tuple)):
            return self.encode(tokens)
        if tokens.device.type != 'cuda':
            raise _lib.DsError('B200CLIPTextEncoder: token ids must live on the CUDA device (no CPU fallback)')
        if tokens.dim() != 2:
            raise ValueError(f'expected token ids [B, T], got {tuple(tokens.shape)}')
        ids = tokens.to(torch.int32).contiguous()
        B, T = ids.shape
        h, pl = self._plan(B, T)
        if out is None:
            out = torch.empty(B, T, self.cfg['hidden_size'], device=ids.device, dtype=torch.float32)
        self.total_launches += self.native.run(h, (ids.data_ptr(), out.data_ptr(), None, None, None, None),
                                               torch.cuda.current_stream(ids.device).cuda_stream)
        return out

    forward = __call__

    def encode(self, text):
        """FrozenCLIPEmbedder.encode (modules.py:148-159): tokenise with the reference's tokenizer (padding to max_length), then run."""
        if self.tokenizer is None:
            raise _lib.DsError('B200CLIPTextEncoder.encode needs the tokenizer of the reference module (from_reference keeps it)')
        enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True, return_overflowing_tokens=False,
                             padding='max_length', return_tensors='pt')
        return self(enc['input_ids'].to(self.device))

    def debug_read(self, B, T, name, numel, dtype=torch.float32):
        self._plan(B, T)
        return self.native.debug_read((B, T), name, numel, dtype)

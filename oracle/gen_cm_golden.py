"""Generate tests/golden/ref_cm.npz with the REAL reference Consistency-Models U-Net (models/cm/unet.py) inside CMPrecond
(models/networks_edm.py:504-549), in this container:

    python oracle/gen_cm_golden.py

The net is cm_net.TINY_SETTING (64 base channels x (2, 2, 2), 32x32, attention at 16x16 and 8x8, ResBlock up/down sampling) with the
seeded, de-zeroed weights of cm_net.init_state_dict, run on seeded inputs on CPU fp32.  Its outputs pin oracle/cm_oracle.py
(tests/test_cm_host.py).  The reference's QKVFlashAttention calls flash_attn's v1 `FlashAttention`, which needs a GPU; a sys.modules
stub supplies plain softmax(q k^T / sqrt(d)) v on the same `b s three h d` layout and records that layout, so the importer's qkv row
permutation is checked against the reference rearrange.  /root/reference is only imported, never copied.
"""
import math
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference/diff-solvers-main')

SEEN = []


class _FlashAttention(torch.nn.Module):
    """flash_attn.flash_attention.FlashAttention (v1) on the CPU: qkv [b, s, 3, h, d] -> ([b, s, h, d], None)."""

    def __init__(self, attention_dropout=0.0, **_):
        super().__init__()

    def forward(self, qkv, key_padding_mask=None, need_weights=False, causal=False):
        SEEN.append(qkv.detach().clone())
        q, k, v = qkv.unbind(2)                                   # [b, s, h, d]
        d = q.shape[-1]
        p = torch.softmax(torch.einsum('bqhd,bkhd->bhqk', q, k) / math.sqrt(d), dim=-1)
        return torch.einsum('bhqk,bkhd->bqhd', p, v), None


def _install_stub():
    fa = types.ModuleType('flash_attn')
    ff = types.ModuleType('flash_attn.flash_attention')
    ff.FlashAttention = _FlashAttention
    fa.flash_attention = ff
    sys.modules.setdefault('flash_attn', fa)
    sys.modules.setdefault('flash_attn.flash_attention', ff)


def main():
    _install_stub()
    from models.cm.cm_model_loader import create_model
    from models.cm.unet import QKVFlashAttention
    from models.networks_edm import CMPrecond
    from diff_sampler_b200 import cm_net

    out = {}
    setting = dict(cm_net.TINY_SETTING)
    kw = {k: v for k, v in setting.items() if k != 'use_fp16'}
    model = create_model(**kw, use_fp16=False).eval()
    sd = cm_net.init_state_dict(setting, seed=0, dezero=True)
    model.load_state_dict(sd, strict=True)
    net = CMPrecond(model).eval()
    taps = []
    model.middle_block.register_forward_hook(lambda m, i, o: taps.append(o.detach().clone()))
    g = torch.Generator().manual_seed(7)
    B, R = 2, setting['image_size']
    x = torch.randn(B, 3, R, R, generator=g)
    for tag, sig in (('s2', torch.tensor([2.0])), ('s80', torch.tensor([80.0])), ('s0p002', torch.tensor([0.002])),
                     ('per', torch.tensor([0.5, 11.0]))):
        xs = x * sig.reshape(-1, 1, 1, 1)
        with torch.no_grad():
            D = net(xs, sig)
        out[f'cm/{tag}/x'] = xs.numpy()
        out[f'cm/{tag}/sigma'] = sig.numpy()
        out[f'cm/{tag}/D'] = D.numpy()
        out[f'cm/{tag}/middle'] = taps[-1].numpy()
        print(tag, 'max|D|', float(D.abs().max()))

    # the qkv layout QKVFlashAttention hands to FlashAttention: rows of the qkv conv -> [three][head][d]
    SEEN.clear()
    heads, d, L = 2, 16, 3
    qkv = torch.arange(3 * heads * d, dtype=torch.float32)[None, :, None].expand(1, 3 * heads * d, L).contiguous()
    QKVFlashAttention(heads * d, heads)(qkv)
    out['qkv/heads'] = np.array(heads)
    out['qkv/layout'] = SEEN[-1][0, 0].numpy()                  # [3, heads, d]: the conv row each (three, h, d) slot reads
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'ref_cm.npz'), **out)


if __name__ == '__main__':
    main()

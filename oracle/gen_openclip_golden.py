"""Writes tests/golden/ref_openclip.npz: a small seeded transformers CLIPModel (exact GELU, argmax text pooling) in open_clip's
state-dict layout, its image and text embeddings, and open_clip's transform (Pillow bicubic Resize, CenterCrop, ToTensor, Normalize)
of seeded uint8 images: a downscale, an upscale and both non-square orientations, each from NCHW and from the NHWC view.

    python oracle/gen_openclip_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diff_sampler_b200.openclip_net import openclip_state_dict_from_transformers   # noqa: E402
from diff_sampler_b200.openclip_plan import OPENAI_MEAN, OPENAI_STD                  # noqa: E402

CROP = 16                                   # transform output size of the image cases
IMAGE_CASES = [(40, 40), (10, 10), (24, 36), (36, 24)]
VISION = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, image_size=28, patch_size=14,
              hidden_act='gelu', layer_norm_eps=1e-5)
TEXT = dict(vocab_size=100, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, max_position_embeddings=16,
            hidden_act='gelu', layer_norm_eps=1e-5, eos_token_id=2)


def transform(S):
    from torchvision import transforms as T
    return T.Compose([T.Resize(S, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(S), T.ToTensor(),
                      T.Normalize(OPENAI_MEAN, OPENAI_STD)])


def main():
    from transformers import CLIPConfig, CLIPModel
    from torchvision import transforms as T
    torch.manual_seed(0)
    model = CLIPModel(CLIPConfig(text_config=TEXT, vision_config=VISION, projection_dim=32)).double().eval()
    sd = openclip_state_dict_from_transformers(model.state_dict())
    out = {f'sd/{k}': v.detach().float().numpy() for k, v in sd.items()}      # initialised in fp32: exact
    g = torch.Generator().manual_seed(1)
    pix = torch.randn(3, 3, 28, 28, generator=g, dtype=torch.float64)
    ids = torch.zeros(3, 16, dtype=torch.long)
    for b, n in enumerate((5, 9, 14)):
        ids[b, 0] = 98
        ids[b, 1:n] = torch.randint(1, 98, (n - 1,), generator=g)
        ids[b, n] = 99
    with torch.no_grad():
        out['pixels'] = pix.numpy()
        out['ids'] = ids.numpy()
        out['image_embeds'] = model.visual_projection(model.vision_model(pixel_values=pix).pooler_output).numpy()
        out['text_embeds'] = model.text_projection(model.text_model(input_ids=ids).pooler_output).numpy()
    tf, to_pil = transform(CROP), T.ToPILImage()
    for i, (H, W) in enumerate(IMAGE_CASES):
        u8 = torch.randint(0, 256, (2, 3, H, W), generator=torch.Generator().manual_seed(10 + i), dtype=torch.uint8)
        out[f'img/{H}x{W}'] = u8.numpy()
        out[f'pre/{H}x{W}'] = torch.stack([tf(to_pil(x)) for x in u8]).numpy()
        nhwc = u8.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        assert torch.equal(torch.stack([tf(to_pil(x)) for x in nhwc]), torch.from_numpy(out[f'pre/{H}x{W}']))
    path = os.path.join(ROOT, 'tests', 'golden', 'ref_openclip.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, sum(v.nbytes for v in out.values()), 'bytes')


if __name__ == '__main__':
    main()

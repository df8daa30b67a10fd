"""Throughput of the native CLIP score at ViT-g-14 dimensions (seeded random weights): encode_image images/s at batch 250 in fp16x3
and fp16, encode_text prompts/s, and transformers' CLIPModel of the same shapes run eagerly on the same GPU (fp32, which may use TF32,
and fp16).  Prints the card, its power limit and maximum SM clock, and the results as one JSON line.

    python tools/clip_score_probe.py [--batch 250] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diff_sampler_b200.openclip_net import B200OpenCLIP      # noqa: E402
from oracle import openclip_oracle as O                      # noqa: E402


def _timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=250)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--size', type=int, default=512)
    a = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    print('card:', card)
    dev = torch.device('cuda')
    cfg = dict(O.VIT_G_14)
    sd = O.make_weights(cfg, seed=0)
    u8 = torch.randint(0, 256, (a.batch, a.size, a.size, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8).to(dev)
    x = u8.permute(0, 3, 1, 2)
    ids = O.make_ids(a.batch, 77, cfg['vocab_size'], seed=1).to(dev)
    res = dict(card=card, batch=a.batch, size=a.size)
    for prec in ('fp16x3', 'fp16'):
        clip = B200OpenCLIP(sd, precision=prec)
        ti = _timed(lambda: clip.encode_image(x), a.iters)
        tt = _timed(lambda: clip.encode_text(ids), a.iters)
        res[f'native_{prec}_images_per_s'] = a.batch / ti
        res[f'native_{prec}_prompts_per_s'] = a.batch / tt
        print(f'native {prec}: {a.batch / ti:.1f} images/s, {a.batch / tt:.1f} prompts/s')
        del clip
        torch.cuda.empty_cache()
    import transformers
    conf = transformers.CLIPConfig(
        text_config=dict(vocab_size=cfg['vocab_size'], hidden_size=cfg['text_width'], intermediate_size=cfg['text_mlp'],
                         num_hidden_layers=cfg['text_layers'], num_attention_heads=cfg['text_heads'], max_position_embeddings=77,
                         hidden_act='gelu', eos_token_id=2),
        vision_config=dict(hidden_size=cfg['vision_width'], intermediate_size=cfg['vision_mlp'], num_hidden_layers=cfg['vision_layers'],
                           num_attention_heads=cfg['vision_heads'], image_size=224, patch_size=14, hidden_act='gelu'),
        projection_dim=cfg['embed_dim'])
    with torch.device(dev):
        model = transformers.CLIPModel(conf).eval()
    pix = torch.randn(a.batch, 3, 224, 224, device=dev)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    for name, dt in (('fp32', torch.float32), ('fp16', torch.float16)):
        m = model.to(dt)
        with torch.no_grad():
            chunks = [slice(i, i + 64) for i in range(0, a.batch, 64)]      # clip_score.py's max_batch_size
            ti = _timed(lambda: [m.visual_projection(m.vision_model(pixel_values=pix[c].to(dt)).pooler_output) for c in chunks], a.iters)
            tt = _timed(lambda: [m.text_projection(m.text_model(input_ids=ids[c].long()).pooler_output) for c in chunks], a.iters)
        res[f'eager_{name}_images_per_s'] = a.batch / ti
        res[f'eager_{name}_prompts_per_s'] = a.batch / tt
        print(f'eager CLIPModel {name}: {a.batch / ti:.1f} images/s (tower only, preprocessing excluded), {a.batch / tt:.1f} prompts/s')
    print(json.dumps(res))


if __name__ == '__main__':
    main()

"""Op-by-op replay of the CLIP-score plans (open_clip image and text towers) on the GPU against the float64 plan interpreter, as
tests/test_gpu_plan_ops.py replays the benchmarked plans: every op stores only inside its spans, writes every element the reference
writes, finitely and within its class tolerance.  This catches what the end-to-end embedding tests cannot: the patch-embedding GEMM
writes rows 1 .. L-1 of each sample and the class-token gather right after it writes row 0, so a stray store into row 0 would be
overwritten before anything reads it; the im2col's K padding (588 -> 640) must come out zero; the wide-head attention kernel reads
Q, K and V^T through per-head tensor maps that must stop at the head and the pitch padding.

The image input, the im2col and the pooled heads' gathers restate their reference bit for bit, so they are held to error 0; the L2
normalisation and the score keep the default 1e-5 bound.

Two workloads at full tower widths and two layers per tower (every layer has the same descriptors, so depth adds time, not
coverage), batch 3, both precisions:
  vit_g_14       ViT-g-14: 16 heads of 88, 257 tokens (V^T pitch 264); 512 x 768 images with NHWC strides (the samplers' output)
  vit_h_14_378   ViT-H-14 at 378 px (DFN5B): 16 heads of 80, 730 tokens (V^T pitch 736); 300 x 224 NCHW images (upscaled)
Both share the text tower of ViT-g-14 (1024 wide, 16 causal heads of 64)."""
import collections
import functools

import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import openclip_plan as OP
from oracle import openclip_oracle as O

import openclip_interp as OI

pytestmark = pytest.mark.gpu

B = 3
MODELS = {
    'vit_g_14': (dict(O.VIT_G_14, vision_layers=2, text_layers=2), 88, (512, 768), True),
    'vit_h_14_378': (dict(O.VIT_G_14, image_size=378, vision_width=1280, vision_mlp=5120, vision_layers=2, text_layers=2), 80,
                     (300, 224), False),
}
NPASS = {'fp16x3': 3, 'fp16': 1}
EXACT = ('clip_input', 'im2col')                 # and the clip_head gathers
RESULTS = {}                                     # (model, precision) -> {tower: replay result}


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


@functools.lru_cache(maxsize=1)
def _weights(model):
    cfg0, hw, _, _ = MODELS[model]
    sd = O.make_weights(cfg0, seed=13)
    cfg = OP.openclip_config(sd, vision_head_width=hw)
    return cfg, OP.pack_openclip_weights(sd, cfg)


def _workload(model, npass, tower):
    """(plan, weight blob bytes, {io slot: host tensor}) of one tower."""
    cfg, wb = _weights(model)
    _, _, (H, W), nhwc = MODELS[model]
    d = torch.zeros(B, cfg['embed_dim'])
    if tower == 'text':
        ids = O.make_ids(B, cfg['context_length'], cfg['vocab_size'], seed=5, lengths=[1, 76, 40])   # EOT at 1, 76 and 40
        return OP.compile_text_plan(cfg, wb, B, cfg['context_length'], npass), wb.bytes(), {S.DS_IO_X: ids, S.DS_IO_D: d}
    u8 = torch.randint(0, 256, (B, 3, H, W), generator=torch.Generator().manual_seed(H + W), dtype=torch.uint8)
    strides = None
    if nhwc:
        u8 = u8.permute(0, 2, 3, 1).contiguous()                                  # stored [B][H][W][3], read through NCHW strides
        strides = tuple(u8.permute(0, 3, 1, 2).stride())
    pl = OP.compile_image_plan(cfg, wb, B, H, W, npass, strides)
    return pl, wb.bytes(), {S.DS_IO_X: u8, S.DS_IO_CTX: OP.bicubic_tables(H, W, cfg['image_size'])[0], S.DS_IO_D: d}


@pytest.mark.parametrize('model,precision', [(m, p) for m in MODELS for p in NPASS])
def test_plan_ops_against_the_interpreter(lib, monkeypatch, model, precision):
    import test_gpu_plan_ops as TPO
    OI.install(monkeypatch)
    plans = {}

    def workload(name):
        tower = name.split('/')[-1]
        w = _workload(model, NPASS[precision], tower)
        plans[tower] = w[0]
        return w
    monkeypatch.setattr(TPO, 'workload', workload)
    cfg, _ = _weights(model)
    RESULTS[(model, precision)] = out = {}
    for tower in ('image', 'text'):
        name = f'{model}/{precision}/{tower}'
        res = out[tower] = TPO.replay(lib, name)
        pl = plans[tower]
        print(f"\n{'workload':10s} {'op':>4s} {'type':11s} {'tag':>5s} {'shape':44s} {'max err':>10s} {'bound':>10s} {'ratio':>7s}")
        for r in res['rows']:
            print(TPO._fmt(name, r))
        print(f"{name}: {res['n_ops']} ops, {res['seconds']:.1f} s, peak device memory {res['peak'] / 2 ** 30:.2f} GiB")
        compared = {r['type'] for r in res['rows']}
        assert not res['skips'] and len(res['rows']) == res['n_ops'] and compared == res['types'], sorted(res['types'] - compared)
        bad = [r for r in res['rows'] if r['ratio'] > 1.0 or r['problems']]
        assert not bad, '\n'.join(TPO._fmt(name, r) for r in bad[:20])
        exact = [r for r in res['rows'] if r['type'] in EXACT
                 or (r['type'] == 'clip_head' and int(pl.ops_array[r['i']].u.clip_head.mode) == S.DS_CLIP_GATHER)]
        assert len(exact) == (4 if tower == 'image' else 1), [r['type'] for r in exact]   # image: class row and pooled row gathers
        assert all(r['err'] == 0.0 for r in exact), '\n'.join(TPO._fmt(name, r) for r in exact if r['err'] != 0.0)
        if tower == 'image':                     # the plan runs the wide kernel over all tokens at this head width
            L = (cfg['image_size'] // cfg['patch_size']) ** 2 + 1
            hd = cfg['vision_width'] // cfg['vision_heads']
            attn = [pl.ops_array[r['i']].u.attn for r in res['rows'] if r['type'] == 'attn']
            assert attn and all((int(a.pad0), int(a.L), int(a.Lk)) == (hd, L, L) for a in attn)


def test_plan_ops_report():
    if not RESULTS:
        pytest.skip('no workload of this module ran')
    print('\nworst ratio (error / bound) per op type')
    rows = [(f'{m}/{p}/{t}', res) for (m, p), towers in RESULTS.items() for t, res in towers.items()]
    types = sorted({t for _, res in rows for t in res['types']})
    print(f"{'workload':26s} {'ops':>4s} {'secs':>6s} " + ' '.join(f'{t:>11s}' for t in types))
    for name, res in rows:
        worst = collections.defaultdict(float)
        for r in res['rows']:
            worst[r['type']] = max(worst[r['type']], r['ratio'])
        print(f"{name:26s} {res['n_ops']:4d} {res['seconds']:6.1f} "
              + ' '.join(f'{worst[t]:11.3f}' if t in res['types'] else f"{'-':>11s}" for t in types))

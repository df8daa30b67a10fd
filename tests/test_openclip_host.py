"""CLIP score on the host: the float64 oracle against transformers' CLIPModel (committed golden), the open_clip-layout import, the
preprocessing restatement against Pillow + torchvision bit for bit, both plans on the float64 plan interpreter against the oracle,
every new launcher rule, the descriptor sizes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import openclip_plan as OP
from diff_sampler_b200.openclip_net import openclip_state_dict_from_transformers
from oracle import openclip_oracle as O

import openclip_interp as OI

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_openclip.npz')


@pytest.fixture(scope='module')
def ref():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope='module')
def built():
    import __graft_entry__
    __graft_entry__.build()
    from diff_sampler_b200 import _lib
    return _lib


def _sd(ref):
    return {k[3:]: torch.from_numpy(v).double() for k, v in ref.items() if k.startswith('sd/')}


def test_oracle_matches_clipmodel(ref):
    sd = _sd(ref)
    ei = O.image_features(sd, torch.from_numpy(ref['pixels']), heads=2)
    et = O.text_features(sd, torch.from_numpy(ref['ids']), heads=2)
    want_i, want_t = torch.from_numpy(ref['image_embeds']), torch.from_numpy(ref['text_embeds'])
    assert (ei - want_i).abs().max() < 1e-12 * want_i.abs().max()
    assert (et - want_t).abs().max() < 1e-12 * want_t.abs().max()
    s = 100 * (O.normalize(ei) * O.normalize(et)).sum(-1)
    s_want = 100 * (O.normalize(want_i) * O.normalize(want_t)).sum(-1)
    assert (s - s_want).abs().max() < 1e-10


def test_open_clip_named_module_maps_to_the_same_function(ref):
    """A module with open_clip's parameter names, built from nn.MultiheadAttention / LayerNorm / GELU, computes the oracle's function
    from the mapped state dict (the layout B200OpenCLIP reads)."""
    sd = _sd(ref)
    W = sd['transformer.resblocks.0.ln_1.weight'].shape[0]

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ln_1, self.ln_2 = torch.nn.LayerNorm(W), torch.nn.LayerNorm(W)
            self.attn = torch.nn.MultiheadAttention(W, 2, batch_first=True)
            self.mlp = torch.nn.Sequential()
            self.mlp.add_module('c_fc', torch.nn.Linear(W, 2 * W))
            self.mlp.add_module('gelu', torch.nn.GELU())
            self.mlp.add_module('c_proj', torch.nn.Linear(2 * W, W))

        def forward(self, x, mask):
            h = self.ln_1(x)
            x = x + self.attn(h, h, h, need_weights=False, attn_mask=mask)[0]
            return x + self.mlp(self.ln_2(x))

    blocks = torch.nn.ModuleList([Block() for _ in range(2)]).double()
    blocks.load_state_dict({k[len('transformer.resblocks.'):]: v for k, v in sd.items() if k.startswith('transformer.resblocks.')})
    ids = torch.from_numpy(ref['ids']).long()
    T = ids.shape[1]
    x = sd['token_embedding.weight'][ids] + sd['positional_embedding'][:T]
    mask = torch.full((T, T), float('-inf'), dtype=torch.float64).triu(1)
    with torch.no_grad():
        for b in blocks:
            x = b(x, mask)
        x = torch.nn.functional.layer_norm(x, (W,), sd['ln_final.weight'], sd['ln_final.bias'], 1e-5)
        got = x[torch.arange(x.shape[0]), ids.argmax(-1)] @ sd['text_projection']
    want = torch.from_numpy(ref['text_embeds'])
    assert (got - want).abs().max() < 1e-12 * want.abs().max()


def test_transformers_state_dict_mapping_round_trip():
    transformers = pytest.importorskip('transformers')
    conf = transformers.CLIPConfig(text_config=dict(vocab_size=50, hidden_size=64, intermediate_size=128, num_hidden_layers=1,
                                                    num_attention_heads=1, max_position_embeddings=8, hidden_act='gelu'),
                                   vision_config=dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1,
                                                      image_size=28, patch_size=14, hidden_act='gelu'), projection_dim=16)
    m = transformers.CLIPModel(conf)
    sd = openclip_state_dict_from_transformers(m.state_dict())
    cfg = OP.openclip_config(sd, 64, 64)
    assert (cfg['image_size'], cfg['vision_layers'], cfg['text_layers'], cfg['embed_dim'], cfg['context_length']) == (28, 1, 1, 16, 8)
    assert torch.equal(sd['visual.proj'], m.visual_projection.weight.t())


@pytest.mark.parametrize('case', ['40x40', '10x10', '24x36', '36x24'])
def test_preprocess_matches_committed_pillow_transform(ref, case):
    u8 = torch.from_numpy(ref[f'img/{case}'])
    want = torch.from_numpy(ref[f'pre/{case}'])
    assert torch.equal(O.preprocess(u8, 16), want)
    assert torch.equal(O.preprocess(u8.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2), 16), want)


@pytest.mark.parametrize('H,W', [(512, 512), (256, 256), (64, 64), (512, 768), (768, 512), (224, 300), (333, 257)])
def test_preprocess_is_bit_identical_to_pillow(H, W):
    pytest.importorskip('PIL')
    T = pytest.importorskip('torchvision.transforms')
    tf = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                    T.Normalize(OP.OPENAI_MEAN, OP.OPENAI_STD)])
    u8 = torch.randint(0, 256, (2, 3, H, W), generator=torch.Generator().manual_seed(H * 1000 + W), dtype=torch.uint8)
    want = torch.stack([tf(T.ToPILImage()(x)) for x in u8])
    assert torch.equal(O.preprocess(u8), want)


def _small():
    cfg = dict(O.SMALL)
    sd = O.make_weights(cfg, seed=3)
    return cfg, sd, OP.pack_openclip_weights(sd, cfg)


@pytest.mark.parametrize('H,W,nhwc', [(40, 60, False), (100, 70, True)])
def test_image_plan_on_the_interpreter(monkeypatch, H, W, nhwc):
    OI.install(monkeypatch)
    cfg, sd, wb = _small()
    B = 2
    u8 = torch.randint(0, 256, (B, 3, H, W), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    x = u8.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2) if nhwc else u8
    strides = tuple(int(s) for s in x.stride())
    pl = OP.compile_image_plan(cfg, wb, B, H, W, 3, strides)
    tab = OP.bicubic_tables(H, W, cfg['image_size'])[0]
    out = torch.zeros(B, cfg['embed_dim'])
    base = x.as_strided((x.numel(),), (1,), 0) if nhwc else x.reshape(-1)
    mem = OI.run_plan(pl, wb.bytes(), {S.DS_IO_X: base, S.DS_IO_D: out, S.DS_IO_CTX: tab})
    img = OI.PI.read_buffer(mem, pl, 'img', (B, cfg['image_size'], cfg['image_size'], 3))
    assert torch.equal(img.permute(0, 3, 1, 2), O.preprocess(u8, cfg['image_size']))
    want = O.normalize(O.image_features(sd, O.preprocess(u8, cfg['image_size']), cfg['vision_heads']))
    err = (out.double() - want).abs().max().item()
    print(f'image plan on the interpreter: {err:.2e}')
    assert err < 2e-5


def test_text_plan_on_the_interpreter(monkeypatch):
    OI.install(monkeypatch)
    cfg, sd, wb = _small()
    ids = O.make_ids(3, 77, cfg['vocab_size'], seed=2)
    pl = OP.compile_text_plan(cfg, wb, 3, 77, 3)
    out = torch.zeros(3, cfg['embed_dim'])
    OI.run_plan(pl, wb.bytes(), {S.DS_IO_X: ids, S.DS_IO_D: out})
    want = O.normalize(O.text_features(sd, ids, cfg['text_heads']))
    err = (out.double() - want).abs().max().item()
    print(f'text plan on the interpreter: {err:.2e}')
    assert err < 2e-5


def test_every_plan_op_passes_the_launcher_checks(built):
    cfg = dict(O.VIT_G_14)
    cfg.update(vision_layers=1, text_layers=1)
    sd = O.make_weights(dict(cfg, vocab_size=1000), seed=0)
    cfg['vocab_size'] = 1000
    wb = OP.pack_openclip_weights(sd, cfg)
    for pl in (OP.compile_image_plan(cfg, wb, 3, 512, 768), OP.compile_text_plan(cfg, wb, 3, 77)):
        for i in range(pl.n_ops):
            op = pl.ops_array[i]
            assert built.op_check(getattr(op.u, S.ALL_UNION_FIELD[op.type])) is None, (i, op.type)
        assert any(op.type == S.DS_OP_ATTN for op in pl.ops_array)
    attn = [pl.ops_array[i].u.attn for i in range(pl.n_ops) if pl.ops_array[i].type == S.DS_OP_ATTN]
    assert all(int(a.pad0) == 0 for a in attn)          # the text tower's 64-wide heads


def _with(desc, **kw):
    d = type(desc).from_buffer_copy(desc)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _attn():
    return S.AttnDesc(q=1, k=1, vt=1, out=1, B=2, nh=16, L=257, Lk=257, q_pitch=2816, q_c0=0, k_pitch=2816, k_c0=1408, vt_pitch=264,
                      o_pitch=1408, nplanes=2, scale=88 ** -0.5, causal=0, pad0=88)


def _clip_input():
    return S.ClipInputDesc(src=1, tab=1, out=1, sn=3 * 64 * 64, sc=64 * 64, sy=64, sx=1, B=2, H=64, W=64, S=224, ky=5, kx=5,
                           mean=OP.OPENAI_MEAN, std=OP.OPENAI_STD)


def _clip_head():
    return S.ClipHeadDesc(src=1, src2=0, ids=1, out=1, src_stride=77 * 1024, out_stride=1024, B=2, C=1024, T=77, row=0,
                          mode=S.DS_CLIP_GATHER, scale=0.0)


def _gelu():
    return S.GegluDesc(src=1, out=1, rows=4, I=64, nplanes=2, fmt=0, mode=2)


RULES = [   # (make, rule, a breaking change, its nearest valid neighbour)
    (_attn, 'attn: head_dim', dict(pad0=90, q_pitch=2880, k_pitch=2880, k_c0=1440, o_pitch=1440),
     dict(pad0=96, q_pitch=3072, k_pitch=3072, k_c0=1536, o_pitch=1536)),
    (_attn, 'attn: head_dim', dict(pad0=136, q_pitch=4352, k_pitch=4352, k_c0=2176, o_pitch=2176),
     dict(pad0=128, q_pitch=4096, k_pitch=4096, k_c0=2048, o_pitch=2048)),
    (_attn, 'attn: wide causal', dict(causal=1), dict(causal=0)),
    (_clip_input, 'clip_input: shape', dict(S=0), dict(S=1)),
    (_clip_input, 'clip_input: taps', dict(ky=0), dict(ky=1)),
    (_clip_input, 'clip_input: taps', dict(kx=6), dict(kx=5)),
    (_clip_input, 'clip_input: tables', dict(tab=0), dict(tab=2)),
    (_clip_input, 'clip_input: std', dict(std=(0.5, 0.0, 0.5)), dict(std=(0.5, 0.5, 0.5))),
    (_clip_head, 'clip_head: mode', dict(mode=3), dict(mode=S.DS_CLIP_L2NORM)),
    (_clip_head, 'clip_head: shape', dict(C=0), dict(C=1)),
    (_clip_head, 'clip_head: row', dict(T=0), dict(ids=0, T=0)),
    (_clip_head, 'clip_head: operands', dict(mode=S.DS_CLIP_SCORE), dict(mode=S.DS_CLIP_SCORE, src2=1)),
    (_gelu, 'geglu: mode', dict(mode=3), dict(mode=1)),
    (_gelu, 'geglu: GELU fmt', dict(fmt=1), dict(fmt=0, nplanes=1)),
]


@pytest.mark.parametrize('make,rule,bad,good', RULES, ids=[f'{r[1]}-{i}' for i, r in enumerate(RULES)])
def test_each_rule_refuses_what_breaks_it_and_accepts_its_neighbour(built, make, rule, bad, good):
    assert built.op_check(make()) is None
    assert built.op_check(_with(make(), **bad)) == rule
    assert built.op_check(_with(make(), **good)) is None


def test_descriptor_sizes(built):
    lib = built.load()
    assert C.sizeof(S.PlanOp) == 528 == lib.ds_sizeof(0)
    assert C.sizeof(S.AttnDesc) == lib.ds_sizeof(S.DS_OP_ATTN) and C.sizeof(S.GegluDesc) == lib.ds_sizeof(S.DS_OP_GEGLU)
    for t in (S.DS_OP_CLIP_INPUT, S.DS_OP_CLIP_HEAD):
        assert lib.ds_sizeof(t) == C.sizeof(S.SIZEOF_CHECKS[t])


def test_bicubic_taps_match_the_tables():
    for H, W in ((512, 512), (64, 64), (512, 768), (1000, 240)):
        tab, ky, kx = OP.bicubic_tables(H, W, 224)
        assert (ky, kx) == OP.table_taps(H, W, 224)
        assert tab.numel() == 4 * 224 + 224 * (ky + kx)

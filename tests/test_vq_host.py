"""VQ first-stage decode without a GPU: the state-dict parse, the plan the quantizing decoder compiles to, and that plan run on the CPU
plan interpreter against the float64 restatement (tests/vq_ref.py) over the decoder oracle."""
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
from diff_sampler_b200 import vae_plan
from oracle import plan_interp as PI
from oracle import vae_oracle as VO
import vq_ref as VQ


def _compile(name, B, R, **kw):
    P, cfg = VQ.make_params(name)
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    return P, cfg, mods, meta, wb, vae_plan.compile_vae_plan(mods, meta, wb, B, R, **kw)


def test_vq_f4_structure():
    """The VQ-f4 first stage of lsun_bedroom_ldm / ffhq_ldm: three levels of 128/256/512 channels, the mid attention over 512 channels,
    3 latent channels, 8192 codes, x4 upsampling."""
    P, cfg = VQ.make_params('vq_f4')
    mods, meta = vae_plan.vae_structure(P)
    omods, c_end = VO.structure(cfg)
    assert mods == omods
    assert meta == dict(z_channels=3, embed_dim=3, out_ch=3, c_end=c_end, upscale=4, n_embed=8192)
    assert ('attn', 'decoder.mid.attn_1', 512) in mods


def test_codebook_must_match_embed_dim():
    P, _ = VQ.make_params('tiny_vq')
    P['quantize.embedding.weight'] = torch.randn(16, 4)
    with pytest.raises(ValueError, match='embed_dim'):
        vae_plan.vae_structure(P)
    P, _ = VO.make_params('tiny_vae')
    mods, meta = vae_plan.vae_structure(P)
    assert 'n_embed' not in meta
    with pytest.raises(ValueError, match='codebook'):
        vae_plan.compile_vae_plan(mods, meta, vae_plan.pack_vae_weights(mods, meta, P), 1, 8, quantize=True)


def test_quantizing_plan_differs_from_the_plain_one_only_in_its_input_op():
    """Quantization is a mode of the input op: the plan with it equals the force_not_quantize plan op for op and in its arena, except
    that the first prep_input carries the codebook (and, when asked, the index buffer appended to the arena)."""
    P, cfg, mods, meta, wb, plain = _compile('tiny_vq', 2, 8)
    for dbg in (False, True):
        q = vae_plan.compile_vae_plan(mods, meta, wb, 2, 8, quantize=True, debug_indices=dbg)
        assert q.n_ops == plain.n_ops and q.meta == dict(plain.meta, quantize=True)
        assert {k: v for k, v in q.arena_offsets.items() if k != 'vq_idx'} == plain.arena_offsets
        assert ('vq_idx' in q.arena_offsets) == dbg
        k = [i for i in range(q.n_ops) if q.ops_array[i].type == S.DS_OP_PREP_INPUT]
        assert k == [1]                                            # after the statistics memset, before post_quant_conv
        for i in range(q.n_ops):
            a, b = q.ops_array[i], plain.ops_array[i]
            if i != k[0]:
                assert bytes(a) == bytes(b), i
                continue
            d, e = a.u.prep_input, b.u.prep_input
            assert not e.codebook and not e.idx and e.n_embed == 0
            assert d.codebook == wb.ref('quantize:e') and d.n_embed == 512 and d.C == 3
            assert bool(d.idx) == dbg
            d.codebook, d.idx, d.n_embed = 0, 0, 0
            assert bytes(a) == bytes(b)


def test_vq_decoder_plan_on_the_cpu_interpreter():
    """The quantizing decoder plan, run op by op on the interpreter (the input op by its float64 restatement), reproduces the oracle
    module by module, the chosen indices included, and every byte each op changes lies inside its write spans."""
    B, R = 2, 8
    P, cfg, mods, meta, wb, pl = _compile('tiny_vq', B, R, quantize=True, debug_indices=True)
    z, gap = VQ.latents_near_codes(P, cfg, B, R)
    assert gap.min().item() > VQ.MIN_GAP
    out = torch.zeros(B, meta['out_ch'], R * meta['upscale'], R * meta['upscale'])
    io = {S.DS_IO_X: z, S.DS_IO_D: out, S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0 / cfg['scale_factor'], 0.0]])}
    mem = PI.Memory(pl.arena_bytes, wb.bytes(), io)
    regions = {S.SPACE_ARENA: mem.arena, (S.SPACE_IO, S.DS_IO_D): out.reshape(-1).view(torch.uint8)}
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        before = {k: r.clone() for k, r in regions.items()}
        VQ.run_op(mem, op)
        inside = {k: torch.zeros(r.numel(), dtype=torch.bool) for k, r in regions.items()}
        for s in VQ.vq_writes(op):
            space, off = s.ref >> 60, s.ref & PI.MASK60
            key = space if space == S.SPACE_ARENA else (space, off)
            if key in inside:
                o = off if space == S.SPACE_ARENA else 0
                inside[key][o:o + s.nbytes] = True
        for k, r in regions.items():
            assert not ((r != before[k]) & ~inside[k]).any(), (i, S.UNION_FIELD[op.type], k)
    taps = {}
    with torch.no_grad():
        ref = VQ.decode(P, cfg, z, taps=taps)
        _, want_idx = VQ.quantize(P, cfg, z)
    got_idx = PI.read_buffer(mem, pl, 'vq_idx', (B, R * R), torch.int32)
    assert torch.equal(got_idx.long(), want_idx)
    for mname, t in taps.items():
        n, c, h, w = t.shape
        mine = PI.read_buffer(mem, pl, 'h:' + mname, (n, h, w, c)).permute(0, 3, 1, 2)
        assert (mine - t).abs().max().item() < 3e-5 * max(1.0, t.abs().max().item()), mname
    assert (out - ref).abs().max().item() < 3e-5


def test_force_not_quantize_plan_on_the_cpu_interpreter():
    """decode(z, force_not_quantize=True) of a VQ first stage is the plain decoder plan over z itself."""
    B, R = 1, 8
    P, cfg, mods, meta, wb, pl = _compile('tiny_vq', B, R)
    z = torch.randn(B, 3, R, R, generator=torch.Generator().manual_seed(4))
    out = torch.zeros(B, 3, R * 2, R * 2)
    PI.run_plan(pl, wb.bytes(), {S.DS_IO_X: z, S.DS_IO_D: out, S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0, 0.0]])})
    with torch.no_grad():
        ref = VQ.decode(P, cfg, z, force_not_quantize=True)
    assert (out - ref).abs().max().item() < 3e-5

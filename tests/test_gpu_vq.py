"""VQ first-stage decode on the GPU: the quantizing input kernel against a float64 brute force, and B200VAEDecoder on a VQ first stage
(VQModelInterface.decode) against the float64 restatement of tests/vq_ref.py over the decoder oracle."""
import pytest
import torch

from diff_sampler_b200 import _cstructs as S
import vq_ref as VQ

pytestmark = pytest.mark.gpu

TOL = 1e-3                       # image parity gate of tests/test_gpu_parity.py


def dev():
    return torch.device('cuda:0')


@pytest.mark.parametrize('C,n_embed,HW', [(3, 8192, 4096), (8, 1000, 4096), (5, 1, 4096), (3, 1500, 4095)])
def test_vq_prep_input_kernel(C, n_embed, HW):
    """Nearest codebook row per pixel of coef * x (randn codes and pixels, so near ties occur): the index equals the float64 argmin
    wherever the best-to-second gap exceeds vq_ref.MIN_GAP and is within it of the best elsewhere; every output pixel is exactly
    the chosen row split into fp16 hi + lo, zero past C; nothing is written past the planes or the index buffer.  1500 codes end in
    a partial shared-memory chunk; 3 x 4095 pixels leave the last block partly idle."""
    from diff_sampler_b200 import _lib
    g = torch.Generator().manual_seed(C)
    B, pad = 3, 4096
    x = torch.randn(B, C, HW, generator=g).to(dev())
    coef = torch.tensor([[0.0, 0.0, s, 0.0] for s in (1.0, 0.5, 2.0)]).to(dev())
    e = torch.randn(n_embed, C, generator=g).to(dev())
    n = B * HW * 64
    o = torch.full((2 * n + pad,), -1, dtype=torch.int16, device=dev())         # 0xFFFF: fp16 NaN
    idx = torch.full((B * HW + pad,), -1, dtype=torch.int32, device=dev())
    _lib.op_launch(S.PrepInputDesc(x=x.data_ptr(), coef=coef.data_ptr(), coef_stride=4, B=B, C=C, HW=HW, nplanes=2, out=o.data_ptr(),
                                   codebook=e.data_ptr(), idx=idx.data_ptr(), n_embed=n_embed))
    torch.cuda.synchronize()
    assert (o[2 * n:] == -1).all() and (idx[B * HW:] == -1).all()
    got = idx[:B * HW].long()
    assert ((got >= 0) & (got < n_embed)).all()
    v = (x * coef[:, 2][:, None, None]).permute(0, 2, 1).reshape(-1, C)
    best, d1, d2 = VQ.nearest(v, e)
    clear = (d2 - d1) > VQ.MIN_GAP
    mism = (got != best) & clear
    print(f'C{C} n_embed {n_embed}: {int((~clear).sum())} of {B * HW} pixels within {VQ.MIN_GAP} of a tie, {int((got != best).sum())} '
          f'differ from the float64 argmin, {int(mism.sum())} of them clear')
    assert not mism.any()
    dv = ((v.double() - e.double()[got]) ** 2).sum(1)
    assert (dv - d1).max().item() <= VQ.MIN_GAP
    planes = o[:2 * n].view(torch.float16).reshape(2, B * HW, 64)
    row = e[got]
    hi = row.half()
    lo = (row - hi.float()).half()
    assert torch.equal(planes[0, :, :C], hi) and torch.equal(planes[1, :, :C], lo)
    assert (planes[:, :, C:] == 0).all()


def _decoder(name, **kw):
    from diff_sampler_b200.vae_net import B200VAEDecoder
    P, cfg = VQ.make_params(name)
    return P, cfg, B200VAEDecoder(P, scale_factor=cfg['scale_factor'], device=dev(), **kw)


@pytest.mark.parametrize('name,B,R', [('tiny_vq', 2, 8), ('vq_f4', 1, 64)])
def test_vq_decoder_parity(name, B, R):
    """decode_first_stage of a VQ first stage through B200VAEDecoder vs the float64 reference on the GPU, on latents checked first to
    have no near-tie pixel: the chosen codebook rows exactly, per-module activations, the image.  vq_f4 is the LSUN-Bedroom / FFHQ
    VQ-f4 at full size, 64 -> 256."""
    P, cfg, vae = _decoder(name, debug_indices=True)
    z, gap = VQ.latents_near_codes(P, cfg, B, R)
    assert gap.min().item() > VQ.MIN_GAP
    taps = {}
    with torch.no_grad():
        ref = VQ.decode(P, cfg, z.to(dev()), taps=taps)
        _, want_idx = VQ.quantize(P, cfg, z.to(dev()))
    got = vae.decode(z.to(dev()))
    torch.cuda.synchronize()
    assert torch.equal(vae.debug_read(B, R, 'vq_idx', B * R * R, torch.int32).long().reshape(B, R * R), want_idx.cpu())
    for mname, t in taps.items():
        n, c, h, w = t.shape
        mine = vae.debug_read(B, R, 'h:' + mname, n * c * h * w).reshape(n, h, w, c).permute(0, 3, 1, 2)
        print(f'{mname:32s} max|ref| {t.abs().max().item():9.4f}  err {(mine.double() - t.cpu()).abs().max().item():.3e}')
    err = (got.double() - ref).abs().max().item()
    print(f'{name}: image err {err:.3e} (max|x| {ref.abs().max().item():.2f}); launches {vae.total_launches}')
    assert got.shape == ref.shape == (B, 3, R * vae.meta['upscale'], R * vae.meta['upscale']) and err < TOL


def test_vq_decoder_force_not_quantize():
    """force_not_quantize decodes z as given (ddpm.py:761-762); the default quantizes, and the two plans live side by side."""
    P, cfg, vae = _decoder('tiny_vq')
    z = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(6)).to(dev())
    with torch.no_grad():
        ref_plain = VQ.decode(P, cfg, z, force_not_quantize=True)
    got_plain = vae.decode(z, force_not_quantize=True)
    got_q = vae.decode(z)
    torch.cuda.synchronize()
    assert (got_plain.double() - ref_plain).abs().max().item() < TOL
    assert (got_q - got_plain).abs().max().item() > 10 * TOL


def test_vq_decoder_from_reference():
    """from_reference on a LatentDiffusion stand-in whose first stage holds a whole VQModelInterface state dict (encoder, quant_conv,
    the codebook, decoder) decodes exactly as the direct construction."""
    from diff_sampler_b200.vae_net import B200VAEDecoder
    P, cfg, direct = _decoder('tiny_vq')
    full = dict(P)
    full['encoder.conv_in.weight'] = torch.randn(64, 3, 3, 3)
    full['quant_conv.weight'] = torch.randn(3, 3, 1, 1)

    class FirstStage(torch.nn.Module):
        def state_dict(self, *a, **k):
            return dict(full)

    class LDM:
        first_stage_model = FirstStage()
        scale_factor = cfg['scale_factor']

    vae = B200VAEDecoder.from_reference(LDM(), device=dev())
    assert vae.is_vq and vae.meta == direct.meta
    z, _ = VQ.latents_near_codes(P, cfg, 2, 8, seed=8)
    z = z.to(dev())
    assert torch.equal(vae.decode(z), direct.decode(z))


def test_vq_decoder_plan_ops_against_the_interpreter():
    """Every op of the full-size VQ-f4 decode plan (batch 1, 64 -> 256, indices kept), launched alone on the plan's own activations
    against the float64 interpreter, as tests/test_gpu_plan_ops.py replays the benchmarked plans: each op's spans are pre-filled with
    0xFF, the interpreter (the quantizing input op by its restatement in vq_ref) runs on a snapshot, the kernel on the live arena.
    Outside its spans nothing may change; inside, every element the reference wrote must be written and within the op class's bound,
    and every element it left must keep the fill.  The chosen indices must equal the reference's exactly."""
    from diff_sampler_b200 import _lib, vae_plan
    from oracle import plan_interp as PI
    from plan_spans import reads_own_output, resolve
    from test_gpu_plan_ops import _check_span, _elements, _equal_chunked, _unwritten_bytes, _values
    P, cfg = VQ.make_params('vq_f4')
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    B, R = 1, 64
    pl = vae_plan.compile_vae_plan(mods, meta, wb, B, R, quantize=True, debug_indices=True)
    z, gap = VQ.latents_near_codes(P, cfg, B, R)
    assert gap.min().item() > VQ.MIN_GAP
    arena = torch.zeros(pl.arena_bytes, dtype=torch.uint8, device=dev())
    weights = torch.frombuffer(bytearray(wb.bytes()), dtype=torch.uint8).to(dev())
    io = {S.DS_IO_X: z.to(dev()), S.DS_IO_D: torch.zeros(B, 3, 4 * R, 4 * R, device=dev()),
          S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 1.0 / cfg['scale_factor'], 0.0]], device=dev())}

    def regions(ar, iod):
        r = {S.SPACE_ARENA: ar}
        r.update({(S.SPACE_IO, k): v.reshape(-1).view(torch.uint8) for k, v in iod.items()})
        return r

    def locate(reg, span):
        space, off = span.ref >> 60, span.ref & PI.MASK60
        if space == S.SPACE_ARENA:
            return reg[S.SPACE_ARENA][off:off + span.nbytes]
        return reg[(space, off)][:span.nbytes]

    live = regions(arena, io)
    bad, types = [], set()
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        types.add(S.UNION_FIELD[op.type])
        spans = VQ.vq_writes(op)
        fill = not reads_own_output(op)
        pre = [locate(live, s).clone() for s in spans]
        if fill:
            for s in spans:
                locate(live, s).fill_(255)
        snap_arena, snap_io = arena.clone(), {k: v.clone() for k, v in io.items()}
        ref = PI.Memory(0, None, snap_io, device=dev(), arena=snap_arena, weights=weights)
        ref.stored = []
        VQ.run_op(ref, op)
        _lib.op_launch(resolve(op, arena, weights, io))
        torch.cuda.synchronize()
        snap = regions(snap_arena, snap_io)
        got = [locate(live, s).clone() for s in spans]
        want = [locate(snap, s) for s in spans]
        for s, w in zip(spans, want):
            locate(live, s).copy_(w)
        for key in live:
            at = _equal_chunked(live[key], snap[key])
            assert at is None, f'op {i} ({S.UNION_FIELD[op.type]}): store outside its spans, {key} byte {at}'
        worst = 0.0
        for k, s in enumerate(spans):
            if s.fmt == 'i32':                                     # the chosen indices: all written, exactly the reference's
                if not torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)):
                    bad.append(f'op {i}: indices differ from the reference')
                continue
            pat_g, _ = _elements(s, got[k])
            pat_w, _ = _elements(s, want[k])
            written = ~pat_w if fill else torch.ones_like(pat_w)
            if fill and ((pat_w & ~pat_g).any() or (~pat_w & pat_g).any()):
                bad.append(f'op {i} span {k}: written elements differ from the reference\'s')
            if s.fmt != 'zero':
                vals = _values(s, got[k])
                if not torch.isfinite(vals[written[:vals.numel()]]).all():
                    bad.append(f'op {i} span {k}: non-finite value where the reference wrote one')
            worst = max(worst, _check_span(op, s, got[k], want[k], written, ref.stored, spans, got, want)[2])
        if worst > 1.0:
            bad.append(f'op {i} ({S.UNION_FIELD[op.type]} tag {op.tag}): error / bound {worst:.3f}')
        for s, p, g in zip(spans, pre, got):
            dst = locate(live, s)
            dst.copy_(torch.where(_unwritten_bytes(s, g), p, g) if fill and s.fmt != 'i32' else g)
        del snap_arena, snap_io, ref, snap, got, want, pre
    print(f'vq_f4 decode plan: {pl.n_ops} ops, types {sorted(types)}')
    assert 'prep_input' in types and not bad, '\n'.join(bad[:20])

"""The 64-wide and paired-head fused attention kernels (attn_kernel, attn_pair_kernel) and the unfused path (QK^T GEMM -> row softmax
-> P.V GEMM) against float64, at every key count, query count, layout and logit pattern they accept.

Every operand is fp16 hi + lo planes; the references are computed in float64 from the values those planes hold.  Every byte a
kernel promises not to touch is NaN: the Q / K channels outside the heads' window of each row, the V^T columns Lk .. vt_pitch, the
output channels outside the heads and a guard before and after each buffer.  After a launch the inputs must be bit for bit
unchanged, the outputs finite inside their window and still NaN outside it.

ATTN_CASES and SOFTMAX_CASES are plain constants: tests/test_attention_shapes.py checks without a GPU that every attention and
softmax the compiled plans launch falls into a class these lists run."""
import collections

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
GUARD = 4096                                    # fp16 / fp32 elements of NaN before and after every buffer

# ------------------------------------------------------------------------------------------ the fused kernels' case list
# kind -> (head width, pad0 of the descriptor, channels per head slot).  d40 is SD-1.5's 40-wide head zero-padded to 64.
KINDS = {'d64': (64, 0, 64), 'd40': (40, 0, 64), 'pair': (32, 32, 32)}
ATTN_LKS = [1, 2, 63, 64, 65, 77, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 4096, 4097]
ATTN_LS = [1, 9, 77, 127, 128, 129, 257, 1024, 4096]
CROSS_LKS = [77, 1, 129, 1025, 64, 257, 65]
CAUSAL_LS = [1, 9, 77, 128, 129, 1024, 1025]
PAIR_COUNTS = [1, 7, 14]                        # head pairs: the unconditional LDMs' 14 / 21 / 28 heads are padded to even counts
LOGIT_SHAPES = [(129, 129, 'qk'), (77, 1025, 'sep'), (1024, 4097, 'sep'), (255, 255, 'qk'), (9, 257, 'sep')]
LOGITS = ['late40', 'late200', 'deep', 'equal']


def _heads(kind, i, Lk):
    """Head count of case i: 2 heads of 64 / 40, or 1, 7, 14 head pairs in turn (1 pair from 4096 keys on)."""
    if kind != 'pair':
        return 2
    return 2 * (1 if Lk >= 4096 else PAIR_COUNTS[i % len(PAIR_COUNTS)])


def _attn_cases():
    """(kind, nh, B, L, Lk, layout, causal, logits): the sweep this module runs and test_attention_shapes.py checks the plans against."""
    cases = []
    for kind in KINDS:
        for i, Lk in enumerate(ATTN_LKS):                                  # key counts: self-attention from one [q | k] buffer
            cases.append((kind, _heads(kind, i, Lk), 1 if Lk >= 4096 else 2, Lk, Lk, 'qk', 0, 'randn'))
        for i, L in enumerate(ATTN_LS):                                    # query counts: cross-attention from separate buffers
            for j in range(2):
                Lk = CROSS_LKS[(2 * i + j) % len(CROSS_LKS)]
                cases.append((kind, _heads(kind, i + j, Lk), 1 if L >= 4096 else 3, L, Lk, 'sep', 0, 'randn'))
        for i, L in enumerate(CAUSAL_LS):                                  # causal self-attention, both layouts
            cases.append((kind, _heads(kind, i, L), 2, L, L, 'qk' if i % 2 == 0 else 'sep', 1, 'randn'))
        for i, (L, Lk, layout) in enumerate(LOGIT_SHAPES):                  # logit patterns (_operands)
            for logits in LOGITS:
                cases.append((kind, _heads(kind, i, Lk), 1 if Lk >= 4096 else 2, L, Lk, layout, 0, logits))
    # cross-attention with whole query tiles and key blocks
    cases += [('d40', 2, 2, 1024, 64, 'sep', 0, 'randn'), ('pair', 14, 2, 128, 256, 'sep', 0, 'randn')]
    # more than 3000 CTAs: 32 x 12 heads x 8 query tiles (attn_kernel), 32 x 14 pairs x 8 tiles (pair kernel); 2 CTAs for 132 SMs
    cases += [('d64', 12, 32, 1024, 65, 'sep', 0, 'randn'), ('pair', 28, 32, 1024, 1024, 'qk', 0, 'randn'),
              ('d40', 2, 1, 128, 128, 'qk', 0, 'randn'), ('pair', 2, 1, 128, 77, 'sep', 0, 'randn')]
    return cases


ATTN_CASES = _attn_cases()


def attn_class(kernel, hd, self_attn, causal, L, Lk):
    """The class an attention belongs to for the shape inventory: kernel, head width, self / cross, causal, whether the last
    query tile (128 rows) and the last key block (64 keys) are whole."""
    return (kernel, hd, bool(self_attn), bool(causal), 'whole' if L % 128 == 0 else 'part', 'whole' if Lk % 64 == 0 else 'part')


def case_class(case):
    kind, nh, B, L, Lk, layout, causal, logits = case
    hd, pad0, slot = KINDS[kind]
    return attn_class('pair' if pad0 == 32 else 'attn', slot, layout == 'qk', causal, L, Lk)


# ------------------------------------------------------------------------------------------ the softmax launcher's case list
SOFTMAX_LS = [4, 76, 77, 80, 252, 256, 260, 1020, 1024, 1028, 4092, 4096, 4100, 8188, 8192, 8196, 9216, 16384]
# (pitch_in, pitch_out) as gaps past L: None = 0 in the descriptor (rows of L), 0 = pitch L written out; (3, 51) is the SD-1.5
# cross-attention's 77 keys in score rows of 80 and probability rows of 128
SOFTMAX_PITCHES = [(None, None), (0, 0), (None, 4), (4, None), (4, 4), (3, 51)]
SOFTMAX_CASES = [(L, gi, go) for L in SOFTMAX_LS for gi, go in SOFTMAX_PITCHES]


def softmax_kernel(L, pitch_in, pitch_out):
    """The kernel ds_softmax_launch (csrc/elementwise.cu) picks for a row length and the descriptor's pitches (0 = L)."""
    dense = pitch_in in (0, L) and pitch_out in (0, L) and L % 4 == 0
    if dense and L <= 1024:
        return 'reg2' if L <= 256 else 'reg8'
    if dense and L <= 8192:
        return 'cta4' if L <= 4096 else 'cta8'
    pin, pout = pitch_in or L, pitch_out or L
    return 'warp_f4' if L % 4 == 0 and pin % 4 == 0 and pout % 4 == 0 else 'warp_scalar'


def softmax_class(L, pitch_in, pitch_out):
    """Kernel and the pitch gaps (elements past L; 0 for a pitch of 0 or L)."""
    return (softmax_kernel(L, pitch_in, pitch_out), (pitch_in or L) - L, (pitch_out or L) - L)


def _pitch(L, gap):
    return 0 if gap is None else L + gap


def softmax_case_class(case):
    L, gi, go = case
    return softmax_class(L, _pitch(L, gi), _pitch(L, go))


# ------------------------------------------------------------------------------------------ helpers
RATIOS = collections.defaultdict(dict)          # (kernel, layout or causal) -> Lk -> worst error / bound


def _split(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def _guarded(n, dtype=torch.float16):
    buf = torch.full((2 * GUARD + n,), float('nan'), dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + n]


class _Inputs:
    """Places fp32 operands as fp16 planes in guarded NaN buffers and remembers them, to check afterwards that none changed."""

    def __init__(self):
        self.bufs = []

    def planes(self, x):
        hi, lo = _split(x)
        buf, inner = _guarded(2 * x.numel())
        inner.view(2, -1).copy_(torch.stack([hi, lo]).reshape(2, -1))
        self.bufs.append((buf, buf.clone()))
        return inner, (hi.double() + lo.double())

    def unchanged(self):
        for buf, before in self.bufs:
            assert torch.equal(buf.view(torch.int16), before.view(torch.int16)), 'an input buffer changed'


def _operands(kind, nh, B, L, Lk, logits, v_mean, g):
    """q [B][L][nh][d], k, v [B][Lk][nh][d] (fp32 on the device) for a logit pattern:
    randn    q, k, v standard normal;
    late40 / late200   channel 0 of every head carries a bias: q = 1 there and the last key's k = (G + 10) / scale, so every row's
             maximum is the last key, at least G above all others, and arrives in the last key block;
    deep     the same bias channel puts keys 0 .. 63 110 below the rest: more than 126 log2 units under the row maximum;
    equal    all keys equal: each row's logits are one value, its weights uniform."""
    hd = KINDS[kind][0]
    scale = hd ** -0.5
    q = torch.randn(B, L, nh, hd, generator=g, device=DEV)
    k = torch.randn(B, Lk, nh, hd, generator=g, device=DEV)
    v = torch.randn(B, Lk, nh, hd, generator=g, device=DEV) + v_mean
    if logits in ('late40', 'late200', 'deep'):
        q[..., 0] = 1.0                                                    # exact in fp16: the bias products carry no rounding
        k[..., 0] = 0.0
        if logits == 'deep':
            k[:, :64, :, 0] = -110.0 / scale
        else:
            k[:, Lk - 1, :, 0] = (int(logits[4:]) + 10) / scale
    elif logits == 'equal':
        k[:] = k[:, :1]
    return q, k, v, scale


def _fused_case(case):
    """Launch one ATTN_CASES entry and compare with float64.  Returns error / bound, bound = 2e-5 max(1, max |O|).  From 4096 keys
    on the values have mean 1, so that O sums up a large total over the whole key range.
    layout 'qk': the plan's [q | k] rows (L == Lk, q_pitch = k_pitch = 2 C, k_c0 = C, vt_pitch = Lk rounded up to 8, o_pitch = C);
    'sep': Q and K in buffers of their own with q_c0 = 16, k_c0 = 40, pitches C + 40 and C + 48, 8 more V^T columns, o_pitch C + 16."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    kind, nh, B, L, Lk, layout, causal, logits = case
    hd, pad0, slot = KINDS[kind]
    g = torch.Generator(device=DEV).manual_seed(7 * L + Lk)
    q, k, v, scale = _operands(kind, nh, B, L, Lk, logits, 1.0 if Lk >= 4096 else 0.0, g)
    C = nh * slot
    if layout == 'qk':
        assert L == Lk
        q_c0, k_c0, qp, kp, vp, op = 0, C, 2 * C, 2 * C, -(-Lk // 8) * 8, C
    else:
        q_c0, k_c0, qp, kp, vp, op = 16, 40, C + 40, C + 48, -(-Lk // 8) * 8 + 8, C + 16

    def heads(x):                                                          # [B][rows][nh][hd] -> [B][rows][C]: slots, zero padded
        t = torch.zeros(*x.shape[:2], nh, slot, device=DEV)
        t[..., :hd] = x
        return t.reshape(*x.shape[:2], C)

    def operand(rows, pitch, c0, x):                                       # fp32 [B][rows][pitch], NaN outside the heads
        t = torch.full((B, rows, pitch), float('nan'), device=DEV)
        t[:, :, c0:c0 + C] = heads(x)
        return t
    qf = operand(L, qp, q_c0, q)
    kf = operand(Lk, kp, k_c0, k)
    if layout == 'qk':
        qf[:, :, k_c0:k_c0 + C] = kf[:, :, k_c0:k_c0 + C]
    vf = torch.full((B, C, vp), float('nan'), device=DEV)
    vf[:, :, :Lk] = heads(v).transpose(1, 2)
    inp = _Inputs()
    qd, q64 = inp.planes(qf)
    kd, k64 = (qd, q64) if layout == 'qk' else inp.planes(kf)
    vd, v64 = inp.planes(vf)
    obuf, od = _guarded(2 * B * L * op)
    _lib.op_launch(S.AttnDesc(q=qd.data_ptr(), k=kd.data_ptr(), vt=vd.data_ptr(), out=od.data_ptr(), B=B, nh=nh, L=L, Lk=Lk,
                              q_pitch=qp, q_c0=q_c0, k_pitch=kp, k_c0=k_c0, vt_pitch=vp, o_pitch=op, nplanes=2, scale=scale,
                              causal=causal, pad0=pad0))
    torch.cuda.synchronize()
    inp.unchanged()
    out = od.view(2, B, L, op)
    assert torch.isfinite(out[..., :C]).all(), 'non-finite output: a NaN sentinel was read, or a row was left unwritten'
    assert torch.isnan(out[..., C:]).all() and torch.isnan(obuf[:GUARD]).all() and torch.isnan(obuf[GUARD + od.numel():]).all(), \
        'a store outside the output window'
    got = (out[0].double() + out[1].double())[..., :C].reshape(B, L, nh, slot).transpose(1, 2)
    if hd < slot:
        assert (got[..., hd:] == 0).all(), 'padded head channels are not exactly 0'
    qs = q64[:, :, q_c0:q_c0 + C].reshape(B, L, nh, slot)[..., :hd].transpose(1, 2)
    ks = k64[:, :, k_c0:k_c0 + C].reshape(B, Lk, nh, slot)[..., :hd].transpose(1, 2)
    vs = v64[:, :, :Lk].reshape(B, nh, slot, Lk)[:, :, :hd].transpose(2, 3)
    s = scale * qs @ ks.transpose(2, 3)
    if causal:
        s = s + torch.full((L, Lk), float('-inf'), dtype=torch.float64, device=DEV).triu(1)
    if logits.startswith('late'):                                          # the construction did what it claims
        top = s.topk(min(2, Lk), dim=3)
        assert (top.indices[..., 0] == Lk - 1).all()
        assert Lk == 1 or (top.values[..., 0] - top.values[..., 1]).min() > int(logits[4:])
    if logits == 'deep' and Lk > 64:
        assert (s.amax(dim=3) - s[..., :64].amax(dim=3)).min() * 1.4426950408889634 > 126
    want = torch.softmax(s, dim=3) @ vs
    err = (got[..., :hd] - want).abs().max().item()
    ratio = err / (2e-5 * max(1.0, want.abs().max().item()))
    key = ('pair' if pad0 == 32 else f'attn d{hd}', 'causal' if causal else layout)
    RATIOS[key][Lk] = max(RATIOS[key].get(Lk, 0.0), ratio)
    print(f'{kind:4s} nh {nh:2d} B {B:2d} L {L:4d} Lk {Lk:4d} {layout:3s}{" causal" if causal else ""} {logits:7s}: '
          f'err {err:.2e}, {ratio:.3f} of the bound')
    return ratio


def _case_id(c):
    kind, nh, B, L, Lk, layout, causal, logits = c
    return f'{kind}-nh{nh}-B{B}-L{L}-Lk{Lk}-{layout}{"-causal" if causal else ""}-{logits}'


@pytest.mark.parametrize('case', ATTN_CASES, ids=[_case_id(c) for c in ATTN_CASES])
def test_fused_attention_against_float64(case):
    assert _fused_case(case) < 1.0


# ------------------------------------------------------------------------------------------ ds_softmax_launch
def _softmax_rows(pattern, rows, L, g):
    if pattern == 'spread80':
        return torch.rand(rows, L, generator=g, device=DEV) * 160 - 80
    if pattern == 'randn3':
        return torch.randn(rows, L, generator=g, device=DEV) * 3
    return torch.randn(rows, 1, generator=g, device=DEV).expand(rows, L).contiguous()      # all-equal rows: uniform weights


@pytest.mark.parametrize('L,gi,go', SOFTMAX_CASES, ids=[f'L{L}-in{gi}-out{go}' for L, gi, go in SOFTMAX_CASES])
def test_softmax_launcher_against_float64(L, gi, go):
    """Each of ds_softmax_launch's six kernels on both sides of every dispatch edge.  Logits spread over +-80, normal with
    standard deviation 3, and all-equal rows; 1, 7, 37 and 4099 rows; one and two output planes.  hi + lo within 2e-6 of float64
    softmax, and the hi plane on its own within half an fp16 ulp (+ 2e-6) of it: the fp16 rounding of the float64 value.
    Score and probability pitch gaps, the unwritten lo plane and the guards stay NaN."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    pin, pout = _pitch(L, gi), _pitch(L, go)
    kern = softmax_kernel(L, pin, pout)
    g = torch.Generator(device=DEV).manual_seed(L + 10 * (gi or 0) + (go or 0))
    runs = [(37, p, n) for p in ('spread80', 'randn3', 'equal') for n in (1, 2)] + [(1, 'spread80', 2), (7, 'randn3', 2),
                                                                                   (4099, 'spread80', 2)]
    worst_hi = worst_sum = 0.0
    for rows, pattern, npl in runs:
        si, so = pin or L, pout or L
        x = _softmax_rows(pattern, rows, L, g)
        sbuf, sd = _guarded(rows * si, torch.float32)
        sd.view(rows, si)[:, :L] = x
        before = sbuf.clone()
        pbuf, pd = _guarded(2 * rows * so)
        _lib.op_launch(S.SoftmaxDesc(S=sd.data_ptr(), P=pd.data_ptr(), rows=rows, L=L, nplanes=npl, pitch_in=pin, pitch_out=pout))
        torch.cuda.synchronize()
        assert torch.equal(sbuf.view(torch.int32), before.view(torch.int32)), 'the scores changed'
        P = pd.view(2, rows, so)
        assert torch.isnan(pbuf[:GUARD]).all() and torch.isnan(pbuf[GUARD + pd.numel():]).all(), 'a store outside P'
        assert torch.isnan(P[:, :, L:]).all(), 'a store into the probability rows\' pitch gap'
        if npl == 1:
            assert torch.isnan(P[1]).all(), 'a store into the lo plane of a one-plane softmax'
        hi = P[0, :, :L]
        assert torch.isfinite(hi).all(), 'an unwritten probability'
        ref = torch.softmax(x.double(), dim=1)
        ulp = torch.finfo(torch.float16).eps * torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))))
        r_hi = ((hi.double() - ref).abs() / (0.5 * ulp + 2e-6)).max().item()
        r_sum = 0.0
        if npl == 2:
            lo = P[1, :, :L]
            assert torch.isfinite(lo).all()
            r_sum = ((hi.double() + lo.double()) - ref).abs().max().item() / 2e-6
        worst_hi, worst_sum = max(worst_hi, r_hi), max(worst_sum, r_sum)
        assert r_hi <= 1 and r_sum <= 1, (rows, pattern, npl, r_hi, r_sum)
    print(f'softmax {kern:11s} L {L:5d} pitch_in {pin:5d} pitch_out {pout:5d}: hi + lo {worst_sum:.3f} of 2e-6, '
          f'hi {worst_hi:.3f} of half an fp16 ulp + 2e-6')


# ------------------------------------------------------------------------------------------ the unfused path, as the plans emit it
def _sd_tokens_pitch():
    from diff_sampler_b200 import ldm_plan
    return ldm_plan.CTX_TOKENS_PITCH


# (name, B, nh, d, L, Lk, vt_pitch, s_pitch); vt_pitch None = the plan's 77-token pitch (ldm_plan.CTX_TOKENS_PITCH: the P.V GEMM's K
# runs over vt_pitch, a multiple of 64)
UNFUSED_SHAPES = [('vae', 1, 1, 512, 1024, 1024, 1024, None), ('vae', 2, 1, 512, 1024, 1024, 1024, None),
                  ('vae', 1, 1, 512, 4096, 4096, 4096, None), ('vae', 2, 1, 512, 4096, 4096, 4096, None),
                  ('sd_cross', 2, 8, 64, 1024, 77, None, 80),
                  ('sd_cross', 2, 8, 128, 1024, 77, None, 80), ('sd_cross', 2, 8, 192, 256, 77, None, 80),
                  ('sd_self', 2, 8, 192, 256, 256, 256, None), ('edm', 3, 4, 64, 256, 256, 256, None), ('edm', 3, 2, 64, 64, 64, 64, None)]


@pytest.mark.parametrize('name,B,nh,d,L,Lk,vt_pitch,s_pitch', UNFUSED_SHAPES, ids=[f'{s[0]}-B{s[1]}-nh{s[2]}-d{s[3]}-L{s[4]}-Lk{s[5]}-vt{s[6]}'
                                                                                   for s in UNFUSED_SHAPES])
def test_unfused_attention_chain(name, B, nh, d, L, Lk, vt_pitch, s_pitch):
    """The three ops PlanBuilder.attention(fused=False, ...) emits -- QK^T into S, the row softmax into P, P.V into O -- with the
    descriptors it builds, launched one after the other on NaN-initialised buffers.  S and P keep their pitch gaps NaN (the
    softmax never writes P's columns Lk .. vt_pitch, and the P.V product must not read them); V^T's columns past Lk are NaN too.
    Each stage against float64 on the previous stage's output, and O end to end against float64 attention."""
    from diff_sampler_b200 import _lib
    from diff_sampler_b200 import plan as planner
    vt_pitch = vt_pitch or _sd_tokens_pitch()
    C = nh * d
    self_attn = L == Lk and name != 'sd_cross'
    pb = planner.PlanBuilder(planner.WeightBlob(), B)
    q, k = ('qk', 'qk') if self_attn else ('q2', 'k2')
    qp = 2 * C if self_attn else C
    pb.need(q, 2 * B * L * qp * 2)
    if not self_attn:
        pb.need(k, 2 * B * Lk * C * 2)
    pb.need('vt', 2 * B * C * vt_pitch * 2)
    pb.need('o', 2 * B * L * C * 2)
    pb.attention(False, q, k, 'o', nh, L, Lk, d, d ** -0.5, vt_pitch, s_pitch=s_pitch)
    assert len(pb.ops) == 3
    g = torch.Generator(device=DEV).manual_seed(L + Lk + d + B)
    inp = _Inputs()
    if self_attn:
        qk = torch.randn(B, L, 2 * C, generator=g, device=DEV)
        qd, q64 = inp.planes(qk)
        q64, k64 = q64[..., :C], q64[..., C:]
        kd = qd
    else:
        qd, q64 = inp.planes(torch.randn(B, L, C, generator=g, device=DEV))
        kd, k64 = inp.planes(torch.randn(B, Lk, C, generator=g, device=DEV))
    vt = torch.full((B, C, vt_pitch), float('nan'), device=DEV)
    vt[:, :, :Lk] = torch.randn(B, C, Lk, generator=g, device=DEV) + 0.5
    vd, v64 = inp.planes(vt)
    sp = s_pitch or Lk
    sbuf, Sd = _guarded(pb.sizes['S'] // 4, torch.float32)
    pbuf, Pd = _guarded(pb.sizes['P'] // 2)
    obuf, Od = _guarded(2 * B * L * C)
    ptr = {q: qd, k: kd, 'vt': vd, 'S': Sd, 'P': Pd, 'o': Od}

    def R(nm, extra=0):
        return ptr[nm].data_ptr() + int(extra)
    descs = [build(R) for _, build in pb.ops]
    for dsc in descs:
        _lib.op_launch(dsc)
    torch.cuda.synchronize()
    inp.unchanged()
    scale = d ** -0.5
    qh = q64.reshape(B, L, nh, d).transpose(1, 2)
    kh = k64.reshape(B, Lk, nh, d).transpose(1, 2)
    vh = v64[:, :, :Lk].reshape(B, nh, d, Lk).transpose(2, 3)
    Sm = Sd[:B * nh * L * sp].view(B, nh, L, sp)
    assert torch.isnan(Sm[..., Lk:]).all() and torch.isnan(sbuf[:GUARD]).all() and torch.isnan(sbuf[GUARD + Sd.numel():]).all()
    s_ref = scale * qh @ kh.transpose(2, 3)
    e_s = (Sm[..., :Lk].double() - s_ref).abs().max().item() / (3e-5 * s_ref.abs().max().item())
    pw = Pd[:2 * B * nh * L * vt_pitch].view(2, B, nh, L, vt_pitch)
    assert torch.isnan(pw[..., Lk:]).all() and torch.isnan(pbuf[:GUARD]).all() and torch.isnan(pbuf[GUARD + Pd.numel():]).all()
    p_got = pw[0, ..., :Lk].double() + pw[1, ..., :Lk].double()
    e_p = (p_got - torch.softmax(Sm[..., :Lk].double(), dim=3)).abs().max().item() / 2e-6
    O = Od.view(2, B, L, C)
    assert torch.isfinite(O).all() and torch.isnan(obuf[:GUARD]).all() and torch.isnan(obuf[GUARD + Od.numel():]).all()
    o_got = (O[0].double() + O[1].double()).reshape(B, L, nh, d).transpose(1, 2)
    o_stage = p_got @ vh
    e_o = (o_got - o_stage).abs().max().item() / (3e-5 * max(1.0, o_stage.abs().max().item()))
    want = torch.softmax(s_ref, dim=3) @ vh
    e_all = (o_got - want).abs().max().item() / (2e-5 * max(1.0, want.abs().max().item()))
    RATIOS[('unfused', name)][Lk] = max(RATIOS[('unfused', name)].get(Lk, 0.0), e_all)
    print(f'unfused {name:8s} B {B} nh {nh} d {d:3d} L {L:4d} Lk {Lk:4d} s_pitch {sp:4d} vt_pitch {vt_pitch:4d}: of the bounds '
          f'S {e_s:.3f}, P {e_p:.3f}, O {e_o:.3f}, end to end {e_all:.3f}')
    assert e_s < 1 and e_p < 1 and e_o < 1 and e_all < 1


def test_attention_error_table():
    """Worst error / bound per kernel and key count over the cases above that ran."""
    if not RATIOS:
        pytest.skip('no attention case of this module ran')
    lks = sorted({lk for r in RATIOS.values() for lk in r})
    print('\nworst error / bound by key count')
    print(f"{'kernel':22s} " + ' '.join(f'{lk:>6d}' for lk in lks))
    for key in sorted(RATIOS):
        r = RATIOS[key]
        print(f"{' '.join(key):22s} " + ' '.join(f'{r[lk]:6.3f}' if lk in r else f"{'-':>6s}" for lk in lks))

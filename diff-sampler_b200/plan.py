"""Plan compiler: lowers one EDM denoiser (NetSpec + parameter dict) at one batch size into
  * a packed weight blob (fp16 hi/lo K-major GEMM operands + fp32 vectors), built once per net, and
  * a flat list of ds_plan_op records over a workspace arena, built once per (batch, sigma-mode),
which the native executor (csrc/engine.cu) runs.  Pure host logic — no GPU needed to compile a plan.

WeightBlob and PlanBuilder are shared with the other plan compilers (ldm_plan.py, vae_plan.py, clip_plan.py).

Reference forward being lowered: networks_edm.py:482-496 (EDMPrecond), :312-355 / :427-453 (U-Nets), :158-179 (UNetBlock).
"""
import math

import torch

from . import _cstructs as S
from . import gemm_desc as G

ALIGN = 1024
F4, H2 = 4, 2
NPL = 2                 # fp16 planes per activation operand (hi, lo)


def _groups(c):
    """GroupNorm group count of the reference: min(32, C // 4)  (networks_edm.py:91)."""
    return min(32, c // 4)


def _align(n, a=ALIGN):
    return (n + a - 1) // a * a


def io(slot):
    """Reference to one of the io pointers the caller passes per forward (DS_IO_*)."""
    return S.ref(S.SPACE_IO, slot)


class WeightBlob:
    def __init__(self):
        self.chunks = []
        self.off = {}
        self.size = 0

    def add(self, name, t):
        t = t.detach().contiguous().cpu()
        raw = t.numpy().tobytes() if t.dtype != torch.float16 else t.view(torch.int16).numpy().tobytes()
        o = _align(self.size)
        if o > self.size:
            self.chunks.append(b'\0' * (o - self.size))
        self.chunks.append(raw)
        self.size = o + len(raw)
        self.off[name] = o
        return o

    def add_gemm(self, key, w, skip_w=None, bias=None, f8=False):
        """Conv2d [Cout, Cin, k, k] or linear [N, K] weight (+ a 1x1 skip weight appended along K) as the packed B operand `key`:w of
        the GEMM kernel -- fp16 hi/lo planes, or the fp16 + 2 x e4m3 layout of the f8 mode -- and its bias `key`:b.
        Returns (packed weight, f8 shift or None)."""
        if w.dim() == 2:
            w = w.reshape(w.shape[0], w.shape[1], 1, 1)
        packed, shift = G.pack_conv_weight_f8(w, skip_w) if f8 else (G.pack_conv_weight(w, skip_w), None)
        self.add(key + ':w', packed)
        if bias is not None:
            self.add(key + ':b', bias)
        return packed, shift

    def add_norm(self, key, P, src=None):
        """Norm gain and bias `key`:g / `key`:b from the parameters `src`.weight / `src`.bias (src defaults to key; P: name -> tensor)."""
        src = src or key
        self.add(key + ':g', P(src + '.weight'))
        self.add(key + ':b', P(src + '.bias'))

    def ref(self, name, extra=0):
        return S.ref(S.SPACE_WEIGHTS, self.off[name] + extra)

    def bytes(self):
        return b''.join(self.chunks)


def _resolve(R, x):
    """Arena name, (arena name, byte offset), an already resolved reference (io / weights), or None (-> 0)."""
    if x is None:
        return 0
    if isinstance(x, str):
        return R(x)
    if isinstance(x, tuple):
        return R(*x)
    return x


class Plan:
    def __init__(self, ops_array, n_ops, arena_bytes, arena_offsets, meta):
        self.ops_array = ops_array
        self.n_ops = n_ops
        self.arena_bytes = arena_bytes
        self.arena_offsets = arena_offsets
        self.meta = meta


class PlanBuilder:
    """Collects one plan over the weight blob `wb` for a batch of B samples.

    Arena: named buffers, laid out in the order each name is first needed; a name needed again (scratch shared between layers) is
    sized to the largest request.  Ops: callables build(R) -> descriptor, materialised by finish() once the arena is laid out;
    R(name, extra=0) is the arena reference.  Each op is stamped with the current `tag` (None: with its own index)."""

    def __init__(self, wb, B, npass=3, tag=0):
        self.wb, self.B, self.npass, self.tag = wb, B, npass, tag
        self.sizes = {}
        self.ops = []
        self._slots = self._n_slots = 0

    def need(self, name, nbytes):
        self.sizes[name] = max(self.sizes.get(name, 0), int(nbytes))
        return name

    def emit(self, build):
        self.ops.append((len(self.ops) if self.tag is None else self.tag, build))

    def finish(self, **meta):
        offsets, total = {}, 0
        for name, nbytes in self.sizes.items():
            offsets[name] = total
            total += _align(nbytes)

        def R(name, extra=0):
            return S.ref(S.SPACE_ARENA, offsets[name] + int(extra))
        arr = (S.PlanOp * len(self.ops))()
        for op, (tag, build) in zip(arr, self.ops):
            desc = build(R)
            op.type = S.OP_TYPE_OF[type(desc)]
            op.tag = tag
            setattr(op.u, S.ALL_UNION_FIELD[op.type], desc)
        meta.update(n_ops=len(self.ops), n_gemm=sum(1 for op in arr if op.type == S.DS_OP_GEMM))
        return Plan(arr, len(self.ops), total, offsets, meta)

    # ---- GroupNorm ------------------------------------------------------------------------------------------------------------
    def stats(self, n_slots):
        """The 'stats' buffer: fp64 {sum, sumsq} per (sample, group) for up to n_slots GroupNorms, zeroed by a memset op."""
        nbytes = n_slots * self.B * 32 * 2 * 8
        self.need('stats', nbytes)
        self.emit(lambda R: S.MemsetDesc(ptr=R('stats'), bytes=nbytes))
        self._n_slots = n_slots

    def stats_slot(self):
        """Byte offset of the next GroupNorm's sums in 'stats'."""
        assert self._slots < self._n_slots
        self._slots += 1
        return (self._slots - 1) * self.B * 32 * 2 * 8

    def gn_stats(self, slot, parts, hw, groups=32):
        """Accumulate the fp64 sums of the (virtually concatenated) fp32 NHWC tensors `parts` = [(arena name, channels), ...]."""
        (n0, c0), (n1, c1) = parts[0], (parts[1] if len(parts) > 1 else (None, 0))
        self.emit(lambda R: S.GnStatsDesc(src0=R(n0), src1=_resolve(R, n1), C0=c0, C1=c1, HW=hw, B=self.B, groups=groups,
                                          sums=R('stats', slot)))

    def gn_apply(self, parts, H, norm, eps, out, *, W=None, B=None, groups=32, slot=None, coef=False, silu=1, ada=None, ada_stride=0,
                 resample=0, raw=None, raw_f32=None, fmt=0, phase_pitch=0):
        """GroupNorm of `parts` (as gn_stats; an input may also be an io reference) with the gain / bias `norm`:g / `norm`:b (+ SiLU)
        into the activation operand `out`: fp16 planes, or the f8 operand image (fmt=1).  The statistics are the sums of stats slot
        `slot`, or the coefficient table 'gncoef' (coef=True).  raw / raw_f32 also receive the input un-normalised (fp16 planes /
        fp32); resample 1 / 2 / 3 = 2x2 average pooling / nearest x2 / space-to-depth (phase_pitch: channels per phase, 0 = C).
        norm=None: no normalisation."""
        (n0, c0), (n1, c1) = parts[0], (parts[1] if len(parts) > 1 else (None, 0))
        assert norm is None or (c0 + c1) % groups == 0
        Wt = self.wb.ref
        self.emit(lambda R: S.GnApplyDesc(
            src0=_resolve(R, n0), src1=_resolve(R, n1), C0=c0, C1=c1, H=H, W=W or H, B=B or self.B, groups=groups,
            sums=R('stats', slot) if slot is not None and not coef else 0, coef=R('gncoef') if coef else 0,
            gamma=Wt(norm + ':g') if norm else 0, beta=Wt(norm + ':b') if norm else 0, eps=eps, silu=silu,
            ada=_resolve(R, ada), ada_stride=ada_stride, resample=resample, nplanes=NPL, out_act=_resolve(R, out),
            out_raw=_resolve(R, raw), out_raw_f32=_resolve(R, raw_f32), fmt=fmt, pad0=phase_pitch))

    def group_norm(self, parts, H, norm, eps, out, **apply_kw):
        """GroupNorm from sums: a statistics pass into a fresh stats slot, then gn_apply."""
        slot = self.stats_slot()
        self.gn_stats(slot, parts, H * H)
        self.gn_apply(parts, H, norm, eps, out, slot=slot, **apply_kw)

    def to_planes(self, src, C, H, W, B, dst, fmt=0, resample=0, groups=32, phase_pitch=0):
        """fp32 NHWC -> the fp16 hi/lo planes (or, fmt=1, the f8 operand image) of a GEMM operand, without normalisation."""
        self.gn_apply([(src, C)], H, None, 0.0, None, W=W, B=B, groups=groups, silu=0, resample=resample, raw=dst, fmt=fmt,
                      phase_pitch=phase_pitch)

    # ---- attention --------------------------------------------------------------------------------------------------------------
    def vt_gemm(self, w, src, C, N, L, pitch, bias=None):
        """V^T[b][n][key] = sum_c Wv[n][c] src[b][key][c] (+ bias[n]) into 'vt' (rows of `pitch` keys), the layout the P.V product
        reads: the weight's fp16 planes `w` [2][N][C] are the M operand, the B batch entries' L rows of `src` the N operand.  C % 64 != 0:
        the K loop runs to C rounded up to 64, both operands' last block zero-filled by TMA."""
        W = self.wb.ref
        K = -(-C // 64) * 64
        self.emit(lambda R: G.rows_gemm(W(w), N, C, 1, R(src), L, C, self.B, K, num_z=self.B, nh=1, m_valid=N, n_valid=L,
                                        npass=self.npass, b_z_per_zb=1, out_h16=R('vt'), o_zb=N * pitch, ldo=pitch,
                                        o_plane=self.B * N * pitch, bias_m=W(bias) if bias else 0)[0])

    def attention(self, fused, q, k, out, nh, L, Lk, d, scale, vt_pitch, causal=0, s_pitch=None, pairs=False):
        """softmax(scale Q K^T) V for nh heads of width d over the B batch entries: L queries, Lk keys, V^T in 'vt' (rows of vt_pitch
        keys), O into the fp16 planes `out` [B][L][nh d].  q == k: one [q heads | k heads] buffer of pitch 2 nh d, else two of nh d.
        fused: the fused kernel (csrc/attention.cu, 64-wide heads, or pairs=True: 32-wide heads two per CTA, nh even); otherwise QK^T into 'S' (rows of s_pitch, default Lk), the row
        softmax into 'P' (rows of vt_pitch) and the P.V GEMM."""
        B, C = self.B, nh * d
        qp, kc0 = (2 * C, C) if q == k else (C, 0)
        if fused:
            self.emit(lambda R: S.AttnDesc(q=R(q), k=R(k), vt=R('vt'), out=R(out), B=B, nh=nh, L=L, Lk=Lk, q_pitch=qp, q_c0=0,
                                           k_pitch=qp, k_c0=kc0, vt_pitch=vt_pitch, o_pitch=C, nplanes=NPL, scale=scale, causal=causal,
                                           pad0=32 if pairs else 0))
            return
        sp = s_pitch or Lk
        self.need('S', B * nh * L * sp * F4)
        self.need('P', NPL * B * nh * L * vt_pitch * H2)
        self.emit(lambda R: G.rows_gemm(R(q), L, qp, B, R(k), Lk, qp, B, d, num_z=B * nh, nh=nh, m_valid=L, n_valid=Lk, npass=self.npass,
                                        a_c_per_zh=d, a_n_per_zb=1, b_k0=kc0, b_k_per_zh=d, b_z_per_zb=1, out_f32=R('S'),
                                        o_zb=nh * L * sp, o_zh=L * sp, ldo=sp, scale=scale)[0])
        self.emit(lambda R: S.SoftmaxDesc(S=R('S'), P=R('P'), rows=B * nh * L, L=Lk, nplanes=NPL, pitch_in=s_pitch or 0,     # 0: Lk
                                          pitch_out=0 if vt_pitch == Lk else vt_pitch))
        self.emit(lambda R: G.rows_gemm(R('P'), L, vt_pitch, B * nh, R('vt'), C, vt_pitch, B, vt_pitch, num_z=B * nh, nh=nh, m_valid=L,
                                        n_valid=d, npass=self.npass, a_n_per_zb=nh, a_n_per_zh=1, b_row_per_zh=d, b_z_per_zb=1,
                                        out_h16=R(out), o_zb=L * C, o_zh=d, ldo=C, o_plane=B * L * C, a_k_valid=Lk, b_k_valid=Lk)[0])


def _qkv_split(w, b, heads):
    """Reorder the reference's interleaved qkv channels ([head][c][q|k|v], networks_edm.py:174) into
    [q heads | k heads] rows and separate v rows."""
    c3 = w.shape[0]
    cc = c3 // 3
    d = cc // heads
    idx = torch.arange(c3).reshape(heads, d, 3)
    qi, ki, vi = idx[:, :, 0].reshape(-1), idx[:, :, 1].reshape(-1), idx[:, :, 2].reshape(-1)
    w2 = w.reshape(c3, -1)
    return torch.cat([w2[qi], w2[ki]]), torch.cat([b[qi], b[ki]]), w2[vi], b[vi]


def pack_weights(spec, params, f8=False, f8_min_channels=0):
    """Everything the kernels read that does not depend on the batch size.  f8=True packs the block convolutions (conv0, conv1 +
    skip) and the head conv in the fp16 + 2 x e4m3 operand layout of the f8 GEMM mode (csrc/ops.h); everything else keeps fp16 hi/lo
    planes (the attention GEMMs share their operand planes, the stem conv reads the 3-channel input).
    f8_min_channels > 0 keeps blocks with fewer input or output channels in fp16x3: the narrow, high-resolution levels average the e4m3
    rounding over the fewest terms and dominate the f8 error (FFHQ-64: the 128-channel 64x64 levels, tests/study_fp8_corrections.py)."""
    pf = spec.prefix
    P = lambda k: params[pf + k].detach().float().cpu()
    has = lambda k: (pf + k) in params
    wb = WeightBlob()
    info = {}

    def add_conv(key, w, skip_w=None, bias=None, as_f8=False):
        packed, shift = wb.add_gemm(key, w, skip_w, bias, f8=as_f8)
        info[key] = dict(cout=w.shape[0], f8_shift=shift) if as_f8 else dict(cout=w.shape[0], cout_pad=packed.shape[1], ktot=packed.shape[2])

    add_conv(spec.stem, P(spec.stem + '.weight'), bias=P(spec.stem + '.bias'))
    aff_w, aff_b = [], []
    for b in spec.enc + spec.dec:
        n = b.name
        wb.add_norm(n + '.norm0', P)
        blk_f8 = f8 and min(b.cin, b.cout) >= f8_min_channels
        add_conv(n + '.conv0', P(n + '.conv0.weight'), bias=P(n + '.conv0.bias'), as_f8=blk_f8)
        wb.add_norm(n + '.norm1', P)
        bias1 = P(n + '.conv1.bias')
        skip_w = None
        if b.skip == 'conv':
            skip_w = P(n + '.skip.weight')
            bias1 = bias1 + P(n + '.skip.bias')
        add_conv(n + '.conv1', P(n + '.conv1.weight'), skip_w, bias=bias1, as_f8=blk_f8)
        aff_w.append(P(n + '.affine.weight'))
        aff_b.append(P(n + '.affine.bias'))
        if b.heads:
            wb.add_norm(n + '.norm2', P)
            wqk, bqk, wv, bv = _qkv_split(P(n + '.qkv.weight'), P(n + '.qkv.bias'), b.heads)
            add_conv(n + '.qk', wqk.reshape(wqk.shape[0], wqk.shape[1], 1, 1), bias=bqk)
            wb.add(n + '.v:w', G.split_planes(wv))            # [2][C][C] used as the M operand
            wb.add(n + '.v:b', bv)
            add_conv(n + '.proj', P(n + '.proj.weight'), bias=P(n + '.proj.bias'))
    wb.add('affine:w', torch.cat(aff_w, dim=0))
    wb.add('affine:w16', G.split_planes(torch.cat(aff_w, dim=0)))     # [2][aff_total][emb]: N operand of the batched-embedding GEMM
    wb.add('affine:b', torch.cat(aff_b, dim=0))
    for k in ('map_layer0', 'map_layer1'):
        wb.add(k + ':w', P(k + '.weight'))
        wb.add(k + ':b', P(k + '.bias'))
    if spec.label_dim:
        wb.add('map_label:w', P('map_label.weight'))
        if has('map_label.bias'):
            wb.add('map_label:b', P('map_label.bias'))
    wb.add_norm(spec.head_norm, P)
    # the head conv has 3 output channels: its cost is reading the A operand, which the f8 layout cuts from 3 to 2 tile loads per 64 channels
    add_conv(spec.head_conv, P(spec.head_conv + '.weight'), bias=P(spec.head_conv + '.bias'),
             as_f8=f8 and P(spec.head_conv + '.weight').shape[1] >= f8_min_channels)
    return wb, info


def compile_plan(spec, wb, winfo, B, nsig, nlab, npass=3, fuse_stats=True, flash_attn=True, f8=False):
    """Lower the forward pass for batch B.  nsig in {1, B}: number of sigma values (embedding rows);
    nlab in {0, 1, B}: rows of class labels supplied.  f8: the block convolutions run in the f8 GEMM mode (weights must have been
    packed with pack_weights(f8=True))."""
    assert nsig in (1, B) and nlab in (0, 1, B)
    assert not f8 or npass == 3

    def is_f8(key):
        """This GEMM was packed for the f8 mode (pack_weights decides per block: f8_min_channels)."""
        return f8 and 'f8_shift' in winfo[key]

    def f8_args(key):
        return dict(f8=True, acc_scale=2.0 ** -winfo[key]['f8_shift']) if is_f8(key) else {}
    pb = PlanBuilder(wb, B, npass)
    emit, W = pb.emit, wb.ref
    nE = max(nsig, nlab, 1)
    R0 = spec.img_resolution

    # Fused GroupNorm statistics (fuse_stats=True): the GEMM that writes an fp32 tensor also stores, per 32-row slab and channel
    # quad, the partial {sum, sumsq} (ds_gemm_desc.st_quads); a tiny ds_gn_finalize per GroupNorm folds slabs and quads into the
    # fp64 sums gn_apply reads.  The partials are independent of the consumer's grouping, so one buffer per tensor serves both the
    # next block and the decoder block that concatenates it as a skip.  No atomics, no pass over the tensor itself.
    prod_of = {}            # buffer name -> (op index of the GEMM that wrote it, Cout, rows)
    quads_of = {}           # producer op index -> arena name of its quad-partial buffer
    unit_of = {}            # producer op index -> channels per partial (4 = quads, 2 = pairs: some consumer has 6/18/30-channel groups)

    def emit_producer(name, cout, m_rows, build):
        pid = len(pb.ops)
        prod_of[name] = (pid, cout, m_rows)

        def materialise(R):
            d = build(R)
            if pid in quads_of:
                d.st_quads = R(quads_of[pid])
                d.st_unit = unit_of[pid]
            return d
        emit(materialise)

    def need_stats(slot, parts, hw, norm=None, eps=0.0, ada=None, ada_stride=0):
        """GroupNorm statistics over the (virtually concatenated) fp32 tensors `parts` = [(buffer, channels), ...] for `slot`.
        norm (the weight key of the gain / bias, with eps and the adaptive scale `ada`) additionally asks for the per-(sample, channel)
        coefficient table y = x * a + b in the scratch buffer 'gncoef' (ds_gn_finalize_desc.coef), which lets gn_apply skip its fp64
        prologue and run the persistent variant; returns True when the table is produced."""
        assert len(parts) <= 2
        c_total = sum(c for _, c in parts)
        g = _groups(c_total)
        cpg = c_total // g
        (n0, c0), (n1, c1) = parts[0], (parts[1] if len(parts) > 1 else (None, 0))
        # partial granularity each producer must write for this consumer: 4 channels (quads) when the groups -- and, for a virtual concat
        # whose first source does not end on a group boundary, both pieces of the straddling group -- are multiples of 4, else 2 (pairs)
        rem = c0 % cpg if n1 else 0
        pieces = [cpg] + ([rem, cpg - rem] if rem else [])
        unit = 4 if all(p % 4 == 0 for p in pieces) else (2 if all(p % 2 == 0 for p in pieces) else 0)
        fusable = (fuse_stats and hw % 32 == 0 and unit and all(c % unit == 0 for _, c in parts)
                   and all(name in prod_of and prod_of[name][1] == c for name, c in parts))
        want_coef = norm is not None and c_total <= 2048        # the persistent gn_apply covers up to 256 eight-channel columns
        if want_coef:
            pb.need('gncoef', B * c_total * 2 * F4)

        def coef_args(R):
            if not want_coef:
                return {}
            return dict(gamma=W(norm + ':g'), beta=W(norm + ':b'), ada=_resolve(R, ada), ada_stride=ada_stride, eps=eps, HW=hw,
                        coef=R('gncoef'))
        if not fusable:
            pb.gn_stats(slot, parts, hw, groups=g)
            if want_coef:       # coefficient table from the sums the separate statistics pass accumulated
                emit(lambda R: S.GnFinalizeDesc(quads0=0, quads1=0, C0=c0, C1=c1, slabs_per_sample=0, B=B, groups=g, sums=R('stats', slot),
                                                **coef_args(R)))
            return want_coef
        bufs, pids = [], []
        for name, c in parts:
            pid, cout, m_rows = prod_of[name]
            unit_of[pid] = min(unit_of.get(pid, 4), unit)           # a producer serves all its consumers at the finest unit any of them needs
            quads_of[pid] = pb.need('quads:' + name, (m_rows // 32) * (cout // unit_of[pid]) * 2 * F4)
            bufs.append(quads_of[pid])
            pids.append(pid)
        # unit_of is final only once the whole net is lowered: read it when the descriptors are materialised
        emit(lambda R: S.GnFinalizeDesc(quads0=R(bufs[0]), quads1=R(bufs[1]) if len(bufs) > 1 else 0, C0=c0, C1=c1,
                                        slabs_per_sample=hw // 32, B=B, groups=g, sums=R('stats', slot), unit0=unit_of[pids[0]],
                                        unit1=unit_of[pids[1]] if len(pids) > 1 else 4, **coef_args(R)))
        return want_coef

    def group_norm(parts, H, norm, eps, silu, fmt=0, ada=None):
        """GroupNorm (+ SiLU) of `parts` at H x H into 'act'."""
        slot = pb.stats_slot()
        ada_stride = aff_stride if ada else 0
        coef = need_stats(slot, parts, H * H, norm, eps, ada, ada_stride)
        pb.gn_apply(parts, H, norm, eps, 'act', groups=_groups(sum(c for _, c in parts)), slot=slot, coef=coef, silu=silu, ada=ada,
                    ada_stride=ada_stride, fmt=fmt)

    # ---------------- embedding ----------------------------------------------------------------------------------
    pb.need('coef', nsig * 4 * F4)
    pb.need('emb0', nsig * spec.noise_channels * F4)
    pb.need('e1', nE * spec.emb_channels * F4)
    pb.need('e2', nE * spec.emb_channels * F4)
    pb.need('e3', nE * spec.emb_channels * F4)
    pb.need('aff', nE * spec.aff_total * F4)
    pb.stats(2 * len(spec.enc + spec.dec) + sum(1 for b in spec.enc + spec.dec if b.heads) + 1)
    emit(lambda R: S.PosembDesc(sigma=io(S.DS_IO_SIGMA), nsig=nsig, num_channels=spec.noise_channels,
                                endpoint=1 if spec.kind == 'song' else 0, swap_sincos=1 if spec.kind == 'song' else 0,
                                sigma_data=spec.sigma_data, coef=R('coef'), emb=R('emb0'),
                                noise_scale=0.0 if spec.noise_scale == 1 else spec.noise_scale))     # 0: the kernel's default of 1
    nc, ec = spec.noise_channels, spec.emb_channels
    if spec.kind == 'song':
        src, src_rows = 'emb0', nsig
        if spec.label_dim and nlab:
            pb.need('emb0b', nE * nc * F4)
            emit(lambda R: S.LinearDesc(in_=io(S.DS_IO_LABELS), in_stride=spec.label_dim if nlab > 1 else 0, W=W('map_label:w'),
                                        b=W('map_label:b'), add=R('emb0'), add_stride=nc if nsig > 1 else 0, out=R('emb0b'),
                                        n_rows=nE, in_f=spec.label_dim, out_f=nc, act=0, in_scale=math.sqrt(spec.label_dim)))
            src, src_rows = 'emb0b', nE
        emit(lambda R: S.LinearDesc(in_=R(src), in_stride=nc if src_rows > 1 else 0, W=W('map_layer0:w'), b=W('map_layer0:b'),
                                    out=R('e1'), n_rows=src_rows, in_f=nc, out_f=ec, act=1, in_scale=1.0))
        emit(lambda R: S.LinearDesc(in_=R('e1'), in_stride=ec if src_rows > 1 else 0, W=W('map_layer1:w'), b=W('map_layer1:b'),
                                    out=R('e2'), n_rows=src_rows, in_f=ec, out_f=ec, act=1, in_scale=1.0))
        emb_buf, emb_rows = 'e2', src_rows
    else:
        with_label = bool(spec.label_dim and nlab)
        emit(lambda R: S.LinearDesc(in_=R('emb0'), in_stride=nc if nsig > 1 else 0, W=W('map_layer0:w'), b=W('map_layer0:b'),
                                    out=R('e1'), n_rows=nsig, in_f=nc, out_f=ec, act=1, in_scale=1.0))
        emit(lambda R: S.LinearDesc(in_=R('e1'), in_stride=ec if nsig > 1 else 0, W=W('map_layer1:w'), b=W('map_layer1:b'),
                                    out=R('e2'), n_rows=nsig, in_f=ec, out_f=ec, act=0 if with_label else 1, in_scale=1.0))
        emb_buf, emb_rows = 'e2', nsig
        if with_label:
            emit(lambda R: S.LinearDesc(in_=io(S.DS_IO_LABELS), in_stride=spec.label_dim if nlab > 1 else 0, W=W('map_label:w'), b=0,
                                        add=R('e2'), add_stride=ec if nsig > 1 else 0, out=R('e3'), n_rows=nE, in_f=spec.label_dim,
                                        out_f=ec, act=1, in_scale=1.0))
            emb_buf, emb_rows = 'e3', nE
    if emb_rows >= 32 and ec % 64 == 0:
        # per-sample conditioning (class labels / per-sample sigma): [rows x emb] x [emb x aff_total] is a real GEMM (ImageNet-64 at
        # batch 256: 20 GFLOP) -> fp16 planes of the embedding + the wgmma kernel
        pb.need('emb_planes', NPL * emb_rows * ec * H2)
        pb.to_planes(emb_buf, ec, emb_rows, 1, 1, 'emb_planes', groups=1)
        emit(lambda R: G.rows_gemm(R('emb_planes'), emb_rows, ec, 1, W('affine:w16'), spec.aff_total, ec, 1, ec, num_z=1, nh=1,
                                   m_valid=emb_rows, n_valid=spec.aff_total, npass=npass, out_f32=R('aff'), ldo=spec.aff_total,
                                   bias_n=W('affine:b'))[0])
    else:
        emit(lambda R: S.LinearDesc(in_=R(emb_buf), in_stride=ec if emb_rows > 1 else 0, W=W('affine:w'), b=W('affine:b'), out=R('aff'),
                                    n_rows=emb_rows, in_f=ec, out_f=spec.aff_total, act=0, in_scale=1.0))
    aff_stride = spec.aff_total if emb_rows > 1 else 0

    # ---------------- stem ---------------------------------------------------------------------------------------
    HW0 = R0 * R0
    pb.need('in_planes', NPL * B * HW0 * 64 * H2)
    emit(lambda R: S.PrepInputDesc(x=io(S.DS_IO_X), coef=R('coef'), coef_stride=4 if nsig > 1 else 0, B=B, C=spec.img_channels,
                                   HW=HW0, nplanes=NPL, out=R('in_planes')))
    pb.need('x:' + spec.stem, B * HW0 * spec.stem_cout * F4)
    emit_producer('x:' + spec.stem, spec.stem_cout, B * HW0, lambda R: G.conv_gemm(R('in_planes'), B, R0, R0, 64, W(spec.stem + ':w'), spec.stem_cout, taps=9,
                                                          npass=npass, out_f32=R('x:' + spec.stem), bias=W(spec.stem + ':b'))[0])

    def lower_block(b, x0, c0, x1, c1):
        """x0/x1: arena names of the (virtually concatenated) fp32 NHWC inputs."""
        pb.tag += 1
        n = b.name
        Hi, Ho = b.res_in, b.res_out
        cin, cout = b.cin, b.cout
        assert c0 + c1 == cin
        resample = 1 if b.down else (2 if b.up else 0)
        Mo = B * Ho * Ho
        parts = [(x0, c0)] + ([(x1, c1)] if x1 else [])
        s0 = pb.stats_slot()
        k0 = need_stats(s0, parts, Hi * Hi, n + '.norm0' if resample == 0 else None, b.eps)
        pb.need('act', NPL * Mo * max(cin, cout) * H2)
        want_raw = b.skip == 'conv'
        want_rawf = b.skip == 'resample'
        if want_raw:
            pb.need('raw', NPL * Mo * cin * H2)
        if want_rawf:
            pb.need('rawf', Mo * cin * F4)
        pb.gn_apply(parts, Hi, n + '.norm0', b.eps, 'act', groups=_groups(cin), slot=s0, coef=k0, resample=resample,
                    raw='raw' if want_raw else None, raw_f32='rawf' if want_rawf else None, fmt=1 if is_f8(n + '.conv0') else 0)
        pb.need('y', Mo * cout * F4)
        emit_producer('y', cout, Mo, lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cin, W(n + '.conv0:w'), cout, taps=9, npass=npass, out_f32=R('y'),
                                                 bias=W(n + '.conv0:b'), rowvec=0 if b.adaptive_scale else R('aff', b.aff_off * F4),
                                                 rowvec_stride=aff_stride, **f8_args(n + '.conv0'))[0])
        group_norm([('y', cout)], Ho, n + '.norm1', b.eps, 1, fmt=1 if is_f8(n + '.conv1') else 0,
                   ada=('aff', b.aff_off * F4) if b.adaptive_scale else None)
        xout = pb.need('x:' + n, Mo * cout * F4)
        mid = pb.need('xmid', Mo * cout * F4) if b.heads else xout
        if b.skip == 'identity':
            assert x1 is None
            res_name = x0
        elif b.skip == 'resample':
            res_name = 'rawf'
        else:
            res_name = None
        emit_producer(mid, cout, Mo, lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cout, W(n + '.conv1:w'), cout, taps=9, npass=npass,
                                                 a2_ptr=R('raw') if want_raw else 0, C2=cin if want_raw else 0, out_f32=R(mid),
                                                 bias=W(n + '.conv1:b'), residual=R(res_name) if res_name else 0, ldr=cout,
                                                 scale=b.skip_scale, **f8_args(n + '.conv1'))[0])
        if b.heads:
            nh = b.heads
            d = cout // nh
            L = Ho * Ho
            group_norm([(mid, cout)], Ho, n + '.norm2', b.eps, 0)
            pb.need('qk', NPL * B * L * 2 * cout * H2)
            pb.need('vt', NPL * B * cout * L * H2)
            pb.need('o', NPL * B * L * cout * H2)
            emit(lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cout, W(n + '.qk:w'), 2 * cout, taps=1, npass=npass, out_h16=R('qk'),
                                       bias=W(n + '.qk:b'))[0])
            pb.vt_gemm(n + '.v:w', 'act', cout, cout, L, L, bias=n + '.v:b')
            # fused: one kernel per attention layer, the L x L score matrix never leaves the SM; L % 8 == 0 for the V^T row pitch
            pb.attention(flash_attn and d == 64 and L % 8 == 0, 'qk', 'qk', 'o', nh, L, L, d, 1.0 / math.sqrt(d), L)
            emit_producer(xout, cout, Mo, lambda R: G.conv_gemm(R('o'), B, Ho, Ho, cout, W(n + '.proj:w'), cout, taps=1, npass=npass, out_f32=R(xout),
                                                      bias=W(n + '.proj:b'), residual=R(mid), ldr=cout, scale=b.skip_scale)[0])
        if n == spec.bottleneck_block:
            emit(lambda R: S.ChanmeanDesc(src=R(xout), out=io(S.DS_IO_BOTTLENECK), rows=B * Ho * Ho, C=cout))
        return xout

    # ---------------- encoder / decoder --------------------------------------------------------------------------
    skips = [('x:' + spec.stem, spec.stem_cout)]
    cur, cur_c = 'x:' + spec.stem, spec.stem_cout
    for b in spec.enc:
        cur = lower_block(b, cur, cur_c, None, 0)
        cur_c = b.cout
        skips.append((cur, cur_c))
    for b in spec.dec:
        if b.concat:
            sk, sc = skips.pop()
            assert sc == b.concat
            cur = lower_block(b, cur, cur_c, sk, sc)
        else:
            cur = lower_block(b, cur, cur_c, None, 0)
        cur_c = b.cout
    # ---------------- head: GN -> SiLU -> conv3x3 -> EDM combine ----------------------------------------------------
    pb.tag += 1
    pb.need('act', NPL * B * HW0 * cur_c * H2)
    fin_c = cur_c
    group_norm([(cur, fin_c)], R0, spec.head_norm, spec.head_eps, 1, fmt=1 if is_f8(spec.head_conv) else 0)
    emit(lambda R: G.conv_gemm(R('act'), B, R0, R0, fin_c, W(spec.head_conv + ':w'), spec.img_channels, taps=9, npass=npass,
                               bias=W(spec.head_conv + ':b'),
                               edm=(io(S.DS_IO_X), R('coef'), 4 if nsig > 1 else 0, spec.img_channels, io(S.DS_IO_D)),
                               **f8_args(spec.head_conv))[0])
    return pb.finish(B=B, nsig=nsig, nlab=nlab, npass=npass, f8=bool(f8))

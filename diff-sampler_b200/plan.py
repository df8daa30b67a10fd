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
        self.f8_shift = {}          # GEMM key -> S of its weight packed for the f8 mode (acc_scale 2^-S)

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
        the GEMM kernel -- fp16 hi/lo planes, or the fp16 + 2 x e4m3 layout of the f8 mode -- and its bias `key`:b."""
        if w.dim() == 2:
            w = w.reshape(w.shape[0], w.shape[1], 1, 1)
        if f8:
            packed, self.f8_shift[key] = G.pack_conv_weight_f8(w, skip_w)
        else:
            packed = G.pack_conv_weight(w, skip_w)
        self.add(key + ':w', packed)
        if bias is not None:
            self.add(key + ':b', bias)

    def add_norm(self, key, P, src=None):
        """Norm gain and bias `key`:g / `key`:b from the parameters `src`.weight / `src`.bias (src defaults to key; P: name -> tensor)."""
        src = src or key
        self.add(key + ':g', P(src + '.weight'))
        self.add(key + ':b', P(src + '.bias'))

    def add_res_block(self, key, P, norm0, conv0, norm1, conv1, skip=None, f8=False):
        """The weights PlanBuilder.res_block reads under `key`, from the parameters named by the other arguments (P: name -> tensor):
        the GroupNorms `norm0` / `norm1` and the 3x3 convolutions `conv0` / `conv1`; a 1x1 `skip` convolution is appended to conv1
        along K, its bias folded into conv1's.  f8: both convolutions in the f8 GEMM mode."""
        self.add_norm(key + '.norm0', P, norm0)
        self.add_gemm(key + '.conv0', P(conv0 + '.weight'), bias=P(conv0 + '.bias'), f8=f8)
        self.add_norm(key + '.norm1', P, norm1)
        bias1 = P(conv1 + '.bias')
        if skip:
            bias1 = bias1 + P(skip + '.bias')
        self.add_gemm(key + '.conv1', P(conv1 + '.weight'), P(skip + '.weight') if skip else None, bias=bias1, f8=f8)

    def add_attn_block(self, key, P, norm, qk, v, proj):
        """The weights PlanBuilder.attn_block reads under `key`: the GroupNorm parameters `norm` (P: name -> tensor), and the (weight,
        bias) pairs of the [q heads | k heads] rows, the v rows and the output projection, in the head layout the plan runs."""
        self.add_norm(key + '.norm', P, norm)
        self.add_gemm(key + '.qk', qk[0], bias=qk[1])
        self.add(key + '.v:w', G.split_planes(v[0]))            # [2][N][C]: the M operand of the V^T GEMM
        self.add(key + '.v:b', v[1])
        self.add_gemm(key + '.proj', proj[0], bias=proj[1])

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
    sized to the largest request.  The block methods below reserve their scratch as they go, so a caller whose arena must keep another
    order reserves those names first.  Ops: callables build(R) -> descriptor, materialised by finish() once the arena is laid out;
    R(name, extra=0) is the arena reference.  Each op is stamped with the current `tag` (None: with its own index).

    Fixed per plan: f8 -- the GEMMs whose weight was packed for the f8 mode run in it; gn_groups(C) -- the group count of a C-channel
    GroupNorm; gn_coef -- GroupNorms with a gain over at most 2048 channels get the per-(sample, channel) coefficient table;
    gn_fuse -- the statistics of a GEMM output come from partial sums its producer stores (need_stats)."""

    def __init__(self, wb, B, npass=3, tag=0, f8=False, gn_groups=lambda c: 32, gn_coef=False, gn_fuse=False):
        self.wb, self.B, self.npass, self.tag = wb, B, npass, tag
        self.f8, self.gn_groups, self.gn_coef, self.gn_fuse = f8, gn_groups, gn_coef, gn_fuse
        self.sizes = {}
        self.ops = []
        self._slots = 0
        self.prod_of = {}           # buffer name -> (op index of the GEMM that wrote it, Cout, rows)
        self.quads_of = {}          # producer op index -> arena name of its partial-sum buffer
        self.unit_of = {}           # producer op index -> channels per partial (4 = quads, 2 = pairs: some consumer has 6/18/30-channel groups)

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

    def is_f8(self, key):
        """GEMM `key` runs in the f8 mode: an f8 plan, and the weight was packed for it (pack_weights may keep narrow blocks fp16x3)."""
        return self.f8 and key in self.wb.f8_shift

    def f8_args(self, key):
        return dict(f8=True, acc_scale=2.0 ** -self.wb.f8_shift[key]) if self.is_f8(key) else {}

    def producer(self, name, cout, m_rows, build):
        """emit() for the GEMM that writes the fp32 tensor `name` [m_rows][cout]: with gn_fuse, a GroupNorm of `name` has it store
        partial sums (need_stats)."""
        pid = len(self.ops)
        self.prod_of[name] = (pid, cout, m_rows)

        def materialise(R):
            d = build(R)
            if pid in self.quads_of:
                d.st_quads = R(self.quads_of[pid])
                d.st_unit = self.unit_of[pid]
            return d
        self.emit(materialise)

    # ---- GroupNorm ------------------------------------------------------------------------------------------------------------
    def stats(self):
        """The 'stats' buffer: fp64 {sum, sumsq} per (sample, group), one slot per GroupNorm of the plan, zeroed by a memset op here.
        Its size is the slots taken once the plan is lowered."""
        self.need('stats', 0)
        self.emit(lambda R: S.MemsetDesc(ptr=R('stats'), bytes=self.sizes['stats']))

    def stats_slot(self):
        """Byte offset of the next GroupNorm's sums in 'stats'."""
        assert 'stats' in self.sizes, 'stats() reserves and zeroes the buffer first'
        nbytes = self.B * 32 * 2 * 8
        self._slots += 1
        self.need('stats', self._slots * nbytes)
        return (self._slots - 1) * nbytes

    def need_stats(self, slot, parts, hw, groups, norm=None, eps=0.0, ada=None, ada_stride=0):
        """GroupNorm statistics over the (virtually concatenated) fp32 tensors `parts` = [(buffer, channels), ...] into `slot`.
        gn_fuse: when every part was written by a producer() GEMM, that GEMM also stores, per 32-row slab and channel quad, the partial
        {sum, sumsq} (ds_gemm_desc.st_quads), and a tiny ds_gn_finalize folds slabs and quads into the fp64 sums gn_apply reads.  The
        partials are independent of the consumer's grouping, so one buffer per tensor serves both the next block and the decoder block
        that concatenates it as a skip.  No atomics, no pass over the tensor itself.  Otherwise a gn_stats pass over the tensors.
        gn_coef and norm (the weight key of the gain / bias, with eps and the adaptive scale `ada`): the finalize also writes the
        per-(sample, channel) coefficient table y = x * a + b into the scratch buffer 'gncoef' (ds_gn_finalize_desc.coef), which lets
        gn_apply skip its fp64 prologue and run the persistent variant; returns True when the table is produced."""
        assert len(parts) <= 2
        B, W = self.B, self.wb.ref
        c_total = sum(c for _, c in parts)
        cpg = c_total // groups
        (n0, c0), (n1, c1) = parts[0], (parts[1] if len(parts) > 1 else (None, 0))
        # partial granularity each producer must write for this consumer: 4 channels (quads) when the groups -- and, for a virtual concat
        # whose first source does not end on a group boundary, both pieces of the straddling group -- are multiples of 4, else 2 (pairs)
        rem = c0 % cpg if n1 else 0
        pieces = [cpg] + ([rem, cpg - rem] if rem else [])
        unit = 4 if all(p % 4 == 0 for p in pieces) else (2 if all(p % 2 == 0 for p in pieces) else 0)
        fusable = (self.gn_fuse and hw % 32 == 0 and unit and all(c % unit == 0 for _, c in parts)
                   and all(name in self.prod_of and self.prod_of[name][1] == c for name, c in parts))
        want_coef = self.gn_coef and norm is not None and c_total <= 2048     # the persistent gn_apply covers up to 256 eight-channel columns
        if want_coef:
            self.need('gncoef', B * c_total * 2 * F4)

        def coef_args(R):
            if not want_coef:
                return {}
            return dict(gamma=W(norm + ':g'), beta=W(norm + ':b'), ada=_resolve(R, ada), ada_stride=ada_stride, eps=eps, HW=hw,
                        coef=R('gncoef'))
        if not fusable:
            self.emit(lambda R: S.GnStatsDesc(src0=R(n0), src1=_resolve(R, n1), C0=c0, C1=c1, HW=hw, B=B, groups=groups,
                                              sums=R('stats', slot)))
            if want_coef:       # coefficient table from the sums the separate statistics pass accumulated
                self.emit(lambda R: S.GnFinalizeDesc(quads0=0, quads1=0, C0=c0, C1=c1, slabs_per_sample=0, B=B, groups=groups,
                                                     sums=R('stats', slot), **coef_args(R)))
            return want_coef
        bufs, pids = [], []
        for name, c in parts:
            pid, cout, m_rows = self.prod_of[name]
            self.unit_of[pid] = min(self.unit_of.get(pid, 4), unit)    # a producer serves all its consumers at the finest unit any needs
            self.quads_of[pid] = self.need('quads:' + name, (m_rows // 32) * (cout // self.unit_of[pid]) * 2 * F4)
            bufs.append(self.quads_of[pid])
            pids.append(pid)
        # unit_of is final only once the whole net is lowered: read it when the descriptors are materialised
        self.emit(lambda R: S.GnFinalizeDesc(quads0=R(bufs[0]), quads1=R(bufs[1]) if len(bufs) > 1 else 0, C0=c0, C1=c1,
                                             slabs_per_sample=hw // 32, B=B, groups=groups, sums=R('stats', slot),
                                             unit0=self.unit_of[pids[0]], unit1=self.unit_of[pids[1]] if len(pids) > 1 else 4,
                                             **coef_args(R)))
        return want_coef

    def gn_apply(self, parts, H, norm, eps, out, *, W=None, B=None, groups=32, slot=None, coef=False, silu=1, ada=None, ada_stride=0,
                 resample=0, raw=None, raw_f32=None, fmt=0, phase_pitch=0):
        """GroupNorm of `parts` (as need_stats; an input may also be an io reference) with the gain / bias `norm`:g / `norm`:b (+ SiLU)
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

    def group_norm(self, parts, H, norm, eps, out, *, ada=None, ada_stride=0, **apply_kw):
        """GroupNorm (+ SiLU) of `parts` at H x H into `out`: the statistics of a fresh stats slot (need_stats), then gn_apply."""
        groups = self.gn_groups(sum(c for _, c in parts))
        slot = self.stats_slot()
        coef = self.need_stats(slot, parts, H * H, groups, norm, eps, ada, ada_stride)
        self.gn_apply(parts, H, norm, eps, out, groups=groups, slot=slot, coef=coef, ada=ada, ada_stride=ada_stride, **apply_kw)

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
        fused: the fused kernel (csrc/attention.cu, 64-wide heads, or pairs=True: 32-wide heads two per CTA, nh even, or d in 72 .. 128:
        unpadded wide heads); otherwise QK^T into 'S' (rows of s_pitch, default Lk), the row
        softmax into 'P' (rows of vt_pitch) and the P.V GEMM."""
        B, C = self.B, nh * d
        qp, kc0 = (2 * C, C) if q == k else (C, 0)
        if fused:
            self.emit(lambda R: S.AttnDesc(q=R(q), k=R(k), vt=R('vt'), out=R(out), B=B, nh=nh, L=L, Lk=Lk, q_pitch=qp, q_c0=0,
                                           k_pitch=qp, k_c0=kc0, vt_pitch=vt_pitch, o_pitch=C, nplanes=NPL, scale=scale, causal=causal,
                                           pad0=32 if pairs else (d if d > 64 else 0)))
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


    # ---- blocks -----------------------------------------------------------------------------------------------------------------
    def res_block(self, key, parts, H, cout, out, *, eps, skip, skip_scale=1.0, resample=0, emb=None, ada=None, emb_stride=0):
        """ResBlock `key` (WeightBlob.add_res_block) over the (virtually concatenated) fp32 NHWC tensors `parts` at H x H: GroupNorm + SiLU
        (resample 1 / 2: 2x2 average pooling / nearest x2) -> conv3x3 (+ the row vector `emb`) -> GroupNorm (ada: adaptive scale / shift
        rows) + SiLU -> conv3x3 + skip, times skip_scale, into `out`, which the caller reserves.  skip: 'conv' (1x1, appended along K),
        'identity' (parts[0]) or 'resample' (the resampled input).  emb_stride: row stride of emb / ada (0: one row for the batch).
        A resampling GroupNorm gets no coefficient table: gn_apply reads the table only without resample."""
        B, W = self.B, self.wb.ref
        cin = sum(c for _, c in parts)
        Ho = {1: H // 2, 2: 2 * H}.get(resample, H)
        M = B * Ho * Ho
        conv0, conv1 = key + '.conv0', key + '.conv1'
        s0 = self.stats_slot()
        k0 = self.need_stats(s0, parts, H * H, self.gn_groups(cin), key + '.norm0' if resample == 0 else None, eps)
        self.need('act', NPL * M * max(cin, cout) * H2)
        if skip == 'conv':
            self.need('raw', NPL * M * cin * H2)
        if skip == 'resample':
            self.need('rawf', M * cin * F4)
        self.gn_apply(parts, H, key + '.norm0', eps, 'act', groups=self.gn_groups(cin), slot=s0, coef=k0, resample=resample,
                      raw='raw' if skip == 'conv' else None, raw_f32='rawf' if skip == 'resample' else None, fmt=int(self.is_f8(conv0)))
        self.need('y', M * cout * F4)
        self.producer('y', cout, M, lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cin, W(conv0 + ':w'), cout, taps=9, npass=self.npass,
                                                          out_f32=R('y'), bias=W(conv0 + ':b'), rowvec=_resolve(R, emb),
                                                          rowvec_stride=emb_stride, **self.f8_args(conv0))[0])
        self.group_norm([('y', cout)], Ho, key + '.norm1', eps, 'act', ada=ada, ada_stride=emb_stride if ada else 0,
                        fmt=int(self.is_f8(conv1)))
        assert skip != 'identity' or len(parts) == 1
        residual = {'identity': parts[0][0], 'resample': 'rawf'}.get(skip)
        self.producer(out, cout, M, lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cout, W(conv1 + ':w'), cout, taps=9, npass=self.npass,
                                                          a2_ptr=R('raw') if skip == 'conv' else 0, C2=cin if skip == 'conv' else 0,
                                                          out_f32=R(out), bias=W(conv1 + ':b'), residual=_resolve(R, residual), ldr=cout,
                                                          scale=skip_scale, **self.f8_args(conv1))[0])

    def attn_block(self, key, src, C, H, out, *, eps, heads, d, scale, fused, pairs=False, skip_scale=1.0):
        """Attention block `key` (WeightBlob.add_attn_block) over the fp32 NHWC tensor `src` [B][H][H][C]: GroupNorm -> the [q | k] 1x1
        GEMM and the V^T GEMM -> attention over `heads` heads of width d (attention()) -> 1x1 projection + src, times skip_scale,
        into `out`."""
        B, W, L = self.B, self.wb.ref, H * H
        hp = heads * d
        self.need('act', NPL * B * L * C * H2)
        self.group_norm([(src, C)], H, key + '.norm', eps, 'act', silu=0)
        self.need('qk', NPL * B * L * 2 * hp * H2)
        self.need('vt', NPL * B * hp * L * H2)
        self.need('o', NPL * B * L * hp * H2)
        self.emit(lambda R: G.conv_gemm(R('act'), B, H, H, C, W(key + '.qk:w'), 2 * hp, taps=1, npass=self.npass, out_h16=R('qk'),
                                        bias=W(key + '.qk:b'))[0])
        self.vt_gemm(key + '.v:w', 'act', C, hp, L, L, bias=key + '.v:b')
        self.attention(fused, 'qk', 'qk', 'o', heads, L, L, d, scale, L, pairs=pairs)
        self.need(out, B * L * C * F4)
        self.producer(out, C, B * L, lambda R: G.conv_gemm(R('o'), B, H, H, hp, W(key + '.proj:w'), C, taps=1, npass=self.npass,
                                                           out_f32=R(out), bias=W(key + '.proj:b'), residual=R(src), ldr=C,
                                                           scale=skip_scale)[0])

    def upsample_conv(self, key, src, cin, H, cout, out):
        """Nearest x2 upsampling of the fp32 NHWC tensor `src` [B][H][H][cin], then the 3x3 convolution `key` into `out`."""
        B, W, Ho = self.B, self.wb.ref, 2 * H
        self.need('act', NPL * B * Ho * Ho * cin * H2)
        self.to_planes(src, cin, H, H, B, 'act', fmt=int(self.is_f8(key)), resample=2)
        self.need(out, B * Ho * Ho * cout * F4)
        self.emit(lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cin, W(key + ':w'), cout, taps=9, npass=self.npass, out_f32=R(out),
                                        bias=W(key + ':b'), **self.f8_args(key))[0])

    def head_conv(self, src, C, H, norm, eps, key, cout, **epilogue):
        """GroupNorm + SiLU of the fp32 NHWC tensor `src` [B][H][H][C], then the 3x3 convolution `key` to `cout` channels through
        conv_gemm's output epilogue `epilogue` (edm=... or nchw_out=...; arena names in it are resolved)."""
        B, W = self.B, self.wb.ref
        self.need('act', NPL * B * H * H * C * H2)
        self.group_norm([(src, C)], H, norm, eps, 'act', fmt=int(self.is_f8(key)))
        self.emit(lambda R: G.conv_gemm(R('act'), B, H, H, C, W(key + ':w'), cout, taps=9, npass=self.npass, bias=W(key + ':b'),
                                        **{k: tuple(_resolve(R, x) for x in v) for k, v in epilogue.items()},
                                        **self.f8_args(key))[0])

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
    rounding over the fewest terms and dominate the f8 error (FFHQ-64: the 128-channel 64x64 levels, tests/study_fp8_corrections.py).
    Returns (blob, info); info holds nothing the lowering reads (the f8 shifts are in blob.f8_shift)."""
    pf = spec.prefix
    P = lambda k: params[pf + k].detach().float().cpu()
    has = lambda k: (pf + k) in params
    wb = WeightBlob()
    wb.add_gemm(spec.stem, P(spec.stem + '.weight'), bias=P(spec.stem + '.bias'))
    aff_w, aff_b = [], []
    for b in spec.enc + spec.dec:
        n = b.name
        wb.add_res_block(n, P, n + '.norm0', n + '.conv0', n + '.norm1', n + '.conv1', n + '.skip' if b.skip == 'conv' else None,
                         f8=f8 and min(b.cin, b.cout) >= f8_min_channels)
        aff_w.append(P(n + '.affine.weight'))
        aff_b.append(P(n + '.affine.bias'))
        if b.heads:
            wqk, bqk, wv, bv = _qkv_split(P(n + '.qkv.weight'), P(n + '.qkv.bias'), b.heads)
            wb.add_attn_block(n, P, n + '.norm2', (wqk, bqk), (wv, bv), (P(n + '.proj.weight'), P(n + '.proj.bias')))
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
    wb.add_gemm(spec.head_conv, P(spec.head_conv + '.weight'), bias=P(spec.head_conv + '.bias'),
                f8=f8 and P(spec.head_conv + '.weight').shape[1] >= f8_min_channels)
    return wb, {}


def compile_plan(spec, wb, winfo, B, nsig, nlab, npass=3, fuse_stats=True, flash_attn=True, f8=False):
    """Lower the forward pass for batch B.  nsig in {1, B}: number of sigma values (embedding rows);
    nlab in {0, 1, B}: rows of class labels supplied.  f8: the block convolutions run in the f8 GEMM mode (weights must have been
    packed with pack_weights(f8=True)).  winfo: pack_weights' info.  Every GroupNorm with a gain reads the coefficient table;
    fuse_stats: GroupNorm statistics from the GEMM epilogues (PlanBuilder.need_stats)."""
    assert nsig in (1, B) and nlab in (0, 1, B)
    assert not f8 or npass == 3
    pb = PlanBuilder(wb, B, npass, f8=f8, gn_groups=_groups, gn_coef=True, gn_fuse=fuse_stats)
    emit, W = pb.emit, wb.ref
    nE = max(nsig, nlab, 1)
    R0 = spec.img_resolution

    # ---------------- embedding ----------------------------------------------------------------------------------
    pb.need('coef', nsig * 4 * F4)
    pb.need('emb0', nsig * spec.noise_channels * F4)
    pb.need('e1', nE * spec.emb_channels * F4)
    pb.need('e2', nE * spec.emb_channels * F4)
    pb.need('e3', nE * spec.emb_channels * F4)
    pb.need('aff', nE * spec.aff_total * F4)
    pb.stats()
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
    pb.producer('x:' + spec.stem, spec.stem_cout, B * HW0, lambda R: G.conv_gemm(R('in_planes'), B, R0, R0, 64, W(spec.stem + ':w'),
                                                                            spec.stem_cout, taps=9, npass=npass,
                                                                            out_f32=R('x:' + spec.stem), bias=W(spec.stem + ':b'))[0])

    def lower_block(b, parts):
        """Block b over the (virtually concatenated) fp32 NHWC inputs `parts`: the ResBlock, then the attention block if it has one."""
        pb.tag += 1
        n = b.name
        Ho = b.res_out
        assert sum(c for _, c in parts) == b.cin
        aff = ('aff', b.aff_off * F4)
        xout = 'x:' + n
        mid = 'xmid' if b.heads else xout
        pb.res_block(n, parts, b.res_in, b.cout, mid, eps=b.eps, skip=b.skip, skip_scale=b.skip_scale,
                     resample=1 if b.down else (2 if b.up else 0), emb=None if b.adaptive_scale else aff,
                     ada=aff if b.adaptive_scale else None, emb_stride=aff_stride)
        pb.need(xout, B * Ho * Ho * b.cout * F4)
        if b.heads:
            pb.need(mid, B * Ho * Ho * b.cout * F4)
            d = b.cout // b.heads
            # fused: one kernel per attention layer, the L x L score matrix never leaves the SM; L % 8 == 0 for the V^T row pitch
            pb.attn_block(n, mid, b.cout, Ho, xout, eps=b.eps, heads=b.heads, d=d, scale=1.0 / math.sqrt(d),
                          fused=flash_attn and d == 64 and Ho * Ho % 8 == 0, skip_scale=b.skip_scale)
        if n == spec.bottleneck_block:
            emit(lambda R: S.ChanmeanDesc(src=R(xout), out=io(S.DS_IO_BOTTLENECK), rows=B * Ho * Ho, C=b.cout))
        return xout

    # ---------------- encoder / decoder --------------------------------------------------------------------------
    skips = [('x:' + spec.stem, spec.stem_cout)]
    cur, cur_c = 'x:' + spec.stem, spec.stem_cout
    for b in spec.enc:
        cur = lower_block(b, [(cur, cur_c)])
        cur_c = b.cout
        skips.append((cur, cur_c))
    for b in spec.dec:
        parts = [(cur, cur_c)]
        if b.concat:
            sk, sc = skips.pop()
            assert sc == b.concat
            parts.append((sk, sc))
        cur = lower_block(b, parts)
        cur_c = b.cout
    # ---------------- head: GN -> SiLU -> conv3x3 -> EDM combine ----------------------------------------------------
    pb.tag += 1
    pb.head_conv(cur, cur_c, R0, spec.head_norm, spec.head_eps, spec.head_conv, spec.img_channels,
                 edm=(io(S.DS_IO_X), 'coef', 4 if nsig > 1 else 0, spec.img_channels, io(S.DS_IO_D)))
    return pb.finish(B=B, nsig=nsig, nlab=nlab, npass=npass, f8=bool(f8))

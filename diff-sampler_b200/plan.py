"""Plan compiler: lowers one EDM denoiser (NetSpec + parameter dict) at one batch size into
  * a packed weight blob (fp16 hi/lo K-major GEMM operands + fp32 vectors), built once per net, and
  * a flat list of ds_plan_op records over a workspace arena, built once per (batch, sigma-mode),
which the native executor (csrc/engine.cu) runs.  Pure host logic — no GPU needed to compile a plan.

Reference forward being lowered: networks_edm.py:482-496 (EDMPrecond), :312-355 / :427-453 (U-Nets), :158-179 (UNetBlock).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _cstructs as S
from . import gemm_desc as G

ALIGN = 1024


def _groups(c):
    """GroupNorm group count of the reference: min(32, C // 4)  (networks_edm.py:91)."""
    return min(32, c // 4)


def _align(n, a=ALIGN):
    return (n + a - 1) // a * a


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

    def ref(self, name, extra=0):
        return S.ref(S.SPACE_WEIGHTS, self.off[name] + extra)

    def bytes(self):
        return b''.join(self.chunks)


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
        if as_f8:
            packed, shift = G.pack_conv_weight_f8(w, skip_w)
            info[key] = dict(cout=w.shape[0], f8_shift=shift)
        else:
            packed = G.pack_conv_weight(w, skip_w)
            info[key] = dict(cout=w.shape[0], cout_pad=packed.shape[1], ktot=packed.shape[2])
        wb.add(key + ':w', packed)
        if bias is not None:
            wb.add(key + ':b', bias.float())

    add_conv(spec.stem, P(spec.stem + '.weight'), bias=P(spec.stem + '.bias'))
    aff_w, aff_b = [], []
    for b in spec.enc + spec.dec:
        n = b.name
        wb.add(n + '.norm0:g', P(n + '.norm0.weight'))
        wb.add(n + '.norm0:b', P(n + '.norm0.bias'))
        blk_f8 = f8 and min(b.cin, b.cout) >= f8_min_channels
        add_conv(n + '.conv0', P(n + '.conv0.weight'), bias=P(n + '.conv0.bias'), as_f8=blk_f8)
        wb.add(n + '.norm1:g', P(n + '.norm1.weight'))
        wb.add(n + '.norm1:b', P(n + '.norm1.bias'))
        bias1 = P(n + '.conv1.bias')
        skip_w = None
        if b.skip == 'conv':
            skip_w = P(n + '.skip.weight')
            bias1 = bias1 + P(n + '.skip.bias')
        add_conv(n + '.conv1', P(n + '.conv1.weight'), skip_w, bias=bias1, as_f8=blk_f8)
        aff_w.append(P(n + '.affine.weight'))
        aff_b.append(P(n + '.affine.bias'))
        if b.heads:
            wb.add(n + '.norm2:g', P(n + '.norm2.weight'))
            wb.add(n + '.norm2:b', P(n + '.norm2.bias'))
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
    wb.add(spec.head_norm + ':g', P(spec.head_norm + '.weight'))
    wb.add(spec.head_norm + ':b', P(spec.head_norm + '.bias'))
    # the head conv has 3 output channels: its cost is reading the A operand, which the f8 layout cuts from 3 to 2 tile loads per 64 channels
    add_conv(spec.head_conv, P(spec.head_conv + '.weight'), bias=P(spec.head_conv + '.bias'),
             as_f8=f8 and P(spec.head_conv + '.weight').shape[1] >= f8_min_channels)
    return wb, info


class _Arena:
    """Bump allocator with named buffers; scratch names are shared (sized to the largest request)."""

    def __init__(self):
        self.sizes = {}
        self.order = []
        self.offsets = None

    def need(self, name, nbytes):
        if name not in self.sizes:
            self.sizes[name] = 0
            self.order.append(name)
        self.sizes[name] = max(self.sizes[name], int(nbytes))
        return name

    def finalize(self):
        off = 0
        self.offsets = {}
        for n in self.order:
            self.offsets[n] = off
            off += _align(self.sizes[n])
        self.total = off
        return off

    def ref(self, name, extra=0):
        return S.ref(S.SPACE_ARENA, self.offsets[name] + int(extra))


class Plan:
    def __init__(self, ops_array, n_ops, arena_bytes, arena_offsets, meta):
        self.ops_array = ops_array
        self.n_ops = n_ops
        self.arena_bytes = arena_bytes
        self.arena_offsets = arena_offsets
        self.meta = meta


def compile_plan(spec, wb, winfo, B, nsig, nlab, npass=3, fuse_stats=True, flash_attn=True, f8=False, gn_coef=True, pair_stats=True):
    """Lower the forward pass for batch B.  nsig in {1, B}: number of sigma values (embedding rows);
    nlab in {0, 1, B}: rows of class labels supplied.  f8: the block convolutions run in the f8 GEMM mode (weights must have been
    packed with pack_weights(f8=True)).  gn_coef: GroupNorm coefficient tables + persistent gn_apply (False = the round-1 lowering)."""
    assert nsig in (1, B) and nlab in (0, 1, B)
    assert not f8 or npass == 3

    def is_f8(key):
        """This GEMM was packed for the f8 mode (pack_weights decides per block: f8_min_channels)."""
        return f8 and 'f8_shift' in winfo[key]

    def f8_args(key):
        return dict(f8=True, acc_scale=2.0 ** -winfo[key]['f8_shift']) if is_f8(key) else {}
    A = _Arena()
    ops = []        # list of (type, tag, builder(R) -> desc)
    F4, H2 = 4, 2
    npl = 2
    nE = max(nsig, nlab, 1)
    R0 = spec.img_resolution
    io = lambda slot: S.ref(S.SPACE_IO, slot)
    W = wb.ref
    tag = [0]

    def emit(builder):
        ops.append((tag[0], builder))

    # Fused GroupNorm statistics (fuse_stats=True): the GEMM that writes an fp32 tensor also stores, per 32-row slab and channel
    # quad, the partial {sum, sumsq} (ds_gemm_desc.st_quads); a tiny ds_gn_finalize per GroupNorm folds slabs and quads into the
    # fp64 sums gn_apply reads.  The partials are independent of the consumer's grouping, so one buffer per tensor serves both the
    # next block and the decoder block that concatenates it as a skip.  No atomics, no pass over the tensor itself.
    prod_of = {}            # buffer name -> (op index of the GEMM that wrote it, Cout, rows)
    quads_of = {}           # producer op index -> arena name of its quad-partial buffer
    unit_of = {}            # producer op index -> channels per partial (4 = quads, 2 = pairs: some consumer has 6/18/30-channel groups)

    def emit_producer(name, cout, m_rows, build):
        pid = len(ops)
        prod_of[name] = (pid, cout, m_rows)

        def materialise(R):
            d = build(R)
            if pid in quads_of:
                d.st_quads = R(quads_of[pid])
                d.st_unit = unit_of[pid]
            return d
        emit(materialise)

    def need_stats(slot, parts, hw, norm=None):
        """GroupNorm statistics over the (virtually concatenated) fp32 tensors `parts` = [(buffer, channels), ...] for `slot`.
        norm = dict(gamma, beta, eps, ada, ada_stride) (weight / arena references as callables of R) additionally asks for the
        per-(sample, channel) coefficient table y = x * a + b in the scratch buffer 'gncoef' (ds_gn_finalize_desc.coef), which lets
        gn_apply skip its fp64 prologue and run the persistent variant; returns True when the table is produced."""
        assert len(parts) <= 2
        c_total = sum(c for _, c in parts)
        g = _groups(c_total)
        cpg = c_total // g
        (n0, c0), (n1, c1) = parts[0], (parts[1] if len(parts) > 1 else (None, 0))
        # partial granularity each producer must write for this consumer: 4 channels (quads) when the groups -- and, for a virtual concat
        # whose first source does not end on a group boundary, both pieces of the straddling group -- are multiples of 4, else 2 (pairs)
        rem = c0 % cpg if n1 else 0
        pieces = [cpg] + ([rem, cpg - rem] if rem else [])
        unit = 4 if all(p % 4 == 0 for p in pieces) else (2 if all(p % 2 == 0 for p in pieces) and pair_stats else 0)
        fusable = (fuse_stats and hw % 32 == 0 and unit and all(c % unit == 0 for _, c in parts)
                   and all(name in prod_of and prod_of[name][1] == c for name, c in parts))
        want_coef = norm is not None and gn_coef and c_total <= 2048        # the persistent gn_apply covers up to 256 eight-channel columns
        if want_coef:
            A.need('gncoef', B * c_total * 2 * F4)

        def coef_args(R):
            if not want_coef:
                return {}
            return dict(gamma=norm['gamma'](R), beta=norm['beta'](R), ada=norm['ada'](R) if norm.get('ada') else 0,
                        ada_stride=norm.get('ada_stride', 0), eps=norm['eps'], HW=hw, coef=R('gncoef'))
        if not fusable:
            emit(lambda R: S.GnStatsDesc(src0=R(n0), src1=R(n1) if n1 else 0, C0=c0, C1=c1, HW=hw, B=B, groups=g, sums=R('stats', slot)))
            if want_coef:       # coefficient table from the sums the separate statistics pass accumulated
                emit(lambda R: S.GnFinalizeDesc(quads0=0, quads1=0, C0=c0, C1=c1, slabs_per_sample=0, B=B, groups=g, sums=R('stats', slot),
                                                **coef_args(R)))
            return want_coef
        bufs, pids = [], []
        for name, c in parts:
            pid, cout, m_rows = prod_of[name]
            unit_of[pid] = min(unit_of.get(pid, 4), unit)           # a producer serves all its consumers at the finest unit any of them needs
            quads_of[pid] = A.need('quads:' + name, (m_rows // 32) * (cout // unit_of[pid]) * 2 * F4)
            bufs.append(quads_of[pid])
            pids.append(pid)
        # unit_of is final only once the whole net is lowered: read it when the descriptors are materialised
        emit(lambda R: S.GnFinalizeDesc(quads0=R(bufs[0]), quads1=R(bufs[1]) if len(bufs) > 1 else 0, C0=c0, C1=c1,
                                        slabs_per_sample=hw // 32, B=B, groups=g, sums=R('stats', slot), unit0=unit_of[pids[0]],
                                        unit1=unit_of[pids[1]] if len(pids) > 1 else 4, **coef_args(R)))
        return want_coef

    def stat_args(R, slot, coef=False):
        """gn_apply reads either the coefficient table (resample == 0 uses) or the fp64 sums."""
        return dict(sums=0, coef=R('gncoef')) if coef else dict(sums=R('stats', slot))

    # ---------------- embedding ----------------------------------------------------------------------------------
    A.need('coef', nsig * 4 * F4)
    A.need('emb0', nsig * spec.noise_channels * F4)
    A.need('e1', nE * spec.emb_channels * F4)
    A.need('e2', nE * spec.emb_channels * F4)
    A.need('e3', nE * spec.emb_channels * F4)
    A.need('aff', nE * spec.aff_total * F4)
    n_stats = 2 * len(spec.enc + spec.dec) + sum(1 for b in spec.enc + spec.dec if b.heads) + 1
    A.need('stats', n_stats * B * 32 * 2 * 8)
    emit(lambda R: S.MemsetDesc(ptr=R('stats'), bytes=n_stats * B * 32 * 2 * 8))
    emit(lambda R: S.PosembDesc(sigma=io(S.DS_IO_SIGMA), nsig=nsig, num_channels=spec.noise_channels,
                                endpoint=1 if spec.kind == 'song' else 0, swap_sincos=1 if spec.kind == 'song' else 0,
                                sigma_data=spec.sigma_data, coef=R('coef'), emb=R('emb0')))
    nc, ec = spec.noise_channels, spec.emb_channels
    if spec.kind == 'song':
        src, src_rows = 'emb0', nsig
        if spec.label_dim and nlab:
            A.need('emb0b', nE * nc * F4)
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
        # batch 256: 20 GFLOP) -> fp16 planes of the embedding (gn_apply in pass-through mode) + the wgmma kernel
        A.need('emb_planes', npl * emb_rows * ec * H2)
        emit(lambda R: S.GnApplyDesc(src0=R(emb_buf), src1=0, C0=ec, C1=0, H=emb_rows, W=1, B=1, groups=1, sums=0, gamma=0, beta=0, eps=0.0,
                                     silu=0, ada=0, ada_stride=0, resample=0, nplanes=npl, out_act=0, out_raw=R('emb_planes'), out_raw_f32=0))
        emit(lambda R: G.rows_gemm(R('emb_planes'), emb_rows, ec, 1, W('affine:w16'), spec.aff_total, ec, 1, ec, num_z=1, nh=1,
                                   m_valid=emb_rows, n_valid=spec.aff_total, npass=npass, out_f32=R('aff'), ldo=spec.aff_total,
                                   bias_n=W('affine:b'))[0])
    else:
        emit(lambda R: S.LinearDesc(in_=R(emb_buf), in_stride=ec if emb_rows > 1 else 0, W=W('affine:w'), b=W('affine:b'), out=R('aff'),
                                    n_rows=emb_rows, in_f=ec, out_f=spec.aff_total, act=0, in_scale=1.0))
    aff_stride = spec.aff_total if emb_rows > 1 else 0

    # ---------------- stem ---------------------------------------------------------------------------------------
    HW0 = R0 * R0
    A.need('in_planes', npl * B * HW0 * 64 * H2)
    emit(lambda R: S.PrepInputDesc(x=io(S.DS_IO_X), coef=R('coef'), coef_stride=4 if nsig > 1 else 0, B=B, C=spec.img_channels,
                                   HW=HW0, nplanes=npl, out=R('in_planes')))
    A.need('x:' + spec.stem, B * HW0 * spec.stem_cout * F4)
    emit_producer('x:' + spec.stem, spec.stem_cout, B * HW0, lambda R: G.conv_gemm(R('in_planes'), B, R0, R0, 64, W(spec.stem + ':w'), spec.stem_cout, taps=9,
                                                          npass=npass, out_f32=R('x:' + spec.stem), bias=W(spec.stem + ':b'))[0])

    stat_i = [0]

    def stats_slot():
        i = stat_i[0]
        stat_i[0] += 1
        return i * B * 32 * 2 * 8

    def lower_block(b, x0, c0, x1, c1):
        """x0/x1: arena names of the (virtually concatenated) fp32 NHWC inputs."""
        tag[0] += 1
        n = b.name
        Hi, Ho = b.res_in, b.res_out
        cin, cout = b.cin, b.cout
        assert c0 + c1 == cin
        resample = 1 if b.down else (2 if b.up else 0)
        Mo = B * Ho * Ho
        s0 = stats_slot()
        k0 = need_stats(s0, [(x0, c0)] + ([(x1, c1)] if x1 else []), Hi * Hi,
                        norm=dict(gamma=lambda R: W(n + '.norm0:g'), beta=lambda R: W(n + '.norm0:b'), eps=b.eps) if resample == 0 else None)
        A.need('act', npl * Mo * max(cin, cout) * H2)
        want_raw = b.skip == 'conv'
        want_rawf = b.skip == 'resample'
        if want_raw:
            A.need('raw', npl * Mo * cin * H2)
        if want_rawf:
            A.need('rawf', Mo * cin * F4)
        emit(lambda R: S.GnApplyDesc(src0=R(x0), src1=R(x1) if x1 else 0, C0=c0, C1=c1, H=Hi, W=Hi, B=B, groups=_groups(cin), **stat_args(R, s0, k0),
                                     gamma=W(n + '.norm0:g'), beta=W(n + '.norm0:b'), eps=b.eps, silu=1, ada=0, ada_stride=0,
                                     resample=resample, nplanes=npl, out_act=R('act'), out_raw=R('raw') if want_raw else 0,
                                     out_raw_f32=R('rawf') if want_rawf else 0, fmt=1 if is_f8(n + '.conv0') else 0))
        A.need('y', Mo * cout * F4)
        emit_producer('y', cout, Mo, lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cin, W(n + '.conv0:w'), cout, taps=9, npass=npass, out_f32=R('y'),
                                                 bias=W(n + '.conv0:b'), rowvec=0 if b.adaptive_scale else R('aff', b.aff_off * F4),
                                                 rowvec_stride=aff_stride, **f8_args(n + '.conv0'))[0])
        s1 = stats_slot()
        k1 = need_stats(s1, [('y', cout)], Ho * Ho,
                        norm=dict(gamma=lambda R: W(n + '.norm1:g'), beta=lambda R: W(n + '.norm1:b'), eps=b.eps,
                                  ada=(lambda R: R('aff', b.aff_off * F4)) if b.adaptive_scale else None,
                                  ada_stride=aff_stride if b.adaptive_scale else 0))
        emit(lambda R: S.GnApplyDesc(src0=R('y'), src1=0, C0=cout, C1=0, H=Ho, W=Ho, B=B, groups=_groups(cout), **stat_args(R, s1, k1),
                                     gamma=W(n + '.norm1:g'), beta=W(n + '.norm1:b'), eps=b.eps, silu=1,
                                     ada=R('aff', b.aff_off * F4) if b.adaptive_scale else 0,
                                     ada_stride=aff_stride if b.adaptive_scale else 0, resample=0, nplanes=npl, out_act=R('act'),
                                     out_raw=0, out_raw_f32=0, fmt=1 if is_f8(n + '.conv1') else 0))
        xout = A.need('x:' + n, Mo * cout * F4)
        mid = A.need('xmid', Mo * cout * F4) if b.heads else xout
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
            s2 = stats_slot()
            k2 = need_stats(s2, [(mid, cout)], L, norm=dict(gamma=lambda R: W(n + '.norm2:g'), beta=lambda R: W(n + '.norm2:b'), eps=b.eps))
            emit(lambda R: S.GnApplyDesc(src0=R(mid), src1=0, C0=cout, C1=0, H=Ho, W=Ho, B=B, groups=_groups(cout), **stat_args(R, s2, k2),
                                         gamma=W(n + '.norm2:g'), beta=W(n + '.norm2:b'), eps=b.eps, silu=0, ada=0, ada_stride=0,
                                         resample=0, nplanes=npl, out_act=R('act'), out_raw=0, out_raw_f32=0))
            A.need('qk', npl * B * L * 2 * cout * H2)
            A.need('vt', npl * B * cout * L * H2)
            A.need('o', npl * B * L * cout * H2)
            emit(lambda R: G.conv_gemm(R('act'), B, Ho, Ho, cout, W(n + '.qk:w'), 2 * cout, taps=1, npass=npass, out_h16=R('qk'),
                                       bias=W(n + '.qk:b'))[0])
            emit(lambda R: G.rows_gemm(W(n + '.v:w'), cout, cout, 1, R('act'), L, cout, B, cout, num_z=B, nh=1, m_valid=cout,
                                       n_valid=L, npass=npass, b_z_per_zb=1, out_h16=R('vt'), o_zb=cout * L, ldo=L,
                                       o_plane=B * cout * L, bias_m=W(n + '.v:b'))[0])
            if flash_attn and d == 64 and npl == 2 and L % 8 == 0:
                # one fused kernel per attention layer: the L x L score matrix never leaves the SM (attention.cu)
                emit(lambda R: S.AttnDesc(q=R('qk'), k=R('qk'), vt=R('vt'), out=R('o'), B=B, nh=nh, L=L, Lk=L, q_pitch=2 * cout, q_c0=0,
                                          k_pitch=2 * cout, k_c0=cout, vt_pitch=L, o_pitch=cout, nplanes=npl, scale=1.0 / math.sqrt(d)))
            else:
                A.need('S', B * nh * L * L * F4)
                A.need('P', npl * B * nh * L * L * H2)
                emit(lambda R: G.rows_gemm(R('qk'), L, 2 * cout, B, R('qk'), L, 2 * cout, B, d, num_z=B * nh, nh=nh, m_valid=L, n_valid=L,
                                           npass=npass, a_c_per_zh=d, a_n_per_zb=1, b_k0=cout, b_k_per_zh=d, b_z_per_zb=1,
                                           out_f32=R('S'), o_zb=nh * L * L, o_zh=L * L, ldo=L, scale=1.0 / math.sqrt(d))[0])
                emit(lambda R: S.SoftmaxDesc(S=R('S'), P=R('P'), rows=B * nh * L, L=L, nplanes=npl))
                emit(lambda R: G.rows_gemm(R('P'), L, L, B * nh, R('vt'), cout, L, B, L, num_z=B * nh, nh=nh, m_valid=L, n_valid=d,
                                           npass=npass, a_n_per_zb=nh, a_n_per_zh=1, b_row_per_zh=d, b_z_per_zb=1, out_h16=R('o'),
                                           o_zb=L * cout, o_zh=d, ldo=cout, o_plane=B * L * cout)[0])
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
    tag[0] += 1
    sh = stats_slot()
    A.need('act', npl * B * HW0 * cur_c * H2)
    fin, fin_c = cur, cur_c
    kh = need_stats(sh, [(fin, fin_c)], HW0, norm=dict(gamma=lambda R: W(spec.head_norm + ':g'), beta=lambda R: W(spec.head_norm + ':b'),
                                                       eps=spec.head_eps))
    emit(lambda R: S.GnApplyDesc(src0=R(fin), src1=0, C0=fin_c, C1=0, H=R0, W=R0, B=B, groups=_groups(fin_c), **stat_args(R, sh, kh),
                                 gamma=W(spec.head_norm + ':g'), beta=W(spec.head_norm + ':b'), eps=spec.head_eps, silu=1, ada=0,
                                 ada_stride=0, resample=0, nplanes=npl, out_act=R('act'), out_raw=0, out_raw_f32=0,
                                 fmt=1 if is_f8(spec.head_conv) else 0))
    emit(lambda R: G.conv_gemm(R('act'), B, R0, R0, fin_c, W(spec.head_conv + ':w'), spec.img_channels, taps=9, npass=npass,
                               bias=W(spec.head_conv + ':b'),
                               edm=(io(S.DS_IO_X), R('coef'), 4 if nsig > 1 else 0, spec.img_channels, io(S.DS_IO_D)),
                               **f8_args(spec.head_conv))[0])
    assert stat_i[0] <= n_stats

    total = A.finalize()
    R = A.ref
    arr = (S.PlanOp * len(ops))()
    for i, (tg, builder) in enumerate(ops):
        desc = builder(R)
        arr[i].type = S.OP_TYPE_OF[type(desc)]
        arr[i].tag = tg
        setattr(arr[i].u, S.UNION_FIELD[arr[i].type], desc)
    meta = dict(B=B, nsig=nsig, nlab=nlab, npass=npass, f8=bool(f8), n_ops=len(ops),
                n_gemm=sum(1 for i in range(len(ops)) if arr[i].type == S.DS_OP_GEMM))
    return Plan(arr, len(ops), total, dict(A.offsets), meta)

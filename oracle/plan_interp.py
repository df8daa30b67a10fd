"""ORACLE — test infrastructure, not product code.

CPU interpreter for the plans the product's compilers emit (diff-sampler_b200/plan.py, ldm_plan.py, vae_plan.py): executes a
`ds_plan_op` array op by op with torch on the host, reading and writing the same byte-addressed arena / weight blob / io slots the
native executor (csrc/engine.cu) uses, with each op's arithmetic restated from its kernel (csrc/*.cu) in float64.

What it is for: a plan is pure data (pointers, strides, tile shapes, operand formats).  Running it here checks that data -- buffer
reuse, operand layouts, K ordering of packed weights, the f8 operand images, row-segment tiles -- against the network oracles WITHOUT
a GPU, so a new lowering can be debugged before it ever reaches the hardware.  It does not model tiling, pipelines or rounding of the
tensor cores: a GEMM is evaluated exactly on the operand values its planes hold.  Only tests/ may import this.
"""
import math

import numpy as np
import torch

from diff_sampler_b200 import _cstructs as S

MASK60 = (1 << 60) - 1
F8_A16, F8_LO8, F8_HI8 = S.DS_F8_SH_A16, S.DS_F8_SH_LO8, S.DS_F8_SH_HI8


class Memory:
    """The three address spaces of a plan.  By default a zeroed host arena and a host copy of the weight blob; `device` places them
    elsewhere, and `arena` / `weights` (uint8 tensors) wrap existing buffers instead (e.g. a live device arena or a snapshot of it).
    Every tensor an op creates is made on `device`.  `stored`, when a list, receives (ref, fmt, float64 values, index) for every
    fp16-plane or f8-image store: the values before they are rounded into the planes."""
    def __init__(self, arena_bytes, weight_blob, io, device='cpu', arena=None, weights=None):
        self.device = torch.device(device)
        self.arena = torch.zeros(int(arena_bytes), dtype=torch.uint8, device=self.device) if arena is None else arena
        if weights is None:
            weights = torch.frombuffer(bytearray(weight_blob), dtype=torch.uint8).to(self.device)
        self.weights = weights
        self.io = io                                           # slot -> contiguous torch tensor (fp32) or None
        self.stored = None

    def raw(self, ref):
        ref = int(ref)
        space, off = ref >> 60, ref & MASK60
        if space == S.SPACE_ARENA:
            return self.arena, off
        if space == S.SPACE_WEIGHTS:
            return self.weights, off
        if space == S.SPACE_IO:
            t = self.io.get(off)
            if t is None:
                return None, 0
            return t.reshape(-1).view(torch.uint8), 0
        raise ValueError(f'bad pointer reference {ref:#x}')

    def view(self, ref, dtype, count, byte_offset=0):
        """1-D typed view of `count` elements at the referenced address (+ byte_offset)."""
        buf, off = self.raw(ref)
        if buf is None:
            return None
        esz = torch.empty(0, dtype=dtype).element_size()
        a = off + int(byte_offset)
        return buf[a:a + int(count) * esz].view(dtype)


def _strided(buf1d, shape, strides_elems, offset_elems=0):
    """Strided window into a 1-D typed view (as_strided takes an ABSOLUTE storage offset, hence the view's own offset is added)."""
    return torch.as_strided(buf1d, tuple(int(s) for s in shape), tuple(int(s) for s in strides_elems),
                            buf1d.storage_offset() + int(offset_elems))


def _split16(x):
    hi = x.to(torch.float16)
    lo = (x - hi.to(x.dtype)).to(torch.float16)
    return hi, lo


def _e4m3(x, shift):
    return (x * 2.0 ** shift).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


# ------------------------------------------------------------------------------------------------ operand readers
def _planes_f16(mem, ref, n_elems_per_plane, nplanes, plane_stride_elems=None):
    """fp16 hi (+ lo) planes -> float64 values."""
    ps = n_elems_per_plane if plane_stride_elems is None else plane_stride_elems
    hi = mem.view(ref, torch.float16, n_elems_per_plane).double()
    if nplanes > 1:
        hi = hi + mem.view(ref, torch.float16, n_elems_per_plane, byte_offset=2 * ps).double()
    return hi


def _store_planes(mem, ref, values, nplanes, fmt=0, plane_elems=None, index=None):
    """Write float values as fp16 hi/lo planes (fmt 0) or the f8 operand image (fmt 1) at element positions `index` (default all)."""
    v = values.reshape(-1).to(torch.float64)
    n = v.numel() if plane_elems is None else int(plane_elems)
    idx = slice(None) if index is None else index.reshape(-1)
    if mem.stored is not None:
        mem.stored.append((int(ref), fmt, v, index))
    if fmt == 0:
        hi = v.to(torch.float32).to(torch.float16)
        mem.view(ref, torch.float16, n)[idx] = hi
        if nplanes > 1:
            lo = (v.to(torch.float32) - hi.float()).to(torch.float16)
            mem.view(ref, torch.float16, n, byte_offset=2 * n)[idx] = lo
        return
    v32 = v.to(torch.float32)
    hi = (v32 * 2.0 ** F8_A16).clamp(-65504.0, 65504.0).to(torch.float16)
    hf = hi.float() / 2.0 ** F8_A16
    mem.view(ref, torch.float16, n)[idx] = hi
    mem.view(ref, torch.uint8, n, byte_offset=2 * n)[idx] = _e4m3(v32 - hf, F8_LO8).view(torch.uint8)
    mem.view(ref, torch.uint8, n, byte_offset=3 * n)[idx] = _e4m3(hf, F8_HI8).view(torch.uint8)


# ------------------------------------------------------------------------------------------------ GEMM
def _conv_A(mem, d, ptr, C, Bn, plane_n, passes):
    """Implicit-GEMM A operand of conv mode for tensor `ptr` with C physical channels: returns {name: [M, K] float64} for the
    requested planes ('hi', 'lo' as fp16 planes; 'lo8', 'hi8' as e4m3 byte planes behind the fp16 plane)."""
    H, W = int(d.conv_H), int(d.conv_W)
    out = {}
    for name in passes:
        if name in ('hi', 'lo'):
            t = mem.view(ptr, torch.float16, (plane_n + Bn) * H * W * C if name == 'lo' else Bn * H * W * C)
            x = t[(plane_n * H * W * C if name == 'lo' else 0):][:Bn * H * W * C].reshape(Bn, H, W, C).double()
        else:
            base = 2 * Bn * H * W * C + (Bn * H * W * C if name == 'hi8' else 0)
            x = mem.view(ptr, torch.float8_e4m3fn, Bn * H * W * C, byte_offset=base).reshape(Bn, H, W, C).to(torch.float32).double()
        out[name] = x
    return out


def _im2col(x, d, cpb_ch, taps, use_taps=True):
    """x: [Bn, H, W, C] -> [Bn*H*W, taps * cpb_ch] with the desc's tap shifts / channel bases, zero outside the image / channel extent."""
    Bn, H, W, C = x.shape
    cols = []
    for t in range(taps):
        dh, dw, cb = (int(d.tap_dh[t]), int(d.tap_dw[t]), int(d.tap_cb[t])) if use_taps else (0, 0, 0)
        sh = torch.zeros(Bn, H, W, cpb_ch, dtype=x.dtype, device=x.device)
        h0, h1 = max(0, -dh), min(H, H - dh)
        w0, w1 = max(0, -dw), min(W, W - dw)
        cc = max(0, min(cpb_ch, C - cb))
        if h1 > h0 and w1 > w0 and cc > 0:
            sh[:, h0:h1, w0:w1, :cc] = x[:, h0 + dh:h1 + dh, w0 + dw:w1 + dw, cb:cb + cc]
        cols.append(sh.reshape(Bn * H * W, cpb_ch))
    return torch.cat(cols, dim=1)


def _gemm(mem, d):
    f8 = bool(d.f8 & 1)
    m_valid, n_valid = int(d.m_valid), int(d.n_valid)
    nh = max(int(d.nh), 1)
    results = []                                                     # per z: [m_valid, n_valid] float64 accumulators
    if d.a_mode == 0:
        assert d.num_z == 1
        H, W = int(d.conv_H), int(d.conv_W)
        Bn = m_valid // (H * W)
        assert Bn * H * W == m_valid
        if W > 128:
            assert W % 128 == 0, 'rows wider than an M tile must be whole 128-pixel segments'
        C = int(d.a_dims[0])
        assert tuple(int(v) for v in d.a_strides) == (C * 2, W * C * 2, H * W * C * 2), 'conv A operand must be dense NHWC'
        taps, cpb = int(d.taps), int(d.cpb)
        ktot = int(d.b_dims[0])
        rows_b = int(d.b_dims[1])
        assert int(d.b_strides[0]) == ktot * 2
        k_main, k_aux = taps * cpb * 64, int(d.a2_c)
        assert ktot == k_main + k_aux, (ktot, k_main, k_aux)
        names = ('hi', 'lo8', 'hi8') if f8 else (('hi', 'lo') if d.npass == 3 else ('hi',))
        A = _conv_A(mem, d, d.a_ptr, C, Bn, int(d.a_plane_n), names)
        A2 = _conv_A(mem, d, d.a2_ptr, k_aux, Bn, int(d.a2_plane_n), names) if k_aux else None

        def amat(name, blk):                                        # blk: channels per tap block (64-multiple for fp16, 128-multiple for e4m3)
            m = _im2col(A[name], d, blk, taps)
            if A2 is not None:
                kb = -(-k_aux // (128 if name in ('lo8', 'hi8') else 64)) * (128 if name in ('lo8', 'hi8') else 64)
                m = torch.cat([m, _im2col(A2[name], d, kb, 1, use_taps=False)], dim=1)
            return m
        nrows = min(rows_b, n_valid)
        if f8:
            w16 = mem.view(d.b_ptr, torch.float16, rows_b * ktot).reshape(rows_b, ktot).double()
            cpb8 = (cpb + 1) // 2
            k8 = taps * cpb8 * 128 + (-(-k_aux // 128) * 128 if k_aux else 0)
            whi8 = mem.view(d.b_ptr, torch.float8_e4m3fn, rows_b * k8, byte_offset=rows_b * ktot * 2).reshape(rows_b, k8).float().double()
            wlo8 = mem.view(d.b_ptr, torch.float8_e4m3fn, rows_b * k8, byte_offset=rows_b * ktot * 2 + rows_b * k8).reshape(rows_b, k8).float().double()
            acc = amat('hi', cpb * 64) @ w16[:nrows].T + amat('lo8', cpb8 * 128) @ whi8[:nrows].T + amat('hi8', cpb8 * 128) @ wlo8[:nrows].T
        else:
            bh = mem.view(d.b_ptr, torch.float16, rows_b * ktot).reshape(rows_b, ktot).double()
            acc = amat('hi', cpb * 64) @ bh[:nrows].T
            if d.npass == 3:
                bl = mem.view(d.b_ptr, torch.float16, rows_b * ktot, byte_offset=int(d.b_strides[1]) * int(d.b_plane_batch)).reshape(rows_b, ktot).double()
                acc = acc + amat('lo', cpb * 64) @ bh[:nrows].T + amat('hi', cpb * 64) @ bl[:nrows].T
        if nrows < n_valid:
            acc = torch.cat([acc, torch.zeros(m_valid, n_valid - nrows, dtype=acc.dtype, device=acc.device)], dim=1)
        results.append(acc)
    else:
        assert not f8
        K = int(d.cpb) * 64
        a_kv, a_rows = int(d.a_dims[0]), int(d.a_dims[1])
        a_pitch = int(d.a_strides[0]) // 2
        a_bstride = int(d.a_strides[2]) // 2
        a_tot = int(d.a_dims[3])
        b_kv, b_rows, b_tot = int(d.b_dims[0]), int(d.b_dims[1]), int(d.b_dims[2])
        b_pitch, b_bstride = int(d.b_strides[0]) // 2, int(d.b_strides[1]) // 2
        abuf = mem.view(d.a_ptr, torch.float16, a_tot * a_bstride)
        bbuf = mem.view(d.b_ptr, torch.float16, (b_tot - 1) * b_bstride + b_rows * b_pitch)

        def a_block(batch, c_off):
            x = torch.zeros(m_valid, K, dtype=torch.float64, device=mem.device)
            rows = min(m_valid, a_rows)
            cc = max(0, min(K, a_kv - c_off))
            if cc > 0:
                x[:rows, :cc] = _strided(abuf, (rows, cc), (a_pitch, 1), batch * a_bstride + c_off).double()
            return x

        def b_block(batch, k_off, row_off):
            x = torch.zeros(n_valid, K, dtype=torch.float64, device=mem.device)
            rows = max(0, min(n_valid, b_rows - row_off))
            cc = max(0, min(K, b_kv - k_off))
            if rows > 0 and cc > 0:
                x[:rows, :cc] = _strided(bbuf, (rows, cc), (b_pitch, 1), batch * b_bstride + row_off * b_pitch + k_off).double()
            return x
        for z in range(int(d.num_z)):
            zb, zh = divmod(z, nh)
            an = zb * int(d.a_n_per_zb) + zh * int(d.a_n_per_zh)
            bz = zb * int(d.b_z_per_zb) + zh * int(d.b_z_per_zh)
            ac, bk, br = zh * int(d.a_c_per_zh), int(d.b_k0) + zh * int(d.b_k_per_zh), zh * int(d.b_row_per_zh)
            ah, bh = a_block(an, ac), b_block(bz, bk, br)
            acc = ah @ bh.T
            if d.npass == 3:
                acc = acc + a_block(an + int(d.a_plane_n), ac) @ bh.T + ah @ b_block(bz + int(d.b_plane_batch), bk, br).T
            results.append(acc)
    # ---- epilogue -------------------------------------------------------------------------------------------------------------
    acc_scale = float(d.acc_scale) if d.acc_scale else 1.0
    rows = torch.arange(m_valid, device=mem.device)
    for z, acc in enumerate(results):
        zb, zh = divmod(z, nh)
        r = acc * acc_scale
        if d.bias_n:
            r = r + mem.view(d.bias_n, torch.float32, n_valid).double()[None, :]
        if d.bias_m:
            r = r + mem.view(d.bias_m, torch.float32, m_valid).double()[:, None]
        if d.rowvec:
            rs = int(d.rowvec_stride)
            nsamp = (m_valid - 1) // max(int(d.rows_per_sample), 1) + 1
            rv = mem.view(d.rowvec, torch.float32, (nsamp - 1) * rs + n_valid)
            samp = rows // max(int(d.rows_per_sample), 1)
            r = r + _strided(rv, (nsamp, n_valid), (rs, 1)).double()[samp if rs else torch.zeros_like(samp)]
        if d.residual:
            ldr = int(d.ldr)
            res = mem.view(d.residual, torch.float32, (m_valid - 1) * ldr + n_valid)
            r = r + _strided(res, (m_valid, n_valid), (ldr, 1)).double()
        r = r * float(d.scale)
        if d.st_quads:
            u = 2 if int(d.st_unit) == 2 else 4
            assert m_valid % 32 == 0 and n_valid % u == 0
            q = r.reshape(m_valid // 32, 32, n_valid // u, u)
            part = torch.stack([q.sum(dim=(1, 3)), (q * q).sum(dim=(1, 3))], dim=-1)             # [slabs, quads, 2]
            mem.view(d.st_quads, torch.float32, part.numel())[:] = part.reshape(-1).float()
        if d.edm_out:
            HW = int(d.rows_per_sample)
            Cimg = int(d.edm_C)
            nsamp = m_valid // HW
            img = r[:, :Cimg].reshape(nsamp, HW, Cimg).permute(0, 2, 1)                           # [n, c, hw]
            out = mem.view(d.edm_D, torch.float32, nsamp * Cimg * HW)
            if d.edm_out == 2:
                out[:] = img.reshape(-1).float()
            else:
                coef = mem.view(d.edm_coef, torch.float32, (nsamp - 1) * int(d.edm_coef_stride) + 4)
                cs = torch.stack([coef[n * int(d.edm_coef_stride) + 0] for n in range(nsamp)]).double()
                co = torch.stack([coef[n * int(d.edm_coef_stride) + 1] for n in range(nsamp)]).double()
                x = mem.view(d.edm_x, torch.float32, nsamp * Cimg * HW).reshape(nsamp, Cimg, HW).double()
                out[:] = (cs[:, None, None] * x + co[:, None, None] * img).reshape(-1).float()
            continue
        ldo = int(d.ldo)
        base = zb * int(d.o_zb) + zh * int(d.o_zh)
        span = (m_valid - 1) * ldo + n_valid
        if d.out_f32:
            o = mem.view(d.out_f32, torch.float32, base + span)
            _strided(o, (m_valid, n_valid), (ldo, 1), base)[:] = r.float()
        if d.out_h16:
            hi, lo = _split16(r.float())
            o = mem.view(d.out_h16, torch.float16, base + span)
            _strided(o, (m_valid, n_valid), (ldo, 1), base)[:] = hi
            if d.o_plane:
                o2 = mem.view(d.out_h16, torch.float16, base + span, byte_offset=2 * int(d.o_plane))
                _strided(o2, (m_valid, n_valid), (ldo, 1), base)[:] = lo


# ------------------------------------------------------------------------------------------------ GroupNorm / elementwise
def _src_cat(mem, d, n_pix_total):
    x = mem.view(d.src0, torch.float32, n_pix_total * int(d.C0)).reshape(n_pix_total, int(d.C0)).double()
    if d.C1:
        x = torch.cat([x, mem.view(d.src1, torch.float32, n_pix_total * int(d.C1)).reshape(n_pix_total, int(d.C1)).double()], dim=1)
    return x


def _gn_stats(mem, d):
    B, HW, C, G = int(d.B), int(d.HW), int(d.C0) + int(d.C1), int(d.groups)
    x = _src_cat(mem, d, B * HW).reshape(B, HW, G, C // G)
    s = mem.view(d.sums, torch.float64, B * G * 2).reshape(B, G, 2)
    s[:, :, 0] += x.sum(dim=(1, 3))
    s[:, :, 1] += (x * x).sum(dim=(1, 3))


def _gn_finalize(mem, d):
    B, G, slabs = int(d.B), int(d.groups), int(d.slabs_per_sample)
    C0, C1 = int(d.C0), int(d.C1)
    C = C0 + C1
    if d.quads0:
        u0, u1 = (2 if int(d.unit0) == 2 else 4), (2 if int(d.unit1) == 2 else 4)
        # per-channel view of the partials (each unit's sums attributed to its first channel) so that any grouping can be summed
        def per_channel(ptr, Cx, u):
            q = mem.view(ptr, torch.float32, B * slabs * (Cx // u) * 2).reshape(B, slabs, Cx // u, 2).double().sum(dim=1)
            out = torch.zeros(B, Cx, 2, dtype=torch.float64, device=mem.device)
            out[:, ::u, :] = q
            return out
        pc = per_channel(d.quads0, C0, u0)
        if C1:
            pc = torch.cat([pc, per_channel(d.quads1, C1, u1)], dim=1)
        cpg = C // G
        rem = C0 % cpg
        assert cpg % u0 == 0 and rem % u0 == 0 and (not C1 or (cpg % u1 == 0 and (cpg - rem) % u1 == 0 or rem == 0 and cpg % u1 == 0))
        mem.view(d.sums, torch.float64, B * G * 2)[:] = pc.reshape(B, G, cpg, 2).sum(dim=2).reshape(-1)
    if d.coef:
        # per-(sample, channel) {a, b}: y = x * a + b, in fp32 as the kernel computes them (elementwise.cu gn_finalize_kernel)
        s = mem.view(d.sums, torch.float64, B * G * 2).reshape(B, G, 2)
        cnt = (C // G) * int(d.HW)
        mu = s[:, :, 0] / cnt
        var = (s[:, :, 1] / cnt - mu * mu).clamp_min(0.0)
        rstd = (1.0 / torch.sqrt(var + float(d.eps))).float()
        mu_c = mu.float().repeat_interleave(C // G, dim=1)
        a = rstd.repeat_interleave(C // G, dim=1) * mem.view(d.gamma, torch.float32, C)[None, :]
        b = mem.view(d.beta, torch.float32, C)[None, :].expand(B, C).clone()
        if d.ada:
            st = int(d.ada_stride)
            ada = mem.view(d.ada, torch.float32, (B - 1) * st + 2 * C)
            ada = _strided(ada, (B, 2 * C), (st, 1))
            sc, sh = ada[:, :C] + 1.0, ada[:, C:]
            a = a * sc
            b = b * sc + sh
        out = mem.view(d.coef, torch.float32, B * C * 2).reshape(B, C, 2)
        out[:, :, 0] = a
        out[:, :, 1] = b - mu_c * a


def _gn_apply(mem, d):
    B, H, W, C, G = int(d.B), int(d.H), int(d.W), int(d.C0) + int(d.C1), int(d.groups)
    x = _src_cat(mem, d, B * H * W).reshape(B, H, W, C)
    y = None
    if d.coef:
        assert int(d.resample) == 0 and not d.sums
        cf = mem.view(d.coef, torch.float32, B * C * 2).reshape(B, C, 2).double()
        y = x * cf[:, None, None, :, 0] + cf[:, None, None, :, 1]
        if d.silu:
            y = y * torch.sigmoid(y)
    elif d.sums:
        s = mem.view(d.sums, torch.float64, B * G * 2).reshape(B, G, 2)
        cnt = (C // G) * H * W
        mu = s[:, :, 0] / cnt
        var = (s[:, :, 1] / cnt - mu * mu).clamp_min(0.0)
        rstd = 1.0 / torch.sqrt(var + float(d.eps))
        mu_c = mu.repeat_interleave(C // G, dim=1)[:, None, None, :]
        rstd_c = rstd.repeat_interleave(C // G, dim=1)[:, None, None, :]
        a = mem.view(d.gamma, torch.float32, C).double()[None, None, None, :] * rstd_c
        b = mem.view(d.beta, torch.float32, C).double()[None, None, None, :].expand(B, 1, 1, C)
        if d.ada:
            st = int(d.ada_stride)
            ada = mem.view(d.ada, torch.float32, (B - 1) * st + 2 * C)
            ada = _strided(ada, (B, 2 * C), (st, 1)).double()
            sc, sh = ada[:, :C] + 1.0, ada[:, C:]
            a = a * sc[:, None, None, :]
            b = b * sc[:, None, None, :] + sh[:, None, None, :]
        y = (x - mu_c) * a + b
        if d.silu:
            y = y * torch.sigmoid(y)
    rs = int(d.resample)

    def resample(t):
        if rs == 1:
            return t.reshape(B, H // 2, 2, W // 2, 2, C).mean(dim=(2, 4))
        if rs == 2:
            return t.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        if rs == 3:                                                   # space-to-depth, phase-major channels
            return t.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4 * C)
        return t
    npl, fmt = int(d.nplanes), int(d.fmt)
    if d.out_act:
        assert y is not None
        _store_planes(mem, d.out_act, resample(y), npl, fmt)
    if d.out_raw:
        _store_planes(mem, d.out_raw, resample(x), npl, fmt)
    if d.out_raw_f32:
        r = resample(x)
        mem.view(d.out_raw_f32, torch.float32, r.numel())[:] = r.reshape(-1).float()


def _softmax(mem, d):
    rows, L = int(d.rows), int(d.L)
    pin, pout = int(d.pitch_in) or L, int(d.pitch_out) or L
    s = _strided(mem.view(d.S, torch.float32, (rows - 1) * pin + L), (rows, L), (pin, 1)).double()
    p = torch.softmax(s, dim=1).float()
    hi, lo = _split16(p)
    n = rows * pout
    _strided(mem.view(d.P, torch.float16, n), (rows, L), (pout, 1))[:] = hi
    if d.nplanes > 1:
        _strided(mem.view(d.P, torch.float16, n, byte_offset=2 * n), (rows, L), (pout, 1))[:] = lo


def _posemb(mem, d):
    n, ch = int(d.nsig), int(d.num_channels)
    sig = mem.view(d.sigma, torch.float32, n).double()
    half = ch // 2
    i = torch.arange(half, dtype=torch.float64, device=mem.device)
    emb = mem.view(d.emb, torch.float32, n * ch).reshape(n, ch)
    if d.mode == 1:
        a = sig[:, None] * torch.exp(-math.log(10000.0) * i / half)[None, :]
        emb[:, :half], emb[:, half:] = torch.cos(a).float(), torch.sin(a).float()
        return
    sd = float(d.sigma_data)
    s2 = sig * sig + sd * sd
    c_noise = torch.log(sig) / 4
    coef = mem.view(d.coef, torch.float32, n * 4).reshape(n, 4)
    coef[:, 0], coef[:, 1], coef[:, 2], coef[:, 3] = (sd * sd / s2).float(), (sig * sd / torch.sqrt(s2)).float(), (1 / torch.sqrt(s2)).float(), c_noise.float()
    a = c_noise[:, None] * ((1.0 / 10000.0) ** (i / (half - (1 if d.endpoint else 0))))[None, :]
    cs, sn = torch.cos(a).float(), torch.sin(a).float()
    if d.swap_sincos:
        emb[:, :half], emb[:, half:] = sn, cs
    else:
        emb[:, :half], emb[:, half:] = cs, sn


def _linear(mem, d):
    n, fi, fo = int(d.n_rows), int(d.in_f), int(d.out_f)
    ist = int(d.in_stride)
    xin = mem.view(getattr(d, 'in_'), torch.float32, (n - 1) * ist + fi)
    x = _strided(xin, (n, fi), (ist, 1)).double() * float(d.in_scale)
    Wm = mem.view(d.W, torch.float32, fo * fi).reshape(fo, fi).double()
    v = x @ Wm.T
    if d.b:
        v = v + mem.view(d.b, torch.float32, fo).double()[None, :]
    if d.add:
        ast = int(d.add_stride)
        v = v + _strided(mem.view(d.add, torch.float32, (n - 1) * ast + fo), (n, fo), (ast, 1)).double()
    if d.act == 1:
        v = v * torch.sigmoid(v)
    mem.view(d.out, torch.float32, n * fo)[:] = v.reshape(-1).float()


def _prep_input(mem, d):
    B, C, HW = int(d.B), int(d.C), int(d.HW)
    xb = int(d.x_batch) if d.x_batch > 0 else B
    x = mem.view(d.x, torch.float32, xb * C * HW).reshape(xb, C, HW).double()
    cst = int(d.coef_stride)
    coef = mem.view(d.coef, torch.float32, (xb - 1) * cst + 4)
    out = torch.zeros(B, HW, 64, dtype=torch.float64, device=mem.device)
    for n in range(B):
        nx = n % xb
        out[n, :, :C] = (float(coef[nx * cst + 2]) * x[nx]).T
    _store_planes(mem, d.out, out, int(d.nplanes))


def _layernorm(mem, d):
    rows, C = int(d.rows), int(d.C)
    x = mem.view(d.src, torch.float32, rows * C).reshape(rows, C).double()
    y = torch.nn.functional.layer_norm(x, (C,), mem.view(d.gamma, torch.float32, C).double(), mem.view(d.beta, torch.float32, C).double(), float(d.eps))
    if int(d.fmt) == 2:                                        # fp32 result
        mem.view(d.out, torch.float32, rows * C)[:] = y.reshape(-1).float()
        return
    _store_planes(mem, d.out, y, int(d.nplanes), int(d.fmt))


def _geglu(mem, d):
    rows, I = int(d.rows), int(d.I)
    if int(d.mode) == 1:                                       # quick-GELU on [rows][I]
        x = mem.view(d.src, torch.float32, rows * I).reshape(rows, I).double()
        _store_planes(mem, d.out, x * torch.sigmoid(1.702 * x), int(d.nplanes), 0)
        return
    x = mem.view(d.src, torch.float32, rows * 2 * I).reshape(rows, 2 * I).double()
    _store_planes(mem, d.out, x[:, :I] * torch.nn.functional.gelu(x[:, I:]), int(d.nplanes), int(d.fmt))


def _chanmean(mem, d):
    if not d.out:
        return
    out = mem.view(d.out, torch.float32, int(d.rows))
    if out is None:
        return
    out[:] = mem.view(d.src, torch.float32, int(d.rows) * int(d.C)).reshape(int(d.rows), int(d.C)).double().mean(dim=1).float()


def _attn(mem, d):
    B, nh, L, Lk = int(d.B), int(d.nh), int(d.L), int(d.Lk)
    qp, kp, vp, op = int(d.q_pitch), int(d.k_pitch), int(d.vt_pitch), int(d.o_pitch)
    q = _planes_f16(mem, d.q, B * L * qp, 2).reshape(B, L, qp)
    k = _planes_f16(mem, d.k, B * Lk * kp, 2).reshape(B, Lk, kp)
    vt = _planes_f16(mem, d.vt, B * nh * 64 * vp, 2).reshape(B, nh * 64, vp)
    out = torch.zeros(B, L, op, dtype=torch.float64, device=mem.device)
    for h in range(nh):
        qs = q[:, :, int(d.q_c0) + h * 64:int(d.q_c0) + (h + 1) * 64]
        ks = k[:, :, int(d.k_c0) + h * 64:int(d.k_c0) + (h + 1) * 64]
        sc = float(d.scale) * qs @ ks.transpose(1, 2)
        if int(d.causal):
            sc = sc + torch.full((L, Lk), float('-inf'), dtype=torch.float64, device=mem.device).triu(1)
        p = torch.softmax(sc, dim=2)
        out[:, :, h * 64:(h + 1) * 64] = p @ vt[:, h * 64:(h + 1) * 64, :Lk].transpose(1, 2)
    idx = None
    if op != nh * 64:
        raise NotImplementedError('attention output pitch != nh * 64')
    _store_planes(mem, d.out, out, 2, index=idx)


def _embed(mem, d):
    rows, T, C_, V = int(d.rows), int(d.T), int(d.C), int(d.vocab)
    ids = mem.view(d.ids, torch.int32, rows).long().clamp(0, V - 1)
    tok = mem.view(d.tok, torch.float32, V * C_).reshape(V, C_)
    pos = mem.view(d.pos, torch.float32, T * C_).reshape(T, C_)
    mem.view(d.out, torch.float32, rows * C_)[:] = (tok[ids] + pos[torch.arange(rows, device=mem.device) % T]).reshape(-1)


_DISPATCH = {
    S.DS_OP_GEMM: ('gemm', _gemm), S.DS_OP_GN_STATS: ('gn_stats', _gn_stats), S.DS_OP_GN_APPLY: ('gn_apply', _gn_apply),
    S.DS_OP_SOFTMAX: ('softmax', _softmax), S.DS_OP_POSEMB: ('posemb', _posemb), S.DS_OP_LINEAR: ('linear', _linear),
    S.DS_OP_PREP_INPUT: ('prep_input', _prep_input), S.DS_OP_CHANMEAN: ('chanmean', _chanmean), S.DS_OP_LAYERNORM: ('layernorm', _layernorm),
    S.DS_OP_GEGLU: ('geglu', _geglu), S.DS_OP_GN_FINALIZE: ('gn_finalize', _gn_finalize), S.DS_OP_ATTN: ('attn', _attn),
    S.DS_OP_EMBED: ('embed', _embed),
}


def run_op(mem, op):
    """Execute one ds_plan_op (pointer fields still plan references) on `mem`."""
    with torch.no_grad():
        if op.type == S.DS_OP_MEMSET:
            mem.view(op.u.memset.ptr, torch.uint8, int(op.u.memset.bytes))[:] = 0
            return
        field, fn = _DISPATCH[op.type]
        fn(mem, getattr(op.u, field))


def run_plan(plan, weight_blob, io):
    """Execute `plan` (diff_sampler_b200.plan.Plan) on the host.  io: {DS_IO_* slot: contiguous fp32 CPU tensor}; output tensors
    (e.g. DS_IO_D) are written in place.  Returns the Memory (arena readable through plan.arena_offsets)."""
    mem = Memory(plan.arena_bytes, weight_blob, io)
    for i in range(plan.n_ops):
        run_op(mem, plan.ops_array[i])
    return mem


def read_buffer(mem, plan, name, shape, dtype=torch.float32):
    n = int(np.prod(shape))
    return mem.view(S.ref(S.SPACE_ARENA, plan.arena_offsets[name]), dtype, n).reshape(shape).clone()

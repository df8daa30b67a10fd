"""Builders for ds_gemm_desc (csrc/ops.h): how each contraction of the denoiser maps onto the one
wgmma kernel.  Pure integer/shape logic — importable and testable without a GPU.

Pointer arguments are either absolute device addresses (tests) or plan references (plan.py)."""
from . import _cstructs as S

H16 = 2  # bytes per fp16


NUM_SMS = 132                            # H100 SXM


def _tile_cost(bn):
    """Relative cost of one 64-wide K step of a 128 x bn tile: a fixed part per K step (the 16 KB activation tile through TMA and the
    shared-memory port) plus a part per weight row, so narrow tiles are far from proportionally cheaper.  A tile-selection model,
    not a measurement."""
    return 690.0 + bn


def pick_bn(n):
    """N tile (any multiple of 16 up to 256): narrow outputs get the smallest covering tile; otherwise the tiling with the least
    total cost tiles x _tile_cost(bn), ties to less padding: 192 -> 192, 320 -> 160x2, 384 -> 192x2, 576 -> 192x3, 640 -> 224x3,
    1280 -> 256x5."""
    for bn in (32, 64):
        if n <= bn:
            return bn, 1
    best = None
    for bn in range(256, 63, -16):
        tiles = -(-n // bn)
        key = (tiles * _tile_cost(bn), tiles * bn - n, -bn)
        if best is None or key < best[0]:
            best = (key, bn, tiles)
    return best[1], best[2]


def fill_bn(n, m_tiles, num_z=1):
    """N tile for a problem with few tiles (small batch / low resolution): the persistent grid runs ceil(tiles / NUM_SMS) waves, so
    140 tiles cost two full waves.  Choose the multiple of 16 that minimises waves x per-tile cost.  Large problems keep pick_bn's tiling.
    The packed weight keeps pick_bn's padded row count; rows past it are zero-filled by TMA."""
    bn, tiles = pick_bn(n)
    if m_tiles * tiles * num_z >= 4 * NUM_SMS or bn <= 64:
        return bn, tiles
    best = None
    for cand in range(256, 63, -16):
        nt = -(-n // cand)
        waves = -(-(m_tiles * nt * num_z) // NUM_SMS)
        key = (waves * _tile_cost(cand), nt * cand - n, -cand)
        if best is None or key < best[0]:
            best = (key, cand, nt)
    return best[1], best[2]


def padded_rows(n):
    """Row count of a weight packed by pack_conv_weight / pack_conv_weight_f8: pick_bn's whole N tiles."""
    bn, tiles = pick_bn(n)
    return bn * tiles


def split_planes_rows(n_valid, bn):
    tiles = -(-n_valid // bn)
    return tiles, tiles * bn


def conv_box(H, W):
    """TMA box (64, bw, bh, bn) covering 128 consecutive NHWC pixels: whole rows for W <= 128, a 128-pixel row segment for wider
    images (W a multiple of 128)."""
    if W > 128:
        assert W % 128 == 0, f'unsupported width {W}'
        return 128, 1, 1
    assert 128 % W == 0, f'unsupported width {W}'
    bw = W
    bh = min(H, 128 // W)
    bn = 128 // (bw * bh)
    assert bw * bh * bn == 128
    return bw, bh, bn


def conv_gemm(a_ptr, Bn, H, W, C, w_ptr, Cout, *, taps=9, npass=3, a_planes=2, w_planes=2, a2_ptr=0, C2=0,
              out_f32=0, out_h16=0, o_planes=2, ldo=None, bias=0, rowvec=0, rowvec_stride=0, residual=0, ldr=None, scale=1.0,
              edm=None, nchw_out=None, bn=None, s2d=False, f8=False, acc_scale=1.0):
    """3x3 (taps=9) or 1x1 (taps=1) convolution over NHWC fp16 planes [a_planes][Bn][H][W][C] with the
    packed weight matrix [w_planes][Cout_pad][taps*C + C2] (K ordered tap-major, then the aux/skip block).
    Output rows are NHWC pixels: out[pixel][cout] (+ fused epilogue).
    edm = (x, coef, coef_stride, C, D): D = c_skip x + c_out y as NCHW fp32 (the EDM combine); nchw_out = (C, D): y as NCHW fp32.
    f8=True: both operands are in the fp16 + 2 x e4m3 layout of csrc/ops.h (activations from ds_gn_apply fmt=1, weights from
    pack_conv_weight_f8); acc_scale = 2^-S of that packed weight.
    C and C2 need only be multiples of 8: the K loop runs over whole 64-channel blocks, TMA zero-fills the channels past C (C2) in
    the last block and pack_conv_weight pads each tap (the skip block) to a multiple of 64.  s2d: the space-to-depth input holds
    each phase at a pitch of C rounded up to 64 channels, the gap zeroed (ds_gn_apply_desc.pad0)."""
    assert C % 8 == 0 and C2 % 8 == 0
    cpad, c2pad = -(-C // 64) * 64, -(-C2 // 64) * 64
    if f8:
        assert npass == 3 and not s2d
        a_planes = w_planes = 1          # one fp16 plane; the e4m3 planes sit behind it (the kernel derives their tensor maps)
    elif npass == 3:
        assert a_planes == 2 and w_planes == 2
    d = S.GemmDesc()
    bw, bh, bnn = conv_box(H, W)
    BN, n_tiles = (bn, -(-Cout // bn)) if bn else fill_bn(Cout, -(-(Bn * H * W) // 128))
    cout_pad = padded_rows(Cout)         # rows of the packed weight; tiles past it read TMA zero fill
    ktot = taps * cpad + c2pad
    d.a_ptr = a_ptr
    cphys = 4 * cpad if s2d else C       # physical channel extent of the activation tensor
    d.a_dims[:] = [cphys, W, H, a_planes * Bn]
    d.a_strides[:] = [cphys * H16, W * cphys * H16, H * W * cphys * H16]
    d.a_box[:] = [64, bw, bh, bnn]
    d.a_plane_n = Bn
    d.a2_ptr = a2_ptr
    d.a2_c = C2
    d.a2_plane_n = Bn
    d.nkb_aux = c2pad // 64
    d.b_ptr = w_ptr
    d.b_dims[:] = [ktot, cout_pad, w_planes]
    d.b_strides[:] = [ktot * H16, cout_pad * ktot * H16]
    d.b_plane_batch = 1
    d.BN = BN
    d.m_tiles = -(-(Bn * H * W) // 128)
    d.n_tiles = n_tiles
    d.num_z = 1
    d.nh = 1
    d.taps = taps
    d.cpb = cpad // 64
    d.npass = npass
    d.a_mode = 0
    d.conv_H, d.conv_W = H, W
    if taps == 9:
        for t in range(9):
            kh, kw = t // 3, t % 3
            if s2d:     # stride-2 conv over a space-to-depth input: (shift, phase) of input offset kh-1 in {-1, 0, +1}
                sh, ph = [(-1, 1), (0, 0), (0, 1)][kh]
                sw, pw = [(-1, 1), (0, 0), (0, 1)][kw]
                d.tap_dh[t], d.tap_dw[t], d.tap_cb[t] = sh, sw, (ph * 2 + pw) * cpad
            else:
                d.tap_dh[t], d.tap_dw[t], d.tap_cb[t] = kh - 1, kw - 1, 0
    d.m_valid = Bn * H * W
    d.n_valid = Cout
    d.out_f32 = out_f32
    d.out_h16 = out_h16
    d.ldo = ldo if ldo is not None else Cout
    d.o_plane = (Bn * H * W * d.ldo) if (out_h16 and o_planes == 2) else 0
    d.bias_n = bias
    d.rowvec = rowvec
    d.rowvec_stride = rowvec_stride
    d.rows_per_sample = H * W
    d.residual = residual
    d.ldr = ldr if ldr is not None else Cout
    d.scale = scale
    d.f8 = 1 if f8 else 0
    d.acc_scale = acc_scale
    if edm is not None:
        d.edm_out = 1
        d.edm_x, d.edm_coef, d.edm_coef_stride, d.edm_C, d.edm_D = edm
    if nchw_out is not None:
        d.edm_out = 2
        d.edm_C, d.edm_D = nchw_out
    return d, dict(BN=BN, n_tiles=n_tiles, cout_pad=cout_pad, ktot=ktot)


def rows_gemm(a_ptr, a_rows, a_pitch, a_batches, b_ptr, b_rows, b_pitch, b_batches, K, *, num_z, nh=1, m_valid, n_valid,
              npass=3, a_planes=2, b_planes=2, a_c_per_zh=0, a_n_per_zb=0, a_n_per_zh=0, b_k0=0, b_k_per_zh=0, b_row_per_zh=0,
              b_z_per_zb=0, b_z_per_zh=0, out_f32=0, out_h16=0, o_zb=0, o_zh=0, ldo=0, o_plane=0, bias_n=0, bias_m=0,
              residual=0, ldr=0, scale=1.0, bn=None, a_k_valid=None, b_k_valid=None, relu=0):
    """Batched row-major product  D_z[m][n] = sum_k A_z[m][k] * B_z[n][k].
    A: fp16 planes [a_planes][a_batches][a_rows][a_pitch]; B: fp16 planes [b_planes][b_batches][b_rows][b_pitch].
    z = zb*nh + zh selects the batch entry / column window of each operand (see csrc/ops.h).  relu=1: max(v, 0) before the stores."""
    assert K % 64 == 0
    d = S.GemmDesc()
    BN, n_tiles = (bn, -(-n_valid // bn)) if bn else fill_bn(n_valid, -(-m_valid // 128), num_z)
    d.a_ptr = a_ptr
    d.a_dims[:] = [a_k_valid or a_pitch, a_rows, 1, a_planes * a_batches]       # K beyond the valid extent is zero-filled by TMA
    d.a_strides[:] = [a_pitch * H16, a_rows * a_pitch * H16, a_rows * a_pitch * H16]
    d.a_box[:] = [64, 128, 1, 1]
    d.a_plane_n = a_batches
    d.b_ptr = b_ptr
    d.b_dims[:] = [b_k_valid or b_pitch, b_rows, b_planes * b_batches]
    d.b_strides[:] = [b_pitch * H16, b_rows * b_pitch * H16]
    d.b_plane_batch = b_batches
    d.BN = BN
    d.m_tiles = -(-m_valid // 128)
    d.n_tiles = n_tiles
    d.num_z = num_z
    d.nh = nh
    d.taps = 1
    d.cpb = K // 64
    d.npass = npass
    d.a_mode = 1
    d.conv_H = d.conv_W = 1
    d.a_c_per_zh, d.a_n_per_zb, d.a_n_per_zh = a_c_per_zh, a_n_per_zb, a_n_per_zh
    d.b_k0, d.b_k_per_zh, d.b_row_per_zh, d.b_z_per_zb, d.b_z_per_zh = b_k0, b_k_per_zh, b_row_per_zh, b_z_per_zb, b_z_per_zh
    d.m_valid, d.n_valid = m_valid, n_valid
    d.out_f32, d.out_h16 = out_f32, out_h16
    d.o_zb, d.o_zh, d.ldo, d.o_plane = o_zb, o_zh, ldo, o_plane
    d.bias_n, d.bias_m = bias_n, bias_m
    d.rows_per_sample = 1
    d.residual, d.ldr = residual, ldr
    d.scale = scale
    d.relu = relu
    return d, dict(BN=BN, n_tiles=n_tiles)


def pack_conv_weight(weight, skip_weight=None, cin_pad=None, bn=None):
    """torch CPU: Conv2d weight [Cout, Cin, k, k] (+ optional 1x1 skip weight [Cout, C2, 1, 1]) ->
    fp16 planes [2][Cout_pad][taps*Cin_pad + C2], K ordered (kh, kw, cin) then the skip block."""
    import torch
    cout, cin, kh, kw = weight.shape
    cin_pad = cin_pad or -(-cin // 64) * 64
    w = torch.zeros(cout, kh, kw, cin_pad, dtype=torch.float32)
    w[..., :cin] = weight.detach().float().permute(0, 2, 3, 1)
    w = w.reshape(cout, kh * kw * cin_pad)
    if skip_weight is not None:
        c2 = skip_weight.shape[1]
        c2_pad = -(-c2 // 64) * 64
        sk = torch.zeros(cout, c2_pad, dtype=torch.float32)
        sk[:, :c2] = skip_weight.detach().float().reshape(cout, c2)
        w = torch.cat([w, sk], dim=1)
    BN, n_tiles = (bn, -(-cout // bn)) if bn else pick_bn(cout)
    cout_pad = BN * n_tiles
    wp = torch.zeros(cout_pad, w.shape[1], dtype=torch.float32)
    wp[:cout] = w
    hi = wp.half()
    lo = (wp - hi.float()).half()
    return torch.stack([hi, lo]).contiguous()


def describe(d):
    """Algorithmic work of one ds_gemm_desc launch (bench.py roofline): label, FLOPs (2 M N K over the valid extents, counted once per
    product whatever the number of precision passes) and the bytes the launch has to move through HBM when every operand is read
    once and every output written once: 4 B per A element in all layouts (fp16 hi + lo, or fp16 + 2 x e4m3), the packed weights,
    fp32 / fp16-plane outputs, the residual."""
    m, n, z = int(d.m_valid), int(d.n_valid), max(int(d.num_z), 1)
    k_main = int(d.taps) * int(d.cpb) * 64
    k_aux = int(d.a2_c)
    k = k_main + k_aux
    flops = 2.0 * m * n * k * z
    a_bytes = 4 * m * (int(d.cpb) * 64 + k_aux) * z if d.a_mode == 0 else 4 * m * k * z
    w_bytes = 4 * n * k * (z if d.a_mode == 1 else 1)
    out_bytes = m * n * z * ((4 if d.out_f32 else 0) + (4 if d.out_h16 and d.o_plane else (2 if d.out_h16 else 0)))
    if d.edm_out:
        out_bytes = 2 * 4 * m * int(d.edm_C)                       # read x, write D (NCHW fp32)
    res_bytes = 4 * m * n * z if d.residual else 0
    if d.a_mode == 0:
        label = f"conv{'3x3' if d.taps == 9 else '1x1'} {int(d.cpb) * 64}{'+' + str(k_aux) if k_aux else ''}->{n} @{int(d.conv_H)}x{int(d.conv_W)} x{m // max(int(d.conv_H) * int(d.conv_W), 1)}"
    else:
        label = f'gemm {m}x{n}x{k} z{z}'
    return dict(label=label + (' f8' if d.f8 & 1 else ''), flops=flops, bytes=float(a_bytes + w_bytes + out_bytes + res_bytes),
                m=m, n=n, k=k, z=z, f8=bool(d.f8 & 1))


E4M3_MAX = 448.0


def _e4m3_bytes(x, shift):
    """fp32 -> e4m3 (saturating, round to nearest even) of x * 2^shift, as uint8."""
    import torch
    return (x * 2.0 ** shift).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def f8_weight_shift(*weights):
    """S of an f8 GEMM (csrc/ops.h): the e4m3 copy of w_hi uses the largest power of two that keeps max|w| inside e4m3."""
    import math
    wmax = max(float(w.detach().abs().max()) for w in weights if w is not None)
    b1 = int(math.floor(math.log2(E4M3_MAX / wmax))) if wmax > 0 else 0
    return S.DS_F8_SH_LO8 + b1


def pack_conv_weight_f8(weight, skip_weight=None, bn=None):
    """Operand B of an f8 GEMM (csrc/ops.h): uint8 blob
        [fp16 (w * 2^b)][Cout_pad][taps*Cin64 + C2_64]  |  [2][Cout_pad][taps*Cin128 + C2_128] e4m3: (w_hi * 2^b1), (w_lo * 2^b2)
    with b = S - A16, b1 = S - LO8, b2 = S - HI8; K ordered (kh, kw, cin) per plane, channels padded per tap to 64 (fp16) or
    128 (e4m3).  Returns (blob, S); the GEMM's acc_scale is 2^-S."""
    import torch
    cout, cin, kh, kw = weight.shape
    Sh = f8_weight_shift(weight, skip_weight)
    b, b1, b2 = Sh - S.DS_F8_SH_A16, Sh - S.DS_F8_SH_LO8, Sh - S.DS_F8_SH_HI8
    BN, n_tiles = (bn, -(-cout // bn)) if bn else pick_bn(cout)
    cout_pad = BN * n_tiles

    def kmajor(t, pad):
        """[cout, cin, kh, kw] (+ skip [cout, c2, 1, 1]) fp32 -> [cout_pad, K] with per-tap channel padding to `pad`."""
        cp = -(-cin // pad) * pad
        w = torch.zeros(cout, kh, kw, cp, dtype=torch.float32)
        w[..., :cin] = t.permute(0, 2, 3, 1)
        w = w.reshape(cout, kh * kw * cp)
        return w

    def with_skip(main, skip, pad):
        w = kmajor(main, pad)
        if skip is not None:
            c2 = skip.shape[1]
            c2p = -(-c2 // pad) * pad
            sk = torch.zeros(cout, c2p, dtype=torch.float32)
            sk[:, :c2] = skip.reshape(cout, c2)
            w = torch.cat([w, sk], dim=1)
        out = torch.zeros(cout_pad, w.shape[1], dtype=torch.float32)
        out[:cout] = w
        return out

    wf = weight.detach().float()
    sf = skip_weight.detach().float() if skip_weight is not None else None
    hi16 = lambda t: (t * 2.0 ** b).clamp(-65504.0, 65504.0).half()
    w_hi = hi16(wf)
    s_hi = hi16(sf) if sf is not None else None
    w_hi_f = w_hi.float() / 2.0 ** b                              # the value the fp16 plane represents
    s_hi_f = s_hi.float() / 2.0 ** b if sf is not None else None
    plane16 = with_skip(w_hi.float(), s_hi.float() if sf is not None else None, 64).half()      # exact: already fp16 values
    hi8 = _e4m3_bytes(with_skip(w_hi_f, s_hi_f, 128), b1)
    lo8 = _e4m3_bytes(with_skip(wf - w_hi_f, (sf - s_hi_f) if sf is not None else None, 128), b2)
    blob = torch.cat([plane16.contiguous().view(torch.uint8).reshape(-1), hi8.reshape(-1), lo8.reshape(-1)]).contiguous()
    return blob, Sh


def act_planes_f8(x):
    """fp32 activations [..., C] -> the uint8 image of an f8 GEMM's A operand (csrc/ops.h): fp16 plane of x * 2^A16, then the e4m3
    planes (x - hi) * 2^LO8 and hi * 2^HI8.  This is what ds_gn_apply writes with fmt == 1; host copy for tests and documentation."""
    import torch
    hi = (x * 2.0 ** S.DS_F8_SH_A16).clamp(-65504.0, 65504.0).half()
    hf = hi.float() / 2.0 ** S.DS_F8_SH_A16
    lo8 = _e4m3_bytes(x - hf, S.DS_F8_SH_LO8)
    hi8 = _e4m3_bytes(hf, S.DS_F8_SH_HI8)
    return torch.cat([hi.contiguous().view(torch.uint8).reshape(-1), lo8.reshape(-1), hi8.reshape(-1)]).contiguous()


def decode_act_planes_f8(buf, shape):
    """Inverse view of act_planes_f8: (hi, lo8, hi8) as fp32 tensors of `shape`, unscaled."""
    import torch
    n = 1
    for d in shape:
        n *= d
    hi = buf[:2 * n].view(torch.float16).float().reshape(shape) / 2.0 ** S.DS_F8_SH_A16
    lo8 = buf[2 * n:3 * n].view(torch.float8_e4m3fn).float().reshape(shape) / 2.0 ** S.DS_F8_SH_LO8
    hi8 = buf[3 * n:4 * n].view(torch.float8_e4m3fn).float().reshape(shape) / 2.0 ** S.DS_F8_SH_HI8
    return hi, lo8, hi8


def decode_conv_weight_f8(blob, shift, cout, cin, taps, c2=0, bn=None):
    """Inverse view of pack_conv_weight_f8: the three weight planes as fp32 [cout, taps, cin] (+ skip [cout, c2]), unscaled."""
    import torch
    BN, n_tiles = (bn, -(-cout // bn)) if bn else pick_bn(cout)
    cout_pad = BN * n_tiles
    c64, c128 = -(-cin // 64) * 64, -(-cin // 128) * 128
    s64, s128 = -(-c2 // 64) * 64, -(-c2 // 128) * 128
    k16, k8 = taps * c64 + s64, taps * c128 + s128
    n16 = cout_pad * k16 * 2
    p16 = blob[:n16].view(torch.float16).float().reshape(cout_pad, k16) / 2.0 ** (shift - S.DS_F8_SH_A16)
    h8 = blob[n16:n16 + cout_pad * k8].view(torch.float8_e4m3fn).float().reshape(cout_pad, k8) / 2.0 ** (shift - S.DS_F8_SH_LO8)
    l8 = blob[n16 + cout_pad * k8:n16 + 2 * cout_pad * k8].view(torch.float8_e4m3fn).float().reshape(cout_pad, k8) / 2.0 ** (shift - S.DS_F8_SH_HI8)

    def cut(p, cp, sp):
        main = p[:cout, :taps * cp].reshape(cout, taps, cp)[:, :, :cin]
        skip = p[:cout, taps * cp:taps * cp + sp][:, :c2]
        return main, skip
    return cut(p16, c64, s64), cut(h8, c128, s128), cut(l8, c128, s128)


def split_planes(x):
    """fp32 tensor -> stacked fp16 (hi, lo) planes with hi + lo ~= x to ~2^-22."""
    import torch
    hi = x.half()
    lo = (x - hi.float()).half()
    return torch.stack([hi, lo]).contiguous()

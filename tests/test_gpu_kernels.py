"""Kernel-level parity (GPU): each hand-written kernel, called through the C ABI (ds_op_launch /
ds_solver_update / ds_dyn_threshold), against plain PyTorch fp32/fp64 math on the same inputs."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu



@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


def dev():
    return torch.device('cuda:0')


def sync():
    torch.cuda.synchronize()


def planes(x):
    from diff_sampler_b200.gemm_desc import split_planes
    return split_planes(x)


# --------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize('npass', [1, 3])
@pytest.mark.parametrize('M,N,K', [(128, 128, 64), (300, 200, 128), (1000, 384, 320), (64, 64, 64)])
def test_rows_gemm(lib, npass, M, N, K):
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(0)
    A = torch.randn(M, K, device=dev())
    Bm = torch.randn(N, K, device=dev())
    Ap, Bp = planes(A), planes(Bm)
    out = torch.full((M, N), float('nan'), device=dev())
    d, _ = G.rows_gemm(Ap.data_ptr(), M, K, 1, Bp.data_ptr(), N, K, 1, K, num_z=1, m_valid=M, n_valid=N, npass=npass,
                       out_f32=out.data_ptr(), ldo=N)
    lib.op_launch(d)
    sync()
    if npass == 1:
        ref = Ap[0].double() @ Bp[0].double().t()
        tol = 1e-4
    else:
        ref = A.double() @ Bm.double().t()
        tol = 2e-5
    err = (out.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f'rows_gemm npass={npass} M{M} N{N} K{K}: max err {err:.3e} (scale {scale:.2f})')
    assert not torch.isnan(out).any()
    assert err <= tol * scale


@pytest.mark.parametrize('npass', [1, 3])
@pytest.mark.parametrize('Bn,H,W,Cin,Cout', [(3, 32, 32, 64, 128), (3, 16, 16, 128, 192), (3, 8, 8, 64, 256), (2, 64, 64, 64, 64),
                                             (5, 8, 8, 128, 3)])
def test_conv3x3(lib, npass, Bn, H, W, Cin, Cout):
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(1)
    x = torch.randn(Bn, Cin, H, W, device=dev())
    w = torch.randn(Cout, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
    xa = planes(x.permute(0, 2, 3, 1).contiguous())                 # [2][Bn][H][W][C]
    wp = G.pack_conv_weight(w.cpu()).to(dev())
    out = torch.full((Bn * H * W, Cout), float('nan'), device=dev())
    d, info = G.conv_gemm(xa.data_ptr(), Bn, H, W, Cin, wp.data_ptr(), Cout, taps=9, npass=npass, out_f32=out.data_ptr())
    lib.op_launch(d)
    sync()
    if npass == 1:
        ref = F.conv2d(xa[0].permute(0, 3, 1, 2).double(), wp[0][:Cout].double().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2), padding=1)
        tol = 1e-4
    else:
        ref = F.conv2d(x.double(), w.double(), padding=1)
        tol = 2e-5
    ref = ref.permute(0, 2, 3, 1).reshape(Bn * H * W, Cout)
    err = (out.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f'conv3x3 npass={npass} {Bn}x{H}x{W} {Cin}->{Cout} BN={info["BN"]}: max err {err:.3e} (scale {scale:.2f})')
    assert not torch.isnan(out).any()
    assert err <= tol * scale


def test_conv_fused_epilogue(lib):
    """conv1 of a UNetBlock: 3x3 conv + 1x1 skip appended on K + bias + per-sample embedding + residual, * skip_scale,
    fp32 and fp16-plane outputs (networks_edm.py:169-171)."""
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(2)
    Bn, H, W, Cin, C2, Cout = 4, 16, 16, 128, 64, 128
    x = torch.randn(Bn, Cin, H, W, device=dev())
    orig = torch.randn(Bn, C2, H, W, device=dev())
    w = torch.randn(Cout, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
    ws = torch.randn(Cout, C2, 1, 1, device=dev()) / C2 ** 0.5
    bias = torch.randn(Cout, device=dev())
    emb = torch.randn(Bn, Cout, device=dev())
    res = torch.randn(Bn, Cout, H, W, device=dev())
    xa = planes(x.permute(0, 2, 3, 1).contiguous())
    oa = planes(orig.permute(0, 2, 3, 1).contiguous())
    wp = G.pack_conv_weight(w.cpu(), ws.cpu()).to(dev())
    res_nhwc = res.permute(0, 2, 3, 1).contiguous()
    out = torch.full((Bn * H * W, Cout), float('nan'), device=dev())
    out_h = torch.zeros(2, Bn * H * W, Cout, dtype=torch.float16, device=dev())
    d, _ = G.conv_gemm(xa.data_ptr(), Bn, H, W, Cin, wp.data_ptr(), Cout, taps=9, npass=3, a2_ptr=oa.data_ptr(), C2=C2,
                       out_f32=out.data_ptr(), out_h16=out_h.data_ptr(), bias=bias.data_ptr(), rowvec=emb.data_ptr(),
                       rowvec_stride=Cout, residual=res_nhwc.data_ptr(), scale=0.70710678)
    lib.op_launch(d)
    sync()
    ref = F.conv2d(x.double(), w.double(), padding=1) + F.conv2d(orig.double(), ws.double())
    ref = (ref + bias.double()[None, :, None, None] + emb.double()[:, :, None, None] + res.double()) * 0.70710678
    ref = ref.permute(0, 2, 3, 1).reshape(Bn * H * W, Cout)
    err = (out.double() - ref).abs().max().item()
    errh = ((out_h[0].double() + out_h[1].double()) - ref).abs().max().item()
    print(f'fused epilogue: f32 err {err:.3e}  h16-planes err {errh:.3e}')
    assert err < 5e-5 * ref.abs().max().item()
    assert errh < 5e-5 * ref.abs().max().item()


@pytest.mark.parametrize('L,d,nh', [(256, 256, 1), (64, 64, 3), (1024, 64, 2)])
def test_attention_gemms(lib, L, d, nh):
    """S = Q K^T / sqrt(d) and O = P V through the batched rows mode (networks_edm.py:108, :176)."""
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(3)
    Bn = 2
    Cc = nh * d
    qk = torch.randn(Bn, L, 2 * Cc, device=dev())          # [b][l][q heads | k heads]
    vt = torch.randn(Bn, Cc, L, device=dev())              # V^T: [b][head*d + c][l]
    qkp, vtp = planes(qk), planes(vt)
    Smat = torch.full((Bn * nh, L, L), float('nan'), device=dev())
    scale = 1.0 / d ** 0.5
    dS, _ = G.rows_gemm(qkp.data_ptr(), L, 2 * Cc, Bn, qkp.data_ptr(), L, 2 * Cc, Bn, d, num_z=Bn * nh, nh=nh, m_valid=L, n_valid=L,
                        a_c_per_zh=d, a_n_per_zb=1, b_k0=Cc, b_k_per_zh=d, b_z_per_zb=1, out_f32=Smat.data_ptr(),
                        o_zb=nh * L * L, o_zh=L * L, ldo=L, scale=scale)
    lib.op_launch(dS)
    sync()
    q = qk[:, :, :Cc].reshape(Bn, L, nh, d).permute(0, 2, 1, 3).double()
    k = qk[:, :, Cc:].reshape(Bn, L, nh, d).permute(0, 2, 1, 3).double()
    refS = (q @ k.transpose(-1, -2) * scale).reshape(Bn * nh, L, L)
    errS = (Smat.double() - refS).abs().max().item()
    print(f'QK^T L{L} d{d} nh{nh}: err {errS:.3e}')
    assert errS < 3e-5 * refS.abs().max().item()

    Pm = torch.softmax(Smat, dim=-1)
    Pp = planes(Pm)
    O = torch.zeros(2, Bn, L, Cc, dtype=torch.float16, device=dev())
    dO, _ = G.rows_gemm(Pp.data_ptr(), L, L, Bn * nh, vtp.data_ptr(), Cc, L, Bn, L, num_z=Bn * nh, nh=nh, m_valid=L, n_valid=d,
                        a_n_per_zb=nh, a_n_per_zh=1, b_row_per_zh=d, b_z_per_zb=1, out_h16=O.data_ptr(), o_zb=L * Cc, o_zh=d,
                        ldo=Cc, o_plane=Bn * L * Cc)
    lib.op_launch(dO)
    sync()
    v = vt.reshape(Bn, nh, d, L).double()
    refO = (Pm.reshape(Bn, nh, L, L).double() @ v.transpose(-1, -2)).permute(0, 2, 1, 3).reshape(Bn, L, Cc)
    errO = ((O[0].double() + O[1].double()) - refO).abs().max().item()
    print(f'PV   L{L} d{d} nh{nh}: err {errO:.3e}')
    assert errO < 3e-5 * max(1.0, refO.abs().max().item())


def test_vt_gemm_bias_m(lib):
    """V^T = Wv . n2^T with the weight as the M operand and a bias along M."""
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(4)
    Bn, L, Cc = 3, 64, 192
    Wv = torch.randn(Cc, Cc, device=dev()) / Cc ** 0.5
    bv = torch.randn(Cc, device=dev())
    n2 = torch.randn(Bn, L, Cc, device=dev())
    Wp, n2p = planes(Wv), planes(n2)
    Vt = torch.zeros(2, Bn, Cc, L, dtype=torch.float16, device=dev())
    dV, _ = G.rows_gemm(Wp.data_ptr(), Cc, Cc, 1, n2p.data_ptr(), L, Cc, Bn, Cc, num_z=Bn, nh=1, m_valid=Cc, n_valid=L,
                        b_z_per_zb=1, out_h16=Vt.data_ptr(), o_zb=Cc * L, ldo=L, o_plane=Bn * Cc * L, bias_m=bv.data_ptr())
    lib.op_launch(dV)
    sync()
    ref = (Wv.double() @ n2.double().transpose(1, 2)) + bv.double()[None, :, None]
    err = ((Vt[0].double() + Vt[1].double()) - ref).abs().max().item()
    print(f'Vt gemm err {err:.3e}')
    assert err < 3e-5 * ref.abs().max().item()


def test_edm_output_fold(lib):
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(5)
    Bn, H, W, Cin, Cimg = 3, 16, 16, 128, 3
    a = torch.randn(Bn, Cin, H, W, device=dev())
    w = torch.randn(Cimg, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
    b = torch.randn(Cimg, device=dev())
    x = torch.randn(Bn, Cimg, H, W, device=dev())
    coef = torch.rand(Bn, 4, device=dev()) + 0.5
    xa = planes(a.permute(0, 2, 3, 1).contiguous())
    wp = G.pack_conv_weight(w.cpu()).to(dev())
    D = torch.full((Bn, Cimg, H, W), float('nan'), device=dev())
    d, _ = G.conv_gemm(xa.data_ptr(), Bn, H, W, Cin, wp.data_ptr(), Cimg, taps=9, npass=3, bias=b.data_ptr(),
                       edm=(x.data_ptr(), coef.data_ptr(), 4, Cimg, D.data_ptr()))
    lib.op_launch(d)
    sync()
    Fx = F.conv2d(a.double(), w.double(), b.double(), padding=1)
    ref = coef[:, 0].double()[:, None, None, None] * x.double() + coef[:, 1].double()[:, None, None, None] * Fx
    err = (D.double() - ref).abs().max().item()
    print(f'edm fold err {err:.3e}')
    assert err < 3e-5 * ref.abs().max().item()


# --------------------------------------------------------------------------------------------- GroupNorm
@pytest.mark.parametrize('C0,C1,H,W,resample,ada,silu', [
    (128, 0, 16, 16, 0, False, True), (256, 128, 8, 8, 0, False, True), (192, 0, 16, 16, 1, True, True),
    (576, 384, 8, 8, 2, True, True), (256, 0, 32, 32, 0, False, False), (1344, 0, 8, 8, 0, False, True)])
def test_groupnorm_apply(lib, C0, C1, H, W, resample, ada, silu):
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(6)
    Bn, Cc, G = 3, C0 + C1, 32
    x0 = torch.randn(Bn, H, W, C0, device=dev()) * 1.7 + 0.3
    x1 = torch.randn(Bn, H, W, C1, device=dev()) * 0.6 - 0.2 if C1 else None
    gamma = torch.randn(Cc, device=dev())
    beta = torch.randn(Cc, device=dev())
    adav = torch.randn(Bn, 2 * Cc, device=dev()) * 0.3 if ada else None
    sums = torch.zeros(Bn, G, 2, dtype=torch.float64, device=dev())
    ds = S.GnStatsDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, HW=H * W, B=Bn, groups=G,
                       sums=sums.data_ptr())
    lib.op_launch(ds)
    Ho, Wo = (H // 2, W // 2) if resample == 1 else ((H * 2, W * 2) if resample == 2 else (H, W))
    act = torch.zeros(2, Bn, Ho, Wo, Cc, dtype=torch.float16, device=dev())
    raw = torch.zeros(2, Bn, Ho, Wo, Cc, dtype=torch.float16, device=dev())
    rawf = torch.zeros(Bn, Ho, Wo, Cc, device=dev())
    da = S.GnApplyDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, H=H, W=W, B=Bn, groups=G,
                       sums=sums.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-6, silu=int(silu),
                       ada=adav.data_ptr() if ada else 0, ada_stride=2 * Cc if ada else 0, resample=resample, nplanes=2,
                       out_act=act.data_ptr(), out_raw=raw.data_ptr(), out_raw_f32=rawf.data_ptr())
    lib.op_launch(da)
    sync()
    xc = torch.cat([x0, x1], dim=-1) if C1 else x0
    xn = xc.permute(0, 3, 1, 2).double()
    y = F.group_norm(xn, G, gamma.double(), beta.double(), eps=1e-6)
    if ada:
        sc, sh = adav[:, :Cc].double(), adav[:, Cc:].double()
        y = y * (sc[:, :, None, None] + 1) + sh[:, :, None, None]
    if silu:
        y = F.silu(y)
    r = xn
    if resample == 1:
        y, r = F.avg_pool2d(y, 2), F.avg_pool2d(r, 2)
    elif resample == 2:
        y, r = F.interpolate(y, scale_factor=2, mode='nearest'), F.interpolate(r, scale_factor=2, mode='nearest')
    y, r = y.permute(0, 2, 3, 1), r.permute(0, 2, 3, 1)
    e_act = ((act[0].double() + act[1].double()) - y).abs().max().item()
    e_raw = ((raw[0].double() + raw[1].double()) - r).abs().max().item()
    e_rawf = (rawf.double() - r).abs().max().item()
    print(f'gn C{C0}+{C1} {H}x{W} rs{resample} ada{ada}: act {e_act:.2e} raw {e_raw:.2e} rawf {e_rawf:.2e}')
    assert e_act < 2e-5 * max(1.0, y.abs().max().item())
    assert e_raw < 1e-5 and e_rawf < 1e-6


def test_softmax(lib):
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(7)
    for L in (64, 256, 1024, 2048, 4096, 8192):
        Sm = torch.randn(37, L, device=dev()) * 4
        Pm = torch.zeros(2, 37, L, dtype=torch.float16, device=dev())
        lib.op_launch(S.SoftmaxDesc(S=Sm.data_ptr(), P=Pm.data_ptr(), rows=37, L=L, nplanes=2))
        sync()
        ref = torch.softmax(Sm.double(), -1)
        err = ((Pm[0].double() + Pm[1].double()) - ref).abs().max().item()
        print(f'softmax L{L}: {err:.2e}')
        assert err < 2e-6


def test_posemb_linear_prep(lib):
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(8)
    sig = torch.tensor([80.0, 3.3, 0.002, 0.7], device=dev())
    nc = 128
    coef = torch.zeros(4, 4, device=dev())
    emb = torch.zeros(4, nc, device=dev())
    lib.op_launch(S.PosembDesc(sigma=sig.data_ptr(), nsig=4, num_channels=nc, endpoint=1, swap_sincos=1, sigma_data=0.5,
                               coef=coef.data_ptr(), emb=emb.data_ptr()))
    sync()
    cn = sig.log() / 4
    freqs = (1 / 10000) ** (torch.arange(nc // 2, device=dev(), dtype=torch.float32) / (nc // 2 - 1))
    e = cn.ger(freqs)
    ref = torch.cat([e.sin(), e.cos()], dim=1)
    assert (emb - ref).abs().max().item() < 2e-6
    s2 = sig ** 2 + 0.25
    refc = torch.stack([0.25 / s2, sig * 0.5 / s2.sqrt(), 1 / s2.sqrt(), cn], dim=1)
    assert ((coef - refc).abs() / refc.abs().clamp_min(1e-3)).max().item() < 1e-6

    Wt = torch.randn(300, nc, device=dev()) / nc ** 0.5
    b = torch.randn(300, device=dev())
    out = torch.zeros(4, 300, device=dev())
    lib.op_launch(S.LinearDesc(in_=emb.data_ptr(), in_stride=nc, W=Wt.data_ptr(), b=b.data_ptr(), add=0, add_stride=0,
                               out=out.data_ptr(), n_rows=4, in_f=nc, out_f=300, act=1, in_scale=1.0))
    sync()
    refl = F.silu(emb.double() @ Wt.double().t() + b.double())
    assert (out.double() - refl).abs().max().item() < 1e-5

    x = torch.randn(4, 3, 8, 8, device=dev()) * 10
    o = torch.zeros(2, 4, 64, 64, dtype=torch.float16, device=dev())
    lib.op_launch(S.PrepInputDesc(x=x.data_ptr(), coef=coef.data_ptr(), coef_stride=4, B=4, C=3, HW=64, nplanes=2, out=o.data_ptr()))
    sync()
    refx = (x * coef[:, 2][:, None, None, None]).permute(0, 2, 3, 1).reshape(4, 64, 3).double()
    got = o[0].double() + o[1].double()
    assert (got[:, :, :3] - refx).abs().max().item() < 1e-5
    assert got[:, :, 3:].abs().max().item() == 0


@pytest.mark.parametrize('Bn,H,W,Cout,groups_cat', [(3, 16, 16, 128, 32), (5, 8, 8, 192, 32), (2, 32, 32, 256, 32), (2, 8, 8, 48, 12)])
def test_conv_epilogue_fused_groupnorm_stats(lib, Bn, H, W, Cout, groups_cat):
    """The GEMM epilogue stores, per 32-row slab and channel quad, the {sum, sumsq} partials of the tensor it writes; ds_gn_finalize
    folds them into the per-(sample, group) sums gn_apply reads -- for the tensor alone and as one part of a decoder concat (where a
    group may straddle the two sources, e.g. 192 + 192 channels in 12-wide groups)."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(11)
    Cin = 64
    x = torch.randn(Bn, Cin, H, W, device=dev())
    w = torch.randn(Cout, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
    bias = torch.randn(Cout, device=dev())
    xa = planes(x.permute(0, 2, 3, 1).contiguous())
    wp = G.pack_conv_weight(w.cpu()).to(dev())
    M = Bn * H * W
    out = torch.zeros(M, Cout, device=dev())
    slabs = M // 32
    quads = torch.full((slabs, Cout // 4, 2), float('nan'), device=dev())
    d, _ = G.conv_gemm(xa.data_ptr(), Bn, H, W, Cin, wp.data_ptr(), Cout, taps=9, npass=3, out_f32=out.data_ptr(), bias=bias.data_ptr(),
                       scale=0.5)
    d.st_quads = quads.data_ptr()
    lib.op_launch(d)
    sync()
    y = out.double()
    ys = y.reshape(slabs, 32, Cout // 4, 4)
    rq = torch.stack([ys.sum(dim=(1, 3)), (ys ** 2).sum(dim=(1, 3))], dim=-1)
    eq = (quads.double() - rq).abs().max().item()
    assert eq < 1e-4 * max(1.0, rq.abs().max().item()), eq
    # finalize: the tensor alone (groups = min(32, C/4) as the EDM nets use) ...
    g1 = min(32, Cout // 4)
    while (Cout // g1) % 4:
        g1 //= 2
    sums = torch.full((Bn, g1, 2), float('nan'), dtype=torch.float64, device=dev())
    lib.op_launch(S.GnFinalizeDesc(quads0=quads.data_ptr(), quads1=0, C0=Cout, C1=0, slabs_per_sample=H * W // 32, B=Bn, groups=g1,
                                   sums=sums.data_ptr()))
    yb = y.reshape(Bn, H * W, g1, Cout // g1)
    r1 = torch.stack([yb.sum(dim=(1, 3)), (yb ** 2).sum(dim=(1, 3))], dim=-1)
    # ... and as the first half of a concat [this tensor | this tensor again]
    sums2 = torch.full((Bn, groups_cat, 2), float('nan'), dtype=torch.float64, device=dev())
    lib.op_launch(S.GnFinalizeDesc(quads0=quads.data_ptr(), quads1=quads.data_ptr(), C0=Cout, C1=Cout, slabs_per_sample=H * W // 32, B=Bn,
                                   groups=groups_cat, sums=sums2.data_ptr()))
    sync()
    yc = torch.cat([y, y], dim=1).reshape(Bn, H * W, groups_cat, 2 * Cout // groups_cat)
    r2 = torch.stack([yc.sum(dim=(1, 3)), (yc ** 2).sum(dim=(1, 3))], dim=-1)
    e1 = (sums - r1).abs().max().item()
    e2 = (sums2 - r2).abs().max().item()
    print(f'fused stats: quad partials err {eq:.3e}, finalize err {e1:.3e} / concat {e2:.3e} (max {r2.abs().max().item():.1f})')
    assert e1 < 1e-4 * max(1.0, r1.abs().max().item()) and e2 < 1e-4 * max(1.0, r2.abs().max().item())


@pytest.mark.parametrize('Bn,H,W,Cout,C1,u1', [(3, 16, 16, 192, 0, 4), (2, 8, 8, 576, 0, 4), (2, 16, 16, 128, 64, 2), (4, 8, 8, 192, 144, 4), (2, 32, 32, 48, 0, 4)])
def test_conv_epilogue_pair_partials_for_even_groups(lib, Bn, H, W, Cout, C1, u1):
    """Round 2: ds_gemm_desc.st_unit = 2 stores the GroupNorm partials per channel PAIR, so that consumers whose groups are even but not
    multiples of four channels (ADM: 192 / 32 = 6, 576 / 32 = 18; concatenations: (128 + 64) / 32 = 6 with a group straddling the two
    sources at a pair boundary, (192 + 144) / 28 = 12) get their statistics from the GEMM epilogue too.  The second source may be a
    quad-partial buffer (a producer keeps quads when all ITS consumers allow them): mixed units in one finalize."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(12)
    Cin = 64
    M = Bn * H * W
    slabs = M // 32

    def conv_with_partials(Cc, unit):
        x = torch.randn(Bn, Cin, H, W, device=dev())
        w = torch.randn(Cc, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
        out = torch.zeros(M, Cc, device=dev())
        part = torch.full((slabs, Cc // unit, 2), float('nan'), device=dev())
        d, _ = G.conv_gemm(planes(x.permute(0, 2, 3, 1).contiguous()).data_ptr(), Bn, H, W, Cin, G.pack_conv_weight(w.cpu()).to(dev()).data_ptr(), Cc,
                           taps=9, npass=3, out_f32=out.data_ptr(), scale=0.7)
        d.st_quads, d.st_unit = part.data_ptr(), unit
        lib.op_launch(d)
        sync()
        y = out.double()
        ys = y.reshape(slabs, 32, Cc // unit, unit)
        ref = torch.stack([ys.sum(dim=(1, 3)), (ys ** 2).sum(dim=(1, 3))], dim=-1)
        err = (part.double() - ref).abs().max().item()
        assert err < 1e-4 * max(1.0, ref.abs().max().item()), (Cc, unit, err)
        return y, part
    y0, p0 = conv_with_partials(Cout, 2)
    if C1:
        y1, p1 = conv_with_partials(C1, u1)
    Cc = Cout + C1
    groups = min(32, Cc // 4)
    while Cc % groups:
        groups -= 1
    sums = torch.full((Bn, groups, 2), float('nan'), dtype=torch.float64, device=dev())
    lib.op_launch(S.GnFinalizeDesc(quads0=p0.data_ptr(), quads1=p1.data_ptr() if C1 else 0, C0=Cout, C1=C1, slabs_per_sample=H * W // 32, B=Bn,
                                   groups=groups, unit0=2, unit1=u1, sums=sums.data_ptr()))
    sync()
    yc = (torch.cat([y0, y1], dim=1) if C1 else y0).reshape(Bn, H * W, groups, Cc // groups)
    ref = torch.stack([yc.sum(dim=(1, 3)), (yc ** 2).sum(dim=(1, 3))], dim=-1)
    err = (sums - ref).abs().max().item()
    print(f'pair partials C{Cout}+{C1} groups {groups} ({Cc // groups} channels each): finalize err {err:.3e} (max {ref.abs().max().item():.1f})')
    assert err < 1e-4 * max(1.0, ref.abs().max().item())


def test_fused_stats_rejects_partial_slabs(lib):
    """st_quads needs whole 32-row slabs (here M = 2*4*4 = 32 is fine, 3*4*4 = 48 is not): rc -14, surfaced as DsError."""
    from diff_sampler_b200 import gemm_desc as G
    for Bn, ok_ in ((2, True), (3, False)):
        x = planes(torch.randn(Bn, 4, 4, 64, device=dev()))
        wp = G.pack_conv_weight(torch.randn(64, 64, 3, 3)).to(dev())
        out = torch.zeros(Bn * 16, 64, device=dev())
        quads = torch.zeros(Bn * 16 // 32 + 1, 16, 2, device=dev())
        d, _ = G.conv_gemm(x.data_ptr(), Bn, 4, 4, 64, wp.data_ptr(), 64, taps=9, npass=3, out_f32=out.data_ptr())
        d.st_quads = quads.data_ptr()
        if ok_:
            lib.op_launch(d)
        else:
            with pytest.raises(lib.DsError):
                lib.op_launch(d)
    sync()


# --------------------------------------------------------------------------------------------- fused attention
@pytest.mark.parametrize('B,nh,L,Lk,d', [(2, 3, 256, 256, 64), (1, 2, 192, 77, 40), (3, 1, 64, 64, 64), (1, 8, 1024, 1024, 40),
                                         (2, 2, 320, 200, 64),
                                         # more tiles than SMs (192 > 132), an odd key-block count (3), a single key block,
                                         # many short tiles (L = 64: 300 tiles)
                                         (4, 6, 1024, 1024, 64), (2, 2, 320, 192, 64), (1, 3, 128, 64, 64), (50, 6, 64, 64, 64), (3, 5, 200, 130, 40)])
def test_fused_attention(lib, B, nh, L, Lk, d):
    _fused_attention(lib, B, nh, L, Lk, d, causal=False)


@pytest.mark.parametrize('B,nh,L,d', [(3, 12, 77, 64), (2, 2, 64, 64), (1, 3, 200, 40), (2, 4, 1024, 64), (5, 1, 9, 64)])
def test_fused_attention_causal(lib, B, nh, L, d):
    """Causal self-attention (CLIP text encoder): query l sees keys <= l.  77 tokens put rows without any visible key into the second
    softmax group (weight 2^-inf in the merge); 1024 exercises rows whose later key blocks are entirely masked."""
    _fused_attention(lib, B, nh, L, L, d, causal=True)


def test_fused_attention_long_keys(lib):
    """4096 keys (the SD-1.5 64x64 self-attention, 40-wide heads) with values of non-zero mean: the P V product adds up over the
    whole key range.  Accumulated in one wgmma accumulator its fp32 error grew linearly with the key count and reached 3.4e-5 of
    max |out| on the plan's own activations; each 64-key block now has its own accumulator."""
    _fused_attention(lib, 2, 2, 4096, 4096, 40, causal=False, v_mean=1.0)


def _fused_attention(lib, B, nh, L, Lk, d, causal, v_mean=0.0):
    """attn_kernel (QK^T -> online softmax -> PV in one kernel, head dim padded to 64) against float64 softmax attention on the
    same fp16 hi+lo operands: self-attention shapes, a cross-attention shape (77 keys, pitch 80), partial query / key tiles."""
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(5)
    hp = nh * 64
    q = torch.randn(B, nh, L, d, device=dev()) * 1.5
    k = torch.randn(B, nh, Lk, d, device=dev()) * 1.5
    v = torch.randn(B, nh, Lk, d, device=dev()) + v_mean
    k[:, :, 3] *= 4.0                                    # a dominant key: peaky rows
    scale = d ** -0.5
    qk = torch.zeros(B, max(L, Lk), 2 * hp, device=dev())
    for h in range(nh):
        qk[:, :L, h * 64:h * 64 + d] = q[:, h]
        qk[:, :Lk, hp + h * 64:hp + h * 64 + d] = k[:, h]
    self_attn = (L == Lk)
    if self_attn:
        qa = planes(qk)                                  # [2][B][L][2*hp]: q and k side by side as the nets store them
        q_ptr = k_ptr = qa.data_ptr()
        q_pitch = k_pitch = 2 * hp
        q_c0, k_c0 = 0, hp
    else:
        qa = planes(qk[:, :L, :hp].contiguous())
        ka = planes(qk[:, :Lk, hp:].contiguous())
        q_ptr, k_ptr, q_pitch, k_pitch, q_c0, k_c0 = qa.data_ptr(), ka.data_ptr(), hp, hp, 0, 0
    vt_pitch = (Lk + 7) // 8 * 8
    vt = torch.zeros(B, hp, vt_pitch, device=dev())
    for h in range(nh):
        vt[:, h * 64:h * 64 + d, :Lk] = v[:, h].transpose(1, 2)
    vta = planes(vt)
    out = torch.full((2, B, L, hp), float('nan'), dtype=torch.float16, device=dev())
    lib.op_launch(S.AttnDesc(q=q_ptr, k=k_ptr, vt=vta.data_ptr(), out=out.data_ptr(), B=B, nh=nh, L=L, Lk=Lk, q_pitch=q_pitch, q_c0=q_c0,
                             k_pitch=k_pitch, k_c0=k_c0, vt_pitch=vt_pitch, o_pitch=hp, nplanes=2, scale=scale, causal=int(causal)))
    sync()
    got = (out[0].double() + out[1].double()).reshape(B, L, nh, 64).permute(0, 2, 1, 3)
    # reference on the operands as the kernel sees them (hi + lo), float64
    qd = (planes(q)[0].double() + planes(q)[1].double())
    kd = (planes(k)[0].double() + planes(k)[1].double())
    vd = (planes(v)[0].double() + planes(v)[1].double())
    sc = scale * qd @ kd.transpose(-1, -2)
    if causal:
        sc = sc + torch.full((L, Lk), float('-inf'), dtype=torch.float64, device=dev()).triu(1)
    ref = torch.softmax(sc, dim=-1) @ vd
    err = (got[..., :d] - ref).abs().max().item()
    pad = got[..., d:].abs().max().item() if d < 64 else 0.0
    print(f'fused attention B{B} nh{nh} L{L} Lk{Lk} d{d} causal={causal}: err {err:.3e} (max {ref.abs().max().item():.2f}), pad {pad:.1e}')
    assert err < 2e-5 * max(1.0, ref.abs().max().item()) and pad == 0.0


@pytest.mark.parametrize('C0,C1,H,W,ada,fmt,Bn', [(128, 0, 16, 16, False, 0, 3), (256, 128, 8, 8, False, 0, 5), (192, 0, 16, 16, True, 0, 3),
                                                  (256, 0, 32, 32, False, 1, 40), (576, 384, 8, 8, True, 1, 7), (1344, 0, 8, 8, False, 0, 2),
                                                  (320, 0, 32, 32, False, 0, 16)])
def test_groupnorm_coefficient_table_and_persistent_apply(lib, C0, C1, H, W, ada, fmt, Bn):
    """Round 2: gn_finalize also writes the per-(sample, channel) coefficients y = x * a + b (ds_gn_finalize_desc.coef), and gn_apply with
    ds_gn_apply_desc.coef runs the persistent, evenly split kernel (gn_apply_v3) without the fp64 prologue.  The arithmetic is the one of
    the sums-based kernel (a = rstd * gamma * (1 + scale), b = beta * (1 + scale) + shift - mean * a in fp32), so the outputs must be
    IDENTICAL to the round-1 path on the same statistics -- for hi/lo planes and for the f8 operand image, with and without a second
    source, for channel counts whose 8-channel thread columns do not divide the 256-thread block evenly (192, 1344) and for 10-channel
    groups (C = 320: the LDM GroupNorm32 case, statistics from the separate pass)."""
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(16)
    Cc, G = C0 + C1, 32
    x0 = torch.randn(Bn, H, W, C0, device=dev()) * 1.7 + 0.3
    x1 = torch.randn(Bn, H, W, C1, device=dev()) * 0.6 - 0.2 if C1 else None
    gamma, beta = torch.randn(Cc, device=dev()), torch.randn(Cc, device=dev())
    adav = torch.randn(Bn, 2 * Cc, device=dev()) * 0.3 if ada else None
    sums = torch.zeros(Bn, G, 2, dtype=torch.float64, device=dev())
    lib.op_launch(S.GnStatsDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, HW=H * W, B=Bn, groups=G, sums=sums.data_ptr()))
    coef = torch.full((Bn, Cc, 2), float('nan'), device=dev())
    lib.op_launch(S.GnFinalizeDesc(quads0=0, quads1=0, C0=C0, C1=C1, slabs_per_sample=0, B=Bn, groups=G, sums=sums.data_ptr(),
                                   gamma=gamma.data_ptr(), beta=beta.data_ptr(), ada=adav.data_ptr() if ada else 0, ada_stride=2 * Cc if ada else 0,
                                   eps=1e-6, HW=H * W, coef=coef.data_ptr()))
    outs = []
    for use_coef in (False, True):
        act = torch.zeros(2, Bn, H, W, Cc, dtype=torch.float16, device=dev())
        raw = torch.zeros(2, Bn, H, W, Cc, dtype=torch.float16, device=dev())
        lib.op_launch(S.GnApplyDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, H=H, W=W, B=Bn, groups=G,
                                    sums=0 if use_coef else sums.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-6, silu=1,
                                    ada=adav.data_ptr() if ada else 0, ada_stride=2 * Cc if ada else 0, resample=0, nplanes=2,
                                    out_act=act.data_ptr(), out_raw=raw.data_ptr(), out_raw_f32=0, fmt=fmt, coef=coef.data_ptr() if use_coef else 0))
        sync()
        outs.append((act, raw))
    assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16)), 'normalised planes differ between the sums and the coefficient path'
    assert torch.equal(outs[0][1].view(torch.int16), outs[1][1].view(torch.int16))
    # and the table itself against float64 GroupNorm algebra
    xc = (torch.cat([x0, x1], dim=-1) if C1 else x0).double().reshape(Bn, H * W, G, Cc // G)
    mu = xc.mean(dim=(1, 3))
    var = xc.var(dim=(1, 3), unbiased=False)
    rstd = (1.0 / torch.sqrt(var + 1e-6)).repeat_interleave(Cc // G, dim=1)
    a = rstd * gamma.double()[None]
    b = beta.double()[None].expand(Bn, Cc)
    if ada:
        a = a * (adav[:, :Cc].double() + 1)
        b = b * (adav[:, :Cc].double() + 1) + adav[:, Cc:].double()
    b = b - mu.repeat_interleave(Cc // G, dim=1) * a
    ea, eb = (coef[:, :, 0].double() - a).abs().max().item(), (coef[:, :, 1].double() - b).abs().max().item()
    print(f'gn coef C{C0}+{C1} {H}x{W} B{Bn} ada{ada} fmt{fmt}: identical planes; table err a {ea:.2e} b {eb:.2e}')
    assert ea < 1e-5 * a.abs().max().item() and eb < 1e-5 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize('sd,st', [(0.01, 0.2), (0.0, 0.2), (0.05, 0.0), (0.0, 0.0)])
def test_amed_predictor_kernel(lib, sd, st):
    """ds_amed_predict: the whole AMED predictor + t_mid in one launch, against the torch forward of the same weights
    (amed-solver-main/training/networks.py:121-155; solvers_amed.py:119 for t_mid)."""
    from diff_sampler_b200.amed_predictor import AMEDPredictor
    g = torch.Generator().manual_seed(31)
    W = {'map_layer0.weight': torch.randn(8, 8, generator=g) * 0.5, 'map_layer0.bias': torch.randn(8, generator=g) * 0.1,
         'enc_layer0.weight': torch.randn(128, 64, generator=g) * 0.2, 'enc_layer0.bias': torch.randn(128, generator=g) * 0.1,
         'enc_layer1.weight': torch.randn(4, 128, generator=g) * 0.2, 'enc_layer1.bias': torch.randn(4, generator=g) * 0.1,
         'fc_r.weight': torch.randn(1, 20, generator=g) * 0.4, 'fc_r.bias': torch.randn(1, generator=g) * 0.1}
    if sd:
        W.update({'fc_scale_dir.weight': torch.randn(1, 20, generator=g) * 0.4, 'fc_scale_dir.bias': torch.randn(1, generator=g) * 0.1})
    if st:
        W.update({'fc_scale_time.weight': torch.randn(1, 20, generator=g) * 0.4, 'fc_scale_time.bias': torch.randn(1, generator=g) * 0.1})
    pred = AMEDPredictor(W, scale_dir=sd, scale_time=st).to(dev())
    B = 7
    ts = torch.tensor([80.0, 14.6, 3.1, 0.5, 0.03, 0.002], device=dev())
    for i in range(len(ts) - 1):
        for afs in (False, True):
            enc = None if afs else torch.randn(B, 8, 8, generator=g).to(dev()) * 0.7
            got = pred.predict_native(enc, ts[i], ts[i + 1], B)
            ref = pred(enc if enc is not None else torch.zeros(B, 8, 8, device=dev()), ts[i].reshape(-1, 1, 1, 1), ts[i + 1].reshape(-1, 1, 1, 1))
            ref = list(ref) if isinstance(ref, (tuple, list)) else [ref]
            r = ref[0].reshape(-1)
            rsd = ref[1].reshape(-1) if sd else torch.ones(B, device=dev())
            rst = ref[-1].reshape(-1) if st else torch.ones(B, device=dev())
            tmid = (ts[i + 1] ** r) * (ts[i] ** (1 - r))
            for name, a, b in (('r', got[0], r), ('scale_dir', got[1], rsd), ('scale_time', got[2], rst), ('t_mid', got[3], tmid)):
                err = ((a - b).abs() / b.abs().clamp_min(1e-3)).max().item()
                assert err < 2e-5, (name, i, afs, err)
    sync()
    print(f'amed predictor kernel scale_dir={sd} scale_time={st}: r / scale_dir / scale_time / t_mid within 2e-5 (relative) of the torch forward')


# --------------------------------------------------------------------------------------------- LDM (Stable Diffusion) building blocks
def test_layernorm_geglu_softmax_generic(lib):
    from diff_sampler_b200 import _cstructs as S
    torch.manual_seed(12)
    for Cc in (320, 640, 1280):
        x = torch.randn(50, Cc, device=dev()) * 2 + 0.5
        g, b = torch.randn(Cc, device=dev()), torch.randn(Cc, device=dev())
        out = torch.zeros(2, 50, Cc, dtype=torch.float16, device=dev())
        lib.op_launch(S.LayernormDesc(src=x.data_ptr(), gamma=g.data_ptr(), beta=b.data_ptr(), out=out.data_ptr(), rows=50, C=Cc, nplanes=2, eps=1e-5))
        sync()
        ref = F.layer_norm(x.double(), (Cc,), g.double(), b.double(), 1e-5)
        assert ((out[0].double() + out[1].double()) - ref).abs().max().item() < 2e-5
    xx = torch.randn(33, 2 * 1280, device=dev()) * 2
    o = torch.zeros(2, 33, 1280, dtype=torch.float16, device=dev())
    lib.op_launch(S.GegluDesc(src=xx.data_ptr(), out=o.data_ptr(), rows=33, I=1280, nplanes=2))
    sync()
    a, gate = xx.double().chunk(2, dim=-1)
    assert ((o[0].double() + o[1].double()) - a * F.gelu(gate)).abs().max().item() < 2e-5
    # softmax over 77 valid keys, input pitch 80, output pitch 128
    Sm = torch.randn(21, 80, device=dev()) * 3
    Pm = torch.full((2, 21, 128), 7.0, dtype=torch.float16, device=dev())
    lib.op_launch(S.SoftmaxDesc(S=Sm.data_ptr(), P=Pm.data_ptr(), rows=21, L=77, nplanes=2, pitch_in=80, pitch_out=128))
    sync()
    ref = torch.softmax(Sm[:, :77].double(), -1)
    assert ((Pm[0, :, :77].double() + Pm[1, :, :77].double()) - ref).abs().max().item() < 2e-6
    # LDM timestep embedding
    t = torch.tensor([999.0, 500.5, 3.0], device=dev())
    emb = torch.zeros(3, 320, device=dev())
    lib.op_launch(S.PosembDesc(sigma=t.data_ptr(), nsig=3, num_channels=320, endpoint=0, swap_sincos=0, sigma_data=0.5, mode=1, coef=0,
                               emb=emb.data_ptr()))
    sync()
    import math
    freqs = torch.exp(-math.log(10000) * torch.arange(160, dtype=torch.float32, device=dev()) / 160)
    args = t[:, None] * freqs[None]
    refe = torch.cat([args.cos(), args.sin()], dim=-1)
    assert (emb - refe).abs().max().item() < 2e-4          # arguments up to ~1000 rad: fp32 range reduction differs at the 1e-5 level


@pytest.mark.parametrize('Bn,H,Cin,Cout', [(3, 16, 64, 128), (2, 32, 128, 64)])
def test_stride2_conv_via_space_to_depth(lib, Bn, H, Cin, Cout):
    """LDM Downsample (3x3, stride 2, pad 1): space-to-depth repack + the same GEMM kernel with per-tap (shift, phase) table."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(13)
    x = torch.randn(Bn, Cin, H, H, device=dev())
    w = torch.randn(Cout, Cin, 3, 3, device=dev()) / (3 * Cin ** 0.5)
    xn = x.permute(0, 2, 3, 1).contiguous()
    s2d = torch.zeros(2, Bn, H // 2, H // 2, 4 * Cin, dtype=torch.float16, device=dev())
    lib.op_launch(S.GnApplyDesc(src0=xn.data_ptr(), src1=0, C0=Cin, C1=0, H=H, W=H, B=Bn, groups=32, sums=0, gamma=0, beta=0, eps=0, silu=0,
                                ada=0, ada_stride=0, resample=3, nplanes=2, out_act=0, out_raw=s2d.data_ptr(), out_raw_f32=0))
    wp = G.pack_conv_weight(w.cpu()).to(dev())
    Ho = H // 2
    out = torch.full((Bn * Ho * Ho, Cout), float('nan'), device=dev())
    d, _ = G.conv_gemm(s2d.data_ptr(), Bn, Ho, Ho, Cin, wp.data_ptr(), Cout, taps=9, npass=3, out_f32=out.data_ptr(), s2d=True)
    lib.op_launch(d)
    sync()
    ref = F.conv2d(x.double(), w.double(), stride=2, padding=1).permute(0, 2, 3, 1).reshape(Bn * Ho * Ho, Cout)
    err = (out.double() - ref).abs().max().item()
    print(f'stride-2 conv {Bn}x{H}x{H} {Cin}->{Cout}: err {err:.3e}')
    assert err < 3e-5 * ref.abs().max().item()


def test_cross_attention_gemms_with_77_keys(lib):
    """S = Q K^T and O = P V with 77 context tokens: K extents that are not multiples of 64 rely on TMA zero fill."""
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(14)
    Bn, L, nh, d, T = 2, 256, 2, 64, 77
    Cc = nh * d
    q = torch.randn(Bn, L, Cc, device=dev())
    k = torch.randn(Bn, T, Cc, device=dev())
    vt = torch.zeros(Bn, Cc, 128, device=dev())
    vt[:, :, :T] = torch.randn(Bn, Cc, T, device=dev())
    vt[:, :, T:] = float('nan')                         # garbage beyond the valid keys must never be read
    qp, kp = planes(q), planes(k)
    vtp = torch.stack([vt.half(), (vt - vt.half().float()).half()])
    Smat = torch.full((Bn * nh, L, 80), float('nan'), device=dev())
    dS, _ = G.rows_gemm(qp.data_ptr(), L, Cc, Bn, kp.data_ptr(), T, Cc, Bn, d, num_z=Bn * nh, nh=nh, m_valid=L, n_valid=T,
                        a_c_per_zh=d, a_n_per_zb=1, b_k_per_zh=d, b_z_per_zb=1, out_f32=Smat.data_ptr(), o_zb=nh * L * 80, o_zh=L * 80,
                        ldo=80, scale=d ** -0.5)
    lib.op_launch(dS)
    sync()
    qh = q.reshape(Bn, L, nh, d).permute(0, 2, 1, 3).double()
    kh = k.reshape(Bn, T, nh, d).permute(0, 2, 1, 3).double()
    refS = (qh @ kh.transpose(-1, -2) * d ** -0.5).reshape(Bn * nh, L, T)
    assert (Smat[:, :, :T].double() - refS).abs().max().item() < 3e-5 * refS.abs().max().item()
    Pm = torch.zeros(Bn * nh, L, 128, device=dev())
    Pm[:, :, :T] = torch.softmax(Smat[:, :, :T], -1)
    Pm[:, :, T:] = float('nan')
    Pp = torch.stack([Pm.half(), (Pm - Pm.half().float()).half()])
    O = torch.zeros(2, Bn, L, Cc, dtype=torch.float16, device=dev())
    dO, _ = G.rows_gemm(Pp.data_ptr(), L, 128, Bn * nh, vtp.data_ptr(), Cc, 128, Bn, 128, num_z=Bn * nh, nh=nh, m_valid=L, n_valid=d,
                        a_n_per_zb=nh, a_n_per_zh=1, b_row_per_zh=d, b_z_per_zb=1, out_h16=O.data_ptr(), o_zb=L * Cc, o_zh=d, ldo=Cc,
                        o_plane=Bn * L * Cc, a_k_valid=T, b_k_valid=T)
    lib.op_launch(dO)
    sync()
    v = vt[:, :, :T].reshape(Bn, nh, d, T).double()
    refO = (Pm[:, :, :T].reshape(Bn, nh, L, T).double() @ v.transpose(-1, -2)).permute(0, 2, 1, 3).reshape(Bn, L, Cc)
    got = O[0].double() + O[1].double()
    assert torch.isfinite(got).all()
    assert (got - refO).abs().max().item() < 3e-5 * max(1.0, refO.abs().max().item())


# --------------------------------------------------------------------------------------------- f8 GEMM mode (fp16 hi x hi + e4m3 corrections)
def _f8_reference(x, w, x2=None, w2=None):
    """What the f8 GEMM computes, in float64 from the decoded operand planes (csrc/ops.h): hi x hi + lo8 x w_hi8 + hi8 x w_lo8.
    The operands are packed and decoded on the host; the convolutions run on x's device."""
    from diff_sampler_b200 import gemm_desc as G
    Cout, Cin = w.shape[0], w.shape[1]
    taps = w.shape[2] * w.shape[3]
    blob, shift = G.pack_conv_weight_f8(w.cpu(), None if w2 is None else w2.cpu())
    (m16, s16), (mh8, sh8), (ml8, sl8) = G.decode_conv_weight_f8(blob, shift, Cout, Cin, taps, 0 if w2 is None else w2.shape[1])
    k = w.shape[2]
    as_w = lambda m: m.reshape(Cout, k, k, Cin).permute(0, 3, 1, 2).to(x.device).double()
    xn = x.permute(0, 2, 3, 1).contiguous().cpu()
    abuf = G.act_planes_f8(xn)
    hi, lo8, hi8 = [t.permute(0, 3, 1, 2).to(x.device).double() for t in G.decode_act_planes_f8(abuf, xn.shape)]
    pad = k // 2
    ref = F.conv2d(hi, as_w(m16), padding=pad) + F.conv2d(lo8, as_w(mh8), padding=pad) + F.conv2d(hi8, as_w(ml8), padding=pad)
    a2buf = None
    if w2 is not None:
        x2n = x2.permute(0, 2, 3, 1).contiguous().cpu()
        a2buf = G.act_planes_f8(x2n)
        h2, l2, h82 = [t.permute(0, 3, 1, 2).to(x.device).double() for t in G.decode_act_planes_f8(a2buf, x2n.shape)]
        as_s = lambda m: m.reshape(Cout, -1, 1, 1).to(x.device).double()
        ref = ref + F.conv2d(h2, as_s(s16)) + F.conv2d(l2, as_s(sh8)) + F.conv2d(h82, as_s(sl8))
    return ref, blob, shift, abuf, a2buf


@pytest.mark.parametrize('Bn,H,W,Cin,Cout,C2,taps', [(3, 32, 32, 64, 128, 0, 9), (3, 16, 16, 128, 192, 0, 9), (2, 8, 8, 192, 256, 0, 9),
                                                     (4, 16, 16, 128, 128, 64, 9), (2, 16, 16, 256, 256, 192, 9), (2, 8, 8, 256, 512, 0, 1)])
def test_conv_f8_mode(lib, Bn, H, W, Cin, Cout, C2, taps):
    """f8 GEMM mode: the kernel must reproduce hi x hi + e4m3 corrections of the packed operands to fp32-accumulation accuracy, and
    stay within a few 1e-5 (relative) of the exact convolution -- 3 % of the single-pass fp16 error (tests/study_fp8_corrections.py)."""
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(11)
    k = 3 if taps == 9 else 1
    x = torch.randn(Bn, Cin, H, W, device=dev()) * 1.5
    w = torch.randn(Cout, Cin, k, k, device=dev()) / (k * Cin ** 0.5)
    x2 = torch.randn(Bn, C2, H, W, device=dev()) * 4.0 if C2 else None
    w2 = torch.randn(Cout, C2, 1, 1, device=dev()) / C2 ** 0.5 if C2 else None
    ref, blob, shift, abuf, a2buf = _f8_reference(x, w, x2, w2)
    wp, xa = blob.to(dev()), abuf.to(dev())
    x2a = a2buf.to(dev()) if C2 else None
    out = torch.full((Bn * H * W, Cout), float('nan'), device=dev())
    d, info = G.conv_gemm(xa.data_ptr(), Bn, H, W, Cin, wp.data_ptr(), Cout, taps=taps, npass=3, a2_ptr=x2a.data_ptr() if C2 else 0, C2=C2,
                          out_f32=out.data_ptr(), f8=True, acc_scale=2.0 ** -shift)
    lib.op_launch(d)
    sync()
    exact = F.conv2d(x.double().cpu(), w.double().cpu(), padding=k // 2)
    if C2:
        exact = exact + F.conv2d(x2.double().cpu(), w2.double().cpu())
    to_rows = lambda t: t.permute(0, 2, 3, 1).reshape(Bn * H * W, Cout)
    got = out.double().cpu()
    scale = exact.abs().max().item()
    e_model = (got - to_rows(ref.cpu())).abs().max().item()
    e_exact = (got - to_rows(exact)).abs().max().item()
    print(f'conv f8 {Bn}x{H}x{W} {Cin}(+{C2})->{Cout} taps{taps} BN={info["BN"]} S={shift}: vs operand model {e_model:.3e}, vs exact {e_exact:.3e} '
          f'(scale {scale:.2f})')
    assert not torch.isnan(out).any()
    assert e_model <= 5e-6 * scale          # fp32 accumulation over K up to 2.5k terms (measured 1-2.3e-6)
    assert e_exact <= 1e-4 * scale


@pytest.mark.parametrize('C0,C1,H,W,resample', [(128, 0, 16, 16, 0), (256, 128, 8, 8, 0), (192, 0, 16, 16, 1), (128, 64, 8, 8, 2)])
def test_groupnorm_apply_f8_layout(lib, C0, C1, H, W, resample):
    """ds_gn_apply fmt=1 writes the A operand of the f8 GEMM: fp16 (y * 2^6) | e4m3 ((y - hi) * 2^13) | e4m3 (hi * 2^2)."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(12)
    Bn, Cc, Gr = 3, C0 + C1, 32
    x0 = torch.randn(Bn, H, W, C0, device=dev()) * 1.7 + 0.3
    x1 = torch.randn(Bn, H, W, C1, device=dev()) * 0.6 - 0.2 if C1 else None
    gamma = torch.randn(Cc, device=dev())
    beta = torch.randn(Cc, device=dev())
    sums = torch.zeros(Bn, Gr, 2, dtype=torch.float64, device=dev())
    lib.op_launch(S.GnStatsDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, HW=H * W, B=Bn, groups=Gr,
                                sums=sums.data_ptr()))
    Ho, Wo = (H // 2, W // 2) if resample == 1 else ((H * 2, W * 2) if resample == 2 else (H, W))
    n = Bn * Ho * Wo * Cc
    act = torch.zeros(4 * n, dtype=torch.uint8, device=dev())
    raw = torch.zeros(4 * n, dtype=torch.uint8, device=dev())
    lib.op_launch(S.GnApplyDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, H=H, W=W, B=Bn, groups=Gr,
                                sums=sums.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-6, silu=1, ada=0, ada_stride=0,
                                resample=resample, nplanes=2, out_act=act.data_ptr(), out_raw=raw.data_ptr(), out_raw_f32=0, fmt=1))
    sync()
    xc = torch.cat([x0, x1], dim=-1) if C1 else x0
    xn = xc.permute(0, 3, 1, 2).double()
    y = F.silu(F.group_norm(xn, Gr, gamma.double(), beta.double(), eps=1e-6))
    r = xn
    if resample == 1:
        y, r = F.avg_pool2d(y, 2), F.avg_pool2d(r, 2)
    elif resample == 2:
        y, r = F.interpolate(y, scale_factor=2, mode='nearest'), F.interpolate(r, scale_factor=2, mode='nearest')
    for name, buf, want in (('act', act, y), ('raw', raw, r)):
        want = want.permute(0, 2, 3, 1).cpu()
        hi, lo8, hi8 = [t.double() for t in G.decode_act_planes_f8(buf.cpu(), want.shape)]
        e_hi = (hi - want).abs().max().item()
        e_sum = (hi + lo8 - want).abs().max().item()
        e_h8 = ((hi8 - hi).abs() / hi.abs().clamp_min(2.0 ** -8)).max().item()
        print(f'gn f8 {name} C{C0}+{C1} rs{resample}: |hi - y| {e_hi:.2e}  |hi + lo8 - y| {e_sum:.2e}  rel |hi8 - hi| {e_h8:.3f}')
        m = max(1.0, want.abs().max().item())
        assert e_hi < 6e-4 * m              # fp16: 2^-11 relative
        assert e_sum < 4e-5 * m             # + e4m3 of the residual: 2^-4 of 2^-11
        assert e_h8 < 0.07                  # e4m3: 2^-4 relative


# --------------------------------------------------------------------------------------------- LayerNorm / GEGLU writing the f8 operand image


def test_layernorm_geglu_f8_image(lib):
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(31)
    rows, C = 300, 320
    x = torch.randn(rows, C, device=dev()) * 2.0 + 0.5
    g, b = torch.randn(C, device=dev()), torch.randn(C, device=dev())
    out = torch.zeros(4 * rows * C, dtype=torch.uint8, device=dev())
    lib.op_launch(S.LayernormDesc(src=x.data_ptr(), gamma=g.data_ptr(), beta=b.data_ptr(), out=out.data_ptr(), rows=rows, C=C, nplanes=2,
                                  eps=1e-5, fmt=1))
    I = 640
    src = torch.randn(rows, 2 * I, device=dev()) * 1.5
    out2 = torch.zeros(4 * rows * I, dtype=torch.uint8, device=dev())
    lib.op_launch(S.GegluDesc(src=src.data_ptr(), out=out2.data_ptr(), rows=rows, I=I, nplanes=2, fmt=1))
    sync()
    want_ln = F.layer_norm(x.double(), (C,), g.double(), b.double(), 1e-5).cpu()
    want_gg = (src[:, :I].double() * F.gelu(src[:, I:].double())).cpu()
    for name, buf, want in (('layernorm', out, want_ln), ('geglu', out2, want_gg)):
        hi, lo8, hi8 = [t.double() for t in G.decode_act_planes_f8(buf.cpu(), want.shape)]
        m = max(1.0, want.abs().max().item())
        e_hi, e_sum = (hi - want).abs().max().item(), (hi + lo8 - want).abs().max().item()
        e_h8 = ((hi8 - hi).abs() / hi.abs().clamp_min(2.0 ** -8)).max().item()
        print(f'{name} f8 image: |hi - y| {e_hi:.2e}  |hi + lo8 - y| {e_sum:.2e}  rel |hi8 - hi| {e_h8:.3f}')
        assert e_hi < 6e-4 * m and e_sum < 4e-5 * m and e_h8 < 0.07

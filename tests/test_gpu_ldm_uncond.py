"""The unconditional LSUN-Bedroom / FFHQ latent-diffusion eps-net on the GPU: the pair attention kernel (32-wide heads, two per CTA),
the GEMMs and GroupNorms at channel counts that are not multiples of 64, the denoiser and the samplers against the float64
restatement of tests/ldm_uncond_ref.py."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

import ldm_uncond_ref as U

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    return torch.device('cuda:0')


def _planes(x):
    from diff_sampler_b200.gemm_desc import split_planes
    return split_planes(x)


def _hl(p):
    return p[0].double() + p[1].double()


# --------------------------------------------------------------------------------------------- pair attention kernel
def _attn_operands(B, nh, L, d, hd):
    """q, k, v [B, nh, L, d] and the kernel operands with each head in a slot of hd channels: qk planes [2][B][L][2 nh hd]
    ([q heads | k heads]) and V^T planes [2][B][nh hd][L]."""
    g = torch.Generator(device=_dev()).manual_seed(11 + nh + L)
    q = torch.randn(B, nh, L, d, device=_dev(), generator=g) * 1.5
    k = torch.randn(B, nh, L, d, device=_dev(), generator=g) * 1.5
    v = torch.randn(B, nh, L, d, device=_dev(), generator=g) + 0.5
    k[:, :, 3] *= 4.0
    C = nh * hd
    qk = torch.zeros(B, L, 2 * C, device=_dev())
    vt = torch.zeros(B, C, L, device=_dev())
    for h in range(nh):
        qk[:, :, h * hd:h * hd + d] = q[:, h]
        qk[:, :, C + h * hd:C + h * hd + d] = k[:, h]
        vt[:, h * hd:h * hd + d] = v[:, h].transpose(1, 2)
    return q, k, v, _planes(qk), _planes(vt)


def _launch_attn(qk, vt, B, nh, L, hd, scale):
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    C = nh * hd
    out = torch.full((2, B, L, C), float('nan'), dtype=torch.float16, device=_dev())
    _lib.op_launch(S.AttnDesc(q=qk.data_ptr(), k=qk.data_ptr(), vt=vt.data_ptr(), out=out.data_ptr(), B=B, nh=nh, L=L, Lk=L,
                              q_pitch=2 * C, q_c0=0, k_pitch=2 * C, k_c0=C, vt_pitch=L, o_pitch=C, nplanes=2, scale=scale, causal=0,
                              pad0=32 if hd == 32 else 0))
    torch.cuda.synchronize()
    return _hl(out).reshape(B, L, nh, hd).permute(0, 2, 1, 3)


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('nh', [14, 22, 28])
@pytest.mark.parametrize('L', [64, 256, 1024])
def test_pair_attention_kernel(B, nh, L):
    """attn_pair_kernel against float64 softmax attention on the same fp16 hi + lo operands, and against attn_kernel on the same
    heads zero-padded to 64."""
    d = 32
    scale = d ** -0.5
    q, k, v, qk, vt = _attn_operands(B, nh, L, d, 32)
    got = _launch_attn(qk, vt, B, nh, L, 32, scale)
    qd, kd, vd = (_hl(_planes(t)) for t in (q, k, v))
    ref = torch.softmax(scale * qd @ kd.transpose(-1, -2), dim=-1) @ vd
    err = (got - ref).abs().max().item()
    _, _, _, qk64, vt64 = _attn_operands(B, nh, L, d, 64)
    pad = _launch_attn(qk64, vt64, B, nh, L, 64, scale)[..., :d]
    dpad = (got - pad).abs().max().item()
    print(f'pair attention B{B} nh{nh} L{L}: err {err:.3e} (max {ref.abs().max().item():.2f}), vs padded kernel {dpad:.3e}')
    assert err < 2e-5 * max(1.0, ref.abs().max().item())
    assert dpad < 2e-5 * max(1.0, ref.abs().max().item())


def test_pair_kernel_has_no_stack_frame_or_local_memory():
    lib = os.path.join(ROOT, 'diff-sampler_b200', 'libdiffsampler_b200.so')
    exe = shutil.which('cuobjdump') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not found')
    out = subprocess.run([exe, '-sass', lib], capture_output=True, text=True, check=True).stdout
    code, inside = [], False
    for ln in out.splitlines():
        if 'Function :' in ln:
            inside = 'attn_pair_kernel' in ln
        elif inside and re.match(r'\s*/\*[0-9a-f]{4,}\*/', ln):
            code.append(ln)
    assert any('HGMMA.64x32x16' in ln for ln in code)
    assert not [ln for ln in code if re.search(r'\b(LDL|STL)\b', ln)], 'local memory traffic in attn_pair_kernel'


# --------------------------------------------------------------------------------------------- GEMMs with channel remainders
@pytest.mark.parametrize('C,C2,H', [(224, 0, 32), (672, 672, 16), (1120, 672, 16), (1568, 672, 8), (224, 0, 64)])
def test_conv_gemm_channel_remainder(C, C2, H):
    """3x3 convolution over C channels (+ a 1x1 skip over C2) with C, C2 not multiples of 64: TMA zero-fills the last K block."""
    from diff_sampler_b200 import _lib
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(C + C2)
    B, Cout = 2, 224 if C2 == 0 else 672
    x = torch.randn(B, H, H, C, device=_dev())
    w = torch.randn(Cout, C, 3, 3) / (9 * C) ** 0.5
    x2 = torch.randn(B, H, H, C2, device=_dev()) if C2 else None
    w2 = torch.randn(Cout, C2, 1, 1) / C2 ** 0.5 if C2 else None
    wp = G.pack_conv_weight(w, w2).to(_dev())
    xp = _planes(x)
    x2p = _planes(x2) if C2 else None
    out = torch.full((B * H * H, Cout), float('nan'), device=_dev())
    d, _ = G.conv_gemm(xp.data_ptr(), B, H, H, C, wp.data_ptr(), Cout, taps=9, a2_ptr=x2p.data_ptr() if C2 else 0, C2=C2,
                       out_f32=out.data_ptr())
    _lib.op_launch(d)
    torch.cuda.synchronize()
    xd = _hl(xp).permute(0, 3, 1, 2)
    ref = F.conv2d(xd, w.double().to(_dev()), padding=1)
    if C2:
        ref = ref + F.conv2d(_hl(x2p).permute(0, 3, 1, 2), w2.double().to(_dev()))
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Cout)
    err = (out.double() - ref).abs().max().item()
    print(f'conv C{C} C2{C2} H{H}: err {err:.3e} (max {ref.abs().max().item():.2f})')
    # fp32 accumulation over up to 9 x 1568 + 672 products; a skipped 32-channel remainder would be an O(0.1) error
    assert err < 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('C,H', [(224, 64), (672, 16), (96, 16)])
def test_space_to_depth_downsample_with_phase_pitch(C, H):
    """Stride-2 convolution through gn_apply's space-to-depth repack at a 64-aligned phase pitch (the gap between phases zeroed
    over a buffer that starts as NaN) and conv_gemm(s2d=True)."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    from diff_sampler_b200 import gemm_desc as G
    torch.manual_seed(C)
    B = 2
    cp = -(-C // 64) * 64
    x = torch.randn(B, H, H, C, device=_dev())
    w = torch.randn(C, C, 3, 3) / (9 * C) ** 0.5
    s2d = torch.full((2, B, H // 2, H // 2, 4 * cp), float('nan'), dtype=torch.float16, device=_dev())
    _lib.op_launch(S.GnApplyDesc(src0=x.data_ptr(), C0=C, C1=0, H=H, W=H, B=B, groups=32, eps=0.0, silu=0, resample=3, nplanes=2,
                                 out_raw=s2d.data_ptr(), pad0=cp))
    torch.cuda.synchronize()
    assert not torch.isnan(s2d).any()
    gap = s2d.reshape(2, B, H // 2, H // 2, 4, cp)[..., C:]
    assert gap.abs().max().item() == 0.0
    wp = G.pack_conv_weight(w).to(_dev())
    out = torch.full((B * (H // 2) ** 2, C), float('nan'), device=_dev())
    d, _ = G.conv_gemm(s2d.data_ptr(), B, H // 2, H // 2, C, wp.data_ptr(), C, taps=9, out_f32=out.data_ptr(), s2d=True)
    _lib.op_launch(d)
    torch.cuda.synchronize()
    xd = _hl(_planes(x)).permute(0, 3, 1, 2)
    ref = F.conv2d(xd, w.double().to(_dev()), stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, C)
    err = (out.double() - ref).abs().max().item()
    print(f's2d C{C} H{H}: err {err:.3e}')
    assert err < 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('C0,C1,H', [(224, 0, 64), (672, 0, 16), (896, 672, 16), (1120, 0, 32)])
def test_groupnorm_odd_group_widths(C0, C1, H):
    """GroupNorm32 + SiLU at 7 / 21 / 49 / 35-channel groups (the 1568-channel concat straddles its sources mid-group)."""
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib
    torch.manual_seed(C0 + C1)
    B, C = 2, C0 + C1
    x0 = torch.randn(B, H, H, C0, device=_dev()) * 2 + 0.5
    x1 = torch.randn(B, H, H, C1, device=_dev()) if C1 else None
    gamma = 1 + 0.1 * torch.randn(C, device=_dev())
    beta = 0.1 * torch.randn(C, device=_dev())
    sums = torch.zeros(B, 32, 2, dtype=torch.float64, device=_dev())
    _lib.op_launch(S.GnStatsDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, HW=H * H, B=B, groups=32,
                                 sums=sums.data_ptr()))
    act = torch.full((2, B, H, H, C), float('nan'), dtype=torch.float16, device=_dev())
    _lib.op_launch(S.GnApplyDesc(src0=x0.data_ptr(), src1=x1.data_ptr() if C1 else 0, C0=C0, C1=C1, H=H, W=H, B=B, groups=32,
                                 sums=sums.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=1e-5, silu=1, nplanes=2,
                                 out_act=act.data_ptr()))
    torch.cuda.synchronize()
    x = torch.cat([x0, x1], dim=-1) if C1 else x0
    ref = F.silu(F.group_norm(x.double().permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5)).permute(0, 2, 3, 1)
    err = (_hl(act) - ref).abs().max().item()
    print(f'groupnorm C{C0}+{C1} (group {C // 32}): err {err:.3e}')
    assert err < 2e-5 * max(1.0, ref.abs().max().item())


# --------------------------------------------------------------------------------------------- denoiser
_NETS = {}


def _pair(name, precision='fp16x3', head_pairs=True, cuda_graph=None):
    from diff_sampler_b200.ldm_net import B200LDMNet
    key = (name, precision, head_pairs, cuda_graph)
    if key not in _NETS:
        P, cfg = U.make_params(name)
        nat = B200LDMNet(P, img_resolution=cfg['img_resolution'], img_channels=cfg['in_channels'], guidance_type='uncond',
                         num_head_channels=cfg['num_head_channels'], precision=precision, head_pairs=head_pairs, device=_dev(),
                         cuda_graph=cuda_graph)
        _NETS[key] = (U.OracleUncondNet(P, cfg), nat, cfg)
    return _NETS[key]


def _x(cfg, B, sigma, seed=0):
    g = torch.Generator().manual_seed(seed)
    R = cfg['img_resolution']
    return torch.randn(B, cfg['in_channels'], R, R, generator=g) * sigma


@pytest.mark.parametrize('name', ['tiny_uncond', 'ldm_vq4'])
def test_uncond_denoiser_parity(name):
    """D = x - sigma * eps at batch 2 against float64: fp16x3 (gated at 1e-3 of max |D|) in pair and padded-head modes, and fp16
    (reported); one sigma per call and per-sample sigma; the middle-block read-out against the float64 tap."""
    on, nat, cfg = _pair(name)
    _, pad, _ = _pair(name, head_pairs=False)
    _, n16, _ = _pair(name, precision='fp16')
    B = 2
    for sigma in (14.6, 1.0, 0.05):
        x = _x(cfg, B, sigma, seed=int(sigma * 10))
        on.taps = {}
        ref = on(x.to(_dev()), torch.tensor([sigma]))
        tap = on.taps['middle_block'].mean(dim=1).reshape(B, 64)
        on.taps = None
        scale = max(1.0, ref.abs().max().item())
        bott = torch.zeros(B, 64, device=_dev())
        got = nat(x.to(_dev()), torch.tensor([sigma], device=_dev()), bottleneck=bott)
        gp = pad(x.to(_dev()), torch.tensor([sigma], device=_dev()))
        g16 = n16(x.to(_dev()), torch.tensor([sigma], device=_dev()))
        err, errp, e16 = ((t.double() - ref).abs().max().item() for t in (got, gp, g16))
        eb = (bott.double() - tap).abs().max().item()
        print(f'{name} sigma={sigma}: fp16x3 pairs {err:.3e}, padded {errp:.3e}, fp16 {e16:.3e} (max|D| {scale:.1f}); bottleneck {eb:.3e}')
        assert err < 1e-3 * scale and errp < 1e-3 * scale
        assert eb < 1e-3 * max(1.0, tap.abs().max().item())
    sig = torch.tensor([5.0, 0.3])
    x = _x(cfg, B, 1.0, seed=3) * sig.reshape(-1, 1, 1, 1)
    ref = on(x.to(_dev()), sig)
    got = nat(x.to(_dev()), sig.to(_dev()))
    err = (got.double() - ref).abs().max().item()
    print(f'{name} per-sample sigma: {err:.3e}')
    assert err < 1e-3 * max(1.0, ref.abs().max().item())


def test_uncond_fp16_runs_natively():
    """fp16 (one pass per product) runs the native kernels end to end: the tiny net's plan launched, output finite."""
    _, nat, cfg = _pair('tiny_uncond', precision='fp16')
    x = _x(cfg, 3, 2.0).to(_dev())
    before = nat.total_launches
    out = nat(x, torch.tensor([2.0], device=_dev()))
    assert torch.isfinite(out).all() and nat.total_launches > before


def test_cuda_graph_on_and_off_are_bit_identical():
    _, plain, cfg = _pair('tiny_uncond', cuda_graph=False)
    _, graph, _ = _pair('tiny_uncond', cuda_graph=True)
    B = 2
    for k, sigma in enumerate((10.0, 2.0, 0.5, 0.1)):
        x = _x(cfg, B, sigma, seed=k).to(_dev())
        sig = torch.tensor([sigma], device=_dev())
        bp, bg = torch.zeros(B, 64, device=_dev()), torch.zeros(B, 64, device=_dev())
        a = plain(x, sig, bottleneck=bp if k % 2 else None)
        b = graph(x, sig, bottleneck=bg if k % 2 else None)
        assert torch.equal(a, b) and torch.equal(bp, bg)


def test_fp16f8_is_refused():
    P, cfg = U.make_params('tiny_uncond')
    from diff_sampler_b200.ldm_net import B200LDMNet
    with pytest.raises(ValueError, match='fp16f8'):
        B200LDMNet(P, img_resolution=16, img_channels=3, guidance_type='uncond', num_head_channels=32, precision='fp16f8', device=_dev())


# --------------------------------------------------------------------------------------------- samplers
@pytest.mark.parametrize('solver,kw', [('euler', {}), ('heun', {}), ('dpm_pp', dict(max_order=2, predict_x0=False)),
                                       ('ipndm', dict(max_order=4))])
def test_uncond_samplers_discrete_schedule(solver, kw):
    from oracle import solvers_oracle as SO
    from diff_sampler_b200 import solvers
    on, nat, cfg = _pair('tiny_uncond')
    B = 2
    lat = _x(cfg, B, 1.0, seed=9)
    args = dict(num_steps=6, sigma_min=on.sigma_min, sigma_max=on.sigma_max, schedule_type='discrete', schedule_rho=1, **kw)
    ref = SO.sample(on, lat.double(), solver, **args).double()
    got = getattr(solvers, solver + '_sampler')(nat, lat.to(_dev()), **args).cpu().double()
    err = (got - ref).abs().max().item()
    print(f'uncond {solver} NFE<=10 discrete: err {err:.3e} (max|x| {ref.abs().max().item():.1f})')
    assert err < 2e-3 * max(1.0, ref.abs().max().item())


def test_uncond_gits_grid_and_amed_tap():
    """A GITS-style time grid (t_steps given) through DPM-Solver++, and AMED-DPM++ whose predictor reads the middle-block tap."""
    from diff_sampler_b200 import solvers
    from diff_sampler_b200 import solvers_amed
    on, nat, cfg = _pair('tiny_uncond')
    B = 2
    lat = _x(cfg, B, 1.0, seed=12)
    t_steps = torch.tensor([on.sigma_max, 20.0, 6.0, 1.5, 0.4, on.sigma_min])
    from oracle import solvers_oracle as SO
    ref = SO.sample(on, lat.double(), 'dpm_pp', num_steps=6, t_steps=t_steps, max_order=2, predict_x0=False).double()
    got = solvers.dpm_pp_sampler(nat, lat.to(_dev()), num_steps=6, t_steps=t_steps.to(_dev()), max_order=2, predict_x0=False).cpu().double()
    err = (got - ref).abs().max().item()
    print(f'uncond dpm_pp on a GITS grid: err {err:.3e}')
    assert err < 2e-3 * max(1.0, ref.abs().max().item())
    # AMED-DPM++: the predictor consumes the native bottleneck read-out
    seen = []

    def predictor(enc, t_cur, t_next):
        seen.append(enc.detach().clone())
        r = torch.full((enc.shape[0], 1, 1, 1), 0.5, device=enc.device)
        return r, torch.zeros_like(r), torch.zeros_like(r)
    x = solvers_amed.amed_sampler(nat, lat.to(_dev()), AMED_predictor=predictor, num_steps=4, sigma_min=on.sigma_min, sigma_max=on.sigma_max,
                                  schedule_type='discrete', schedule_rho=1, afs=False)
    assert torch.isfinite(x).all() and seen and seen[0].shape == (B, 8, 8)
    on.taps = {}
    sig0 = torch.tensor([on.sigma_max])
    on(lat.to(_dev()) * on.sigma_max, sig0)
    tap = on.taps['middle_block'].mean(dim=1)
    on.taps = None
    assert (seen[0].double() - tap.reshape(B, 8, 8)).abs().max().item() < 1e-3 * max(1.0, tap.abs().max().item())


def test_tiny_end_to_end_sample_decode_uint8():
    """sample -> VQ-f4 decode -> uint8, with the tiny eps-net and the VQ decoder of tests/vq_ref.py."""
    import vq_ref as VQ
    from diff_sampler_b200 import solvers
    from diff_sampler_b200.vae_net import B200VAEDecoder
    from diff_sampler_b200.dist_utils import to_uint8_nhwc
    on, nat, cfg = _pair('tiny_uncond')
    lat = _x(cfg, 2, 1.0, seed=21)
    z = solvers.dpm_pp_sampler(nat, lat.to(_dev()), num_steps=5, sigma_min=on.sigma_min, sigma_max=on.sigma_max,
                               schedule_type='discrete', schedule_rho=1, max_order=2, predict_x0=False)
    P, vcfg = VQ.make_params('tiny_vq')
    dec = B200VAEDecoder(P, scale_factor=vcfg['scale_factor'], device=_dev())
    img = dec.decode(z)
    u8 = to_uint8_nhwc(img)
    assert u8.dtype == torch.uint8 and u8.shape[0] == 2 and u8.shape[-1] == 3


# --------------------------------------------------------------------------------------------- entry points
def test_from_reference_and_as_native_on_a_reference_layout_standin():
    """A CFGPrecond(guidance_type='uncond') module whose UNetModel says num_heads=-1, num_head_channels=32 (as the LDM-VQ-f4 configs
    build it) goes through as_native -> B200LDMNet.from_reference with 32-wide heads and samples the images of B200LDMNet(P, ...)."""
    import test_gpu_parity as TP
    from diff_sampler_b200 import ldm_net, solvers
    on, direct, cfg = _pair('tiny_uncond')
    P, _ = U.make_params('tiny_uncond')
    mod = TP._module_from_params({'model.model.diffusion_model.' + k: v for k, v in P.items()}, 'CFGPrecond',
                                 {'model.model.diffusion_model': 'UNetModel'}).to(_dev())
    unet = mod.model.model.diffusion_model
    unet.num_heads, unet.num_head_channels = -1, 32
    mod.model.alphas_cumprod = ldm_net.make_alphas_cumprod(*ldm_net.UNCOND_BETAS)
    mod.img_resolution, mod.img_channels, mod.label_dim = cfg['img_resolution'], cfg['in_channels'], 0
    mod.guidance_type, mod.guidance_rate = 'uncond', 1.0
    nat = solvers.as_native(mod)
    assert isinstance(nat, ldm_net.B200LDMNet) and solvers.as_native(mod) is nat and nat.guidance_type == 'uncond'
    heads = {L[3:] for _, ls in nat.st['inp'] + nat.st['mid'] + nat.st['out'] for L in ls if L[0] == 'qkv_attn'}
    assert heads == {(3, 32), (6, 32), (9, 32)}
    assert nat.sigma_max == direct.sigma_max and nat.sigma_min == direct.sigma_min
    mod.sigma_min, mod.sigma_max = nat.sigma_min, nat.sigma_max
    mod.sigma, mod.sigma_inv = nat.sigma, nat.sigma_inv
    lat = _x(cfg, 2, 1.0, seed=4).to(_dev())
    kw = dict(num_steps=4, sigma_min=nat.sigma_min, sigma_max=nat.sigma_max, schedule_type='discrete', schedule_rho=1, max_order=2,
              predict_x0=False)
    assert torch.equal(solvers.dpm_pp_sampler(direct, lat, **kw), solvers.dpm_pp_sampler(mod, lat, **kw))


def test_from_ldm_checkpoint(tmp_path):
    """A file with the released model.ckpt's key layout -> the eps-net and the VQ decoder, equal to the ones built from the tensors."""
    import test_ldm_uncond_host as H
    from diff_sampler_b200.ldm_net import B200LDMNet
    from diff_sampler_b200.vae_net import B200VAEDecoder
    sd, P, V, _ = H._ldm_ckpt_state()
    path = tmp_path / 'model.ckpt'
    torch.save({'state_dict': sd, 'global_step': 7}, path)
    net, vae = B200LDMNet.from_ldm_checkpoint(str(path), img_resolution=32, device=_dev())
    _, direct, cfg = _pair('tiny_uncond')
    x = _x(cfg, 2, 3.0, seed=8).to(_dev())
    sig = torch.tensor([3.0], device=_dev())
    assert torch.equal(net(x, sig), direct(x, sig))
    z = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(2)).to(_dev())
    assert torch.equal(vae.decode(z), B200VAEDecoder(V, scale_factor=1.0, device=_dev()).decode(z))


def test_fullsize_plan_ops_against_the_interpreter(monkeypatch):
    """Every op of the full-size fp16x3 plan with head pairs at batch 2, replayed alone on 0xFF-filled outputs against the float64
    interpreter (tests/ldm_uncond_interp.py for the remainder GEMMs, the phase-pitched repack and pair attention), as
    tests/test_gpu_plan_ops.py does for the benchmarked plans."""
    import ldm_uncond_interp as LI
    import plan_spans
    import test_gpu_plan_ops as TPO
    from diff_sampler_b200 import _cstructs as S
    from diff_sampler_b200 import _lib, ldm_plan
    P, cfg = U.make_params('ldm_vq4')
    st = ldm_plan.ldm_structure(P, 8, 32)
    wb, info = ldm_plan.pack_ldm_weights(st, P)
    B = 2
    pl = ldm_plan.compile_ldm_plan(st, wb, info, B, B, 1, 64)
    g = torch.Generator().manual_seed(11)
    io_host = {S.DS_IO_X: torch.randn(B, 3, 64, 64, generator=g), S.DS_IO_D: torch.zeros(B, 3, 64, 64), S.DS_IO_SIGMA: torch.tensor([417.0]),
               S.DS_IO_LABELS: torch.tensor([[0.0, 0.0, 0.37, 0.0]]), S.DS_IO_BOTTLENECK: torch.zeros(B, 64)}
    monkeypatch.setattr(TPO, 'workload', lambda name: (pl, wb.bytes(), io_host))
    for t, entry in LI.DISPATCH.items():
        monkeypatch.setitem(TPO.PI._DISPATCH, t, entry)
    monkeypatch.setitem(plan_spans._WRITES, S.DS_OP_GN_APPLY, LI.gn_apply_spans(plan_spans._WRITES[S.DS_OP_GN_APPLY]))
    res = TPO.replay(_lib, 'ldm_vq4')

    def limit(r):
        # the fp32 accumulation error of the hi x hi product grows linearly with K on H100 (tests/test_gpu_plan_ops.py): the long-K
        # allowance those tests give f8 GEMMs past K_F8_PLAN_LONG applies to this plan's fp16x3 3x3 convolutions over 1792 channels
        # (K = 16128) too; TOL_X3 is sized for the benchmarked plans' contractions
        m = re.search(r' K(\d+) ', r['shape'])
        if r['type'] == 'gemm' and m and int(m.group(1)) > TPO.K_F8_PLAN_LONG:
            return TPO.TOL_F8_PLAN_LONG_K / TPO.TOL_X3
        return 1.0
    bad = [r for r in res['rows'] if r['ratio'] > limit(r) or r['problems']]
    worst = {}
    for r in res['rows']:
        worst[r['type']] = max(worst.get(r['type'], 0.0), r['ratio'])
    print(f"ldm_vq4: {res['n_ops']} ops, {res['seconds']:.1f} s; worst ratio per type "
          + ', '.join(f'{k} {v:.3f}' for k, v in sorted(worst.items())))
    assert len(res['rows']) == res['n_ops'] and {r['type'] for r in res['rows']} == res['types']
    assert not bad, '\n'.join(TPO._fmt('ldm_vq4', r) for r in bad[:20])

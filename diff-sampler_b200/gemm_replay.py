"""Rebuild the GEMM launches of a compiled plan on seeded device buffers, one launch per distinct configuration.

A configuration (GemmCfg) is what decides how the wgmma kernel runs a ds_gemm_desc: the shape, the N tile, f8 / npass, conv or
rows mode and which epilogue stages are on.  plan_configs() collects them from a plan's descriptors (plan references, so a plan
compiled on the host will do); make_desc() rebuilds one with the N tile pinned and any batch (conv mode) or z count / row count
(rows mode), since with BN fixed the batch only changes how many tiles each persistent CTA walks.  Rows-mode operands are laid
out z-major ([z][rows][K], or one shared batch where the plan shares it); the head windows of the attention products are not
reproduced.  Used by tools/gemm_probe.py (timing) and tests/test_gpu_gemm_tiles.py (accuracy against float64)."""
import collections

from . import _cstructs as S
from . import gemm_desc as G

GemmCfg = collections.namedtuple('GemmCfg', [
    'mode',             # 'conv' (implicit-GEMM convolution, NHWC pixels as rows) or 'rows' (batched row-major product)
    'taps', 'C', 'C2',  # conv: 1 or 9 taps, channels of A (multiple of 64), channels of the K-appended skip operand
    'H', 'W', 's2d',    # conv: image size, stride-2 taps over a space-to-depth input
    'M', 'N', 'K',      # valid rows (conv: pixels of the whole batch; rows: per z), valid columns, rows-mode K (multiple of 64)
    'k_valid',          # rows: valid K extent when below K (the rest is TMA zero fill), else 0
    'num_z', 'nh', 'a_shared', 'b_shared',
    'BN', 'f8', 'npass',
    'o32', 'o16', 'planes',                     # fp32 output, fp16 output, fp16 hi + lo planes
    'bias_n', 'bias_m', 'rowvec', 'residual',   # rowvec: 0 none, 1 one row for all, 2 one row per sample
    'scale', 'st_unit', 'edm',                  # scale != 1; 0 / 2 / 4 channels per statistics partial; edm_out (1 fold, 2 NCHW store)
])

SCALE = 0.70710678                              # the non-unit epilogue scale of a rebuilt launch (UNet skip scale)


def cfg_of(d):
    """The configuration of one ds_gemm_desc (pointer fields may be plan references)."""
    conv = d.a_mode == 0
    K = int(d.cpb) * 64
    return GemmCfg(
        mode='conv' if conv else 'rows', taps=int(d.taps), C=K if conv else 0, C2=int(d.a2_c),
        H=int(d.conv_H) if conv else 0, W=int(d.conv_W) if conv else 0, s2d=any(int(v) for v in d.tap_cb),
        M=int(d.m_valid), N=int(d.n_valid), K=0 if conv else K,
        k_valid=0 if conv or int(d.a_dims[0]) >= K else int(d.a_dims[0]),
        num_z=int(d.num_z), nh=max(int(d.nh), 1),
        a_shared=not conv and d.a_n_per_zb == 0 and d.a_n_per_zh == 0,
        b_shared=not conv and d.b_z_per_zb == 0 and d.b_z_per_zh == 0,
        BN=int(d.BN), f8=bool(d.f8 & 1), npass=int(d.npass),
        o32=bool(d.out_f32), o16=bool(d.out_h16), planes=bool(d.out_h16 and d.o_plane),
        bias_n=bool(d.bias_n), bias_m=bool(d.bias_m), rowvec=(2 if d.rowvec_stride else 1) if d.rowvec else 0,
        residual=bool(d.residual), scale=abs(float(d.scale) - 1.0) > 1e-7,
        st_unit=(2 if int(d.st_unit) == 2 else 4) if d.st_quads else 0, edm=int(d.edm_out))


def plan_configs(pl):
    """Distinct GEMM configurations of a compiled plan, in plan order: {GemmCfg: launches per forward}."""
    out = collections.OrderedDict()
    for i in range(pl.n_ops):
        op = pl.ops_array[i]
        if op.type == S.DS_OP_GEMM:
            c = cfg_of(op.u.gemm)
            out[c] = out.get(c, 0) + 1
    return out


def edm_plan(name, B, f8_min_channels=0, seed=0, dezero=False, norm_jitter=False, with_weights=False):
    """The fp16f8 plan B200Net compiles for an EDM net at batch B (one sigma for the batch, a label per sample), on the host.
    dezero: the weight set bench.py runs (edm_nets.dezero_); norm_jitter: seeded per-channel GroupNorm gains 1 + U(-0.1, 0.1) and
    biases U(-0.1, 0.1) instead of the init's ones and zeros, so that the channels of a group get different coefficients;
    with_weights: return (plan, weight blob bytes)."""
    import torch
    from . import edm_nets, plan as planner
    params, cfg = edm_nets.init_params(name, seed=seed)
    if dezero:
        edm_nets.dezero_(params, cfg['kind'], seed=seed)
    if norm_jitter:
        g = torch.Generator().manual_seed(seed + 4242)
        for k in params:
            if 'norm' in k.rsplit('.', 2)[-2] and params[k].dim() == 1:
                u = torch.rand(params[k].shape, generator=g) * 0.2 - 0.1
                params[k] = (1.0 + u) if k.endswith('.weight') else u
    spec = edm_nets.spec_from_params(params, cfg['img_resolution'], cfg['img_channels'], cfg.get('label_dim', 0))
    spec.sigma_data = 0.5
    wb, info = planner.pack_weights(spec, params, f8=True, f8_min_channels=f8_min_channels)
    pl = planner.compile_plan(spec, wb, info, B, 1, B if spec.label_dim else 0, npass=3, f8=True)
    return (pl, wb.bytes()) if with_weights else pl


def tiles_of(cfg, batch=None):
    """Tiles of the launch make_desc(cfg, batch=...) builds."""
    n_tiles = -(-cfg.N // cfg.BN)
    if cfg.mode == 'conv':
        bn = batch or cfg.M // (cfg.H * cfg.W)
        return -(-(bn * cfg.H * cfg.W) // 128) * n_tiles
    if cfg.num_z > 1:
        return (batch or cfg.num_z) * -(-cfg.M // 128) * n_tiles
    return -(-(batch or cfg.M) // 128) * n_tiles


def ragged_batch(cfg, sms, waves=3):
    """The smallest batch (conv: images; rows: z count, or rows when the plan has a single z) that gives more than `waves` tiles
    per SM and a partial last wave, keeping what the configuration needs: whole 32-row slabs for fused statistics, whole heads."""
    b = 1
    while True:
        t = tiles_of(cfg, b)
        ok = t > waves * sms and t % sms != 0
        if cfg.mode == 'conv':
            ok = ok and not (cfg.st_unit and (b * cfg.H * cfg.W) % 32)
        elif cfg.num_z > 1:
            ok = ok and b % cfg.nh == 0
        else:
            ok = ok and not (cfg.st_unit and b % 32)
        if ok:
            return b
        b += 1


def make_desc(cfg, dev, bn=None, batch=None, pad=False, seed=0):
    """ds_gemm_desc of one configuration on seeded buffers.  Returns (desc, info, bufs): bufs holds every tensor the launch reads
    or writes (keep it alive while the descriptor is used) -- the fp32 originals of the operands ('x', 'w', 'x2', 'w2' in conv
    mode, 'A', 'B' in rows mode), the packed operands, the epilogue inputs and the outputs ('out', 'outh', 'st', 'D'), with their
    layout in 'geom'.  pad=True makes every output wider (ldo > N) and taller (64 more rows per z) than its valid extent and fills
    outputs with NaN, so that a test can see stray and missing stores."""
    import torch
    g = torch.Generator().manual_seed(seed)
    BN = bn or cfg.BN
    N = cfg.N
    nan = float('nan')
    conv = cfg.mode == 'conv'
    if conv:
        Bn = batch or cfg.M // (cfg.H * cfg.W)
        M, nz, mrow = Bn * cfg.H * cfg.W, 1, Bn * cfg.H * cfg.W
    else:
        nz = batch if (batch and cfg.num_z > 1) else cfg.num_z
        M = batch if (batch and cfg.num_z == 1) else cfg.M
        mrow = M
    ldo = (-(-N // 8) * 8 + (8 if pad else 0))
    rows_out = M + (64 if pad else 0)                                  # rows per z of the output buffers
    fill = (lambda shape, dt=torch.float32: torch.full(shape, nan, dtype=dt, device=dev)) if pad else \
           (lambda shape, dt=torch.float32: torch.empty(shape, dtype=dt, device=dev))
    bufs = {}
    rnd = lambda *shape: torch.randn(*shape, generator=g)
    # epilogue inputs: bias along N or M, conditioning rows, residual
    if cfg.bias_n:
        bufs['bias_n'] = rnd(N).to(dev)
    if cfg.bias_m:
        bufs['bias_m'] = rnd(M).to(dev)
    nsamp = Bn if conv else 1
    if cfg.rowvec:
        bufs['rowvec'] = rnd(nsamp if cfg.rowvec == 2 else 1, N).to(dev)
    if cfg.residual:
        bufs['residual'] = rnd(mrow, N).to(dev)
    if cfg.o32:
        bufs['out'] = fill((nz * rows_out, ldo))
    if cfg.o16:
        bufs['outh'] = fill((2 if cfg.planes else 1, nz * rows_out, ldo), torch.float16)
    scale = SCALE if cfg.scale else 1.0
    ptr = lambda k: bufs[k].data_ptr() if k in bufs else 0
    if conv:
        H, W, C, C2, k = cfg.H, cfg.W, cfg.C, cfg.C2, (3 if cfg.taps == 9 else 1)
        cphys = 4 * C if cfg.s2d else C
        bufs['x'] = (rnd(Bn, H, W, cphys) * 1.5).to(dev)
        bufs['w'] = (rnd(N, C, k, k) / (k * C ** 0.5)).to(dev)
        if C2:
            bufs['x2'] = (rnd(Bn, H, W, C2) * 2.0).to(dev)
            bufs['w2'] = (rnd(N, C2, 1, 1) / C2 ** 0.5).to(dev)
        # weights packed at pick_bn's row count, as the plan packs them (conv_gemm's B extent); other N tiles read TMA zero fill
        if cfg.f8:
            blob, shift = G.pack_conv_weight_f8(bufs['w'].cpu(), bufs['w2'].cpu() if C2 else None)
            bufs['wp'], acc = blob.to(dev), 2.0 ** -shift
            bufs['a'] = G.act_planes_f8(bufs['x'].cpu()).to(dev)
            if C2:
                bufs['a2'] = G.act_planes_f8(bufs['x2'].cpu()).to(dev)
        else:
            bufs['wp'], acc = G.pack_conv_weight(bufs['w'].cpu(), bufs['w2'].cpu() if C2 else None).to(dev), 1.0
            bufs['a'] = G.split_planes(bufs['x'])
            if C2:
                bufs['a2'] = G.split_planes(bufs['x2'])
        edm = nchw_out = None
        if cfg.edm:
            bufs['edm_x'] = rnd(Bn, N, H, W).to(dev)
            bufs['edm_coef'] = (torch.rand(Bn, 4, generator=g) + 0.5).to(dev)
            bufs['D'] = fill((Bn * N * H * W + (64 if pad else 0),))
            if cfg.edm == 2:
                nchw_out = (N, ptr('D'))
            else:
                edm = (ptr('edm_x'), ptr('edm_coef'), 4, N, ptr('D'))
        d, info = G.conv_gemm(ptr('a'), Bn, H, W, C, ptr('wp'), N, taps=cfg.taps, npass=cfg.npass, a2_ptr=ptr('a2'), C2=C2,
                              out_f32=ptr('out'), out_h16=ptr('outh'), o_planes=2 if cfg.planes else 1, ldo=ldo, bias=ptr('bias_n'),
                              rowvec=ptr('rowvec'), rowvec_stride=N if cfg.rowvec == 2 else 0, residual=ptr('residual'), ldr=N,
                              scale=scale, edm=edm, nchw_out=nchw_out, bn=BN, s2d=cfg.s2d, f8=cfg.f8, acc_scale=acc)
        d.bias_m = ptr('bias_m')
        d.o_plane = rows_out * ldo if cfg.planes else 0
    else:
        assert not cfg.rowvec and not cfg.f8 and not cfg.edm, 'rows mode has no conditioning rows, f8 passes or image store'
        K = cfg.K
        za, zb = (1 if cfg.a_shared else nz), (1 if cfg.b_shared else nz)
        A, B = rnd(za, M, K), rnd(zb, N, K) / K ** 0.5
        if cfg.k_valid:                                                # columns past the valid K extent must never be read
            A[..., cfg.k_valid:] = nan
            B[..., cfg.k_valid:] = nan
        bufs['A'], bufs['B'] = A.to(dev), B.to(dev)
        bufs['a'], bufs['b'] = G.split_planes(bufs['A']), G.split_planes(bufs['B'])
        nh = cfg.nh
        d, info = G.rows_gemm(ptr('a'), M, K, za, ptr('b'), N, K, zb, K, num_z=nz, nh=nh, m_valid=M, n_valid=N, npass=cfg.npass,
                              a_n_per_zb=0 if cfg.a_shared else nh, a_n_per_zh=0 if cfg.a_shared else 1,
                              b_z_per_zb=0 if cfg.b_shared else nh, b_z_per_zh=0 if cfg.b_shared else 1,
                              out_f32=ptr('out'), out_h16=ptr('outh'), o_zb=nh * rows_out * ldo, o_zh=rows_out * ldo, ldo=ldo,
                              o_plane=nz * rows_out * ldo if cfg.planes else 0, bias_n=ptr('bias_n'), bias_m=ptr('bias_m'),
                              residual=ptr('residual'), ldr=N, scale=scale, bn=BN,
                              a_k_valid=cfg.k_valid or None, b_k_valid=cfg.k_valid or None)
    if cfg.st_unit:
        bufs['st'] = fill((mrow // 32 + (1 if pad else 0), N // cfg.st_unit, 2))
        d.st_quads, d.st_unit = ptr('st'), cfg.st_unit
    bufs['geom'] = dict(M=M, num_z=nz, rows_out=rows_out, ldo=ldo, batch=Bn if conv else nz, scale=scale,
                        acc_scale=float(d.acc_scale))
    return d, info, bufs

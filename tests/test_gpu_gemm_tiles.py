"""The GEMM kernel at the tile widths, ring depths and multi-tile schedules the benchmarked plans run, against float64.

test_gpu_kernels.py lets fill_bn pick the N tile, which on its small problems means BN <= 64, an 8-stage ring and one tile per CTA.
Here the N tile is pinned instead: every BN from 16 to 256, and every GEMM configuration of the plans the benchmark compiles, each
rebuilt (gemm_replay) with a batch that gives every persistent CTA more than three tiles and leaves the last wave partial, so the
operand ring wraps across tiles.  Outputs are wider and taller than their valid extent and pre-filled with NaN: the padding must
stay NaN and every valid element must be written.  One row per launch goes into the coverage table printed at the end."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernels import _f8_reference

pytestmark = pytest.mark.gpu

TOL_X3 = 2e-5          # fp16 hi/lo, three passes: against the exact product
TOL_1P = 1e-4          # single pass: against the product of the fp16 hi planes
TOL_F8_MODEL = 5e-6    # f8: against hi x hi + lo8 x w_hi8 + hi8 x w_lo8 of the decoded operands
TOL_F8_EXACT = 1e-4    # f8: against the exact product
TOL_PLANES = 5e-5      # fp16 hi + lo output planes
TOL_STATS = 1e-4       # GroupNorm partials: of the kernel's own fp32 output
TOL_EDM = 3e-5         # EDM output fold
K_F8_CAL = 2560        # contraction length up to which TOL_F8_MODEL was calibrated (test_conv_f8_mode: K <= 2.5k terms)
TOL_F8_MODEL_LONG_K = 3e-5   # f8 against the operand model beyond K_F8_CAL; see f8_model_tol
CHUNK = 1 << 24        # float64 elements per operand chunk of the reference


def contraction(cfg):
    return cfg.taps * cfg.C + cfg.C2 if cfg.mode == 'conv' else (cfg.k_valid or cfg.K)


def f8_model_tol(cfg):
    """The one bound that depends on K.  In f8 mode the e4m3 corrections accumulate first, on a sum still ~2^-11 of its final size;
    the fp16 hi x hi product then adds K / 16 wgmma steps at full magnitude, and on H100 the fp32 accumulation error of those steps
    grows linearly with K.  Against the operand model (which has no other error) that is all the comparison sees: measured on an
    H100 80GB HBM3 with the seeded operands of gemm_replay, 5.1e-6 at K = 4608 (the CIFAR-10 3x3 512-channel convs), 9-10e-6 at
    K = 13824, 2.1e-5 at K = 23040 (SD-1.5 3x3 2560-channel convs).  Up to K_F8_CAL the calibrated 5e-6 holds; beyond it the fixed
    3e-5 covers every benchmarked plan (K <= 25k).  Every other comparison -- f8 against the exact product included -- keeps its
    tolerance at every K."""
    return TOL_F8_MODEL if contraction(cfg) <= K_F8_CAL else TOL_F8_MODEL_LONG_K

TABLE = []             # one dict per launch


@pytest.fixture(scope='module')
def lib():
    from diff_sampler_b200 import _lib
    return _lib


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev():
    return torch.device('cuda:0')


def base_cfg(**kw):
    from diff_sampler_b200.gemm_replay import GemmCfg
    c = dict(mode='conv', taps=9, C=64, C2=0, H=16, W=16, s2d=False, M=0, N=64, K=0, k_valid=0, num_z=1, nh=1, a_shared=False,
             b_shared=False, BN=64, f8=False, npass=3, o32=True, o16=False, planes=False, bias_n=False, bias_m=False, rowvec=0,
             residual=False, scale=False, st_unit=0, edm=0)
    c.update(kw)
    if c['mode'] == 'conv' and not c['M']:
        c['M'] = c['H'] * c['W']
    return GemmCfg(**c)


def full_epilogue(cfg, unit):
    """Every epilogue stage at once: bias, per-sample conditioning row (conv) or bias along M (rows), residual, scale, fp32 and fp16
    hi/lo outputs, GroupNorm partials."""
    conv = cfg.mode == 'conv'
    return cfg._replace(bias_n=True, bias_m=not conv, rowvec=2 if conv else 0, residual=True, scale=True, o32=True, o16=True,
                        planes=True, st_unit=unit if conv else 0)


# --------------------------------------------------------------------------------------------- float64 references
def _conv_acc(x, wt, d):
    """Implicit-GEMM convolution with the descriptor's tap table: x [b, H, W, Cphys], wt [N, taps, C] -> [b*H*W, N] (float64)."""
    b, H, W, _ = x.shape
    C = wt.shape[2]
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    acc = torch.zeros(b, H, W, wt.shape[0], dtype=torch.float64, device=x.device)
    for t in range(int(d.taps)):
        dh, dw, cb = int(d.tap_dh[t]), int(d.tap_dw[t]), int(d.tap_cb[t])
        acc += xp[:, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W, cb:cb + C] @ wt[:, t, :].t()
    return acc.reshape(b * H * W, -1)


def _conv_refs(cfg, d, bufs):
    """Per batch chunk: (row offset, {name: accumulator [rows, N]}) with 'exact' and, by mode, 'hi' (single pass) or 'model' (f8)."""
    x, w = bufs['x'], bufs['w']
    N, k = w.shape[0], w.shape[2]
    Bn, H, W = x.shape[0], x.shape[1], x.shape[2]
    per_img = H * W * (x.shape[3] + cfg.C2 + N)
    step = max(1, CHUNK // per_img)
    wt = lambda t: t.double().permute(0, 2, 3, 1).reshape(N, k * k, -1)
    for b0 in range(0, Bn, step):
        xs = x[b0:b0 + step]
        x2s = bufs['x2'][b0:b0 + step] if cfg.C2 else None
        out = {}
        exact = _conv_acc(xs.double(), wt(w), d)
        if cfg.C2:
            exact += x2s.double().reshape(-1, cfg.C2) @ bufs['w2'].double().reshape(N, cfg.C2).t()
        out['exact'] = exact
        if cfg.f8:
            ref = _f8_reference(xs.permute(0, 3, 1, 2), w, x2s.permute(0, 3, 1, 2) if cfg.C2 else None, bufs.get('w2'))[0]
            out['model'] = ref.permute(0, 2, 3, 1).reshape(-1, N)
        elif cfg.npass == 1:
            hi = _conv_acc(xs.half().double(), wt(w.half()), d)
            if cfg.C2:
                hi += x2s.half().double().reshape(-1, cfg.C2) @ bufs['w2'].half().double().reshape(N, cfg.C2).t()
            out['hi'] = hi
        yield b0 * H * W, out


def _rows_refs(cfg, bufs):
    """Per z: (z, {name: accumulator [M, N]})."""
    A, B = bufs['A'], bufs['B']
    kv = cfg.k_valid or A.shape[2]
    nz = bufs['geom']['num_z']
    for z in range(nz):
        a, b = A[0 if cfg.a_shared else z, :, :kv], B[0 if cfg.b_shared else z, :, :kv]
        out = {'exact': a.double() @ b.double().t()}
        if cfg.npass == 1:
            out['hi'] = a.half().double() @ b.half().double().t()
        yield z, out


def _epilogue(cfg, bufs, acc, r0):
    """acc (float64 [rows, N], rows r0.. of one z) -> (acc + bias + rowvec + residual) * scale, as the kernel's epilogue."""
    rows = torch.arange(r0, r0 + acc.shape[0], device=acc.device)
    r = acc.clone()
    if cfg.bias_n:
        r += bufs['bias_n'].double()[None, :]
    if cfg.bias_m:
        r += bufs['bias_m'].double()[rows][:, None]
    if cfg.rowvec:
        rv = bufs['rowvec'].double()
        r += rv[rows // (cfg.H * cfg.W)] if cfg.rowvec == 2 else rv[0][None, :]
    if cfg.residual:
        r += bufs['residual'].double()[rows]
    return r * bufs['geom']['scale']


# --------------------------------------------------------------------------------------------- one launch, checked
def run_and_check(lib, sms, cfg, kind, batch=None):
    from diff_sampler_b200.gemm_replay import make_desc
    d, info, bufs = make_desc(cfg, dev(), batch=batch, pad=True)
    conf = lib.gemm_config(d)
    tiles = int(d.num_z) * int(d.m_tiles) * int(d.n_tiles)
    assert conf['grid'] == min(tiles, sms), (conf, tiles)
    lib.op_launch(d)
    torch.cuda.synchronize()
    g = bufs['geom']
    M, N, nz, rows_out, ldo = g['M'], cfg.N, g['num_z'], g['rows_out'], g['ldo']
    primary = 'model' if cfg.f8 else ('hi' if cfg.npass == 1 else 'exact')
    tol = {'exact': TOL_X3, 'hi': TOL_1P, 'model': f8_model_tol(cfg)}[primary]
    errs, over = {}, []

    def note(name, err, scale, t):
        e = err / max(scale, 1e-30)
        errs[name] = max(errs.get(name, 0.0), e)
        if e > t:
            over.append((name, e, t))

    def valid_mask(shape, rows):
        m = torch.zeros(shape, dtype=torch.bool, device=dev())
        m.view(nz, rows_out, ldo)[:, :rows, :N] = True
        return m
    # the reference, per chunk; the scale of each comparison is the largest |reference| of the whole output
    chunks = []
    if cfg.mode == 'conv':
        for r0, accs in _conv_refs(cfg, d, bufs):
            chunks.append((0, r0, {k: _epilogue(cfg, bufs, v, r0) for k, v in accs.items()}))
    else:
        for z, accs in _rows_refs(cfg, bufs):
            chunks.append((z, 0, {k: _epilogue(cfg, bufs, v, 0) for k, v in accs.items()}))
    scale = max(c[2]['exact'].abs().max().item() for c in chunks)
    if 'out' in bufs:
        out = bufs['out']
        ov = out.view(nz, rows_out, ldo)
        for z, r0, refs in chunks:
            got = ov[z, r0:r0 + refs['exact'].shape[0], :N].double()
            assert torch.isfinite(got).all(), (kind, 'fp32 output: a valid element was not written')
            note(primary, (got - refs[primary]).abs().max().item(), scale, tol)
            if cfg.f8:
                note('exact', (got - refs['exact']).abs().max().item(), scale, TOL_F8_EXACT)
        assert torch.isnan(out[~valid_mask(out.shape, M)]).all(), (kind, 'fp32 output: a store landed outside the valid extent')
    if 'outh' in bufs:
        oh = bufs['outh']
        for p in range(oh.shape[0]):
            assert torch.isnan(oh[p][~valid_mask(oh[p].shape, M)].float()).all(), (kind, f'fp16 plane {p}: stray store')
        hv = oh.view(oh.shape[0], nz, rows_out, ldo)
        for z, r0, refs in chunks:
            n = refs['exact'].shape[0]
            got = hv[:, z, r0:r0 + n, :N].double()
            assert torch.isfinite(got).all(), (kind, 'fp16 output: a valid element was not written')
            got = got.sum(0) if cfg.planes else got[0]
            note('planes' if cfg.planes else 'fp16', (got - refs[primary]).abs().max().item(), scale,
                 TOL_PLANES if cfg.planes else 1e-3)
    if 'st' in bufs:
        u = cfg.st_unit
        st = bufs['st']
        y = bufs['out'].view(nz, rows_out, ldo)[0, :M, :N].double().reshape(M // 32, 32, N // u, u)
        ref = torch.stack([y.sum(dim=(1, 3)), (y ** 2).sum(dim=(1, 3))], dim=-1)
        assert torch.isfinite(st[:M // 32]).all(), (kind, 'statistics: a partial was not written')
        assert torch.isnan(st[M // 32:]).all(), (kind, 'statistics: stray store')
        e = (st[:M // 32].double() - ref).abs().max().item()
        note('stats', e, max(1.0, ref.abs().max().item()), TOL_STATS)
    if cfg.edm:
        Bn, H, W = g['batch'], cfg.H, cfg.W
        D = bufs['D']
        nvalid = Bn * N * H * W
        assert torch.isnan(D[nvalid:]).all(), (kind, 'image store outside the batch')
        Dv = D[:nvalid].view(Bn, N, H, W)
        assert torch.isfinite(Dv).all(), (kind, 'image element not written')
        coef = bufs['edm_coef'].double()
        for z, r0, refs in chunks:
            b0, nb = r0 // (H * W), refs['exact'].shape[0] // (H * W)
            got = Dv[b0:b0 + nb].double()
            for name in ((primary, 'exact') if cfg.f8 else (primary,)):
                rr = refs[name].view(nb, H, W, N).permute(0, 3, 1, 2)
                if cfg.edm == 1:
                    cs, co = coef[b0:b0 + nb, 0, None, None, None], coef[b0:b0 + nb, 1, None, None, None]
                    rr = cs * bufs['edm_x'][b0:b0 + nb].double() + co * rr
                t = TOL_F8_EXACT if name == 'exact' and cfg.f8 else (TOL_EDM if cfg.edm == 1 else tol)
                sc = max(scale, rr.abs().max().item())
                note('edm' if name == primary else 'edm_exact', (got - rr).abs().max().item(), sc, t)
    epi = '+'.join(n for n, on in (('bias', cfg.bias_n), ('bias_m', cfg.bias_m), ('rowvec', cfg.rowvec), ('res', cfg.residual),
                                   ('scale', cfg.scale), ('f32', cfg.o32), ('hilo' if cfg.planes else 'h16', cfg.o16),
                                   (f'st{cfg.st_unit}', cfg.st_unit), (f'edm{cfg.edm}', cfg.edm)) if on)
    row = dict(kind=kind, BN=int(d.BN), stages=conf['stages'], grid=conf['grid'], tiles=tiles, per_cta=tiles / conf['grid'],
                      mode=cfg.mode + ('' if cfg.mode == 'rows' else f' {cfg.H}x{cfg.W}'), f8=cfg.f8, npass=cfg.npass,
                      half_block=cfg.f8 and ((cfg.C // 64) % 2 == 1 or (cfg.C2 // 64) % 2 == 1), W=cfg.W, epi=epi,
                      err=errs.get(primary, 0.0), err_exact=errs.get('exact', 0.0) if cfg.f8 else None, K=contraction(cfg),
                      shape=f'C{cfg.C}+{cfg.C2} N{N}' if cfg.mode == 'conv' else f'M{M} N{N} K{cfg.K} z{nz}')
    TABLE.append(row)
    print(_fmt(row))
    assert not over, (kind, cfg, over)
    return errs


def _fmt(r):
    return (f"{r['kind']:18s} {r['BN']:4d} {r['stages']:3d} {r['grid']:4d} {r['tiles']:6d} {r['per_cta']:5.2f} {r['mode']:12s} "
            f"{int(r['f8']):2d} {r['npass']:2d} {r['shape']:22s} {r['K']:6d} {r['epi']:44s} {r['err']:9.2e}"
            + (f" {r['err_exact']:9.2e}" if r['err_exact'] is not None else ''))


# --------------------------------------------------------------------------------------------- 1. N-tile sweep
BNS = list(range(16, 257, 16))


@pytest.mark.parametrize('npass', [3, 1])
@pytest.mark.parametrize('bn', BNS)
def test_tile_sweep_conv(lib, sms, bn, npass):
    """3x3 conv, 64 -> 3 BN - 8 channels: three N tiles, the last one partial; 27 (or 9) ring stages per tile."""
    cfg = base_cfg(BN=bn, N=3 * bn - 8, npass=npass, bias_n=True)
    run_and_check(lib, sms, cfg, f'sweep conv np{npass}', from_batch(cfg, sms))


@pytest.mark.parametrize('unit', [4, 2])
@pytest.mark.parametrize('bn', [128, 192, 256])
def test_tile_sweep_conv_full_epilogue(lib, sms, bn, unit):
    cfg = full_epilogue(base_cfg(BN=bn, N=3 * bn - 8, C2=64), unit)
    run_and_check(lib, sms, cfg, f'sweep conv epi', from_batch(cfg, sms))


@pytest.mark.parametrize('npass', [3, 1])
@pytest.mark.parametrize('bn', BNS)
def test_tile_sweep_rows(lib, sms, bn, npass):
    """Batched rows mode, two heads per batch entry: 200 rows (a partial M tile) x (3 BN - 8) x 192, fp16 hi/lo output at BN >= 128
    with every rows-mode epilogue input."""
    cfg = base_cfg(mode='rows', taps=1, C=0, H=0, W=0, M=200, N=3 * bn - 8, K=192, num_z=2, nh=2, BN=bn, npass=npass, bias_n=True)
    if bn >= 128:
        cfg = full_epilogue(cfg, 0)
    run_and_check(lib, sms, cfg, f'sweep rows np{npass}', from_batch(cfg, sms))


@pytest.mark.parametrize('cin', [192, 256])
@pytest.mark.parametrize('bn', [64, 128, 192, 256])
def test_tile_sweep_f8(lib, sms, bn, cin):
    """f8 mode; Cin = 192 leaves the second 128-channel e4m3 block of every tap half empty, as does the 64-channel skip operand."""
    cfg = base_cfg(BN=bn, N=3 * bn - 8, C=cin, f8=True, bias_n=True)
    if bn >= 128:
        cfg = full_epilogue(cfg._replace(C2=64), 4 if bn != 192 else 2)
    run_and_check(lib, sms, cfg, 'sweep f8', from_batch(cfg, sms))


def from_batch(cfg, sms):
    from diff_sampler_b200.gemm_replay import ragged_batch
    return ragged_batch(cfg, sms)


# --------------------------------------------------------------------------------------------- 2. plan replay
WORKLOADS = ['cifar10', 'ffhq', 'imagenet64', 'sd15', 'sd_vae']
_REPLAYED = set()


def bench_plan(name):
    """The plan of one benchmarked workload, at the batch and precision bench.py runs it: the EDM nets in fp16f8 (FFHQ with f8 only
    in blocks of >= 256 channels), the SD-1.5 eps-net at batch 8 under classifier-free guidance (16 contexts), its VAE decoder."""
    return bench_plan_weights(name, dezero=False)[0]


def bench_plan_weights(name, batch=None, dezero=True):
    """bench_plan with its weights: (plan, weight blob bytes, model config).  batch replaces the benchmark batch (EDM nets: images;
    SD-1.5: prompts, run under guidance as 2 x batch; VAE: latents).  dezero gives the EDM nets the weight set bench.py runs, with
    seeded per-channel GroupNorm gains and biases (the init's are ones and zeros, which would hide a coefficient applied to the
    wrong channel of its group)."""
    from diff_sampler_b200 import gemm_replay
    if name in ('cifar10', 'ffhq', 'imagenet64'):
        from diff_sampler_b200 import edm_nets
        B = batch or {'cifar10': 512}.get(name, 256)
        pl, wb = gemm_replay.edm_plan(name, B, 256 if name == 'ffhq' else 0, dezero=dezero, norm_jitter=dezero, with_weights=True)
        return pl, wb, edm_nets.NET_CONFIGS[name]
    if name == 'sd15':
        from diff_sampler_b200 import ldm_plan
        from oracle import ldm_oracle as LO
        P, cfg = LO.make_params('sd15')
        st = ldm_plan.ldm_structure(P, cfg['num_heads'])
        wb, info = ldm_plan.pack_ldm_weights(st, P, f8=True, f8_linear=True)
        B = batch or 8
        pl = ldm_plan.compile_ldm_plan(st, wb, info, B, 2 * B, 1, cfg['img_resolution'], npass=3, f8=True, f8_linear=True)
        return pl, wb.bytes(), cfg
    from diff_sampler_b200 import vae_plan
    from oracle import vae_oracle as VO
    P, cfg = VO.make_params('sd_vae', seed=0)
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    return vae_plan.compile_vae_plan(mods, meta, wb, batch or 1, 64), wb.bytes(), dict(cfg, **meta)


def replay_key(cfg):
    """A configuration with its batch dimension dropped: that is the free parameter of a replay."""
    if cfg.mode == 'conv':
        return cfg._replace(M=cfg.H * cfg.W)
    return cfg._replace(num_z=cfg.nh) if cfg.num_z > 1 else cfg._replace(M=0)


@pytest.mark.parametrize('workload', WORKLOADS)
def test_plan_replay(lib, sms, workload):
    from diff_sampler_b200.gemm_replay import plan_configs, ragged_batch
    cfgs = plan_configs(bench_plan(workload))
    assert cfgs
    n = 0
    for cfg in cfgs:
        key = replay_key(cfg)
        if key in _REPLAYED:
            continue
        _REPLAYED.add(key)
        run_and_check(lib, sms, cfg, f'plan {workload}', ragged_batch(cfg, sms))
        n += 1
    print(f'{workload}: {len(cfgs)} GEMM configurations, {n} not replayed by an earlier workload')


# --------------------------------------------------------------------------------------------- 3. coverage table
def test_coverage_table(sms):
    if not TABLE:
        pytest.skip('no launch of this module ran')
    print()
    print(f"{'launch':18s} {'BN':>4s} {'stg':>3s} {'grid':>4s} {'tiles':>6s} {'/CTA':>5s} {'mode':12s} {'f8':>2s} {'np':>2s} "
          f"{'shape':22s} {'K':>6s} {'epilogue':44s} {'err':>9s} {'f8 exact':>9s}")
    print('err: output error / max |reference| against the exact product (fp16x3), the fp16 hi planes (single pass) or the operand '
          'model (f8)')
    for r in TABLE:
        print(_fmt(r))
    print('rows-mode replays lay the operands out z-major: the head windows of the plans\' attention products (a_c_per_zh, '
          'b_k_per_zh, b_row_per_zh, b_k0) are not reproduced; test_gpu_kernels.py covers them at the BN fill_bn picks, and '
          'test_gpu_plan_ops.py runs the plans\' own descriptors')
    # each assertion covers what ran (a -k selection may keep only some launches)
    sweep = [r for r in TABLE if r['kind'].startswith('sweep')]
    plan = [r for r in TABLE if r['kind'].startswith('plan')]
    assert all(r['per_cta'] > 3 and r['grid'] == sms for r in sweep)
    if {r['BN'] for r in sweep if r['kind'].startswith('sweep conv np')} >= set(BNS):
        assert {r['stages'] for r in sweep} >= {4, 5, 6, 7, 8}, 'every ring depth'
    if plan:
        assert all(r['per_cta'] >= 3 and r['grid'] == sms for r in plan)
        if any(r['kind'] == 'plan sd_vae' for r in plan):
            assert any(r['W'] > 128 for r in plan if r['kind'] == 'plan sd_vae'), 'the VAE rows wider than one M tile'

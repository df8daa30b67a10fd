"""SHA-256 digests of compiled plans: the op array bytes, arena size and layout, plan meta and the weight blob.  Used by
tests/test_cm_host.py to check that the EDM, CM, LDM, VAE / VQ, CLIP and optimal-denoiser plans -- the tiny interpreter variants,
the compile options and the full-size and benchmarked nets -- compile byte for byte as pinned in tests/golden/plan_digests.json.
Regenerate that file only when a change to those plans is intended:

    python tests/plan_digest.py > tests/golden/plan_digests.json
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def digest(pl, blob):
    h = hashlib.sha256()
    h.update(bytes(memoryview(pl.ops_array).cast('B')))
    h.update(json.dumps([int(pl.arena_bytes), sorted((k, int(v)) for k, v in pl.arena_offsets.items()),
                         sorted((k, repr(v)) for k, v in pl.meta.items())]).encode())
    h.update(hashlib.sha256(blob).digest())
    return h.hexdigest()


def _edm_variants():
    from diff_sampler_b200 import edm_nets, plan as planner
    from oracle import edm_oracle as O
    for name in ('tiny_song', 'tiny_adm', 'tiny_song4'):
        P, St = O.make_net(name, seed=0, dezero=True)
        spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
        spec.sigma_data = 0.5
        for f8 in (False, True):
            wb, info = planner.pack_weights(spec, P, f8=f8)
            blob = wb.bytes()
            for B, nsig, nlab in ((2, 1, 2 if spec.label_dim else 0), (3, 3, 3 if spec.label_dim else 0), (3, 1, 1 if spec.label_dim else 0)):
                for npass in ((3,) if f8 else (3, 1)):
                    pl = planner.compile_plan(spec, wb, info, B, nsig, nlab, npass=npass, f8=f8)
                    yield f'edm/{name}/f8={int(f8)}/B{B}/s{nsig}/l{nlab}/p{npass}', pl, blob


def _edm_options():
    """compile_plan's unfused GroupNorm statistics and unfused attention, and f8 with the narrow blocks kept in fp16x3."""
    from diff_sampler_b200 import edm_nets, plan as planner
    from oracle import edm_oracle as O
    for name in ('tiny_song', 'tiny_adm'):
        P, St = O.make_net(name, seed=0, dezero=True)
        spec = edm_nets.spec_from_params(P, St['img_resolution'], St['img_channels'], St['label_dim'])
        spec.sigma_data = 0.5
        wb, info = planner.pack_weights(spec, P)
        nlab = 2 if spec.label_dim else 0
        for opt in ('fuse_stats', 'flash_attn'):
            yield f'edm/{name}/{opt}=0', planner.compile_plan(spec, wb, info, 2, 1, nlab, npass=3, **{opt: False}), wb.bytes()
        if name == 'tiny_song':
            wb, info = planner.pack_weights(spec, P, f8=True, f8_min_channels=128)
            yield f'edm/{name}/f8=1/min128', planner.compile_plan(spec, wb, info, 2, 1, 0, npass=3, f8=True), wb.bytes()


def _cm_variants():
    """The Consistency-Models nets: the tiny setting in fp16x3 and f8, and the full-size LSUN-256 net."""
    from diff_sampler_b200 import cm_net, plan as planner
    for setting, tag, B, f8s in ((cm_net.TINY_SETTING, 'tiny', 3, (False, True)), (None, 'lsun256', 2, (False,))):
        spec, params = cm_net.convert(cm_net.init_state_dict(setting), setting)
        for f8 in f8s:
            wb, info = planner.pack_weights(spec, params, f8=f8)
            yield f'cm/{tag}/f8={int(f8)}/B{B}', planner.compile_plan(spec, wb, info, B, 1, 0, npass=3, f8=f8), wb.bytes()


def _uncond_ldm_variants():
    """The unconditional LDM eps-net with 32-wide heads in pairs and padded to 64, and the full-size LDM-VQ-f4 net at batch 32."""
    import ldm_uncond_ref as U
    from diff_sampler_b200 import ldm_plan
    for name, B, pairs_opts in (('tiny_uncond', 2, (True, False)), ('ldm_vq4', 32, (True,))):
        P, cfg = U.make_params(name)
        st = ldm_plan.ldm_structure(P, 8, cfg['num_head_channels'])
        for pairs in pairs_opts:
            wb, info = ldm_plan.pack_ldm_weights(st, P, head_pairs=pairs)
            pl = ldm_plan.compile_ldm_plan(st, wb, info, B, B, B, cfg['img_resolution'])
            yield f'ldm_uncond/{name}/pairs={int(pairs)}/B{B}', pl, wb.bytes()


def _vq_variants():
    """The VQ decoder without and with the codebook snap (and its index read-out), and the full-size VQ-f4 decoder at 64 -> 256."""
    import vq_ref as VQ
    from diff_sampler_b200 import vae_plan
    for name, B, R, kws in (('tiny_vq', 2, 8, ({}, {'quantize': True}, {'quantize': True, 'debug_indices': True})),
                            ('vq_f4', 1, 64, ({'quantize': True},))):
        P, _ = VQ.make_params(name)
        mods, meta = vae_plan.vae_structure(P)
        wb = vae_plan.pack_vae_weights(mods, meta, P)
        for kw in kws:
            key = f'vq/{name}/B{B}/R{R}/' + (','.join(sorted(kw)) or 'plain')
            yield key, vae_plan.compile_vae_plan(mods, meta, wb, B, R, **kw), wb.bytes()


def _optimal_variants():
    """The small optimal-denoiser plans (their blob is the dataset: only its layout is part of the plan)."""
    from diff_sampler_b200 import optimal as OPT
    for N, D, B, nsig, knn in ((300, 192, 4, 1, 0), (65, 105, 3, 3, 0), (130, 48, 2, 1, 5), (70, 105, 3, 3, 0), (70, 105, 3, 3, 4)):
        g = OPT._Geometry(N, D)
        wb, _ = OPT.blob_layout(g)
        yield f'optimal/N{N}/D{D}/B{B}/s{nsig}/knn{knn}', OPT.compile_plan(g, wb, B, nsig, 1.0, knn=knn), wb.bytes()


def _small_variants():
    import torch
    from diff_sampler_b200 import clip_plan, ldm_plan, vae_plan
    from oracle import clip_oracle as CO
    from oracle import ldm_oracle as LO
    from oracle import vae_oracle as VO
    P, cfg = LO.make_params('tiny_ldm')
    st = ldm_plan.ldm_structure(P, cfg['num_heads'])
    for f8, f8l in ((False, False), (True, False), (True, True)):
        wb, info = ldm_plan.pack_ldm_weights(st, P, f8=f8, f8_linear=f8l)
        pl = ldm_plan.compile_ldm_plan(st, wb, info, 2, 2, 1, cfg['img_resolution'], npass=3, f8=f8, f8_linear=f8l)
        yield f'ldm/tiny_ldm/f8={int(f8)}/f8l={int(f8l)}', pl, wb.bytes()
    P, cfg = VO.make_params('tiny_vae', seed=0)
    mods, meta = vae_plan.vae_structure(P)
    wb = vae_plan.pack_vae_weights(mods, meta, P)
    yield 'vae/tiny_vae', vae_plan.compile_vae_plan(mods, meta, wb, 2, 8), wb.bytes()
    P, cfg = CO.make_params('tiny_clip', seed=0)
    ccfg = clip_plan.clip_config(P)
    wb = clip_plan.pack_clip_weights(P, ccfg)
    yield 'clip/tiny_clip', clip_plan.compile_clip_plan(ccfg, wb, 2, 24), wb.bytes()
    del torch


def _benchmarked():
    """The five benchmarked plans at their benchmark batch, with bench.py's weight set."""
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_gpu_gemm_tiles import bench_plan_weights
    for name in ('cifar10', 'ffhq', 'imagenet64', 'sd15', 'sd_vae'):
        pl, blob, _ = bench_plan_weights(name)
        yield f'bench/{name}', pl, blob


def all_digests(benchmarked=True):
    out = {}
    gens = [_edm_variants(), _edm_options(), _cm_variants(), _uncond_ldm_variants(), _vq_variants(), _optimal_variants(),
            _small_variants()] + ([_benchmarked()] if benchmarked else [])
    for g in gens:
        for key, pl, blob in g:
            out[key] = digest(pl, blob)
    return out


if __name__ == '__main__':
    print(json.dumps(all_digests(), indent=1, sort_keys=True))

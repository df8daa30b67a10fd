"""SHA-256 digests of compiled plans: the op array bytes, arena size and layout, plan meta and the weight blob.  Used by
tests/test_cm_host.py to check that the EDM, LDM, VAE and CLIP plans -- the tiny interpreter variants and the benchmarked ones --
compile byte for byte as they did before the Consistency-Models lowering (tests/golden/plan_digests.json).  Regenerate that file
only when a change to those plans is intended:

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
    gens = [_edm_variants(), _small_variants()] + ([_benchmarked()] if benchmarked else [])
    for g in gens:
        for key, pl, blob in g:
            out[key] = digest(pl, blob)
    return out


if __name__ == '__main__':
    print(json.dumps(all_digests(), indent=1, sort_keys=True))

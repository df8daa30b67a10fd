"""Writes tests/golden/ref_ldm_uncond.npz from the real reference: its `UNetModel` in the LSUN-Bedroom / FFHQ LDM-VQ-f4 form
(use_spatial_transformer=False, num_head_channels=32: the legacy AttentionBlock) at the tiny_uncond size of tests/ldm_uncond_ref.py,
loaded with that file's non-zero parameter recipe (the reference's zero-initialised proj_out / out.2 would make parity vacuous), under
CFGPrecond(guidance_type='uncond') with the configs' beta schedule.  Stored: D at several sigma and at per-sample sigma, the
middle-block output (AMED's tap, solvers_amed.py:11-12), the 'discrete' schedule, a DPM-Solver++(2M) sample, and the state-dict
names and shapes of the reference UNetModel at the tiny size and at the full lsun_bedrooms-ldm-vq-4.yaml size.

    python tools/gen_ldm_uncond_golden.py          (needs the reference checkout at /root/reference, CPU only)
"""
import os
import sys
import types

import numpy as np
import torch

REF = '/root/reference'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'ref_ldm_uncond.npz')


def main():
    sys.path[:0] = [os.path.join(REF, 'diff-solvers-main'), ROOT, os.path.join(ROOT, 'tests')]
    oc, lc = types.ModuleType('omegaconf'), types.ModuleType('omegaconf.listconfig')
    lc.ListConfig = type('ListConfig', (list,), {})
    oc.listconfig = lc
    sys.modules.setdefault('omegaconf', oc)
    sys.modules.setdefault('omegaconf.listconfig', lc)
    from models.ldm.modules.diffusionmodules.openaimodel import UNetModel
    from models.networks_edm import CFGPrecond
    import solver_utils as RU
    import solvers as RS
    import ldm_uncond_ref as U
    from oracle import edm_oracle as O
    from oracle import ldm_oracle as LO
    import json

    def build(cfg):
        # lsun_bedrooms-ldm-vq-4.yaml:14-34 (attention_resolutions are downsampling factors)
        return UNetModel(image_size=cfg['img_resolution'], in_channels=cfg['in_channels'], out_channels=cfg['out_channels'],
                         model_channels=cfg['model_channels'], attention_resolutions=list(cfg['attention_resolutions']),
                         num_res_blocks=cfg['num_res_blocks'], channel_mult=list(cfg['channel_mult']), num_heads=-1,
                         num_head_channels=cfg['num_head_channels'], use_spatial_transformer=False,
                         use_checkpoint=False).eval().requires_grad_(False)
    shapes = {}
    for name in ('ldm_vq4', 'tiny_uncond'):
        shapes[name] = [[k, list(v.shape)] for k, v in build(U.CONFIGS[name]).state_dict().items()]
    name = 'tiny_uncond'
    P, cfg = U.make_params(name)
    unet = build(cfg)
    sd = unet.state_dict()
    assert list(sd) == list(P), [k for k in sd if k not in P][:5] + [k for k in P if k not in sd][:5]
    for k in sd:
        assert tuple(sd[k].shape) == tuple(P[k].shape), (k, sd[k].shape, P[k].shape)
    unet.load_state_dict(P)

    class Shim(torch.nn.Module):
        def __init__(self, u):
            super().__init__()
            self.u = u
            self.alphas_cumprod = LO.make_alphas_cumprod(*U.BETAS)

        def apply_model(self, x, t, cond):
            return self.u(x, t)
    net = CFGPrecond(Shim(unet), img_resolution=cfg['img_resolution'], img_channels=cfg['in_channels'], guidance_rate=1.0,
                     guidance_type='uncond', label_dim=0).eval()
    taps = []
    unet.middle_block.register_forward_hook(lambda m, i, o: taps.append(o.detach().clone()))
    G = {'sigma_range': np.array([net.sigma_min, net.sigma_max]),
         'state_dict_shapes_json': np.frombuffer(json.dumps(shapes).encode(), dtype=np.uint8)}
    B, R = 2, cfg['img_resolution']
    x = O.stacked_randn(range(B), (cfg['in_channels'], R, R))
    G['x'] = x.numpy()
    with torch.no_grad():
        for sigma in (14.6, 1.0, 0.05):
            taps.clear()
            G[f'D/{sigma}'] = net(x * sigma, torch.tensor([sigma])).numpy()
            G[f'tap/{sigma}'] = taps[-1].mean(dim=1).numpy()
        sig = torch.tensor([5.0, 0.3])
        G['D/persample'] = net(x * sig[:, None, None, None], sig).numpy()
        ts = RU.get_schedule(5, net.sigma_min, net.sigma_max, device=torch.device('cpu'), schedule_type='discrete', schedule_rho=1, net=net)
        G['sched_discrete'] = ts.numpy()
        G['sample_dpmpp'] = RS.dpm_pp_sampler(net, x, num_steps=5, sigma_min=net.sigma_min, sigma_max=net.sigma_max,
                                              schedule_type='discrete', schedule_rho=1, max_order=2, predict_x0=False).numpy()
    np.savez_compressed(OUT, **G)
    print('wrote', OUT, sorted(G))


if __name__ == '__main__':
    torch.set_num_threads(os.cpu_count())
    main()

"""Write tests/golden/ref_opt.npz: diff-analyzer's own get_denoised_opt and optimal_sampler (diff-analyzer-main/solvers.py:19-28,
:773-868), run on the CPU in fp32 over a small seeded dataset, for tests/opt_ref.py's float64 restatement to be pinned to.

    python tools/gen_opt_golden.py /path/to/diff-analyzer-main

The reference is imported from the given directory, never copied."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from opt_ref import golden_dataset, golden_latents, GOLDEN_SIGMAS, GOLDEN_SAMPLER_RUNS   # noqa: E402


def main(ref_dir):
    sys.path.insert(0, ref_dir)
    import solvers as ref
    torch.manual_seed(0)
    ds = golden_dataset()
    lat = golden_latents()
    out = {'dataset': ds.numpy(), 'latents': lat.numpy()}
    for j, s in enumerate(GOLDEN_SIGMAS):
        xs = ds[:4] + s * lat if s < 1 else lat * s
        out[f'opt_x_{j}'] = xs.numpy()
        out[f'opt_d_{j}'] = ref.get_denoised_opt(xs, torch.tensor(s), ds).numpy()
    for name, kw in GOLDEN_SAMPLER_RUNS.items():
        kw = dict(kw)
        if 't_steps' in kw:
            kw['t_steps'] = torch.tensor(kw['t_steps'])
        r = ref.optimal_sampler(None, lat, ds, **kw)
        if isinstance(r, tuple):
            for k, v in zip(('xt', 'den', 'eps'), r):
                out[f'{name}_{k}'] = v.numpy()
        else:
            out[f'{name}_x'] = r.numpy()
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'ref_opt.npz'), **out)
    print('wrote', sorted(out))


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

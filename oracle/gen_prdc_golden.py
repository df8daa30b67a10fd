"""Writes tests/golden/ref_prdc.npz: sfd-main/prdc.py's own compute_prdc (realism included) and compute_nearest_neighbour_distances
on the seeded golden cases of tests/prdc_ref.py (features on a 1/16 grid, stored as their uint8 codes), for the float64 restatement
and the native metrics to be pinned to bit for bit.

    python oracle/gen_prdc_golden.py /path/to/sfd-main

The reference is imported from the given directory, never copied; it needs scikit-learn."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from prdc_ref import features, golden_cases   # noqa: E402


def main(ref_dir):
    sys.path.insert(0, ref_dir)
    import prdc as ref
    out = {}
    for name, r, f, k in golden_cases():
        out[f'{name}/real'], out[f'{name}/fake'], out[f'{name}/k'] = r.numpy(), f.numpy(), np.int64(k)
        R, F = features(r).numpy(), features(f).numpy()            # float64, as prdc.py's get_representations buffers are
        with np.errstate(divide='ignore', invalid='ignore'):
            d = ref.compute_prdc(R, F, k, realism=True)
        for key, v in d.items():
            out[f'{name}/{key}'] = np.asarray(v)
        out[f'{name}/radii'] = ref.compute_nearest_neighbour_distances(R, k)
        out[f'{name}/fake_radii'] = ref.compute_nearest_neighbour_distances(F, k)
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'ref_prdc.npz'), **out)
    print('wrote', len(out), 'arrays')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

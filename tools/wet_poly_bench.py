"""wet_ground_batch with estimation_method='linear' against 'poly' on 32 clouds of 131 072 rows (median of 10 calls, each
ending in a device synchronise; 'poly' includes its copy of NumPy's state back to the host), and the oracle's per-cloud
'poly' on the host.  Prints one JSON object with the card's name and power limit read in the same run; needs a GPU."""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                            # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud                        # noqa: E402

B, N_AZ, REPS = 32, 2048, 10


def main():
    eng = SnowfallEngine(0)
    clouds = [synthetic_cloud(seed=1000 + b, n_azimuth=N_AZ) for b in range(B)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    res = {'card': measure.card(), 'clouds': B, 'rows_per_cloud': int(clouds[0].shape[0])}
    np.random.seed(0)
    for method in ('linear', 'poly'):
        res[f'{method}_ms'] = float(np.median(measure.time_calls(
            lambda: eng.wet_ground_batch(pts, off, estimation_method=method), REPS, 1)))
    eng.check()
    codes = eng.wet_ground_batch(pts, off, estimation_method='poly')['passthrough'].cpu().numpy()
    res['poly_augmented_clouds'] = int((codes == 0).sum())
    if '--no-oracle' not in sys.argv:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import wet_poly_oracle
        plane = eng.wet_ground_batch(pts[:off[1]], off[:2])['plane'][0].cpu().numpy()
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            res['oracle_poly_ms_per_cloud'] = float(np.mean(measure.time_calls(
                lambda: wet_poly_oracle.ground_water_augmentation(clouds[0], plane=(plane[:3], plane[3]),
                                                                  least_populated='first_min'), 3, 0)))
    print(json.dumps(res))


if __name__ == '__main__':
    main()

"""wet_ground_batch with estimation_method='linear' against 'poly' on 32 clouds of 131 072 rows (median of 10 calls, each
ending in a device synchronise; 'poly' includes its copy of NumPy's state back to the host), and the oracle's per-cloud
'poly' on the host.  Prints one JSON object with the card's name and power limit read in the same run; needs a GPU."""
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_snow_sim_b200.engine import SnowfallEngine                            # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud                        # noqa: E402

B, N_AZ, REPS = 32, 2048, 10


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def timed(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    eng = SnowfallEngine(0)
    clouds = [synthetic_cloud(seed=1000 + b, n_azimuth=N_AZ) for b in range(B)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    res = {'card': card(), 'clouds': B, 'rows_per_cloud': int(clouds[0].shape[0])}
    np.random.seed(0)
    for method in ('linear', 'poly'):
        res[f'{method}_ms'] = timed(lambda: eng.wet_ground_batch(pts, off, estimation_method=method))
    eng.check()
    codes = eng.wet_ground_batch(pts, off, estimation_method='poly')['passthrough'].cpu().numpy()
    res['poly_augmented_clouds'] = int((codes == 0).sum())
    if '--no-oracle' not in sys.argv:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import wet_poly_oracle
        plane = eng.wet_ground_batch(pts[:off[1]], off[:2])['plane'][0].cpu().numpy()
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            t0 = time.perf_counter()
            for _ in range(3):
                wet_poly_oracle.ground_water_augmentation(clouds[0], plane=(plane[:3], plane[3]),
                                              least_populated='first_min')
        res['oracle_poly_ms_per_cloud'] = (time.perf_counter() - t0) / 3 * 1e3
    print(json.dumps(res))


if __name__ == '__main__':
    main()

"""Where a solve tile's time goes: the share of each phase of k_solve in the summed warp cycles, on the snowfall bench's
batch (32 clouds x 131 072 points from bench.make_workload, two input batches alternating, full augment() with the
device pre-pass).  Prints one JSON object: the phase shares, tiles per warp, the listed beams per work class and the card
with its power limit.

    python tools/solve_phases.py [--steps 20] [--keep DIR]

The phase clocks exist only in a library built with -DLSS_SOLVE_PHASE_CLOCKS (csrc/solve.cu), so this copies the
repository's sources to a temporary directory, builds the instrumented library there and runs the workload on it; the
tree's own build is left as it is.  --keep DIR builds in DIR instead and keeps it.  Needs a GPU."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ['tile_fetch', 'fill', 'range_sort_claiming', 'pulses', 'piece_sweep', 'piece_eval_argmax', 'stores_stats']
LIST_CLASSES = 128


def class_name(c):
    """work class of csrc/solve.cu (k_scan): 127 - min(127, 2 min(L, 63) + far), far = target beyond 40 m"""
    v = LIST_CLASSES - 1 - c
    return f'L={v // 2}{"+" if v // 2 == 63 else ""},{"far" if v & 1 else "near"}'


def build_copy(dst):
    keep = ('lidar_snow_sim_b200', 'include', 'bench.py', 'tools', 'BASELINE.json')
    for name in keep:
        src = os.path.join(ROOT, name)
        if os.path.isdir(src):
            shutil.copytree(src, os.path.join(dst, name), dirs_exist_ok=True,
                            ignore=shutil.ignore_patterns('_obj', '*.so', '__pycache__'))
        elif os.path.exists(src):
            shutil.copy2(src, dst)
    env = dict(os.environ, LSS_NVCC_FLAGS='-DLSS_SOLVE_PHASE_CLOCKS')
    subprocess.check_call([sys.executable, '-m', 'lidar_snow_sim_b200.build'], cwd=dst, env=env,
                          stdout=subprocess.DEVNULL)


def run(steps):
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    import measure
    from lidar_snow_sim_b200 import _lib
    from lidar_snow_sim_b200.engine import SnowfallEngine
    from lidar_snow_sim_b200.snowfall.sampling import sample_table_set
    dev = torch.device('cuda', 0)
    eng = SnowfallEngine(0)
    tid = eng.upload_tables(sample_table_set(bench.MODE, bench.SNOWFALL_RATE, bench.TERMINAL_VELOCITY,
                                             seed=bench.TABLE_SEED))
    batches = [bench.make_workload(0, bench.BATCH_PER_GPU), bench.make_workload(0, bench.BATCH_PER_GPU, seed0=500000)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in batches[0][0]])]).astype(np.int64)
    pts = [torch.from_numpy(np.concatenate(c)).to(dev) for c, _ in batches]
    outs = [{}, {}]

    def step(k):
        eng.snowfall_batch(tid, pts[k & 1], off, batches[k & 1][1], bench.DIV_DEG, device_prepass=True, out=outs[k & 1])

    words = (__import__('ctypes').c_uint64 * (len(PHASES) + 2 + LIST_CLASSES))()
    for k in range(4):
        step(k)
    _lib.check(eng.lib.lss_debug_solve_phases(eng.h, 1, None, 0), eng.h)
    for k in range(steps):
        step(k)
    _lib.check(eng.lib.lss_debug_solve_phases(eng.h, 1, words, len(words)), eng.h)
    v = [int(x) for x in words]
    cyc = v[:len(PHASES)]
    tiles, warps = v[len(PHASES)], v[len(PHASES) + 1]
    cls = v[len(PHASES) + 2:]
    total = sum(cyc)
    gpu = measure.card()
    out = {'metric': 'k_solve phase shares of the summed warp cycles (clock64 stamps, -DLSS_SOLVE_PHASE_CLOCKS build)',
           'workload': f'bench.make_workload: {bench.BATCH_PER_GPU} clouds x {int(off[-1]) // bench.BATCH_PER_GPU} points, '
                       f'2 batches alternating, {steps} steps',
           'share': {p: c / total for p, c in zip(PHASES, cyc)},
           'fetch_plus_fill_share': (cyc[0] + cyc[1]) / total,
           'cycles_per_tile': {p: c / tiles for p, c in zip(PHASES, cyc)},
           'tiles_per_step': tiles / steps, 'warps_per_launch': warps / steps, 'tiles_per_warp': tiles / warps,
           'listed_beams_per_step': sum(cls) / steps,
           'listed_beams_per_class_per_step': {class_name(c): n / steps for c, n in enumerate(cls) if n},
           'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w']}
    print(json.dumps(out))
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--keep', metavar='DIR', default=None)
    ap.add_argument('--run', action='store_true', help=argparse.SUPPRESS)      # inside the instrumented copy
    args = ap.parse_args()
    if args.run:
        run(args.steps)
        return
    tmp = None if args.keep else tempfile.mkdtemp(prefix='lss_solve_phases_')
    dst = args.keep or tmp
    try:
        os.makedirs(dst, exist_ok=True)
        build_copy(dst)
        subprocess.check_call([sys.executable, os.path.join(dst, 'tools', 'solve_phases.py'), '--run',
                               '--steps', str(args.steps)], cwd=dst)
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()

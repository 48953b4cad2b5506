"""PA-AUG on the host: the parameter parser and the planner with the NumPy restatement of the kernels
(tests/pa_aug_model.py) against the unmodified reference's results (tests/golden/pa_aug.npz,
tools/make_golden_pa_aug.py).  No GPU."""
import os

import numpy as np
import pytest

from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, box_planes, interpret_pa_aug_param, plan_cloud
from pa_aug_model import counts_of, execute, partition

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'pa_aug.npz')
CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']
G = np.load(GOLDEN)
CASES = sorted({int(k[1:].split('_')[0]) for k in G.files if k.startswith('c')})
PARSER = sorted({int(k[6:].split('_')[0]) for k in G.files if k.startswith('parser')})


def case(k):
    p = f'c{k}_'
    c = {f[len(p):]: G[f] for f in G.files if f.startswith(p)}
    c['param'] = None if not bool(c['has_param']) else str(c['param'])
    c['gt_names'] = np.asarray([CLASS_NAMES[int(v) - 1] for v in c['boxes'][:, -1]])
    return c


def rng_state_equal(c):
    _, keys, pos, has_gauss, gauss = np.random.get_state()
    return (np.array_equal(keys, c['st_keys']) and pos == int(c['st_pos']) and has_gauss == int(c['st_gauss'][0])
            and (not has_gauss or gauss == c['st_gauss'][1]))


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize('k', PARSER)
def test_parser(k):
    s = None if bool(G[f'parser{k}_none']) else str(G[f'parser{k}_in'])
    want = str(G[f'parser{k}_out'])
    try:
        got = repr(interpret_pa_aug_param(s))
    except Exception as ex:                                        # noqa: BLE001
        got = type(ex).__name__
    assert got == want


@pytest.mark.parametrize('k', CASES)
def test_plan_and_model_reproduce_reference(k):
    c = case(k)
    pts, boxes, names = c['pts'], c['boxes'], c['gt_names']
    planes = box_planes(boxes, names)
    members, bg = partition(pts, planes, [NUM_PARTITION[n] for n in names], boxes.dtype == np.float64)
    np.random.seed(int(c['seed']))
    if 'exc' in c:
        with pytest.raises(Exception) as ei:
            plan = plan_cloud(counts_of(members), len(bg), boxes, names, len(CLASS_NAMES), c['param'],
                              n_features=pts.shape[1])
            execute(plan, pts, members, bg)
        assert type(ei.value).__name__ == str(c['exc'])
    else:
        plan = plan_cloud(counts_of(members), len(bg), boxes, names, len(CLASS_NAMES), c['param'],
                          n_features=pts.shape[1])
        out = execute(plan, pts, members, bg)
        assert same_bits(out, c['out']), str(c['name'])
        assert plan['mask'] == c['mask'].tolist()
    assert rng_state_equal(c)

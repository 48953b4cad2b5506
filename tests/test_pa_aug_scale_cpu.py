"""PA-AUG at full size on the host: the planner with the NumPy restatement of the kernels (tests/pa_aug_model.py)
against the unmodified reference on the cases of tests/pa_aug_scale_case.py (tests/golden/pa_aug_full.npz): the
partition counts, the output's digest, the mask and NumPy's state after every call, cloud after cloud.  This pins the
restatement the GPU test falls back on to locate a mismatch row by row.  No GPU."""
import numpy as np
import pytest

import pa_aug_scale_case as sc
from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, box_planes
from pa_aug_model import partition
from pa_aug_scale_case import model_run

G = sc.load()
IDS = [G[k]['name'].replace(' ', '_') for k in sorted(G)]


def test_fixture_holds_every_case():
    cs = sc.cases()
    assert [G[k]['name'] for k in sorted(G)] == [c['name'] for c in cs]
    for k, c in enumerate(cs):
        assert (G[k]['param'], G[k]['seed'], len(G[k]['clouds'])) == (c['param'], c['seed'], len(c['clouds']))


@pytest.mark.parametrize('k', sorted(G), ids=IDS)
def test_model_reproduces_reference(k):
    c, g = sc.cases()[k], G[k]
    for i, ((pts, boxes), r) in enumerate(zip(c['clouds'], g['clouds'])):
        assert sc.input_digests(pts, boxes) == r['in_sha'].tolist(), f'cloud {i}: the regenerated inputs differ'
    np.random.seed(c['seed'])
    for i, ((pts, boxes), r) in enumerate(zip(c['clouds'], g['clouds'])):
        if 'exc' in r:
            with pytest.raises(Exception) as ei:
                model_run(pts, boxes, c['param'])
            assert type(ei.value).__name__ == str(r['exc'])
        else:
            counts, n_bg, plan, out = model_run(pts, boxes, c['param'])
            assert np.array_equal(counts, r['counts']) and n_bg == int(r['n_bg']), f'cloud {i}: partition counts'
            assert out.shape == tuple(r['out_shape']) and out.dtype.str == str(r['out_dtype'])
            assert sc.digest(out) == str(r['out_sha']), f'cloud {i}: rows'
            assert plan['mask'] == r['mask'].tolist()
        assert sc.rng_state_equal(r), f'cloud {i}: NumPy state'


def test_fps_tie_case_has_ties_across_threads_and_warps():
    """the FPS tie case is what it claims: one thinned part, whose member list repeats its first 37 rows' coordinates
    256 * FPS_M and 256 * FPS_M + 37 rows on, and the reference's output holds first copies picked at those ties"""
    c = [c for c in sc.cases() if c['name'] == 'fps ties'][0]
    pts, boxes = c['clouds'][0]
    names = sc.names_of(boxes)
    members, bg = partition(pts, box_planes(boxes, names), [8], False)
    sizes = [len(m) for m in members[0]]
    assert sizes[0] == 256 * sc.FPS_M + 100 + 2 * sc.FPS_WARP and sum(sizes) == sizes[0]
    rows = pts[members[0][0]]
    for off in (256 * sc.FPS_M, 256 * sc.FPS_M + sc.FPS_WARP):
        assert np.array_equal(rows[:sc.FPS_WARP, :3], rows[off:off + sc.FPS_WARP, :3])
        assert not np.array_equal(rows[:sc.FPS_WARP, 3], rows[off:off + sc.FPS_WARP, 3])
    np.random.seed(c['seed'])
    _, _, plan, out = model_run(pts, boxes, c['param'])
    assert len(plan['fps']) == 1
    n_fps = plan['fps'][0][2]
    picked = out[:n_fps]
    tied = np.isin(picked[:, :3].astype(np.float32).view(np.uint32).view('V12'),
                   rows[:sc.FPS_WARP, :3].view('V12'))
    assert tied.sum() >= 5                                          # enough tie picks for a wrong rule to show


def test_nan_row_sits_past_every_parts_first_256_members():
    """the NaN row, last in its cloud, is the last member of every part, and every part holds more than 256 rows, so
    the thread of k_pa_fps that reads it reads another row of the part first"""
    c = [c for c in sc.cases() if c['name'] == 'nan row'][0]
    pts, boxes = c['clouds'][0]
    assert np.isnan(pts[-1, 0]) and not np.isnan(pts[:-1]).any()
    names = sc.names_of(boxes)
    members, _ = partition(pts, box_planes(boxes, names), [NUM_PARTITION[n] for n in names], False)
    for parts in members:
        for m in parts:
            assert m[-1] == pts.shape[0] - 1 and len(m) > 256

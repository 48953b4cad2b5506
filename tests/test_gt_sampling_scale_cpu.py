"""The GT-sampling planner and the NumPy restatement of the paste kernels at full size, against the unmodified reference
(tests/golden/gt_sampling_full.npz, the cases of tests/gt_sampling_scale_case.py).  No GPU: the planner runs with the
valid candidates the reference found, and the restated k_gt_mark / k_gt_paste / apply_ops must reproduce the rows'
digest after every queue entry.  The rotation's restatement is held to torch's CPU matmul on every row, signed zeros,
NaN and inf included, and the recorded valid candidates to the compiled boxes_iou_bev_cpu's rule."""
import functools
import json

import numpy as np
import pytest
import torch

import gt_sampling_case as G
import gt_sampling_scale_case as S
from lidar_snow_sim_b200.augmentor import DataAugmentor
from lidar_snow_sim_b200.augmentor import plan as P

GOLD = np.load(S.GOLDEN)
IDS = [c['name'].replace(' ', '_') for c in S.CASES]


def cloud(k, i):
    q = f'c{k}_{i}_'
    return {f[len(q):]: GOLD[f] for f in GOLD.files if f.startswith(q)}


def valid_of(r):
    return [r[f'valid_{j}'] for j in range(int(r['n_classes']))]


def state_equal(r):
    _, keys, pos, has_gauss, gauss = np.random.get_state()
    return (np.array_equal(keys, r['st_keys']) and pos == int(r['st_pos']) and has_gauss == int(r['st_gauss'][0])
            and (not has_gauss or gauss == r['st_gauss'][1]))


@pytest.fixture(scope='module')
def dbroot(tmp_path_factory):
    root = tmp_path_factory.mktemp('gtdb_full')
    for kind in ('main', 'grid'):
        assert S.database_digest(kind) == str(GOLD[f'db_sha_{kind}']), \
            f'the regenerated {kind} database differs from the fixture\'s (not a planner fault)'
        S.write_database(kind, str(root / kind))
    G.write_calib(str(root))
    return root


@functools.lru_cache(maxsize=None)
def _run(k, root):
    """case k through the planner (with the reference's valid candidates) and the restated kernels: per cloud
    (data dict after finish, plan, rows entering the rotation, stage rows' digests, state / groups equal)"""
    case = S.CASES[k]
    aug = DataAugmentor(f'{root}/{case["db"]}', S.augmentor_cfg(case), case['classes'])
    db_rows = aug.sampler._db_host
    calib = G.Calib(f'{root}/calib.txt')
    np.random.seed(case['seed'])
    out = []
    for i, sc in enumerate(S.scenes(k)):
        r = cloud(k, i)
        assert S.input_digest(sc) == str(r['in_sha']), \
            f'{case["name"]} cloud {i}: the regenerated inputs differ from the fixture\'s (not a planner fault)'
        d = S.data_dict(sc, calib, case['classes'])
        pts = d.pop('points')
        plan = P.draw(aug.queue, [d])[0]
        gt_before = d['gt_boxes'].copy()
        P.finish(aug.queue, plan, valid_of(r), final=True)
        stages = S.model_stages(aug.queue, plan, pts, db_rows)
        names = [n for n, _ in aug.queue]
        pre_rot = stages[names.index('random_world_rotation') - 1] if 'random_world_rotation' in names else None
        out.append(dict(d=d, plan=plan, gt_before=gt_before, pre_rot=pre_rot, stage_sha=[S.digest(s) for s in stages],
                        rows=stages[-1][::S.ROW_STRIDE], state=state_equal(r),
                        groups=S.groups_json(aug.sampler.sample_groups) == str(r['groups'])))
    return out


def _first_row(got, want):
    if got.shape != want.shape:
        return f'shapes {got.shape} != {want.shape}'
    bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))[0]
    return f'first differing sampled row {bad[0] * S.ROW_STRIDE}: {got[bad[0]]} != {want[bad[0]]}' if bad.size else ''


@pytest.mark.parametrize('k', range(len(S.CASES)), ids=IDS)
def test_planner_and_restated_kernels_reproduce_every_stage(dbroot, k):
    """every queue entry's rows (by digest), the boxes, names, NumPy's state and sample_groups after every cloud"""
    case = S.CASES[k]
    for i, m in enumerate(_run(k, str(dbroot))):
        r = cloud(k, i)
        want = r['stage_sha'].tolist()
        for j, (g, w) in enumerate(zip(m['stage_sha'], want)):
            assert g == w, f'{case["name"]} cloud {i}: the rows after queue entry {j} differ from the reference\'s' + \
                (f' ({_first_row(m["rows"], r["rows"])})' if j == len(want) - 1 else '')
        assert len(m['stage_sha']) == len(want)
        assert m['stage_sha'][-1] == str(r['out_sha'])
        assert S.digest(m['d']['gt_boxes']) == str(r['boxes_sha']), f'{case["name"]} cloud {i}: boxes'
        assert m['d']['gt_names'].astype(str).tolist() == r['names'].tolist(), f'{case["name"]} cloud {i}: names'
        assert m['state'] and m['groups'], f'{case["name"]} cloud {i}: NumPy state / sample_groups'


def test_fmaf_is_exact():
    """the restated fmaf against exact rational arithmetic, midpoints of float32 and signed zeros included"""
    from fractions import Fraction
    rng = np.random.default_rng(5)
    a = rng.uniform(-4, 4, 4000).astype(np.float32)
    b = rng.uniform(-4, 4, 4000).astype(np.float32)
    c = rng.uniform(-16, 16, 4000).astype(np.float32)
    # a * b + c exactly between two float32: a = 1 + 2^-12, b = 1 + 2^-12, c = -(1 + 2^-11) + k 2^-23 ...
    one = np.float32(1)
    a[:4] = one + np.float32(2.0 ** -12)
    b[:4] = one + np.float32(2.0 ** -12)
    c[:4] = np.float32([0.0, 2.0 ** -23, -(2.0 ** -23), 1.0])
    a[4:8], b[4:8], c[4:8] = np.float32([-0.0, 0.0, -1.5, 1.5]), np.float32([0.5, -0.5, 0.0, -0.0]), \
        np.float32([0.0, -0.0, -0.0, 0.0])
    got = S.fmaf(a, b, c)
    for i in range(a.shape[0]):
        e = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        w = np.float32(float(e))                       # float() rounds the fraction once to double: exact here
        assert abs(Fraction(float(got[i])) - e) <= abs(Fraction(float(w)) - e), i
    assert got[:8].view(np.uint32)[4:].tolist() == np.float32([0.0, -0.0, -0.0, 0.0]).view(np.uint32).tolist()
    # float64 would round 1 + 2^-11 + 2^-24 + 2^-47 ... here: the midpoint case goes through the fractions
    x = np.float32(1 + 2.0 ** -23)
    y = np.float32(1 + 2.0 ** -23)
    z = np.float32(-(2.0 ** -46))                      # x y = 1 + 2^-22 + 2^-46: + z is exactly 1 + 2^-22
    assert S.fmaf(np.array([x]), np.array([y]), np.array([z]))[0] == np.float32(1 + 2.0 ** -22)


def _torch_rot(rows, angle):
    return P.rotate_along_z(np.ascontiguousarray(rows, np.float32), angle)[0][:, :3]


@pytest.mark.parametrize('angle', [0.3187, -0.3187, 0.0, np.pi / 2, np.pi])
def test_rotation_formula_equals_torch_on_signed_zeros(angle):
    """the formula apply_ops uses equals torch.matmul of rotate_points_along_z on every row, bit for bit: 131 072
    random rows, every sign pattern of zeros, NaN and inf rows"""
    rng = np.random.default_rng(int(abs(angle) * 1e4) + 1)
    v = np.float32([0.0, -0.0, 1.5, -1.5, np.nan, np.inf, -np.inf])
    combos = np.array(np.meshgrid(v, v, v)).reshape(3, -1).T.astype(np.float32)
    rows = np.concatenate([combos, S.special_rows(rng)[:, :3],
                           rng.uniform(-70, 70, (131072, 3)).astype(np.float32)])
    rows = np.concatenate([rows, np.zeros((rows.shape[0], 2), np.float32)], 1)
    want, c, s = P.rotate_along_z(rows, angle)
    want = want[:, :3]
    got = S.rotate(rows[:, :3], c, s)
    # with two non-finite coordinates two NaNs meet, and which one x86's BLAS keeps depends on its code path (the same
    # row gives other bits at another position in the batch): there only where the NaNs are is held
    two = (~np.isfinite(rows[:, :3])).sum(axis=1) >= 2
    assert np.array_equal(np.isnan(got[two]), np.isnan(want[two]))
    assert np.array_equal(got[two][~np.isnan(got[two])], want[two][~np.isnan(want[two])])
    bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1) & ~two)[0]
    assert bad.size == 0, f'{bad.size} rows differ, first {rows[bad[0], :3]}: {got[bad[0]]} != {want[bad[0]]}'
    assert (rows[~two, :3] == 0).any(axis=1).sum() > 100 and np.isnan(got[~two]).any()


@pytest.mark.parametrize('k', [k for k, c in enumerate(S.CASES) if c['rot'] is not None], ids=lambda k: IDS[k])
def test_rotation_formula_equals_torch_on_every_case_row(dbroot, k):
    for i, m in enumerate(_run(k, str(dbroot))):
        rows = m['pre_rot'].astype(np.float32)
        angle = [v for kind, v in m['plan'].steps if kind == 'rot'][0]
        _, c, s = P.rotate_along_z(rows[:1], angle)
        got, want = S.rotate(rows[:, :3], c, s), _torch_rot(rows, angle)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f'{S.CASES[k]["name"]} cloud {i}'


@pytest.mark.parametrize('k', [k for k, c in enumerate(S.CASES) if c['db'] == 'main'], ids=lambda k: IDS[k])
def test_recorded_valid_candidates_follow_boxes_iou_bev_cpu(dbroot, k):
    """the reference's valid candidates are those with zero BEV IoU against the gt boxes, the earlier classes' valid
    candidates and the other candidates of their class (boxes_iou_bev_cpu of the compiled reference)"""
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip('oracle/_ref not built (no reference checkout at build time)')
    for i, m in enumerate(_run(k, str(dbroot))):
        existed = m['gt_before'][:, :7]
        for j, ((_, boxes), want) in enumerate(zip(m['plan'].classes, valid_of(cloud(k, i)))):
            iou2 = ref_ops.boxes_iou_bev_cpu(boxes[:, :7], boxes[:, :7])
            iou2[range(boxes.shape[0]), range(boxes.shape[0])] = 0
            iou1 = ref_ops.boxes_iou_bev_cpu(boxes[:, :7], existed) if existed.shape[0] else iou2
            got = np.nonzero((iou1.max(axis=1) + iou2.max(axis=1)) == 0)[0]
            assert got.tolist() == want.tolist(), f'{S.CASES[k]["name"]} cloud {i} class {j}'
            existed = np.concatenate([existed, boxes[got, :7]]).astype(np.float32) if got.size else existed


def test_fixture_holds_the_cases():
    assert [str(GOLD[f'c{k}_name']) for k in range(len(S.CASES))] == [c['name'] for c in S.CASES]
    assert [int(GOLD[f'c{k}_n_clouds']) for k in range(len(S.CASES))] == [c['scenes'] for c in S.CASES]
    k = S.case_index('box limit')
    assert [len(v) for v in valid_of(cloud(k, 0))] == [S.BOX_LIMIT]
    assert [len(v) for v in valid_of(cloud(k + 1, 0))] == [S.BOX_LIMIT + 1]
    assert json.loads(str(cloud(S.case_index('group order'), 0)['groups'])).keys() == {'Cyclist', 'Pedestrian', 'Car'}

"""The device DATA_AUGMENTOR at full size against the unmodified reference (tests/golden/gt_sampling_full.npz, the
cases of tests/gt_sampling_scale_case.py): forward cloud by cloud with rows bit for bit (x and y included, signed zeros
and NaN rows too), forward_batch on the bench workload against the reference's 32 calls, slot-compacted input, a
repeated call, and the 5 688-box limit of k_gt_mark's shared memory.  A mismatch is reported at the first queue entry
and row that differ."""
import copy

import numpy as np
import pytest
import torch

import gt_sampling_case as G
import gt_sampling_scale_case as S
from lidar_snow_sim_b200.augmentor import DataAugmentor
from lidar_snow_sim_b200.augmentor import plan as P
from lidar_snow_sim_b200.engine import default_engine
from test_gt_sampling_scale_cpu import GOLD, IDS, cloud, state_equal, valid_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dbroot(engine, tmp_path_factory):
    root = tmp_path_factory.mktemp('gtdb_full_gpu')
    for kind in ('main', 'grid'):
        assert S.database_digest(kind) == str(GOLD[f'db_sha_{kind}']), \
            f'the regenerated {kind} database differs from the fixture\'s (not a kernel fault)'
        S.write_database(kind, str(root / kind))
    G.write_calib(str(root))
    return root


def augmentor(root, k):
    case = S.CASES[k]
    return DataAugmentor(f'{root}/{case["db"]}', S.augmentor_cfg(case), case['classes'])


def checked_scenes(k):
    scenes = S.scenes(k)
    for i, sc in enumerate(scenes):
        assert S.input_digest(sc) == str(cloud(k, i)['in_sha']), \
            f'{S.CASES[k]["name"]} cloud {i}: the regenerated inputs differ from the fixture\'s (not a kernel fault)'
    return scenes


def snapshot(aug):
    return np.random.get_state(), copy.deepcopy({c: dict(v) for c, v in aug.sampler.sample_groups.items()})


def restore(aug, snap):
    np.random.set_state(snap[0])
    for c, v in snap[1].items():
        aug.sampler.sample_groups[c].update(copy.deepcopy(v))


def first_difference(aug, k, i, sc, calib, snap):
    """rerun cloud i from the state before it with the queue cut after each entry: the first entry whose rows differ
    from the reference's digest, and the first row there that differs from the restatement"""
    r = cloud(k, i)
    full = aug.queue
    try:
        for j in range(len(full)):
            restore(aug, snap)
            aug.queue = full[:j + 1]
            try:
                got = aug.forward(S.data_dict(sc, calib, S.CASES[k]['classes']))['points']
            except NotImplementedError:                              # float64 rows before the rotation
                continue
            if S.digest(got) == str(r['stage_sha'][j]):
                continue
            restore(aug, snap)
            d = S.data_dict(sc, calib, S.CASES[k]['classes'])
            pts = d.pop('points')
            plan = P.draw(full, [d])[0]
            P.finish(full, plan, valid_of(r), final=True)
            want = S.model_stages(full, plan, pts, aug.sampler._db_host_copy)[j].astype(np.float32)
            if got.shape != want.shape:
                return f'queue entry {j} ({full[j][0]}): {got.shape[0]} rows, the restatement {want.shape[0]}'
            bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))[0]
            return (f'queue entry {j} ({full[j][0]}): {bad.size} rows differ from the restatement' +
                    (f', first row {bad[0]}: {got[bad[0]]} != {want[bad[0]]}' if bad.size else ''))
        return 'every queue entry matches alone'
    finally:
        aug.queue = full


def _keep_db_host(aug):
    aug.sampler._db_host_copy = aug.sampler._db_host.copy()


@pytest.mark.parametrize('k', range(len(S.CASES) - 1), ids=IDS[:-1])
def test_forward_matches_reference(dbroot, k):
    """every cloud's rows, boxes, names, NumPy state and sample_groups after forward, the clouds in turn"""
    case = S.CASES[k]
    scenes = checked_scenes(k)
    aug = augmentor(dbroot, k)
    _keep_db_host(aug)
    calib = G.Calib(f'{dbroot}/calib.txt')
    np.random.seed(case['seed'])
    for i, sc in enumerate(scenes):
        r = cloud(k, i)
        snap = snapshot(aug)
        out = aug.forward(S.data_dict(sc, calib, case['classes']))
        if S.digest(out['points']) != str(r['out_sha']):
            pytest.fail(f'{case["name"]} cloud {i}: {first_difference(aug, k, i, sc, calib, snap)}')
        assert S.digest(out['gt_boxes']) == str(r['boxes_sha']), f'{case["name"]} cloud {i}: boxes'
        assert out['gt_names'].astype(str).tolist() == r['names'].tolist(), f'{case["name"]} cloud {i}: names'
        assert state_equal(r), f'{case["name"]} cloud {i}: NumPy state'
        assert S.groups_json(aug.sampler.sample_groups) == str(r['groups']), f'{case["name"]} cloud {i}: groups'


def _batch(scenes, pad=None):
    rows, offs, cnts = [], [0], []
    for b, sc in enumerate(scenes):
        p = sc['pts'].astype(np.float32)
        cnts.append(p.shape[0])
        if pad is not None:
            p = np.concatenate([p, pad[b]])
        rows.append(p)
        offs.append(offs[-1] + p.shape[0])
    counts = torch.tensor(cnts, dtype=torch.int32, device='cuda') if pad is not None else None
    boxes = np.concatenate([sc['boxes'] for sc in scenes])
    names = np.concatenate([sc['names'] for sc in scenes])
    boff = np.concatenate([[0], np.cumsum([len(sc['names']) for sc in scenes])])
    return torch.from_numpy(np.concatenate(rows)).cuda(), np.array(offs), boxes, boff, names, counts


def _check_batch(r, k, aug):
    got = r['points'].cpu().numpy()
    cnt = r['counts'].cpu().numpy()
    for b in range(S.CASES[k]['scenes']):
        w = cloud(k, b)
        o = got[r['offsets'][b]:r['offsets'][b] + cnt[b]]
        assert S.digest(o) == str(w['out_sha']), f'cloud {b}: rows'
        assert S.digest(r['gt_boxes'][b]) == str(w['boxes_sha']), f'cloud {b}: boxes'
        assert r['gt_names'][b].astype(str).tolist() == w['names'].tolist(), f'cloud {b}: names'
    last = cloud(k, S.CASES[k]['scenes'] - 1)
    assert state_equal(last)
    assert S.groups_json(aug.sampler.sample_groups) == str(last['groups'])


def test_batch_matches_reference_calls_in_turn(dbroot):
    """forward_batch on the bench workload (32 x 131 072 rows) equals the reference's 32 sequential calls"""
    k = S.case_index('bench')
    aug = augmentor(dbroot, k)
    args = _batch(checked_scenes(k))
    np.random.seed(S.CASES[k]['seed'])
    r = aug.forward_batch(*args[:5])
    _check_batch(r, k, aug)


def test_slot_compacted_batch_matches_reference(dbroot):
    """counts= with 500 rows behind every count at the centres of database boxes (inside the candidates' removal
    boxes when sampled): the result equals the reference's"""
    k = S.case_index('bench')
    infos, _ = S.database('main')
    centres = np.array([np.asarray(i['box3d_lidar'][:3], np.float32) for c in infos for i in infos[c]])
    rng = np.random.default_rng(21)
    pad = []
    for _ in range(S.CASES[k]['scenes']):
        p = np.zeros((500, S.F), np.float32)
        p[:, :3] = centres[rng.choice(centres.shape[0], 500, replace=False)]
        pad.append(p)
    aug = augmentor(dbroot, k)
    args = _batch(checked_scenes(k), pad)
    np.random.seed(S.CASES[k]['seed'])
    r = aug.forward_batch(*args[:5], counts=args[5])
    _check_batch(r, k, aug)


def test_repeated_call_gives_identical_bits(dbroot):
    k = S.case_index('flip xy')
    res = []
    for _ in range(2):
        aug = augmentor(dbroot, k)
        np.random.seed(S.CASES[k]['seed'])
        r = aug.forward_batch(*_batch(checked_scenes(k))[:5])
        got, cnt = r['points'].cpu().numpy(), r['counts'].cpu().numpy()
        res.append((cnt, [got[o:o + n] for o, n in zip(r['offsets'], cnt)]))      # each slot's counted rows
    assert np.array_equal(res[0][0], res[1][0])
    for a, b in zip(res[0][1], res[1][1]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_one_box_over_the_limit_raises_before_the_paste_kernels(dbroot):
    """5 689 valid sampled boxes in one cloud (the reference takes them; 5 688 is the most k_gt_mark's 200 KB hold):
    ValueError from the library's check, with no launch of the paste call"""
    k = S.case_index('box limit + 1')
    aug = augmentor(dbroot, k)
    sc = checked_scenes(k)[0]
    eng = default_engine()
    seen = {}
    orig = eng.gt_paste_batch

    def paste(*a, **kw):
        seen['before'] = eng.launch_count()
        try:
            return orig(*a, **kw)
        finally:
            seen['after'] = eng.launch_count()
    eng.gt_paste_batch = paste
    try:
        np.random.seed(S.CASES[k]['seed'])
        with pytest.raises(ValueError, match='too many boxes'):
            aug.forward(S.data_dict(sc, None, S.CASES[k]['classes']))
    finally:
        del eng.gt_paste_batch
    assert seen and seen['after'] == seen['before']
    assert [len(v) for v in valid_of(cloud(k, 0))] == [S.BOX_LIMIT + 1]

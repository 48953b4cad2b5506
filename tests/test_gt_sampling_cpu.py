"""The GT-sampling planner's draws and sampler state against the unmodified reference (tests/golden/gt_sampling.npz):
consecutive calls with an exhausted pointer and short slices, LIMIT_WHOLE_SCENE with num_gt >= limit, the PREPARE
filters, and the reference's errors.  No GPU: the planner runs before any launch."""
import json

import numpy as np
import pytest

import gt_sampling_case as G
from lidar_snow_sim_b200.augmentor import DataAugmentor, DataBaseSampler
from lidar_snow_sim_b200.augmentor import plan as P


@pytest.fixture(scope='module')
def golden():
    return np.load(G.GOLDEN)


@pytest.fixture(scope='module')
def dbdir(golden, tmp_path_factory):
    root = tmp_path_factory.mktemp('gtdb')
    G.write_database({k[3:]: golden[k] for k in golden.files if k.startswith('db_')}, str(root))
    return root


def _state_equal(g, k, i):
    st = np.random.get_state()
    return np.array_equal(st[1], g[f'c{k}_st_{i}']) and [st[2], st[3]] == g[f'c{k}_stpos_{i}'].tolist()


def _groups_equal(sampler, g, k, i):
    want = json.loads(str(g[f'c{k}_sg_{i}']))
    got = {c: [v['sample_num'], int(v['pointer']), np.asarray(v['indices']).tolist()]
           for c, v in sampler.sample_groups.items()}
    return got == want


@pytest.mark.parametrize('k', range(len(G.CASES)))
def test_draws_and_sampler_state_match_reference(golden, dbdir, k):
    case = G.CASES[k]
    np.random.seed(case['seed'])
    scenes = G.make_scenes(case)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    calib = object()
    for i, sc in enumerate(scenes):
        d = G.data_dict(sc, calib, G.CLASS_NAMES)
        d.pop('points')
        exc = str(golden[f'c{k}_exc_{i}']) if f'c{k}_exc_{i}' in golden.files else None
        if exc == 'ValueError':
            with pytest.raises(ValueError):
                P.draw(aug.queue, [d])
        else:
            plans = P.draw(aug.queue, [d], snapshot_all=True)
            if exc == 'KeyError':                     # raised after the sampler's draws, before the flip's
                np.random.set_state(plans[0].snapshot[0])
        assert _state_equal(golden, k, i), (case['name'], i)
        assert _groups_equal(aug.sampler, golden, k, i), (case['name'], i)


def test_limit_whole_scene_with_num_gt_at_the_limit(dbdir):
    case = G.CASES[5]
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    d = {'gt_boxes': np.zeros((3, 7), np.float32), 'gt_names': np.array(['Car'] * 3), 'gt_boxes_mask': np.ones(3, bool)}
    np.random.seed(0)
    p = P.draw(aug.queue, [d])[0]
    assert aug.sampler.sample_groups['Car']['sample_num'] == '-1'
    assert len(p.classes) == 1 and p.classes[0][0][0]['name'] == 'Pedestrian'     # only Pedestrian is sampled


def test_prepare_filters(dbdir, golden):
    case = G.CASES[0]
    s = DataBaseSampler(dbdir, G.augmentor_cfg(case)['AUG_CONFIG_LIST'][0], G.CLASS_NAMES)
    n, diff, names = golden['db_npts'], golden['db_difficulty'], golden['db_names']
    for c in G.CLASS_NAMES:
        want = int(((names == c) & (n >= 5) & (diff != -1)).sum())
        assert len(s.db_infos[c]) == want
        assert all(i['num_points_in_gt'] >= 5 and i['difficulty'] != -1 for i in s.db_infos[c])
    assert 'Van' not in s.db_infos


def test_unsupported_entries_raise(dbdir):
    cfg = G.augmentor_cfg(G.CASES[0])
    cfg['AUG_CONFIG_LIST'] = cfg['AUG_CONFIG_LIST'] + [G.Cfg(NAME='random_local_rotation', LOCAL_ROT_ANGLE=0.1)]
    with pytest.raises(NotImplementedError, match='random_local_rotation'):
        DataAugmentor(dbdir, cfg, G.CLASS_NAMES)
    for key in ('USE_SHARED_MEMORY', 'DATABASE_WITH_FAKELIDAR'):
        gt = G.Cfg(G.augmentor_cfg(G.CASES[0])['AUG_CONFIG_LIST'][0], **{key: True})
        with pytest.raises(NotImplementedError, match=key):
            DataBaseSampler(dbdir, gt, G.CLASS_NAMES)
    cfg = G.augmentor_cfg(G.CASES[0])
    cfg['DISABLE_AUG_LIST'] = ['gt_sampling']
    assert [n for n, _ in DataAugmentor(dbdir, cfg, G.CLASS_NAMES).queue][0] == 'random_world_flip'


def test_trig_is_the_c_library():
    import ctypes
    import ctypes.util
    m = ctypes.CDLL(ctypes.util.find_library('m'))
    m.cosf.restype = ctypes.c_float
    m.cosf.argtypes = [ctypes.c_float]
    a = np.float32([0.0, np.pi / 2, -np.pi, 1e-8, 3.1415927])
    c, s = P.c_cos_sin(a)
    assert c.dtype == np.float32 and [m.cosf(float(v)) for v in a] == c.tolist()

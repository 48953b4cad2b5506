"""CPU tests of the DATA_PROCESSOR block: the NumPy restatement of the device shuffle (tests/shuffle_model.py) against
np.random.permutation and its state, and the host halves (feature encoder, box mask) against the unmodified reference
(tests/golden/processor.npz, tools/make_golden_processor.py)."""
import json
import os

import numpy as np
import pytest

import shuffle_model as SM
from lidar_snow_sim_b200.processor import DataProcessor, PointFeatureEncoder, mask_boxes_outside_range_numpy

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'processor.npz')
ENCODING = {'encoding_type': 'absolute_coordinates_encoding', 'used_feature_list': ['x', 'y', 'z', 'intensity'],
            'src_feature_list': ['x', 'y', 'z', 'intensity', 'channel']}
SIZES = [0, 1, 2, 3] + [n for k in (5, 10, 16) for n in (2 ** k - 1, 2 ** k, 2 ** k + 1)] + [100003, 131072]


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize('seed', [0, 5, 1234])
def test_model_equals_numpy_permutation(seed):
    """every size of SIZES in a row, from a state with pos != 624 (and a cached Gaussian for one seed)"""
    np.random.seed(seed)
    np.random.randint(1000, size=seed % 600 + 1)
    if seed == 5:
        np.random.standard_normal()
    st = np.random.get_state()
    assert st[2] != 624
    perms, st_model = SM.permutations(st, SIZES)
    want = [np.random.permutation(n) for n in SIZES]
    for n, p, w in zip(SIZES, perms, want):
        assert np.array_equal(p, w), n
    assert _state_equal(st_model, np.random.get_state())


@pytest.mark.parametrize('n', [1, 2, 3, 63, 64, 65, 1000])
def test_model_single_cloud_from_fresh_block(n):
    """pos == 624 at entry: the first draw twists; n <= 1 draws nothing and leaves the state as it was"""
    np.random.seed(n)
    np.random.randint(2, size=624)
    st = np.random.get_state()
    assert st[2] == 624
    perms, st_model = SM.permutations(st, [n])
    assert np.array_equal(perms[0], np.random.permutation(n))
    assert _state_equal(st_model, np.random.get_state())


def test_reservation_shuffle_equals_sequential_swaps():
    rng = np.random.default_rng(3)
    for n in (2, 17, 5000):
        j = np.array([0] + [rng.integers(0, i + 1) for i in range(1, n)])
        x = np.arange(n)
        for i in range(n - 1, 0, -1):
            x[i], x[j[i]] = x[j[i]], x[i]
        assert np.array_equal(SM.reservation_shuffle(j, n)[0], x)


def test_model_on_golden_masked_rows(golden):
    """the model's permutations applied to the reference's masked rows give the reference's shuffled rows"""
    k_all = sorted(int(k[5:]) for k in golden.files if k.startswith('mask_'))
    for m in range(3):
        cfg = json.loads(str(golden[f'cfg_{m}']))
        st = ('MT19937', golden[f'key_before_{m}'], int(golden[f'pos_before_{m}']),
              int(golden[f'gauss_before_{m}'][0]), float(golden[f'gauss_before_{m}'][1]))
        if cfg['mode'] == 'train':
            perms, st = SM.permutations(st, [golden[f'mask_{k}'].shape[0] for k in k_all])
        else:
            perms = [np.arange(golden[f'mask_{k}'].shape[0]) for k in k_all]
        for k, p in zip(k_all, perms):
            assert np.array_equal(golden[f'mask_{k}'][p], golden[f'c{m}_out_{k}'])
        assert np.array_equal(st[1], golden[f'key_after_{m}']) and st[2] == int(golden[f'pos_after_{m}'])


def test_encoder_matches_reference(golden):
    rng = golden['point_cloud_range']
    enc = PointFeatureEncoder(ENCODING, point_cloud_range=rng)
    assert enc.num_point_features == 4 and enc.columns() == [0, 1, 2, 3]
    for k in sorted(int(k[3:]) for k in golden.files if k.startswith('in_')):
        d = enc.forward({'points': golden[f'in_{k}']})
        want = golden[f'enc_{k}']
        assert d['use_lead_xyz'] is True
        assert d['points'].dtype == want.dtype and np.array_equal(d['points'].view(np.int32), want.view(np.int32))


def test_box_mask_matches_reference(golden):
    rng = golden['point_cloud_range']
    for m in range(3):
        cfg = json.loads(str(golden[f'cfg_{m}']))
        corners = cfg['DATA_PROCESSOR'][0].get('min_num_corners', 1)
        proc = DataProcessor(cfg['DATA_PROCESSOR'], rng, cfg['mode'] == 'train', 4)
        for k in sorted(int(k[6:]) for k in golden.files if k.startswith('boxes_')):
            boxes = golden[f'boxes_{k}']
            mask = mask_boxes_outside_range_numpy(boxes, rng, min_num_corners=corners)
            assert np.array_equal(mask, golden[f'c{m}_box_mask_{k}'])
            assert np.array_equal(proc._box_mask(boxes), golden[f'c{m}_boxes_out_{k}'])


def test_queue_checks():
    rng = np.array([0, -40, -3, 70.4, 40, 1], np.float32)
    vox = {'NAME': 'transform_points_to_voxels', 'VOXEL_SIZE': [0.05, 0.05, 0.1], 'MAX_POINTS_PER_VOXEL': 5,
           'MAX_NUMBER_OF_VOXELS': {'train': 16000, 'test': 40000}}
    p = DataProcessor([{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True}, vox], rng, True, 4)
    assert p.grid_size.tolist() == [1408, 1600, 40] and p.voxel_size == [0.05, 0.05, 0.1]
    for name in ('sample_points', 'downsample_depth_map'):
        with pytest.raises(NotImplementedError):
            DataProcessor([{'NAME': name}], rng, True, 4)
    with pytest.raises(NotImplementedError):
        DataProcessor([vox, {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True}}], rng, True, 4)
    with pytest.raises(NotImplementedError):
        PointFeatureEncoder(dict(ENCODING, filter_sweeps=True, src_feature_list=ENCODING['src_feature_list']
                                 + ['timestamp']))._check_sweeps()

"""The dataset's LISA block (integrations.dense.lisa_block) against a literal transcription of
lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:713-746, both over a LISA stand-in on the CPU oracle: the same draws
from NumPy's global generator, the float32 intensity division, np.round's half-to-even, the cast back into the float32
rows, columns 5+ carried and the label-0 filter."""
import copy
import os

import numpy as np
import pytest

from lidar_snow_sim_b200.integrations.dense import lisa_block
from lidar_snow_sim_b200.synthetic import synthetic_cloud
from oracle import lisa as ol

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'lisa.npz'))
RATES = [2.2383844962893775, 4.816236598076465, 8.847991609353935, 17.90707597031502, 34.97475775452152]


def reference_block(points, dataset_cfg, lisa, rainfall_rates, training=True):
    """dense_dataset.py:713-746, with self.* replaced by the arguments."""
    if training and 'LISA' in dataset_cfg:
        method = dataset_cfg['LISA']
        choices = [0]
        if '8in9' in method:
            choices = [1, 1, 1, 1, 1, 1, 1, 1, 0]
        elif '1in10' in method:
            choices = [1, 0, 0, 0, 0, 0, 0, 0, 0, 0]
        if np.random.choice(choices):
            rainfall_rate = 0
            if 'uniform' in method:
                rainfall_rate = np.random.choice(rainfall_rates)
            before_lisa = np.zeros((points.shape[0], 4))
            before_lisa[:, :3] = copy.deepcopy(points[:, :3])
            before_lisa[:, 3] = copy.deepcopy(points[:, 3] / 255)
            after_lisa = lisa.augment(pc=before_lisa, Rr=rainfall_rate)
            after_lisa[:, 3] = np.round(after_lisa[:, 3] * 255)
            if points.shape[1] < 5:
                points = np.zeros((points.shape[0], points.shape[1] + 1))
            points[:, :5] = after_lisa[:, :5]
            points = points[np.where(points[:, 4] != 0)]
    return points


class OracleLISA:
    """LISA.augment's interface on the CPU oracle (fixed-seed mode); records what it was given."""

    def __init__(self, mode='gunn', signal='strongest'):
        self.mode, self.signal, self.D = mode, signal, G['D']
        self.qext = G['qext_water'] if mode == 'rain' else G['qext_ice']
        self.inputs = []

    def augment(self, pc, Rr, fixed_seed=False):
        self.inputs.append((pc.copy(), Rr))
        a = ol.alpha(self.mode, Rr, self.D, self.qext)
        with np.errstate(divide='ignore', invalid='ignore'):
            return ol.monte_carlo_augment(pc, Rr, self.mode, a, signal=self.signal)


class TieLISA:
    """Returns intensities whose * 255 lies exactly on .5 (and labels 0, 1, 2 in turn): np.round's half-to-even."""

    def augment(self, pc, Rr, fixed_seed=False):
        out = np.zeros((pc.shape[0], pc.shape[1] + 2))
        out[:, :3] = pc[:, :3] * 1.000000001
        out[:, 3] = (np.arange(pc.shape[0]) % 256 + 0.5) / 256 * (256 / 255)
        out[:, 4] = np.arange(pc.shape[0]) % 3
        return out


def _clouds():
    c5 = synthetic_cloud(seed=3, n_azimuth=6)
    c6 = np.column_stack([synthetic_cloud(seed=4, n_azimuth=6), np.arange(384, dtype=np.float32) * 0.5 + 0.25])
    return [c5, c6, c5[:, :4].astype(np.float64)]


@pytest.mark.parametrize('key', ['uniform_8in9', 'uniform_1in10'])
@pytest.mark.parametrize('make', [lambda: OracleLISA('gunn'), lambda: OracleLISA('rain', 'last'), TieLISA])
def test_lisa_block_is_the_dataset_block(key, make):
    cfg = {'LISA': key}
    for seed in (0, 1, 2, 5):
        for pc in _clouds():
            np.random.seed(seed)
            want = reference_block(pc.copy(), cfg, make(), RATES)
            state = np.random.get_state()
            np.random.seed(seed)
            before = pc.copy()
            got = lisa_block(pc, cfg, make(), RATES)
            assert np.array_equal(pc, before)                               # the caller's array is left alone
            assert got.dtype == want.dtype and got.shape == want.shape
            assert np.array_equal(got, want, equal_nan=True)
            assert all(np.array_equal(x, y) for x, y in zip(state, np.random.get_state()))


def test_host_conversions():
    pc = synthetic_cloud(seed=5, n_azimuth=4)
    pc[:7, 3] = [1, 3, 7, 11, 97, 201, 254]
    pc = np.column_stack([pc, np.arange(pc.shape[0], dtype=np.float32) + 0.125])
    lisa = OracleLISA('gunn')
    np.random.seed(0)                                                       # 8in9: the first sample is applied
    got = lisa_block(pc, {'LISA': 'uniform_8in9'}, lisa, RATES)
    before, Rr = lisa.inputs[0]
    assert Rr in RATES
    assert np.array_equal(before[:, 3], (pc[:, 3] / np.float32(255)).astype(np.float64))    # float32 division
    assert not np.array_equal(before[:, 3], pc[:, 3].astype(np.float64) / 255)
    assert got.dtype == np.float32 and set(np.unique(got[:, 4])) <= {1.0, 2.0}
    kept = np.isin(pc[:, 5], got[:, 5])
    assert np.array_equal(got[:, 5], pc[kept, 5])                            # column 5 carried, order kept
    assert kept.sum() < pc.shape[0] or (got[:, 4] != 0).all()
    tie = lisa_block(pc[:, :5].copy(), {'LISA': 'uniform_8in9'}, TieLISA(), RATES)
    i = TieLISA().augment(np.zeros((pc.shape[0], 4)), 1.0)[:, 3] * 255
    exact = i == np.floor(i) + 0.5
    assert exact.any()
    lab = np.arange(pc.shape[0]) % 3 != 0
    want_i = np.round(i)[lab]
    assert np.array_equal(tie[:, 3], want_i.astype(np.float32))
    assert (want_i[exact[lab]] % 2 == 0).all()                               # half to even

"""
DROR on the GPU (csrc/dror.cu through the C ABI, the lidar_snow_sim_b200.dror mirror and integrations.dense.dror_filter)
against the masks frozen from the unmodified reference (tests/golden/dror.npz) and against the oracle (oracle/dror.py) on
ragged batches.  Everything is exact: keep codes, compacted rows and their order, kept and snow counts.
"""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles      # noqa: E402
from oracle import dror as od                                                       # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, 'tests', 'golden', 'dror.npz')


@pytest.fixture(scope='module')
def engine():
    from lidar_snow_sim_b200.engine import SnowfallEngine
    return SnowfallEngine(0)


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def with_snow(pc, seed, n_single=1500, n_pairs=300):
    rng = np.random.default_rng(seed)
    single = rng.uniform((-40, -40, -2), (40, 40, 3), (n_single, 3))
    c = rng.uniform((-40, -40, -2), (40, 40, 3), (n_pairs, 1, 3))
    pairs = (c + rng.normal(0, 0.02, (n_pairs, 2, 3))).reshape(-1, 3)
    snow = np.concatenate([single, pairs]).astype(np.float32)
    rows = rng.choice(pc.shape[0], snow.shape[0], replace=False)
    pc = pc.copy()
    pc[rows, :3] = snow
    return pc


def run(engine, clouds, **kw):
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(clouds), dtype=np.float32)).cuda()
    res = engine.dror_batch(pts, off, **kw)
    engine.check()
    return off, {k: v.cpu().numpy() for k, v in res.items()}


def test_keep_masks_equal_the_reference(engine, gold):
    n = 0
    for key in gold.files:
        if not key.startswith('mask__'):
            continue
        _, name, a, k, s = key.split('__')
        pc = gold[f'pc__{name}']
        want = np.unpackbits(gold[key])[:pc.shape[0]].astype(bool)
        _, res = run(engine, [pc], alpha=float(a), k_min=int(k), sr_min=float(s))
        assert np.array_equal(res['keep'] == 1, want), key
        assert set(np.unique(res['keep'])) <= {0, 1}
        n += 1
    assert n >= 40


def test_ragged_batch_equals_the_oracle(engine):
    rng = np.random.default_rng(7)
    dup = synthetic_cloud(seed=31, n_azimuth=200, shuffle_rows=True)
    dup = with_snow(np.concatenate([dup, dup[:500]]), 1, 400, 100)
    dup = dup[rng.permutation(dup.shape[0])]
    dup[17, 1] = np.nan
    clouds = [np.zeros((0, 5), np.float32),
              np.array([[1, 2, 0, 5, 0]], np.float32),
              np.array([[1, 2, 0, 5, 0], [1, 2, 0.01, 5, 1]], np.float32),
              np.array([[1, 2, 0, 5, 0], [1, 2, 0.01, 5, 1], [1, 2.01, 0, 5, 2]], np.float32),
              dup,
              with_snow(synthetic_cloud(seed=41, n_azimuth=2048), 2),
              with_snow(synthetic_cloud(seed=42, n_azimuth=2048), 3)]
    assert clouds[-1].shape[0] == 131072
    for alpha, k_min, sr_min in ((0.16, 3, 0.04), (0.45, 1, 0.0), (0.08, 0, 0.04), (0.16, 5, 0.0)):
        off, res = run(engine, clouds, alpha=alpha, k_min=k_min, sr_min=sr_min)
        _, again = run(engine, clouds, alpha=alpha, k_min=k_min, sr_min=sr_min)
        for key in ('keep', 'counts', 'n_snow'):
            assert np.array_equal(res[key], again[key]), f'second call differs: {key}'
        for b in range(len(clouds)):
            rows = slice(off[b], off[b] + res['counts'][b])
            assert np.array_equal(res['points'][rows], again['points'][rows]), 'second call differs: points'
        for b, pc in enumerate(clouds):
            codes = od.keep_codes(pc, alpha, 3.0, k_min, sr_min)
            got = res['keep'][off[b]:off[b + 1]]
            assert np.array_equal(got, codes), (b, alpha, k_min, sr_min)
            kept = pc[codes == 1]
            assert res['counts'][b] == kept.shape[0]
            assert res['n_snow'][b] == int((codes == 0).sum())
            assert np.array_equal(res['points'][off[b]:off[b] + kept.shape[0]], kept)
        assert res['keep'][off[4] + 17] == 0                               # the NaN row is snow
        assert res['counts'][1] == (1 if k_min == 0 else 0)


def test_crop_variant(engine, gold):
    from lidar_snow_sim_b200.dror import snow_indices
    pc = gold['pc__large']
    for a in (0.16, 0.45):
        got = snow_indices(pc, alpha=a, crop=True, engine=engine)
        assert np.array_equal(got, gold[f'crop__large__{a}'])
        assert np.array_equal(got, od.snow_indices(pc, alpha=a, crop=True))
    _, res = run(engine, [pc], crop=True)
    assert np.array_equal(res['keep'], od.keep_codes(pc, crop=True))


def test_mirror_signature(engine, gold):
    from lidar_snow_sim_b200.dror import dynamic_radius_outlier_filter
    pc = gold['pc__small']
    want = np.unpackbits(gold['mask__small__0.45__1__0.04'])[:pc.shape[0]].astype(bool)
    got = dynamic_radius_outlier_filter(pc, alpha=0.45, k_min=1, engine=engine)
    assert got.dtype == bool and np.array_equal(got, want)


def test_chained_after_snowfall_on_the_device(engine):
    div = float(np.degrees(3e-3))
    tables = [synthetic_particles(700 + k, 6000) for k in range(64)]
    tid = engine.upload_tables(tables)
    clouds = [with_snow(synthetic_cloud(seed=50 + b, n_azimuth=256), 60 + b, 300, 60) for b in range(3)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    order = np.stack([np.random.default_rng(b).permutation(64) for b in range(3)]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    snow = engine.snowfall_batch(tid, pts, off, order, div, thresh_poly=np.tile([1e-3, -0.2, 14.0], (3, 1)))
    res = engine.dror_batch(snow['points'], off, alpha=0.16, counts=snow['counts'])
    engine.check()
    aug = snow['points'].cpu().numpy()
    cnt = snow['counts'].cpu().numpy()
    keep = res['keep'].cpu().numpy()
    out = res['points'].cpu().numpy()
    for b in range(3):
        host = aug[off[b]:off[b] + cnt[b]]
        codes = od.keep_codes(host, 0.16)
        assert np.array_equal(keep[off[b]:off[b] + cnt[b]], codes)
        assert int(res['counts'][b]) == int((codes == 1).sum())
        assert np.array_equal(out[off[b]:off[b] + int(res['counts'][b])], host[codes == 1])
    engine.free_tables(tid)


@pytest.mark.parametrize('cfg,split', [({'DROR': 0.16}, 'train_clear'), ({'DROR++': 0.45}, 'test_snow'),
                                       ({'DROR++': 0.45}, 'test_clear'), ({'DROR': 0.08, 'DROR++': 0.45}, 'test_snow')])
def test_dataset_path(engine, tmp_path, cfg, split):
    from lidar_snow_sim_b200.integrations.dense import dror_filter
    raw = with_snow(synthetic_cloud(seed=77, n_azimuth=512), 5, 600, 100)
    for alpha in {v for v in cfg.values()}:                               # the reference's .pkl files, from the oracle
        with open(tmp_path / f'alpha_{alpha}.pkl', 'wb') as f:
            pickle.dump(od.snow_indices(raw, alpha), f, protocol=pickle.HIGHEST_PROTOCOL)

    def lookup(alpha):
        with open(tmp_path / f'alpha_{alpha}.pkl', 'rb') as f:
            return pickle.load(f)

    def outcome(fn):
        try:
            return fn()
        except IndexError:
            return IndexError
    want = outcome(lambda: od.apply_dataset_dror(raw, cfg, split, lookup))
    got = outcome(lambda: dror_filter(raw, cfg, split, engine=engine))
    if want is IndexError:
        assert got is IndexError
    else:
        assert got is not IndexError and np.array_equal(got, want)
        if 'DROR' in cfg or 'snow' in split:
            assert got.shape[0] < raw.shape[0]

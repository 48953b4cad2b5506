"""FogAugmentation.batch / after_batch (integrations/dense.py) against the per-sample restatement of foggify
(dense_dataset.py:967-1014): DENSE through BetaRadomization(seed=0) + haze_point_cloud + [:, :n_features] on NumPy's
global state, CVL through foggify_cvl on the fog module's generator, sample after sample."""
import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.fog import simulation as fs
from lidar_snow_sim_b200.fog.haze import BetaRadomization, haze_point_cloud
from lidar_snow_sim_b200.integrations.dense import FogAugmentation, foggify_cvl

pytestmark = pytest.mark.gpu


class Args:
    sensor_type = 'Velodyne HDL-64E S3D'
    fraction_random = 0.05


def clouds(seed, sizes, F=5):
    rs = np.random.RandomState(seed)
    out = []
    for n in sizes:
        r = rs.uniform(0.5, 70.0, n)
        phi = rs.uniform(-np.pi, np.pi, n)
        c = np.zeros((n, F), np.float32)
        c[:, 0], c[:, 1] = r * np.cos(phi), r * np.sin(phi)
        c[:, 2] = rs.uniform(-2, 1, n)
        c[:, 3] = rs.randint(0, 256, n)
        c[:, 4:] = rs.randint(0, 64, (n, F - 4))
        out.append(c)
    return out


def slots(engine, cs, slack):
    off = np.zeros(len(cs) + 1, np.int64)
    off[1:] = np.cumsum([c.shape[0] + s for c, s in zip(cs, slack)])
    pts = np.full((int(off[-1]), cs[0].shape[1]), 7.0, np.float32)
    for b, c in enumerate(cs):
        pts[off[b]:off[b] + c.shape[0]] = c
    cnt = torch.tensor([c.shape[0] for c in cs], dtype=torch.int32, device=engine.device)
    return torch.from_numpy(pts).to(engine.device), off, cnt


def rows_of(res, b):
    o = res['offsets'][b]
    return res['points'][o:o + int(res['counts'][b])].cpu().numpy()


def per_sample_dense(engine, cs, alphas):
    out = []
    for c, alpha in zip(cs, alphas):
        if alpha == '0.000':
            out.append(c.astype(np.float64))
            continue
        B = BetaRadomization(beta=float(alpha), seed=0)
        B.propagate_in_time(10)
        n_features = c.shape[1]
        out.append(haze_point_cloud(c, B, Args(), engine=engine)[:, :n_features])
    return out


@pytest.mark.parametrize('key', ['FOG_AUGMENTATION', 'FOG_AUGMENTATION_AFTER'])
def test_dense_block_equals_per_sample(engine, key):
    cs = clouds(3, [3000, 0, 1, 5000, 257, 4096, 2, 1500])
    cfg = {'FOG_AUGMENTATION': 'DENSE_uniform'} if key == 'FOG_AUGMENTATION' else \
        {'FOG_AUGMENTATION': False, 'FOG_AUGMENTATION_AFTER': 'DENSE_uniform'}
    fog = FogAugmentation(cfg, random_generator=np.random.default_rng(8), engine=engine)
    fog.init_curriculum(0, 1, 1, 100)
    pts, off, cnt = slots(engine, cs, [5 * b for b in range(len(cs))])
    np.random.seed(4)
    res = fog.batch(pts, off, counts=cnt, out_dtype=torch.float64)
    alphas, mor = res['alpha'], res['mor']
    if key == 'FOG_AUGMENTATION_AFTER':
        assert torch.equal(res['points'], pts.double())
        res = fog.after_batch(pts, off, counts=cnt, out_dtype=torch.float64)
    st_batch = np.random.get_state()
    assert any(a != '0.000' for a in alphas)
    want = per_sample_dense(engine, cs, alphas)
    for b in range(len(cs)):
        assert np.array_equal(rows_of(res, b).view(np.uint64), want[b].view(np.uint64))
    st = np.random.get_state()
    assert np.array_equal(st[1], st_batch[1]) and st[2] == st_batch[2]
    assert np.array_equal(mor, np.array([np.inf if a == '0.000' else np.log(20) / float(a) for a in alphas]))
    assert fog.current_iteration == len(cs)


def test_float32_rows_are_the_float64_rows_rounded(engine):
    cs = clouds(5, [2000, 3000])
    cfg = {'FOG_AUGMENTATION': 'DENSE_fixed'}
    pts, off, cnt = slots(engine, cs, [0, 0])
    r64 = FogAugmentation(cfg, engine=engine).batch(pts, off, counts=cnt, out_dtype=torch.float64)
    r32 = FogAugmentation(cfg, engine=engine).batch(pts, off, counts=cnt)
    assert r32['points'].dtype == torch.float32
    for b in range(2):
        assert np.array_equal(rows_of(r32, b), rows_of(r64, b).astype(np.float32))


def test_no_sample_fogs(engine):
    cs = clouds(6, [100, 0, 40])
    fog = FogAugmentation({'FOG_AUGMENTATION': 'DENSE_uniform', 'FOG_ALPHAS': ['0.000']}, engine=engine)
    pts, off, cnt = slots(engine, cs, [3, 0, 1])
    st = np.random.get_state()
    res = fog.batch(pts, off, counts=cnt)
    for b, c in enumerate(cs):
        assert np.array_equal(rows_of(res, b), c)
    assert np.all(np.isinf(res['mor']))
    assert np.array_equal(np.random.get_state()[1], st[1])


def test_cvl_block_equals_per_sample(engine):
    cs = clouds(7, [3000, 1, 2500, 700], F=5)
    cfg = {'FOG_AUGMENTATION': 'CVL_uniform'}
    fog = FogAugmentation(cfg, random_generator=np.random.default_rng(2), engine=engine)
    pts, off, cnt = slots(engine, cs, [0, 4, 9, 1])
    rng0 = fs.RNG.bit_generator.state
    res = fog.batch(pts, off, counts=cnt, out_dtype=torch.float64)
    rng_batch = fs.RNG.bit_generator.state
    fs.RNG.bit_generator.state = rng0
    alphas = res['alpha']
    assert any(a != '0.000' for a in alphas)
    for b, c in enumerate(cs):
        want = foggify_cvl(c, alphas[b], cfg, engine=engine, lut='device')
        assert np.array_equal(rows_of(res, b), np.asarray(want, np.float64))
    assert fs.RNG.bit_generator.state == rng_batch

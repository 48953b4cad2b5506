"""The device fog (csrc/fog.cu, fog_batch_params) at full size against the oracle in rounding='device' (oracle/fog.py:
the device's documented arithmetic where the reference is host-defined), one generator per cloud.

Exact: fog masks, ranks, counts and the min / max responses.  Rows bit for bit without noise and for v1 / v4; the only
exception allowed is a hard-target row whose float64 exp lies within one double ulp of a float32 rounding midpoint
(numpy's and CUDA's float64 exp may round such a value apart), and such rows are found, not tolerated wholesale.  For
v2 / v3 the noise factor goes through pow (device vs host libm): coordinates within a few float64 ulps; the largest
distance measured is printed."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
MAX_POW_ULPS = 8


@pytest.fixture(scope='module')
def engine():
    from lidar_snow_sim_b200.engine import SnowfallEngine
    return SnowfallEngine(0)


@pytest.fixture(scope='module')
def bench_batch():
    import bench
    clouds, _ = bench.make_workload(0, 32)
    return clouds


@pytest.fixture(scope='module')
def lut06():
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'fog.npz'))['lut_0.06']


def run_device(engine, pcs, ps, luts, index, noise, variant, gain, seeds, hard=True):
    """fog_batch_params on the clouds, each cloud's generator default_rng(seeds[b]) stepped as the mirrors step it"""
    from lidar_snow_sim_b200.fog.simulation import _pcg64_state
    off = np.concatenate([[0], np.cumsum([pc.shape[0] for pc in pcs])]).astype(np.int64)
    B = len(pcs)
    gens = [np.random.default_rng(s) for s in seeds]
    for g in gens:
        g.integers(low=1, high=20, size=1)
    args = (torch.from_numpy(np.concatenate(pcs)).cuda(), off, torch.from_numpy(np.stack(luts)).cuda(),
            [p.alpha for p in ps], [p.beta for p in ps], [p.beta_0 for p in ps], index)
    kw = dict(hard=hard, soft=True, gain=gain, noise=noise, noise_variant=variant, want_rank=True)
    if noise and variant == 4:
        cnt = engine.fog_batch_params(*args, **kw)['info'][:, 2].cpu().numpy().astype(np.int64)
        ext = torch.zeros(max(1, int(off[-1])), dtype=torch.float64)
        for b in range(B):
            ext[off[b]:off[b] + cnt[b]] = torch.from_numpy(gens[b].beta(a=2, b=20, size=int(cnt[b])))
        res = engine.fog_batch_params(*args, ext_noise=ext.cuda(), **kw)
    else:
        states = np.stack([_pcg64_state(g) for g in gens]) if noise else None
        res = engine.fog_batch_params(*args, rng_states=states, **kw)
    engine.check()
    return off, {k: v.cpu().numpy() for k, v in res.items()}


def hard_tie_rows(pc, alpha):
    """rows whose float64 exp(-2 alpha r_0) lies within one double ulp of a midpoint between two float32 values"""
    r0 = np.linalg.norm(pc[:, 0:3], axis=1)
    x = np.exp((np.float32(-2 * alpha) * r0).astype(np.float64))
    lo = x.astype(np.float32)
    lo = np.where(lo.astype(np.float64) > x, np.nextafter(lo, np.float32(0)), lo)
    mid = (lo.astype(np.float64) + np.nextafter(lo, np.float32(np.inf)).astype(np.float64)) / 2
    return np.abs(x - mid) <= np.spacing(x)


def ulps(a, b):
    """distance in float64 ulps (0 where both are equal or both NaN)"""
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    d = np.abs(ia - ib).astype(np.float64)
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


def compare(engine, pcs, ps, luts, index, noise, variant, gain, hard=True):
    """device vs oracle for every cloud; returns the largest coordinate distance in float64 ulps"""
    from oracle import fog as ofog
    seeds = list(range(100, 100 + len(pcs)))
    off, res = run_device(engine, pcs, ps, luts, index, noise, variant, gain, seeds, hard)
    worst = 0.0
    for b, pc in enumerate(pcs):
        rng = np.random.default_rng(seeds[b])
        aug, _, info, mask = ofog.simulate_fog(ps[b], pc, noise, luts[index[b]], rng, gain=gain,
                                               noise_variant=f'v{variant}', hard=hard, rounding='device',
                                               want_mask=True)
        s = slice(off[b], off[b + 1])
        got, dmask = res['points'][s], res['fog_mask'][s].astype(bool)
        cnt = int(mask.sum())
        assert np.array_equal(dmask, mask), b
        assert np.array_equal(res['rank'][s][mask], np.arange(cnt)) and np.all(res['rank'][s][~mask] == -1), b
        assert int(res['info'][b, 2]) == info['num_fog_responses'] == cnt, b
        assert res['info'][b, 0] == info['min_fog_response'] and res['info'][b, 1] == info['max_fog_response'], b
        assert np.array_equal(np.isnan(got), np.isnan(aug)), b
        same = (got == aug) | (np.isnan(got) & np.isnan(aug))
        if noise and variant in (2, 3):
            d = ulps(got[:, :3], aug[:, :3])
            worst = max(worst, float(d.max(initial=0)))
            assert d.max(initial=0) <= MAX_POW_ULPS, (b, d.max())
            same[:, :3] = True
        bad = np.flatnonzero(~same.all(axis=1))
        if bad.size:
            # only a non-fog row's hard-target intensity at a detected float32 midpoint, and (without gain) by one count
            assert hard and not gain and not mask[bad].any(), (b, bad[:5])
            assert np.all(same[bad][:, [0, 1, 2] + list(range(4, pc.shape[1]))]), (b, bad[:5])
            assert hard_tie_rows(pc[bad], ps[b].alpha).all(), (b, bad[:5])
            assert np.all(np.abs(got[bad, 3] - aug[bad, 3]) <= 1), (b, bad[:5])
    return worst


@pytest.mark.parametrize('gain', [False, True])
@pytest.mark.parametrize('noise,variant', [(0, 1), (10, 1), (10, 2), (10, 3), (10, 4)])
def test_bench_batch(engine, bench_batch, lut06, noise, variant, gain):
    """the 32 x 131 072-row bench batch (alpha 0.06, the reference's table)"""
    from lidar_snow_sim_b200.fog import ParameterSet
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    worst = compare(engine, bench_batch, [p] * 32, [lut06], [0] * 32, noise, variant, gain)
    print(f'bench batch noise={noise} v{variant} gain={gain}: largest coordinate distance {worst:.0f} float64 ulps')


def test_per_cloud_alphas(engine, bench_batch):
    """fog_batch_params with 32 alphas, the device's tables copied to the oracle"""
    from lidar_snow_sim_b200.fog import ParameterSet
    ps = [ParameterSet(alpha=a, gamma=0.000001) for a in np.linspace(0.004, 0.3, 32)]
    luts = list(engine.fog_integral_tables(ps).cpu().numpy())
    pcs = [c[:32768] for c in bench_batch]
    for noise, variant in ((10, 1), (10, 3)):
        worst = compare(engine, pcs, ps, luts, list(range(32)), noise, variant, gain=True)
        print(f'32 alphas noise={noise} v{variant}: largest coordinate distance {worst:.0f} float64 ulps')


def test_ragged_batch(engine, bench_batch, lut06):
    """clouds of 0, 1, 255, 256, 257 and 65 537 rows"""
    from lidar_snow_sim_b200.fog import ParameterSet
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    src = bench_batch[3]
    pcs = [src[o:o + n] for o, n in zip((0, 5, 300, 1000, 2000, 4000), (0, 1, 255, 256, 257, 65537))]
    for noise, variant in ((10, 1), (10, 4), (0, 1)):
        compare(engine, pcs, [p] * 6, [lut06], [0] * 6, noise, variant, gain=False)
    compare(engine, pcs[1:], [p] * 5, [lut06], [0] * 5, 10, 4, gain=True)   # (gain on an empty cloud raises)


@pytest.mark.parametrize('F', [4, 5, 8, 9, 16])
def test_feature_widths(engine, bench_batch, lut06, F):
    """rows staged through shared memory (F <= 8) and accessed in place (F = 9 .. 16)"""
    from lidar_snow_sim_b200.fog import ParameterSet
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    rs = np.random.RandomState(F)
    pcs = []
    for c in bench_batch[:2]:
        pc = np.zeros((40000, F), np.float32)
        pc[:, :min(F, 5)] = c[:40000, :min(F, 5)]
        pc[:, 5:] = rs.uniform(-3, 3, (40000, max(0, F - 5)))
        pcs.append(pc)
    for noise, variant, gain in ((10, 1, True), (10, 2, False)):
        compare(engine, pcs, [p] * 2, [lut06], [0, 0], noise, variant, gain)


def test_cloud_with_most_rows_fog(engine, bench_batch, lut06):
    """one 131 072-row cloud with more than 100 000 fog points: beta large enough that most responses hit the cap"""
    from lidar_snow_sim_b200.fog import ParameterSet
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    p.beta = p.beta * 1e4
    pc = bench_batch[5]
    off, res = run_device(engine, [pc], [p], [lut06], [0], 10, 1, False, [7])
    assert res['info'][0, 2] > 100000
    compare(engine, [pc], [p], [lut06], [0], 10, 1, gain=False)
    compare(engine, [pc], [p], [lut06], [0], 10, 4, gain=True)

"""The dataset's LISA block with its draws on the device: lisa_block_batch(..., all_modes=True) for LISA's Goodin, fog,
haze and spray modes against B sequential lisa_block calls from the same NumPy state (rows bit for bit, counts,
decisions, rain rates and NumPy's whole state after), against the restatement of the reference
(tests/lisa_average_model.py) on the decisions the device drew, and the device's stream positions against the NumPy
walker (tests/lisa_block_draws_model.py)."""
import numpy as np
import pytest
import torch

import lisa_average_model as LM
import lisa_block_draws_model as WM
from test_lisa_average_cpu import golden_cases, same_state
from test_lisa_average_gpu import f32_conversion

from lidar_snow_sim_b200.integrations.dense import _lisa_choices, lisa_block, lisa_block_batch
from lidar_snow_sim_b200.lisa import LISA

pytestmark = pytest.mark.gpu

RATES = [0.5, 2.0, 2.0, 17.0, 200.0, 0.5]           # duplicates: four distinct candidate rates


def _lisa(engine, gold_dir, mode):
    _, _, D, qext, _ = golden_cases(gold_dir)
    return LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=engine)


def _samples(gold_dir, B, seed):
    """B float32 clouds of the golden mixture (edge rows included), of different sizes, some with NaN rows"""
    _, pc, _, _, _ = golden_cases(gold_dir)
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        rows = f32_conversion(pc[rng.permutation(len(pc))[:int(rng.integers(1, len(pc)))]])
        if b % 3 == 1:
            rows[rng.integers(0, len(rows), 3)] = np.nan
        out.append(rows)
    return out


def _slots(samples, device, empty=()):
    """slot layout with a few spare rows per slot; the slots listed in `empty` hold rows but count 0"""
    lengths = [len(s) + 7 for s in samples]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    pts = np.full((int(off[-1]), samples[0].shape[1]), 3.5, np.float32)
    for b, s in enumerate(samples):
        pts[off[b]:off[b] + len(s)] = s
    counts = np.array([0 if b in empty else len(s) for b, s in enumerate(samples)], np.int32)
    return torch.from_numpy(pts).to(device), off, torch.from_numpy(counts).to(device)


def _sequential(samples, cfg, lisa, rates):
    """B lisa_block calls from NumPy's current state: (outputs, applied, rain rate of each cloud)"""
    drawn = []
    augment = lisa.augment
    lisa.augment = lambda pc, Rr=None, fixed_seed=False: (drawn.append(Rr), augment(pc, Rr, fixed_seed))[1]
    try:
        outs = [lisa_block(p, cfg, lisa, rates) for p in samples]
    finally:
        del lisa.augment
    applied = np.array([o is not p for o, p in zip(outs, samples)], bool)
    rate = np.zeros(len(samples))
    rate[applied] = drawn
    return outs, applied, rate


def _check_block(engine, samples, cfg, lisa, rates, seed, empty=()):
    pts, off, counts = _slots(samples, engine.device, empty)
    seq = [s[:0] if b in empty else s for b, s in enumerate(samples)]
    np.random.seed(seed)
    np.random.standard_normal(seed % 2)                    # odd seeds start with a cached Gaussian
    start = np.random.get_state()
    want, applied, rate = _sequential(seq, cfg, lisa, rates)
    after = np.random.get_state()
    np.random.set_state(start)
    res = lisa_block_batch(pts, off, cfg, lisa, rates, counts=counts, all_modes=True)
    assert same_state(np.random.get_state(), after)
    assert np.array_equal(res['applied'], applied)
    assert np.array_equal(res['rainfall_rate'], rate)
    got_n = res['counts'].cpu().numpy()
    rows = res['points'].cpu().numpy()
    lost = res['n_lost'].cpu().numpy()
    for b, w in enumerate(want):
        assert got_n[b] == len(w), b
        assert lost[b] == len(seq[b]) - len(w), b
        assert np.array_equal(rows[off[b]:off[b] + got_n[b]].view(np.uint32), w.view(np.uint32)), b
    return applied


@pytest.mark.parametrize('mode', ['goodin et al.', 'chu_hogg_fog', 'strong_advection_fog'])
@pytest.mark.parametrize('key', ['uniform_{}_8in9', 'fixed_{}_8in9', 'uniform_{}_1in10', 'fixed_{}_1in10',
                                 'uniform_{}_never'])
def test_block_equals_sequential_lisa_block_calls(engine, gold_dir, mode, key):
    lisa = _lisa(engine, gold_dir, mode)
    cfg = {'LISA': key.format(mode)}
    for B, seed in ((1, 3), (9, 4), (64, 5)):
        applied = _check_block(engine, _samples(gold_dir, B, seed), cfg, lisa, RATES, seed, empty=(2,))
        if key.endswith('never'):
            assert not applied.any()


def test_single_rate_and_a_batch_where_no_sample_is_applied(engine, gold_dir):
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    samples = _samples(gold_dir, 9, 8)
    _check_block(engine, samples, {'LISA': 'uniform_goodin et al._8in9'}, lisa, [17.0], 8)
    for seed in range(40):                                 # 1in10 with few clouds: some seed applies none
        np.random.seed(seed)
        np.random.standard_normal(seed % 2)                # as _check_block starts
        if not any(np.random.choice(_lisa_choices('1in10')) for _ in range(3)):
            break
    assert not _check_block(engine, samples[:3], {'LISA': 'uniform_goodin et al._1in10'}, lisa, RATES, seed).any()


def test_full_size(engine, gold_dir):
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    B, n = 32, 131072
    samples = [synthetic_cloud(seed=200 + b, n_azimuth=n // 64) for b in range(B)]   # x, y, z, I, channel
    applied = _check_block(engine, samples, {'LISA': 'uniform_goodin et al._8in9'}, lisa,
                           [0.5, 2.0, 8.0, 17.0, 34.0, 70.0, 130.0, 200.0], 9)
    assert applied.sum() > B // 2


def test_rows_against_the_reference_restatement(engine, gold_dir):
    """on the decisions the device drew: labels and kept rows exact, values within the Goodin bar"""
    _, _, D, qext, _ = golden_cases(gold_dir)
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    samples = _samples(gold_dir, 9, 12)
    pts, off, counts = _slots(samples, engine.device)
    np.random.seed(12)
    start = np.random.get_state()
    res = lisa_block_batch(pts, off, {'LISA': 'uniform_goodin et al._8in9'}, lisa, RATES, counts=counts,
                           all_modes=True)
    after = np.random.get_state()
    rng = np.random.RandomState()
    rng.set_state(start)
    got_n = res['counts'].cpu().numpy()
    rows = res['points'].cpu().numpy()
    for b, p in enumerate(samples):
        rng.choice(_lisa_choices('8in9'))                  # the draws the device took for this sample
        if not res['applied'][b]:
            assert np.array_equal(rows[off[b]:off[b] + got_n[b]].view(np.uint32), p.view(np.uint32))
            continue
        assert RATES[rng.choice(len(RATES))] == res['rainfall_rate'][b]
        want = LM.dataset_block(p, LM.GOODIN, rng, D, qext, res['rainfall_rate'][b])
        got = rows[off[b]:off[b] + got_n[b]]
        assert got.shape == want.shape and np.array_equal(got[:, 4:], want[:, 4:])
        assert np.allclose(got[:, :4], want[:, :4], rtol=1e-6, atol=1e-6)
    assert same_state(rng.get_state(), after)


def test_stream_positions_against_the_walker_model(engine, gold_dir):
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    samples = _samples(gold_dir, 24, 21)
    pts, off, counts = _slots(samples, engine.device, empty=(5,))
    values, cand = np.unique(RATES, return_inverse=True)
    params = [lisa._average_params(v) for v in values]
    # the detected rows of every cloud under every candidate rate, from the per-cloud entry point
    n_detk = np.stack([engine.lisa_average_cloud_batch(pts, off, 1, q[1], q[3], range_scale=q[2], counts=counts,
                                                       fixed_seed=True)['counts'].cpu().numpy() for q in params],
                      axis=1)
    for seed, has in ((30, 0), (31, 1)):
        np.random.seed(seed)
        np.random.standard_normal(has)
        st = np.random.get_state()
        res = engine.lisa_average_block_batch(pts, off, 1, [q[1] for q in params], params[0][3],
                                              _lisa_choices('8in9'), rate_candidate=cand,
                                              range_scale=[q[2] for q in params], counts=counts)
        engine.check()
        rec, st_want = WM.walk(st, _lisa_choices('8in9'), cand, n_detk)
        assert np.array_equal(res['draws'], rec)
        assert same_state(np.random.get_state(), st_want)


def test_launches_per_call_do_not_depend_on_the_batch(engine, gold_dir):
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    samples = _samples(gold_dir, 64, 40)
    counted = []
    for B in (2, 64):
        pts, off, counts = _slots(samples[:B], engine.device)
        before = engine.launch_count()
        lisa_block_batch(pts, off, {'LISA': 'uniform_goodin et al._8in9'}, lisa, RATES, counts=counts, all_modes=True)
        counted.append(engine.launch_count() - before)
    assert counted[0] == counted[1], counted


@pytest.mark.parametrize('cfg, training', [({'LISA': 'uniform_goodin et al._8in9'}, False), ({}, True)])
def test_no_block_no_draws(engine, gold_dir, cfg, training):
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    pts, off, counts = _slots(_samples(gold_dir, 3, 2), engine.device)
    np.random.seed(2)
    st = np.random.get_state()
    res = lisa_block_batch(pts, off, cfg, lisa, RATES, counts=counts, training=training, all_modes=True)
    assert same_state(np.random.get_state(), st)
    assert res['points'] is pts and res['counts'] is counts
    assert not res['applied'].any() and not res['rainfall_rate'].any()
    assert not res['n_lost'].any()


def test_without_all_modes_it_still_raises(engine, gold_dir):
    lisa = _lisa(engine, gold_dir, 'goodin et al.')
    pts, off, counts = _slots(_samples(gold_dir, 2, 1), engine.device)
    np.random.seed(1)
    st = np.random.get_state()
    with pytest.raises(NotImplementedError):
        lisa_block_batch(pts, off, {'LISA': 'uniform_goodin et al._8in9'}, lisa, RATES, counts=counts)
    assert same_state(np.random.get_state(), st)

"""PA-AUG on the device at full size against the unmodified reference (tests/golden/pa_aug_full.npz, the cases of
tests/pa_aug_scale_case.py): the partition's class totals, every case's rows, masks and NumPy state with each case's
clouds in one batch, a mixed batch against its clouds run alone, slot-compacted input, float32 output and the
256-box limit.  131 072-row clouds take the partition scan past its first 32-tile round, the scatter over hundreds of
tiles and FPS past one row per thread."""
import numpy as np
import pytest
import torch

import pa_aug_scale_case as sc
from lidar_snow_sim_b200.pa_aug import pa_aug_batch
from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, box_planes
from pa_aug_scale_case import model_run
from test_pa_aug_cpu import same_bits

pytestmark = pytest.mark.gpu

G = sc.load()
IDS = [G[k]['name'].replace(' ', '_') for k in sorted(G)]


def cases():
    """the regenerated cases, their inputs checked against the fixture's digests first"""
    cs = sc.cases()
    if getattr(cases, 'checked', False):
        return cs
    for k, c in enumerate(cs):
        for i, ((pts, boxes), r) in enumerate(zip(c['clouds'], G[k]['clouds'])):
            assert sc.input_digests(pts, boxes) == r['in_sha'].tolist(), \
                f'{c["name"]} cloud {i}: the regenerated inputs differ from the fixture\'s (not a kernel fault)'
    cases.checked = True
    return cs


def case_index(name):
    return [G[k]['name'] for k in sorted(G)].index(name)


def batch(clouds, pad=None):
    """(points CUDA, cloud offsets, boxes, box offsets) of clouds in one batch; pad[b] rows after cloud b"""
    rows, offs, boff = [], [0], [0]
    for b, (pts, boxes) in enumerate(clouds):
        p = pts if pad is None else np.concatenate([pts, pad[b]])
        rows.append(p)
        offs.append(offs[-1] + p.shape[0])
        boff.append(boff[-1] + boxes.shape[0])
    return (torch.from_numpy(np.concatenate(rows)).cuda(), np.array(offs, np.int64), np.concatenate([b for _, b in clouds]),
            np.array(boff, np.int64))


def set_state(r):
    np.random.set_state(('MT19937', r['st_keys'], int(r['st_pos']), int(r['st_gauss'][0]), float(r['st_gauss'][1])))


def first_difference(got, c, k, i):
    """where cloud i of case k differs from the reference's sampled rows and from the restatement (run from the state
    the reference had before it)"""
    ref = G[k]['clouds'][i]['rows']
    sampled = got[::sc.ROW_STRIDE]
    if sampled.shape != ref.shape:
        note = 'sampled rows: shapes differ; '
    else:
        d = np.nonzero((sampled.view(np.uint64) != ref.view(np.uint64)).any(axis=1))[0]
        note = f'sampled rows: first differing at row {d[0] * sc.ROW_STRIDE}; ' if d.size else 'sampled rows equal; '
    return note + _model_difference(got, c, k, i)


def _model_difference(got, c, k, i):
    pts, boxes = c['clouds'][i]
    if i == 0:
        np.random.seed(c['seed'])
    else:
        set_state(G[k]['clouds'][i - 1])
    _, _, plan, want = model_run(pts, boxes, c['param'])
    if got.shape != want.shape:
        return f'{got.shape[0]} rows, the restatement {want.shape[0]}'
    bad = np.nonzero((got.view(np.uint64) != want.view(np.uint64)).any(axis=1))[0]
    if bad.size == 0:
        return 'no row differs from the restatement'
    row, dst = int(bad[0]), 0
    for part, segs in enumerate(plan['parts'] + [[plan['bg']]]):
        for kind, ref, n, steps in segs:
            if dst <= row < dst + n:
                where = 'the background' if kind == 'bg' else f'output part {part}'
                return (f'{bad.size} rows differ; first row {row}: {got[row]} != {want[row]}, row {row - dst} of a '
                        f'{kind!r} segment ({ref}, {n} rows, {len(steps)} steps) of {where}')
            dst += n
    return f'{bad.size} rows differ; first row {row}'


@pytest.mark.parametrize('k', sorted(G), ids=IDS)
def test_partition_totals_equal_reference_counts(engine, k):
    """every (box, part) class and the background of every cloud, the parts 4..7 of pedestrians and cyclists 0"""
    c = cases()[k]
    pts, off, boxes, boff = batch(c['clouds'])
    names = sc.names_of(boxes)
    d_planes = torch.from_numpy(box_planes(boxes, names)).cuda()
    d_nparts = torch.tensor([NUM_PARTITION[n] for n in names], dtype=torch.int32, device='cuda')
    totals = engine.pa_partition_batch(pts, off, d_planes, d_nparts, boff, boxes.dtype == np.float64).cpu().numpy()
    assert totals.shape == (8 * boxes.shape[0] + len(c['clouds']),)
    for b, r in enumerate(G[k]['clouds']):
        cls0, M = 8 * int(boff[b]) + b, int(boff[b + 1] - boff[b])
        got = totals[cls0:cls0 + 8 * M].reshape(M, 8)
        bad = np.argwhere(got != r['counts'])
        assert bad.size == 0, f'cloud {b}: {len(bad)} classes differ, first (box, part) {bad[0]}: ' \
                              f'{got[tuple(bad[0])]} != {r["counts"][tuple(bad[0])]}'
        assert totals[cls0 + 8 * M] == int(r['n_bg']), f'cloud {b}: background'


@pytest.mark.parametrize('k', sorted(G), ids=IDS)
def test_batch_matches_reference(engine, k):
    """the case's clouds in one pa_aug_batch call equal the reference called on them in turn: rows (float64, by
    digest), masks and NumPy's state after the last"""
    c = cases()[k]
    pts, off, boxes, boff = batch(c['clouds'])
    np.random.seed(c['seed'])
    r = pa_aug_batch(pts, off, boxes, boff, c['param'], out_dtype=torch.float64, engine=engine)
    got = r['points'].cpu().numpy()
    for i, w in enumerate(G[k]['clouds']):
        o = got[r['offsets'][i]:r['offsets'][i + 1]]
        if sc.digest(o) != str(w['out_sha']):
            pytest.fail(f'{c["name"]} cloud {i}: {first_difference(o, c, k, i)}')
        assert r['gt_boxes_mask'][i] == w['mask'].tolist()
    assert r['counts'].cpu().tolist() == [int(w['out_shape'][0]) for w in G[k]['clouds']]
    assert sc.rng_state_equal(G[k]['clouds'][-1])


def test_mixed_batch_equals_clouds_alone(engine):
    """a cloud with no boxes, one with 1 box, 256 boxes (the shared memory of the largest), 0 rows, and 33 and 513
    tiles: in one batch, each cloud's classes behind the earlier clouds', as when run alone one after another"""
    bench, cs = sc.bench_clouds(), cases()
    one = lambda name: cs[case_index(name)]['clouds'][0]                 # noqa: E731
    clouds = [(bench[0][0], bench[0][1][:0]), (bench[1][0], bench[1][1][:1]), one('256 boxes'), one('zero rows'),
              one('scan 33 tiles'), one('scan 513 tiles')]
    np.random.seed(11)
    want = []
    for cl in clouds:
        want.append(pa_aug_batch(*batch([cl]), sc.DENSE, out_dtype=torch.float64, engine=engine))
    wstate = np.random.get_state()
    np.random.seed(11)
    r = pa_aug_batch(*batch(clouds), sc.DENSE, out_dtype=torch.float64, engine=engine)
    st = np.random.get_state()
    got = r['points'].cpu().numpy()
    for b, w in enumerate(want):
        assert same_bits(got[r['offsets'][b]:r['offsets'][b + 1]], w['points'].cpu().numpy()), f'cloud {b}'
        assert r['gt_boxes_mask'][b] == w['gt_boxes_mask'][0]
    assert np.array_equal(st[1], wstate[1]) and st[2:] == wstate[2:]


def test_slot_compacted_bench_clouds(engine):
    """counts= with rows inside the boxes behind every count: the garbage would change the totals if counted, and the
    result equals the dense call and the reference"""
    k = case_index('bench dense')
    c = cases()[k]
    rng = np.random.default_rng(12)
    pad = [sc.fill_boxes(rng, np.zeros((0, 4), np.float32), boxes, 5) for _, boxes in c['clouds']]
    pts, off, boxes, boff = batch(c['clouds'], pad)
    counts = torch.tensor([p.shape[0] for p, _ in c['clouds']], dtype=torch.int32, device='cuda')
    names = sc.names_of(boxes)
    d_planes = torch.from_numpy(box_planes(boxes, names)).cuda()
    d_nparts = torch.tensor([NUM_PARTITION[n] for n in names], dtype=torch.int32, device='cuda')
    padded = engine.pa_partition_batch(pts, off, d_planes, d_nparts, boff, False).cpu().numpy()
    compact = engine.pa_partition_batch(pts, off, d_planes, d_nparts, boff, False, counts=counts).cpu().numpy()
    want = np.concatenate([np.append(w['counts'].reshape(-1), int(w['n_bg'])) for w in G[k]['clouds']])
    assert np.array_equal(compact, want)
    assert (padded[want != 0] != want[want != 0]).sum() >= 100            # the garbage lies in the boxes' parts
    np.random.seed(c['seed'])
    r = pa_aug_batch(pts, off, boxes, boff, c['param'], counts=counts, out_dtype=torch.float64, engine=engine)
    got = r['points'].cpu().numpy()
    for i, w in enumerate(G[k]['clouds']):
        assert sc.digest(got[r['offsets'][i]:r['offsets'][i + 1]]) == str(w['out_sha']), f'cloud {i}'
        assert r['gt_boxes_mask'][i] == w['mask'].tolist()
    assert sc.rng_state_equal(G[k]['clouds'][-1])


@pytest.mark.parametrize('name', ['bench dense', 'nan row'])
def test_float32_output_is_the_float64_rounded_once(engine, name):
    """out_dtype=torch.float32 equals the float64 result rounded once (NaN payloads as NumPy rounds them), and a
    second identical call gives the same bits"""
    c = cases()[case_index(name)]
    args = batch(c['clouds'])
    res = []
    for dt in (torch.float64, torch.float32, torch.float32):
        np.random.seed(c['seed'])
        res.append(pa_aug_batch(*args, c['param'], out_dtype=dt, engine=engine)['points'].cpu().numpy())
    assert res[1].dtype == np.float32
    assert np.array_equal(res[1].view(np.uint32), res[0].astype(np.float32).view(np.uint32))
    assert np.array_equal(res[1].view(np.uint32), res[2].view(np.uint32))


def test_257_boxes_raise_before_any_draw(engine):
    """the engine's limit is 256 boxes per cloud (the reference has none): ValueError, NumPy's state untouched"""
    pts, boxes = sc.many_boxes_cloud(m=257)
    np.random.seed(13)
    before = np.random.get_state()
    with pytest.raises(ValueError, match='256'):
        pa_aug_batch(*batch([(pts, boxes)]), sc.DENSE, engine=engine)
    after = np.random.get_state()
    assert np.array_equal(after[1], before[1]) and after[2:] == before[2:]

"""
The indexed device stages against plain statements of their rules, on inputs built to reach the edges of their indexes
(tests/index_edges_case.py; tests/test_index_edges_cpu.py checks that they do):

  strongest / last (csrc/select.cu)   forced 32-bit hash collisions inside, behind and just below the window, in the
                                      wrapped window and at diff = 0, -0 / +0, runs of 1 000 duplicates: against
                                      compare_points' own j loop, and a 131 072-row batch against strongest_last_mask.
  DROR (csrc/dror.cu)                 a neighbour one float32 ulp inside / outside the radius in the last cell the
                                      query visits, at every level; rows far past the grid and float32 overflow: against
                                      the full pairwise float32 distance matrix.
  voxels (csrc/voxelize.cu)           rows on and one or two ulps around voxel boundaries, non-finite rows, 5 000 rows
                                      in one voxel, 300-voxel probe chains, chains that wrap, tables at maximum load:
                                      against the literal spconv rule (and the oracle for the 131 072-row clouds).

Every case runs on dense input and on slot-compacted input with adversarial garbage rows behind each cloud's count.
Everything is exact.
"""
import numpy as np
import pytest
import torch

import index_edges_case as C
from oracle import select as osel
from oracle import voxel as V
from test_voxelize import _compare, literal_rule

pytestmark = pytest.mark.gpu


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _offsets(clouds):
    return np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)


def _layout(clouds, slot_compacted, garbage=None, pad=9):
    """(points on the device, offsets, counts or None).  Slot-compacted: `pad` garbage rows behind every cloud, by
    default copies of the cloud's own rows (or of `garbage[b]`), so that a kernel reading past the count is seen."""
    if not slot_compacted:
        return torch.from_numpy(np.concatenate(clouds)).cuda(), _offsets(clouds), None
    rng = np.random.default_rng(len(clouds))
    slots = []
    for b, c in enumerate(clouds):
        src = garbage[b] if garbage is not None else c
        g = src[rng.integers(0, len(src), pad)] if len(src) else rng.normal(0, 10, (pad, c.shape[1]))
        slots.append(np.concatenate([c, g.astype(np.float32)]))
    cnt = torch.tensor([len(c) for c in clouds], dtype=torch.int32, device='cuda')
    return torch.from_numpy(np.concatenate(slots)).cuda(), _offsets(slots), cnt


# ----------------------------------------------------------------------------------------------- strongest / last

def _run_sl(engine, pairs, slot_compacted):
    lasts = [p[0] for p in pairs]
    strongs = [p[1] for p in pairs]
    masters = [s if len(s) > len(l) else l for l, s in zip(lasts, strongs)]
    pl, off_l, cl = _layout(lasts, slot_compacted, masters, pad=7)
    ps, off_s, cs = _layout(strongs, slot_compacted, masters, pad=13)
    res = engine.strongest_last_batch(pl, off_l, ps, off_s, last_counts=cl, strongest_counts=cs, want_mask=True)
    engine.check()
    return res, res['points'].cpu().numpy(), res['mask'].cpu().numpy().astype(bool)


@pytest.mark.parametrize('slot_compacted', [False, True])
def test_strongest_last_on_forced_hash_collisions(engine, slot_compacted):
    cases = C.sl_small_cases()
    res, pts, mask = _run_sl(engine, cases, slot_compacted)
    for b, (last, strongest, planted) in enumerate(cases):
        master, want, *_ = osel.compare_points_loop(last, strongest)
        o, n = int(res['offsets'][b]), int(res['counts'][b])
        got = mask[o:o + len(master)]
        assert np.array_equal(got, want), (b, np.nonzero(got != want)[0][:10])
        assert all(got[i] == w for i, w in planted)
        assert n == int(want.sum()) and _same_bits(pts[o:o + n], master[want]), b
        assert int(res['master_is_strongest'][b]) == int(len(strongest) > len(last))


@pytest.mark.parametrize('slot_compacted', [False, True])
def test_strongest_last_131072_rows_with_planted_collisions(engine, slot_compacted):
    pairs = [C.sl_big_pair(21), C.sl_big_pair(22)]
    res, pts, mask = _run_sl(engine, pairs, slot_compacted)
    for b, (last, strongest, planted) in enumerate(pairs):
        master, want, *_ = osel.strongest_last_mask(last, strongest)
        o, n = int(res['offsets'][b]), int(res['counts'][b])
        assert np.array_equal(mask[o:o + len(master)], want), b
        assert all(want[i] == w for i, w in planted)
        assert n == int(want.sum()) and _same_bits(pts[o:o + n], master[want]), b


# ------------------------------------------------------------------------------------------------------------ DROR

def _run_dror(engine, clouds, k_min, sr_min, slot_compacted, garbage=None):
    pts, off, cnt = _layout(clouds, slot_compacted, garbage)
    res = engine.dror_batch(pts, off, alpha=0.16, beta=3.0, k_min=k_min, sr_min=sr_min, counts=cnt, work_stats=True)
    engine.check()
    out = {k: v.cpu().numpy() for k, v in res.items()}
    for b, pc in enumerate(clouds):
        want = C.dror_brute_codes(pc, 0.16, 3.0, k_min, sr_min)
        o = int(off[b])
        got = out['keep'][o:o + len(pc)]
        assert np.array_equal(got, want), (b, k_min, sr_min, np.nonzero(got != want)[0][:10])
        assert int(out['counts'][b]) == int(want.sum()) and int(out['n_snow'][b]) == int((want == 0).sum())
        assert _same_bits(out['points'][o:o + int(want.sum())], pc[want == 1])
    return out, off


@pytest.mark.parametrize('sr_min', [0.0, 0.04])
@pytest.mark.parametrize('k_min', [0, 1, 3, 5])
def test_dror_neighbour_one_ulp_from_the_radius_in_the_last_cell(engine, k_min, sr_min):
    cases = [C.dror_corner_case(level, inside, k_min, sr_min=sr_min) for level in range(16) for inside in (True, False)]
    clouds = [c for c, _ in cases]
    queries = [c[:1].repeat(3, 0) for c in clouds]                    # garbage: copies of each cloud's query
    for slot_compacted in (False, True):
        out, off = _run_dror(engine, clouds, k_min, sr_min, slot_compacted, queries)
        if k_min >= 1:
            assert [int(out['keep'][off[b]]) for b in range(len(cases))] == [int(i['inside']) for _, i in cases]
        queries_run, cells = int(out['work'][0]), int(out['work'][1])
        assert queries_run == sum(len(c) for c in clouds)
        if k_min == 0:
            assert cells == queries_run                               # every query stops at itself
        else:
            assert cells > queries_run                                # the multi-cell path ran


@pytest.mark.parametrize('k_min,sr_min', [(1, 0.04), (3, 0.0), (0, 0.04)])
def test_dror_rows_past_the_grid_and_overflowing_distances(engine, k_min, sr_min):
    clouds = [C.dror_far_cloud(3), C.dror_far_cloud(4), C.dror_corner_case(15, True, 3, sr_min=sr_min)[0]]
    for slot_compacted in (False, True):
        _run_dror(engine, clouds, k_min, sr_min, slot_compacted)


@pytest.mark.parametrize('k_min', [1, 3, 5])
def test_dror_every_query_exits_in_its_own_cell(engine, k_min):
    clouds = [C.dror_cluster_cloud(4, k_min), C.dror_cluster_cloud(5, k_min, 40)]
    for slot_compacted in (False, True):
        out, _ = _run_dror(engine, clouds, k_min, 0.04, slot_compacted)
        n = sum(len(c) for c in clouds)
        assert out['work'].tolist()[:2] == [n, n] and int(out['work'][3]) == n


# ---------------------------------------------------------------------------------------------------------- voxels

def _voxel_check(engine, clouds, rng, vs, max_points, max_voxels, mask_xy=True, slot_compacted=False, oracle=False):
    pts, off, cnt = _layout(clouds, slot_compacted)
    out = engine.voxelize_batch(pts, off, rng, vs, max_points, max_voxels, counts=cnt, mask_xy_range=mask_xy)
    engine.check()
    for b, pc in enumerate(clouds):
        kept = pc[V.mask_points_by_range(pc, rng)] if mask_xy else pc
        want = V.points_to_voxels(kept, rng, vs, max_points, max_voxels) if oracle else \
            literal_rule(kept, rng, vs, max_points, max_voxels)
        if len(want[0]) == 0:
            want = (np.zeros((0, max_points, pc.shape[1]), np.float32), np.zeros((0, 3), np.int32),
                    np.zeros(0, np.int32))
        _compare(out, b, (kept,) + tuple(want), max_voxels)
    return out


@pytest.mark.parametrize('mask_xy', [True, False])
@pytest.mark.parametrize('max_voxels', [1, 3, 16000])
@pytest.mark.parametrize('max_points', [1, 5, 64])
def test_voxel_boundary_rows(engine, max_points, max_voxels, mask_xy):
    clouds = [C.boundary_cloud(7), C.boundary_cloud(8)]
    for slot_compacted in (False, True):
        _voxel_check(engine, clouds, C.RANGE, C.VSIZE, max_points, max_voxels, mask_xy, slot_compacted)


def test_voxel_grid_size_rounds_half_to_even(engine):
    r = np.random.default_rng(2)
    rng, vs = [0, 0, 0, 2.5, 3.5, 4.5], [1, 1, 1]                      # quotients 2.5, 3.5, 4.5 -> 2, 4, 4
    pc = np.column_stack([r.uniform(-0.5, 5, (3000, 3)), np.arange(3000)]).astype(np.float32)
    pc[:40, 0] = 2.25                                                  # in a third x voxel only if 2.5 rounds up
    for mask_xy in (True, False):
        out = _voxel_check(engine, [pc], rng, vs, 4, 200, mask_xy)
        assert int(out['coords'][0, :int(out['n_voxels'][0]), 3].max()) == 1


@pytest.mark.parametrize('max_points,max_voxels', [(1, 4), (64, 4), (1000, 2)])
def test_voxel_keeps_the_first_points_of_an_overfull_voxel(engine, max_points, max_voxels):
    clouds = [C.one_voxel_cloud(5000, 3), C.one_voxel_cloud(1200, 4)]
    for slot_compacted in (False, True):
        out = _voxel_check(engine, clouds, C.RANGE, C.VSIZE, max_points, max_voxels, True, slot_compacted)
        assert out['num_points'][:, 0].tolist() == [max_points, max_points]


@pytest.mark.parametrize('max_voxels', [100, 16000])
def test_voxel_probe_chains_that_share_a_bucket_and_wrap(engine, max_voxels):
    """chain clouds between clouds at maximum load (every row its own voxel).  The chains depend on the slot size
    (the table has 2 * slot + 1 buckets), so the slot-compacted run builds its clouds at the slot size and overwrites
    the last rows of each slot with garbage."""
    pad = 9
    for slot_compacted in (False, True):
        sizes = (4096, 4096, 2048, 4096)
        full = [C.chain_cloud(sizes[0], 3)[0], C.unique_voxel_cloud(sizes[1], 5), C.unique_voxel_cloud(sizes[2], 6),
                C.chain_cloud(sizes[3], 9)[0]]
        if not slot_compacted:
            _voxel_check(engine, full, C.RANGE, C.VSIZE, 5, max_voxels)
            continue
        valid = [c[:len(c) - pad] for c in full]
        slots = [np.concatenate([c[:len(c) - pad], c[:pad]]) for c in full]
        pts = torch.from_numpy(np.concatenate(slots)).cuda()
        cnt = torch.tensor([len(c) for c in valid], dtype=torch.int32, device='cuda')
        out = engine.voxelize_batch(pts, _offsets(slots), C.RANGE, C.VSIZE, 5, max_voxels, counts=cnt)
        engine.check()
        for b, pc in enumerate(valid):
            kept = pc[V.mask_points_by_range(pc, C.RANGE)]
            _compare(out, b, (kept,) + literal_rule(kept, C.RANGE, C.VSIZE, 5, max_voxels), max_voxels)


@pytest.mark.parametrize('slot_compacted', [False, True])
def test_voxel_131072_row_clouds(engine, slot_compacted):
    clouds = [C.chain_cloud(131072, 3)[0], C.unique_voxel_cloud(131072, 4)]
    if slot_compacted:
        clouds = [c[:-9] for c in clouds]
    for max_voxels in (16000, 131072):
        _voxel_check(engine, clouds, C.RANGE, C.VSIZE, 5, max_voxels, True, slot_compacted, oracle=True)

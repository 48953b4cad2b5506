"""
The inputs of tests/test_index_edges_gpu.py reach the edges they are built for (tests/index_edges_case.py), checked on
the CPU: the restated hashes collide where the cases say they do, every planted strongest/last row has the mask value it
was built for and a walk that trusts the hash or goes below lo_row gets it wrong, every DROR placement passes or fails
the reference's test as intended at the level and in the cell intended, and the voxel boundary rows contain quotients
that a float64 or a reciprocal-multiply floor puts in another voxel.  Without these checks a GPU test could pass
because its input never reached the edge.
"""
import numpy as np
import pytest

import index_edges_case as C
from oracle import dror as od
from oracle import select as osel
from oracle import voxel as V
from test_voxelize import literal_rule


def test_xyz_hash_restatement():
    """-0 hashes as +0; the birthday search returns pairs of different rows with equal hashes."""
    a = np.array([[0.0, 1.5, -2.0], [-0.0, 1.5, -2.0], [0.0, 1.5, -0.0], [1.0, 2.0, 3.0]], np.float32)
    h = C.xyz_hash(a)
    assert h.dtype == np.uint32 and h[0] == h[1] and h[2] != h[0] and h[3] != h[0]
    for zero_x in (False, True):
        A, B = C.colliding_xyz(300 if not zero_x else 8, 11 + zero_x, zero_x)
        assert np.array_equal(C.xyz_hash(A), C.xyz_hash(B))
        assert (A != B).any(axis=1).all()
        assert (np.linalg.norm(A, axis=1) > 3).all() and (np.linalg.norm(B, axis=1) > 3).all()
        if zero_x:
            assert (A[:, 0] == 0).all() and (B[:, 0] == 0).all()
            neg = A.copy()
            neg[:, 0] = -0.0
            assert np.array_equal(C.xyz_hash(neg), C.xyz_hash(B))


def test_voxel_bucket_restatement():
    """wrapping uint64 multiply, the top 32 bits, then % cap"""
    key = np.array([0, 1, 2 ** 40 + 7, 90_111_999], np.uint64)
    want = [((int(k) * 0x9E3779B97F4A7C15) % 2 ** 64 >> 32) % 8193 for k in key]
    assert C.voxel_bucket(key, 8193).tolist() == want


def test_planted_strongest_last_rows_reach_the_walk_edges():
    cases = C.sl_small_cases()
    n_trust = n_past = 0
    for last, strongest, planted in cases:
        master, mask, *_ = osel.compare_points_loop(last, strongest)
        _, model = C.sl_index_model(last, strongest)
        assert np.array_equal(model, mask)                         # the restated index equals the reference ...
        for i, want in planted:
            assert mask[i] == want, i
        hashes = C.xyz_hash(master[[i for i, _ in planted], :3])
        slave = last if len(strongest) > len(last) else strongest
        assert np.isin(hashes, C.xyz_hash(slave[:, :3])).all()     # every planted row's hash has a slave run
        _, trust = C.sl_index_model(last, strongest, trust_hash=True)
        _, past = C.sl_index_model(last, strongest, past_lo=True)
        n_trust += int((trust != mask).sum())                      # ... and a walk that trusts its index does not
        n_past += int((past != mask).sum())
    assert n_trust >= 50 and n_past >= 50
    kinds = {(len(l) == len(s), len(s) > len(l)) for l, s, _ in cases}
    assert kinds == {(True, False), (False, True), (False, False)}  # diff = 0, master strongest, master last


def test_big_strongest_last_pair_plants():
    for seed in (21, 22):
        last, strongest, planted = C.sl_big_pair(seed)
        assert max(len(last), len(strongest)) == 131072 and len(planted) == 450
        master, mask, *_ = osel.strongest_last_mask(last, strongest)
        assert all(mask[i] == want for i, want in planted)
        assert 0 < mask.sum() < len(mask)


@pytest.mark.parametrize('sr_min', [0.0, 0.04])
def test_dror_corner_placements(sr_min):
    """every placement: the neighbour passes (inside) or fails (outside) the reference's test by one float32 ulp of
    the threshold, lies in the diagonally opposite cell at the query's level -- the last cell the query visits -- and
    decides the query's keep code.  Levels 0..15 are all reached (the level-15 cells halve each axis, so no query
    needs level 16); sr_min = 0.04 clamps the radius of the lowest ones."""
    levels = set()
    for level in range(16):
        for inside in (True, False):
            pc, info = C.dror_corner_case(level, inside, 3, sr_min=sr_min)
            p, q = pc[0, :3], pc[-1, :3]
            sr, clamped = od.search_radius(pc[:1], 0.16, 3.0, sr_min)
            d = od.sqdist32(pc[:1], pc[-1:])
            assert bool(od.passes(d, sr, clamped, sr_min)[0]) == inside
            s = np.sqrt(d.astype(np.float32))[0]
            step = np.nextafter(s, np.float32(np.inf) if inside else np.float32(-np.inf))
            assert bool(od.passes(np.array([step * step], np.float32), sr, clamped, sr_min)[0]) != inside or \
                np.float32(np.sqrt(np.float32(step * step))) != step                  # one ulp away flips it
            L = info['level']
            lo = C.dror_quant(p.astype(np.float64) - info['R']) >> L
            hi = C.dror_quant(p.astype(np.float64) + info['R']) >> L
            assert ((hi - lo) <= 1).all() and tuple(hi) == C.dror_cell(q, L)
            assert C.dror_cell(p, L) == tuple(lo) and C.dror_cell(p, L) != C.dror_cell(q, L)
            assert C.dror_brute_codes(pc, k_min=3, sr_min=sr_min)[0] == inside
            levels.add((L, info['clamped']))
    got = {L for L, _ in levels}
    if sr_min == 0.0:
        assert got == set(range(16))
    else:
        assert got == set(range(3, 16)) and (3, True) in levels
    big = max(C.dror_corner_case(15, True, 3, sr_min=sr_min)[1]['query'][:2])
    assert big > 256                                                 # the level-15 query is clamped in x


def test_dror_far_cloud_reaches_clamped_cells_and_overflow():
    pc = C.dror_far_cloud(3)
    q = C.dror_quant(pc[:, :3].astype(np.float64))
    assert ((q == 0) | (q == 65535)).any(axis=1).sum() > 100
    with np.errstate(over='ignore'):
        d = od.sqdist32(pc[:, None, :3].repeat(len(pc), 1).reshape(-1, 3), np.tile(pc[:, :3], (len(pc), 1)))
    assert np.isinf(d).any()
    codes = C.dror_brute_codes(pc, k_min=1)
    assert 0 < codes.sum() < len(pc)


def test_dror_cluster_cloud_exits_in_its_own_cell():
    for k_min in (1, 3, 5):
        pc = C.dror_cluster_cloud(4, k_min)
        qc = C.dror_quant(pc[:, :3].astype(np.float64)).reshape(-1, k_min + 2, 3)
        assert (qc == qc[:, :1]).all()                               # each cluster in one quantum
        assert C.dror_brute_codes(pc, k_min=k_min).all()


def test_dror_brute_codes_equal_the_oracle():
    rng = np.random.default_rng(5)
    pc = np.column_stack([rng.uniform(-5, 5, (1500, 3)), np.zeros((1500, 2))]).astype(np.float32)
    pc[7, 2] = np.nan
    for k_min, sr_min in ((3, 0.04), (1, 0.0)):
        assert np.array_equal(C.dror_brute_codes(pc, 0.16, 3.0, k_min, sr_min), od.keep_codes(pc, 0.16, 3.0, k_min,
                                                                                                  sr_min))


def test_voxel_boundary_rows_reach_the_rounding_edges():
    """float32 floor((x - lo) / vs) differs, on some boundary rows, from the float64 quotient's floor and from a
    float32 multiply by 1 / vs; a row at hi on x or y passes the mask and falls off the grid."""
    lo, hi, vs, gs = C.grid()
    pc = C.boundary_cloud(7)
    fin = np.isfinite(pc[:, :3]).all(axis=1)
    x = pc[fin, :3]
    q32 = np.floor((x - lo) / vs)
    q64 = np.floor((x.astype(np.float64) - lo.astype(np.float64)) / vs.astype(np.float64))
    qrc = np.floor((x - lo) * (np.float32(1) / vs))
    for axis in range(3):
        assert (q32[:, axis] != q64[:, axis]).any(), axis
        assert (q32[:, axis] != qrc[:, axis]).any(), axis
    at_hi = (pc[:, 0] == hi[0]) | (pc[:, 1] == hi[1])
    assert at_hi.sum() >= 4 and V.mask_points_by_range(pc[at_hi], C.RANGE).all()
    assert (np.floor((pc[at_hi, :2] - lo[:2]) / vs[:2]) >= gs[:2]).any(axis=1).all()
    assert np.isnan(pc).any() and np.isposinf(pc).any() and np.isneginf(pc).any()
    assert (np.signbit(pc[:, :3]) & (pc[:, :3] == 0)).any()
    # the literal rule copes with the non-finite rows (skipped) and agrees with the oracle on the rest
    a = V.points_to_voxels(pc[fin], C.RANGE, C.VSIZE, 5, 16000)
    b = literal_rule(pc, C.RANGE, C.VSIZE, 5, 16000)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))


def test_voxel_grid_size_rounds_half_to_even():
    """a range / voxel-size quotient of exactly k + 0.5 rounds to even, as np.round does"""
    for rng, vs, want in (([0, 0, 0, 2.5, 3.5, 1], [1, 1, 1], [2, 4, 1]), ([0, 0, 0, 0.25, 0.75, 4.5], [0.5, 0.5, 1],
                                                                           [0, 2, 4])):
        assert V.grid_size(rng, vs).tolist() == want


def test_voxel_chains_share_a_bucket_and_wrap():
    for n in (4096, 131072):
        pc, same, wrap, cap = C.chain_cloud(n, 3)
        assert cap == 2 * n + 1 and len(pc) == n
        _, _, _, gs = C.grid()
        assert len(np.unique(C.voxel_bucket(same, cap))) == 1 and len(same) == 300
        assert (C.voxel_bucket(wrap, cap) >= cap - 4).all() and len(wrap) == 64
        lo, _, vs, _ = C.grid()
        c = np.floor((pc[:, :3] - lo) / vs).astype(np.int64)
        key = (c[:, 2] * gs[1] + c[:, 1]) * gs[0] + c[:, 0]
        assert np.isin(same, key).all() and np.isin(wrap, key).all()   # the rows land in the keys' voxels
        # the probe sequence of a sequential insert: some chain runs 300 long, some wraps past the table's end
        table = np.full(cap, -1, np.int64)
        longest = wrapped = 0
        for k in dict.fromkeys(key.tolist()):
            h = int(C.voxel_bucket(np.array([k]), cap)[0])
            steps = 0
            while table[h] != -1:
                h = h + 1 if h + 1 < cap else 0
                steps += 1
                wrapped += h == 0
            table[h] = k
            longest = max(longest, steps)
        assert longest >= 299 and wrapped > 0
    u = C.unique_voxel_cloud(4096, 5)
    assert len(np.unique(u[:, :3], axis=0)) == 4096

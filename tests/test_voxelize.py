"""
Point-range mask + voxelisation (SURVEY.md 8f-4): the detector-input stage of the reference's data path
(lib/OpenPCDet/pcdet/datasets/processor/data_processor.py:78-91, 115-143; config dense_dataset.yaml:4,66-78).

The voxel rule is spconv's (third party, absent from the reference tree and from this image): PARITY UNPINNED for that
rule -- oracle/voxel.py restates its published algorithm.  The CPU tests pin the oracle's vectorised restatement to a
literal, loop-by-loop transcription of the rule; the GPU tests compare the CUDA path with the oracle: integer work,
so everything must be bit-exact (voxel order, coordinates, counts, the points kept and their order).
"""
import numpy as np
import pytest
import torch

from oracle import voxel as V
from lidar_snow_sim_b200.synthetic import synthetic_cloud

RANGE = [0, -40, -3, 70.4, 40, 1]           # dense_dataset.yaml:4
VSIZE = [0.05, 0.05, 0.1]                   # dense_dataset.yaml:71


def literal_rule(points, rng, vsize, max_points, max_voxels):
    """spconv 1.x points_to_voxel_3d_np, transcribed literally (float32 scalars, dense coor_to_voxelidx array)."""
    rng = np.asarray(rng, dtype=np.float32)
    vsize = np.asarray(vsize, dtype=np.float32)
    gs = np.round((rng[3:] - rng[:3]) / vsize).astype(np.int32)
    lut = -np.ones(gs[::-1], dtype=np.int32)
    voxels, coors, num = [], [], []
    for i in range(points.shape[0]):
        coor = [0, 0, 0]
        failed = False
        for j in range(3):
            c = np.floor((np.float32(points[i, j]) - rng[j]) / vsize[j])
            if not (c >= 0 and c < gs[j]):          # (a NaN or infinite quotient casts to INT_MIN in C++: skipped)
                failed = True
                break
            coor[2 - j] = int(c)
        if failed:
            continue
        vid = lut[coor[0], coor[1], coor[2]]
        if vid == -1:
            vid = len(voxels)
            if vid >= max_voxels:
                continue
            lut[coor[0], coor[1], coor[2]] = vid
            voxels.append(np.zeros((max_points, points.shape[1]), dtype=np.float32))
            coors.append(coor)
            num.append(0)
        if num[vid] < max_points:
            voxels[vid][num[vid]] = points[i]
            num[vid] += 1
    return np.array(voxels, dtype=np.float32), np.array(coors, dtype=np.int32), np.array(num, dtype=np.int32)


def test_oracle_equals_the_literal_rule():
    pc = synthetic_cloud(seed=5, n_azimuth=96, shuffle_rows=True)
    for vs, mp, mv in ((VSIZE, 5, 16000), ([0.8, 0.8, 0.4], 3, 700), ([2.0, 2.0, 4.0], 32, 10 ** 6)):
        a = V.points_to_voxels(pc, RANGE, vs, mp, mv)
        b = literal_rule(pc, RANGE, vs, mp, mv)
        for x, y in zip(a, b):
            assert x.shape == y.shape and np.array_equal(x, y)
    assert V.grid_size(RANGE, VSIZE).tolist() == [1408, 1600, 40]                  # the reference's PV-RCNN grid
    # mask_points_by_range: x / y only, both ends inclusive (common_utils.py:60-63)
    p = np.array([[0, -40, 9, 1, 0], [70.4, 40, -9, 1, 0], [70.5, 0, 0, 1, 0], [-0.01, 0, 0, 1, 0]], dtype=np.float32)
    assert V.mask_points_by_range(p, RANGE).tolist() == [True, True, False, False]


def _compare(out, b, want, max_voxels):
    pts, vox, co, num = want
    n = int(out['n_voxels'][b])
    assert n == vox.shape[0]
    assert np.array_equal(out['voxels'][b, :n].cpu().numpy(), vox)
    assert np.array_equal(out['coords'][b, :n, 1:].cpu().numpy(), co)
    assert (out['coords'][b, :n, 0].cpu().numpy() == b).all()
    assert np.array_equal(out['num_points'][b, :n].cpu().numpy(), num)
    if n < max_voxels:                                                              # padding rows are zero
        assert not out['voxels'][b, n:].any() and not out['num_points'][b, n:].any()


@pytest.mark.gpu
@pytest.mark.parametrize('vsize,max_points,max_voxels', [(VSIZE, 5, 16000), (VSIZE, 5, 40000), ([0.4, 0.4, 0.5], 5, 6000),
                                                         ([1.6, 1.6, 4.0], 32, 3000)])
def test_batch_matches_the_oracle(engine, vsize, max_points, max_voxels):
    clouds = [synthetic_cloud(seed=40 + b, n_azimuth=n, drop=0.05, shuffle_rows=bool(b & 1)) for b, n in
              enumerate((2048, 512, 3, 1024))]
    clouds[2] = clouds[2][:0]                                                       # an empty cloud in the batch
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    d = torch.from_numpy(np.concatenate(clouds)).cuda()
    out = engine.voxelize_batch(d, off, RANGE, vsize, max_points, max_voxels)
    engine.check()
    for b, c in enumerate(clouds):
        _compare(out, b, V.mask_and_voxelize(c, RANGE, vsize, max_points, max_voxels), max_voxels)
    # deterministic (atomics only feed order-independent reductions)
    out2 = engine.voxelize_batch(d, off, RANGE, vsize, max_points, max_voxels)
    assert all(torch.equal(out[k], out2[k]) for k in out)


@pytest.mark.gpu
def test_augmented_batch_goes_to_voxels_without_leaving_the_device(engine):
    """snowfall -> voxels on the device: the slot-compacted augmentation output (rows + per-cloud counts) is the
    voxeliser's input; equals voxelising the host copy of every augmented cloud with the oracle."""
    from helpers import DIV
    from lidar_snow_sim_b200.synthetic import synthetic_particles
    from lidar_snow_sim_b200.integrations.voxelize import DeviceVoxelizer
    clouds = [synthetic_cloud(seed=90 + b, n_azimuth=512) for b in range(3)]
    tables = [synthetic_particles(3000 + k, 18000) for k in range(64)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    orders = np.stack([np.random.default_rng(b).permutation(64) for b in range(3)]).astype(np.int32)
    tid = engine.upload_tables(tables)
    snow = engine.snowfall_batch(tid, torch.from_numpy(np.concatenate(clouds)).cuda(), off, orders, DIV,
                                 thresh_poly=np.tile([1e-3, -0.2, 9.0], (3, 1)))
    vox = DeviceVoxelizer(RANGE, VSIZE, 5, 16000, engine=engine)
    out = vox.batch(snow['points'], off, counts=snow['counts'])
    engine.check()
    engine.free_tables(tid)
    host = snow['points'].cpu().numpy()
    cnt = snow['counts'].cpu().numpy()
    for b in range(3):
        _compare(out, b, V.mask_and_voxelize(host[off[b]:off[b] + cnt[b]], RANGE, VSIZE, 5, 16000), 16000)
    col = vox.collate(out)
    n = out['n_voxels'].cpu().numpy()
    assert col['voxels'].shape[0] == n.sum() and col['voxel_coords'][n[0], 0].item() == 1
    # the one-cloud, reference-keyed call (DataProcessor API): numpy in, numpy out
    dd = vox({'points': clouds[0], 'use_lead_xyz': True})
    pts, v, c, m = V.mask_and_voxelize(clouds[0], RANGE, VSIZE, 5, 16000)
    assert np.array_equal(dd['points'], pts) and np.array_equal(dd['voxels'], v)
    assert np.array_equal(dd['voxel_coords'], c) and np.array_equal(dd['voxel_num_points'], m)

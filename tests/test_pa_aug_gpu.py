"""PA-AUG on the device against the unmodified reference (tests/golden/pa_aug.npz): PartAwareAugmentation.augment bit
for bit, pa_aug_batch against sequential calls (dense and slot-compacted input), and the dataset block."""
import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.integrations.dense import pa_aug_block, pa_aug_block_batch
from lidar_snow_sim_b200.pa_aug import CLASS_NAMES, PartAwareAugmentation, pa_aug_batch
from test_pa_aug_cpu import CASES, case, rng_state_equal, same_bits

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('k', CASES)
def test_augment_matches_reference(k):
    c = case(k)
    np.random.seed(int(c['seed']))
    aug = PartAwareAugmentation(c['pts'], c['boxes'], c['gt_names'], CLASS_NAMES)
    if 'exc' in c:
        with pytest.raises(Exception) as ei:
            aug.augment(c['param'])
        assert type(ei.value).__name__ == str(c['exc'])
    else:
        out, mask = aug.augment(c['param'])
        assert same_bits(out, c['out']), str(c['name'])
        assert mask == c['mask'].tolist()
    assert rng_state_equal(c)


def _batch_cases():
    ks = [k for k in CASES if 'exc' not in case(k) and case(k)['pts'].shape[1] == 4]
    return [case(k) for k in ks]


def _sequential(cs, param, seed):
    np.random.seed(seed)
    outs, masks = [], []
    for c in cs:
        o, m = PartAwareAugmentation(c['pts'], c['boxes'].astype(np.float32), c['gt_names'], CLASS_NAMES).augment(param)
        outs.append(o)
        masks.append(m)
    return outs, masks, np.random.get_state()


@pytest.mark.parametrize('param', ['dropout1_p05_swap_p10_mix_p10_sparse8_p10_jitter_p10_noise5_p10',
                                   'dropout_p02_swap_p02_mix_p02_sparse40_p02_jitter_p02_noise10_p02'])
@pytest.mark.parametrize('compact', [False, True])
def test_batch_equals_sequential_calls(param, compact):
    cs = _batch_cases()[:12]
    want, wmask, wstate = _sequential(cs, param, 77)
    rows, offs, cnts, boxes, boff = [], [0], [], [], [0]
    rng = np.random.default_rng(3)
    for c in cs:
        p = c['pts']
        cnts.append(p.shape[0])
        if compact:                                                # garbage rows behind the valid ones
            p = np.concatenate([p, rng.uniform(-5, 5, (17, 4)).astype(np.float32)])
        rows.append(p)
        offs.append(offs[-1] + p.shape[0])
        boxes.append(c['boxes'].astype(np.float32))
        boff.append(boff[-1] + c['boxes'].shape[0])
    pts = torch.from_numpy(np.concatenate(rows)).cuda()
    counts = torch.tensor(cnts, dtype=torch.int32, device='cuda') if compact else None
    np.random.seed(77)
    r = pa_aug_batch(pts, offs, np.concatenate(boxes), boff, param, counts=counts, out_dtype=torch.float64)
    st = np.random.get_state()
    got = r['points'].cpu().numpy()
    assert r['counts'].cpu().tolist() == [w.shape[0] for w in want]
    for b, w in enumerate(want):
        assert same_bits(got[r['offsets'][b]:r['offsets'][b + 1]], w)
        assert r['gt_boxes_mask'][b] == wmask[b]
    assert np.array_equal(st[1], wstate[1]) and st[2:] == wstate[2:]
    r32 = pa_aug_batch(pts, offs, np.concatenate(boxes), boff, param, counts=counts)
    assert r32['points'].dtype == torch.float32


def test_batch_raises_where_the_reference_raises():
    cs = _batch_cases()[:3]
    pts = torch.from_numpy(np.concatenate([np.column_stack([c['pts'], np.zeros(len(c['pts']), np.float32)])
                                           for c in cs])).cuda()
    offs = np.concatenate([[0], np.cumsum([len(c['pts']) for c in cs])])
    boxes = np.concatenate([c['boxes'].astype(np.float32) for c in cs])
    boff = np.concatenate([[0], np.cumsum([len(c['boxes']) for c in cs])])
    param = 'swap_p10_jitter_p10'
    np.random.seed(5)
    with pytest.raises(ValueError):
        PartAwareAugmentation(np.column_stack([cs[0]['pts'], np.zeros(len(cs[0]['pts']), np.float32)]),
                              cs[0]['boxes'].astype(np.float32), cs[0]['gt_names'], CLASS_NAMES).augment(param)
    want = np.random.get_state()
    np.random.seed(5)
    with pytest.raises(ValueError):
        pa_aug_batch(pts, offs, boxes, boff, param)
    got = np.random.get_state()
    assert np.array_equal(got[1], want[1]) and got[2:] == want[2:]
    with pytest.raises(IndexError):
        pa_aug_batch(pts, offs, boxes, boff, 'swap')


def _literal_block(data_dict, dataset_cfg, training):
    """dense_dataset.py:938-949 as written, with the reference's PartAwareAugmentation replaced by the engine's"""
    if training and 'PA_AUG_STRING' in dataset_cfg:
        class_names = ['Car', 'Pedestrian', 'Cyclist']
        pa_aug_param = dataset_cfg['PA_AUG_STRING']
        gt_names = np.asarray([class_names[int(c) - 1] for c in data_dict['gt_boxes'][:, -1]])
        pa_aug = PartAwareAugmentation(data_dict['points'], data_dict['gt_boxes'], gt_names, class_names)
        data_dict['points'], gt_boxes_mask = pa_aug.augment(pa_aug_param=pa_aug_param)
        data_dict['gt_boxes'] = data_dict['gt_boxes'][gt_boxes_mask]
    return data_dict


def test_block_and_block_batch():
    cfg = {'PA_AUG_STRING': 'dropout_p02_swap_p02_mix_p02_sparse40_p02_jitter_p02_noise10_p02'}
    cs = _batch_cases()[:4]
    np.random.seed(9)
    want = [_literal_block({'points': c['pts'], 'gt_boxes': c['boxes'].astype(np.float32)}, cfg, True) for c in cs]
    np.random.seed(9)
    got = [pa_aug_block({'points': c['pts'], 'gt_boxes': c['boxes'].astype(np.float32)}, cfg, True) for c in cs]
    for w, g in zip(want, got):
        assert same_bits(g['points'], w['points']) and np.array_equal(g['gt_boxes'], w['gt_boxes'])
    pts = torch.from_numpy(np.concatenate([c['pts'] for c in cs])).cuda()
    offs = np.concatenate([[0], np.cumsum([len(c['pts']) for c in cs])])
    boxes = np.concatenate([c['boxes'].astype(np.float32) for c in cs])
    boff = np.concatenate([[0], np.cumsum([len(c['boxes']) for c in cs])])
    np.random.seed(9)
    r = pa_aug_block_batch(pts, offs, boxes, boff, cfg, out_dtype=torch.float64)
    for b, w in enumerate(want):
        assert same_bits(r['points'][r['offsets'][b]:r['offsets'][b + 1]].cpu().numpy(), w['points'])
        assert np.array_equal(r['gt_boxes'][r['box_offsets'][b]:r['box_offsets'][b + 1]], w['gt_boxes'])
    assert pa_aug_block_batch(pts, offs, boxes, boff, cfg, training=False) is None

"""FogAugmentation's draws (integrations/dense.py) against `DenseDataset.__getitem__`'s fog lines and foggify's
bookkeeping (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:618-671, 1011-1012, init_curriculum :115-119),
restated statement by statement."""
import math

import numpy as np
import pytest

from lidar_snow_sim_b200.integrations.dense import FOG_ALPHAS, FogAugmentation


class Dataset:
    """the dataset's attributes and lines that the fog block reads and writes"""

    def __init__(self, cfg, seed):
        self.dataset_cfg = cfg
        self.curriculum_stage = 0
        self.total_iterations = -1
        self.current_iteration = -1
        self.iteration_increment = -1
        self.random_generator = np.random.default_rng(seed)

    def init_curriculum(self, it, epochs, workers, length):
        self.current_iteration = it
        self.iteration_increment = workers
        self.total_iterations = epochs * length

    def foggify(self, curriculum_stage):
        self.curriculum_stage = curriculum_stage
        self.current_iteration += self.iteration_increment

    def getitem(self, training=True):
        mor = np.inf
        alpha = None
        if training and (self.dataset_cfg.get('FOG_AUGMENTATION') or self.dataset_cfg.get('FOG_AUGMENTATION_AFTER')):
            if self.dataset_cfg.get('FOG_AUGMENTATION'):
                fog_augmentation_string = self.dataset_cfg['FOG_AUGMENTATION']
            else:
                fog_augmentation_string = self.dataset_cfg['FOG_AUGMENTATION_AFTER']
            if 'FOG_ALPHAS' in self.dataset_cfg:
                alphas = self.dataset_cfg['FOG_ALPHAS']
            else:
                alphas = ['0.000', '0.005', '0.010', '0.020', '0.030', '0.060']
            augmentation_method = fog_augmentation_string.split('_')[0]
            augmentation_schedule = fog_augmentation_string.split('_')[-1]
            if augmentation_schedule == 'curriculum':
                progress = self.current_iteration / self.total_iterations
                ratio = 1 / len(alphas)
                curriculum_stage = math.floor(progress / ratio)
            elif augmentation_schedule == 'uniform':
                curriculum_stage = int(self.random_generator.integers(low=0, high=len(alphas)))
            else:
                curriculum_stage = len(alphas) - 1
                if 'FOG_ALPHA' in self.dataset_cfg:
                    a = self.dataset_cfg['FOG_ALPHA']
                    curriculum_stage = min(range(len(alphas)), key=lambda i: abs(float(alphas[i]) - a))
            alpha = alphas[curriculum_stage]
            mor = np.inf if alpha == '0.000' else np.log(20) / float(alpha)
            if self.dataset_cfg.get('FOG_AUGMENTATION'):
                self.foggify(curriculum_stage)
            if 'FOG_AUGMENTATION_AFTER' in self.dataset_cfg:
                self.foggify(curriculum_stage)
            return alpha, augmentation_method, mor
        return alpha, None, mor


CFGS = [
    {'FOG_AUGMENTATION': 'DENSE_uniform'},
    {'FOG_AUGMENTATION': 'CVL_uniform', 'FOG_ALPHAS': ['0.000', '0.030', '0.060']},
    {'FOG_AUGMENTATION': 'DENSE_curriculum'},
    {'FOG_AUGMENTATION': False, 'FOG_AUGMENTATION_AFTER': 'DENSE_curriculum'},
    {'FOG_AUGMENTATION': 'CVL_curriculum', 'FOG_AUGMENTATION_AFTER': 'CVL_uniform'},
    {'FOG_AUGMENTATION': 'DENSE_fixed'},
    {'FOG_AUGMENTATION': 'DENSE_fixed', 'FOG_ALPHA': 0.012},
    {'FOG_AUGMENTATION': False},
]


@pytest.mark.parametrize('cfg', CFGS)
@pytest.mark.parametrize('training', [True, False])
def test_draws_equal_getitem(cfg, training):
    ds = Dataset(cfg, 5)
    fog = FogAugmentation(cfg, random_generator=np.random.default_rng(5))
    ds.init_curriculum(3, 2, 4, 400)
    fog.init_curriculum(3, 2, 4, 400)
    for B in (1, 7, 0, 12):
        want = [ds.getitem(training) for _ in range(B)]
        alphas, methods, mor = fog.draw_batch(B, training)
        assert alphas == [w[0] for w in want]
        assert methods == [w[1] for w in want]
        assert np.array_equal(mor, np.array([w[2] for w in want], dtype=np.float64))
        assert (fog.current_iteration, fog.curriculum_stage) == (ds.current_iteration, ds.curriculum_stage)
        assert fog.random_generator.bit_generator.state == ds.random_generator.bit_generator.state


def test_default_alphas_and_curriculum_end():
    assert FOG_ALPHAS == ['0.000', '0.005', '0.010', '0.020', '0.030', '0.060']
    fog = FogAugmentation({'FOG_AUGMENTATION': 'DENSE_curriculum'})
    fog.init_curriculum(10, 1, 1, 10)                           # progress 1: stage len(alphas), as the reference
    with pytest.raises(IndexError):
        fog.draw_batch(1)


def test_unknown_method_and_schedule():
    with pytest.raises(AssertionError):
        FogAugmentation({'FOG_AUGMENTATION': 'FOO_uniform'}).draw_batch(1)
    with pytest.raises(ValueError):
        FogAugmentation({'FOG_AUGMENTATION': 'DENSE_sometimes'}).draw_batch(1)

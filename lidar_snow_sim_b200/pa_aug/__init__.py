from .augmentation import CLASS_NAMES, PartAwareAugmentation, pa_aug_batch  # noqa: F401
from .plan import interpret_pa_aug_param  # noqa: F401

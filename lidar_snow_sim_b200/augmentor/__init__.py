"""OpenPCDet's DATA_AUGMENTOR (gt_sampling, world flip, rotation and scaling) with the point work on the device."""
from .augmentor import DataAugmentor, DataBaseSampler, run_batch  # noqa: F401

"""DATA_PROCESSOR and POINT_FEATURE_ENCODING of prepare_data on the engine (csrc/processor.cu)."""
from .processor import DataProcessor, PointFeatureEncoder, boxes_to_corners_3d, mask_boxes_outside_range_numpy

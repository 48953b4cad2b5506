from .filter import DROR_LEVELS, dror_level, dynamic_radius_outlier_filter, get_cube_mask, snow_indices  # noqa: F401

"""H100-native (sm_90a) LiDAR snowfall / wet-ground augmentation engine (hot path of SysCV/LiDAR_snow_sim)."""
__version__ = '0.1.0'

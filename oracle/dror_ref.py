"""
TEST INFRASTRUCTURE ONLY -- imports the UNMODIFIED reference lib/cadc_devkit/other/dror.py from /root/reference (this
container only), to generate tests/golden/dror.npz (tools/make_golden_dror.py).  Nothing in the product package, the
`-m gpu` tests, smoke() or bench.py may import this module: /root/reference does not exist on the GPU box.

dror.py imports python-pcl, which is unmaintained and not installed here.  The in-memory `pcl` shim below provides the
three things dynamic_radius_outlier_filter uses, restated from python-pcl / PCL / FLANN (exact search, epsilon 0):
  pcl.PointCloud(array)            float32 (N, 3) copy; .size; pc[i] -> (x, y, z) as Python floats
  .make_kdtree_flann()             KdTreeFLANN over the cloud
  .nearest_k_search_for_point(pc, i, k) -> (indices int32 (k,), squared distances float32 (k,)), ascending, k clamped to
                                   the cloud size; distances are flann::L2_Simple<float>: ((0 + dx*dx) + dy*dy) + dz*dz
found here by brute force.  No reference file is modified.  Parity with PCL's own build is unpinned (DESIGN.md 2, 7.4).
"""
import importlib.util
import os
import sys
import types

import numpy as np

REF_ROOT = '/root/reference'
DROR_PATH = os.path.join(REF_ROOT, 'lib', 'cadc_devkit', 'other', 'dror.py')


def available() -> bool:
    return os.path.exists(DROR_PATH)


def _pcl_shim():
    pcl = types.ModuleType('pcl')

    class KdTreeFLANN:
        def __init__(self, cloud):
            self.xyz = cloud.xyz

        def nearest_k_search_for_point(self, cloud, index, k):
            q = cloud.xyz[index]
            dx = self.xyz[:, 0] - q[0]
            dy = self.xyz[:, 1] - q[1]
            dz = self.xyz[:, 2] - q[2]
            d = ((np.float32(0) + dx * dx) + dy * dy) + dz * dz
            k = min(int(k), d.shape[0])
            order = np.argsort(d, kind='stable')[:k]
            return order.astype(np.int32), d[order].astype(np.float32)

    class PointCloud:
        def __init__(self, array):
            self.xyz = np.ascontiguousarray(np.asarray(array)[:, :3], dtype=np.float32)

        @property
        def size(self):
            return self.xyz.shape[0]

        def __getitem__(self, i):
            return tuple(float(v) for v in self.xyz[i])

        def make_kdtree_flann(self):
            return KdTreeFLANN(self)

    pcl.PointCloud = PointCloud
    return pcl


_dror = None


def load():
    """The unmodified reference module lib/cadc_devkit/other/dror.py, imported with the pcl shim."""
    global _dror
    if _dror is not None:
        return _dror
    if not available():
        raise RuntimeError('reference tree not present (expected in the build container only)')
    sys.dont_write_bytecode = True
    saved = sys.modules.get('pcl')
    sys.modules['pcl'] = _pcl_shim()
    try:
        spec = importlib.util.spec_from_file_location('reference_dror', DROR_PATH)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            del sys.modules['pcl']
        else:
            sys.modules['pcl'] = saved
    _dror = mod
    return mod

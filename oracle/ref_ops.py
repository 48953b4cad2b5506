"""
The reference's compiled box routines, as the oracle of the device GT sampling (test infrastructure, never imported by
the package).  build() compiles OpenPCDet's iou3d_nms and roiaware_pool3d extension sources, unmodified, from the
reference checkout with torch's cpp_extension (nvcc for sm_90a, so the modules' CUDA halves link) into oracle/_ref/.
Only the CPU routines are called: boxes_iou_bev_cpu and points_in_boxes_cpu.

    python -m oracle.ref_ops /path/to/reference        (or REFERENCE_ROOT=/path/to/reference)

Without a reference checkout build() does nothing; load() then finds what an earlier build left in oracle/_ref/.
"""
import glob
import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, '_ref')
DEFAULT_REFERENCE = os.path.join(os.sep, 'root', 'reference')
OPS = {
    'iou3d_nms_cuda': ('pcdet/ops/iou3d_nms/src', ['iou3d_cpu.cpp', 'iou3d_nms_api.cpp', 'iou3d_nms.cpp',
                                                    'iou3d_nms_kernel.cu']),
    'roiaware_pool3d_cuda': ('pcdet/ops/roiaware_pool3d/src', ['roiaware_pool3d.cpp', 'roiaware_pool3d_kernel.cu']),
}


def reference_root():
    root = os.environ.get('REFERENCE_ROOT', DEFAULT_REFERENCE)
    return root if os.path.isdir(os.path.join(root, 'lib', 'OpenPCDet')) else None


def _so(name):
    hits = glob.glob(os.path.join(REF_DIR, name, name + '*.so'))
    return hits[0] if hits else None


def build(root=None, verbose=False):
    """Compile both modules into oracle/_ref/<name>/ unless they are there already.  Returns the names built."""
    root = root or reference_root()
    if root is None:
        return []
    import torch.utils.cpp_extension as ext
    os.environ.setdefault('TORCH_CUDA_ARCH_LIST', '9.0a')
    built = []
    for name, (sub, files) in OPS.items():
        if _so(name):
            continue
        out = os.path.join(REF_DIR, name)
        os.makedirs(out, exist_ok=True)
        src = os.path.join(root, 'lib', 'OpenPCDet', sub)
        # -O2 as setuptools compiles an extension: at -O0 the CPU file's inline check_rect_cross stays an out-of-line
        # weak symbol, and the link binds it to the host stub of the CUDA file's __device__ function of that name
        ext.load(name=name, sources=[os.path.join(src, f) for f in files], build_directory=out, verbose=verbose,
                 extra_cflags=['-O2'], extra_cuda_cflags=['-gencode', 'arch=compute_90a,code=sm_90a'],
                 is_python_module=True)
        built.append(name)
    return built


def load(name):
    """The compiled module `name` from oracle/_ref/ (ImportError when build() has not made it)."""
    import torch  # noqa: F401  (the module links against libtorch)
    so = _so(name)
    if so is None:
        raise ImportError(f'{name} is not built: run oracle.ref_ops.build() with the reference checkout')
    if name in sys.modules:
        return sys.modules[name]
    spec = importlib.util.spec_from_file_location(name, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def available():
    return all(_so(n) for n in OPS)


def boxes_iou_bev_cpu(a, b):
    """iou3d_nms_utils.boxes_bev_iou_cpu: (N, 7), (M, 7) -> (N, M) float32"""
    import numpy as np
    import torch
    ta = torch.from_numpy(np.ascontiguousarray(a)).float().contiguous()
    tb = torch.from_numpy(np.ascontiguousarray(b)).float().contiguous()
    out = ta.new_zeros((ta.shape[0], tb.shape[0]))
    load('iou3d_nms_cuda').boxes_iou_bev_cpu(ta, tb, out)
    return out.numpy()


def points_in_boxes_cpu(points, boxes):
    """roiaware_pool3d_utils.points_in_boxes_cpu: (N, 3), (M, 7) -> (M, N) int32"""
    import numpy as np
    import torch
    tp = torch.from_numpy(np.ascontiguousarray(points)).float().contiguous()
    tb = torch.from_numpy(np.ascontiguousarray(boxes)).float().contiguous()
    out = tp.new_zeros((tb.shape[0], tp.shape[0]), dtype=torch.int)
    load('roiaware_pool3d_cuda').points_in_boxes_cpu(tb, tp, out)
    return out.numpy()


if __name__ == '__main__':
    if len(sys.argv) > 1:
        os.environ['REFERENCE_ROOT'] = sys.argv[1]
    print(build(verbose=True) or 'nothing to build', REF_DIR)

"""
The reference's LISA C++ core (`pylisa`: lib/LISA/src/{Lidar,Lisa,MiniLisa,ParticleDist,Utils}.cpp and
wrappers/wrapper.cpp), compiled unmodified from the reference checkout into oracle/_ref/pylisa/ as the oracle of the
device pylisa (test infrastructure, never imported by the package).  The committed forced include oracle/pylisa_shim.h
makes it reproducible (seeds base, base + 1, ... in construction order) and lets its default constructors build; it
touches no arithmetic.  Flags: -O2 -std=c++17 -fPIC -shared, no -march, no fast-math.

    python -m oracle.pylisa_ref /path/to/reference        (or REFERENCE_ROOT=/path/to/reference)

Without a reference checkout (or without g++ / pybind11) build() does nothing; load() then finds what an earlier build
left in oracle/_ref/pylisa/.
"""
import ctypes
import glob
import importlib.util
import os
import shutil
import subprocess
import sys
import sysconfig

_HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(_HERE, '_ref', 'pylisa')
SHIM = os.path.join(_HERE, 'pylisa_shim.h')
DEFAULT_REFERENCE = os.path.join(os.sep, 'root', 'reference')
SOURCES = ['src/Lidar.cpp', 'src/Lisa.cpp', 'src/MiniLisa.cpp', 'src/ParticleDist.cpp', 'src/Utils.cpp',
           'wrappers/wrapper.cpp']
FLAGS = ['-O2', '-std=c++17', '-fPIC', '-shared', '-pthread']


def reference_root():
    root = os.environ.get('REFERENCE_ROOT', DEFAULT_REFERENCE)
    return root if os.path.isdir(os.path.join(root, 'lib', 'LISA', 'src')) else None


def _so():
    hits = glob.glob(os.path.join(OUT_DIR, 'pylisa*.so'))
    return hits[0] if hits else None


def build(root=None, verbose=False):
    """Compile the module into oracle/_ref/pylisa/ unless it is there already.  Returns True if it was built now."""
    root = root or reference_root()
    cxx = shutil.which('g++')
    if root is None or cxx is None or _so():
        return False
    try:
        import pybind11
    except ImportError:
        return False
    lisa = os.path.join(root, 'lib', 'LISA')
    os.makedirs(OUT_DIR, exist_ok=True)
    so = os.path.join(OUT_DIR, 'pylisa' + sysconfig.get_config_var('EXT_SUFFIX'))
    tmp = so + '.tmp'
    cmd = ([cxx] + FLAGS + ['-include', SHIM, '-I', os.path.join(lisa, 'include'), '-I', pybind11.get_include(),
                            '-I', sysconfig.get_paths()['include']]
           + [os.path.join(lisa, s) for s in SOURCES] + ['-o', tmp])
    if verbose:
        print(' '.join(cmd))
    subprocess.check_call(cmd)
    os.replace(tmp, so)
    return True


def available():
    return _so() is not None


def load():
    """The compiled pylisa module (ImportError when build() has not made it)."""
    so = _so()
    if so is None:
        raise ImportError('pylisa is not built: run oracle.pylisa_ref.build() with the reference checkout')
    if 'pylisa' in sys.modules:
        return sys.modules['pylisa']
    spec = importlib.util.spec_from_file_location('pylisa', so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules['pylisa'] = mod
    return mod


def set_seed(base):
    """The next seed the module hands out (MarshallPalmerRain(), MiniLisa(...), Lisa(...) each take one, in order)."""
    load()
    ctypes.CDLL(_so()).pylisa_set_seed(ctypes.c_uint32(int(base)))


if __name__ == '__main__':
    if len(sys.argv) > 1:
        os.environ['REFERENCE_ROOT'] = sys.argv[1]
    print(build(verbose=True) or 'nothing to build', OUT_DIR)

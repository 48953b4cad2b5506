"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the header declares."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from lidar_snow_sim_b200 import build, _lib
    build.build()
    return _lib.load()


def declared_symbols():
    names = []
    for fn in os.listdir(os.path.join(ROOT, 'include')):
        if fn.endswith('.h'):
            txt = open(os.path.join(ROOT, 'include', fn)).read()
            names += re.findall(r'LSS_API[^;(]*?\b(lss_\w+)\s*\(', txt)
    return sorted(set(names))


def test_exports_every_declared_symbol(lib):
    from lidar_snow_sim_b200 import _lib
    names = declared_symbols()
    assert len(names) >= 16
    bound = {s[0] for s in _lib.SIGNATURES}
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/ but not exported'
        assert n in bound, f'{n} declared in include/ but not bound in _lib.SIGNATURES'
    assert bound <= set(names)


def test_version_and_strings(lib):
    assert lib.lss_version() >= 100
    assert lib.lss_status_string(0) == b'ok'
    assert b'120 m' in lib.lss_status_string(4)


def test_range_grid_matches_numpy(lib, oracle):
    R = np.zeros(1230)
    assert lib.lss_debug_range_grid(ctypes.c_void_p(R.ctypes.data)) == 0
    assert np.array_equal(R, oracle.range_grid())


def test_no_cpu_fallback(lib):
    """Without a GPU the engine must fail loudly, never fall back to host code."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    h = ctypes.c_void_p()
    assert lib.lss_create(0, ctypes.byref(h)) != 0
    from lidar_snow_sim_b200.engine import SnowfallEngine
    with pytest.raises(RuntimeError):
        SnowfallEngine(0)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, 'lidar_snow_sim_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.cpp', '.h')):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', txt, re.M), f'{f} imports the oracle'
                assert 'liboracle' not in txt
                assert '/root/reference' not in txt


def test_focal_offset_matches_python():
    from lidar_snow_sim_b200.calib.hdl64e_s3 import sensor_arrays
    fd = sensor_arrays()[0]
    for v in fd:
        t = 1 - (v * 100) / 13100
        assert (1 - v * 100 / 13100) ** 2 == t * t          # simulation.py:76: pow(x, 2) == x*x for these values


def _header_decl(name):
    """(return type, [parameter declarations]) of `name` in include/lidar_snow_sim.h"""
    txt = open(os.path.join(ROOT, 'include', 'lidar_snow_sim.h')).read()
    m = re.search(r'LSS_API\s+([^;(]*?)\b' + name + r'\s*\(([^;]*?)\)\s*;', txt, re.S)
    assert m, name
    return m.group(1).strip(), [p.strip() for p in m.group(2).split(',') if p.strip()]


def _header_params(name):
    return _header_decl(name)[1]


_CTYPES = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'uint32_t': ctypes.c_uint32, 'uint64_t': ctypes.c_uint64,
           'double': ctypes.c_double, 'lss_status': ctypes.c_int}


def _binds(c_type, bound):
    """whether the ctypes type `bound` is the binding of C type `c_type` (a declaration without its name)"""
    words = c_type.replace('*', ' * ').replace('const', ' ').split()
    if words == ['void']:
        return bound is None
    if words == ['char', '*']:
        return bound is ctypes.c_char_p
    if '*' in words:
        return bound is ctypes.c_void_p or (isinstance(bound, type) and issubclass(bound, ctypes._Pointer))
    return len(words) == 1 and bound is _CTYPES.get(words[0])


def _call_args(text, call):
    """Arguments of the first `call(...)` in text (nesting aware, comments stripped)."""
    i = text.index(call + '(') + len(call) + 1
    depth, args, cur = 1, [], ''
    body = re.sub(r'#[^\n]*|/\*.*?\*/', '', text[i:], flags=re.S)
    for ch in body:
        if ch in '([':
            depth += 1
        elif ch in ')]':
            depth -= 1
            if depth == 0:
                break
        if ch == ',' and depth == 1:
            args.append(cur.strip())
            cur = ''
        else:
            cur += ch
    args.append(cur.strip())
    return [a for a in args if a]


def test_signatures_and_documented_calls_have_the_header_arity():
    """ctypes restypes and argtypes and the raw C-ABI examples of INTEGRATION.md follow the header's declarations: the
    same number of parameters, each bound as its C type (int c_int, int64_t c_int64, a pointer c_void_p or POINTER)."""
    from lidar_snow_sim_b200 import _lib
    for name, restype, argtypes in _lib.SIGNATURES:
        ret, params = _header_decl(name)
        params = [] if params == ['void'] else params
        assert len(params) == len(argtypes), f'{name}: header has {len(params)} parameters, _lib.SIGNATURES {len(argtypes)}'
        assert _binds(ret, restype), f'{name}: returns {ret}, bound as {restype}'
        for k, (p, a) in enumerate(zip(params, argtypes)):
            c_type = re.sub(r'\b\w+$', '', p)                          # without the parameter's name
            assert _binds(c_type, a), f'{name}: parameter {k} is {p!r}, bound as {a}'
    doc = open(os.path.join(ROOT, 'INTEGRATION.md')).read()
    for call, name in (('L.lss_snowfall_batch', 'lss_snowfall_batch'),
                       ('\nlss_snowfall_batch_host_submit', 'lss_snowfall_batch_host_submit')):
        assert len(_call_args(doc, call)) == len(_header_params(name)), f'INTEGRATION.md: {name} example is out of date'

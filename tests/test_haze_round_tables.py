"""The rounding tables of the device's correctly rounded float32 tan and log
(lidar_snow_sim_b200/csrc/haze_round_tables.h, tools/make_haze_round_tables.py): sorted unique arguments, every value the correctly rounded result at 256 bits, and a
rescan of the 2^24-argument chunks that hold entries (and of some that hold none) finding exactly those entries."""
import multiprocessing
import os
import re
import sys

import numpy as np
import pytest

from oracle import haze as oh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'lidar_snow_sim_b200', 'csrc', 'haze_round_tables.h')


def round_tables():
    """{'tan': (arg bits uint32, value bits uint32), 'log': ...} as the header holds them"""
    txt = open(HEADER).read()
    out = {}
    for fn in ('tan', 'log'):
        n = int(re.search(rf'HAZE_{fn.upper()}_N = (\d+);', txt).group(1))
        arrs = []
        for part in ('arg', 'val'):
            body = re.search(rf'haze_{fn}_{part}\[\d+\] = \{{(.*?)\}};', txt, re.S).group(1)
            arrs.append(np.array([int(v, 16) for v in re.findall(r'0x([0-9a-f]{8})u', body)], np.uint32))
        assert arrs[0].size == arrs[1].size == n
        out[fn] = tuple(arrs)
    return out


def _tool():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_haze_round_tables
    return make_haze_round_tables


@pytest.mark.parametrize('fn', ['tan', 'log'])
def test_tables_are_sorted_unique_positive_finite(fn):
    arg, val = round_tables()[fn]
    assert arg.size > 100
    assert np.all(np.diff(arg.astype(np.int64)) > 0)
    assert arg[0] >= 1 and arg[-1] < 0x7f800000
    assert np.all(np.isfinite(val.view(np.float32)))


@pytest.mark.parametrize('fn', ['tan', 'log'])
def test_table_values_are_correctly_rounded_at_256_bits(fn):
    import mpmath
    arg, val = round_tables()[fn]
    mfn = mpmath.tan if fn == 'tan' else mpmath.log
    want = np.array([oh._mp_round(mfn, x) for x in arg.view(np.float32)], np.float32)
    assert np.array_equal(val, want.view(np.uint32))
    # and every entry is a hard case: float64 rounded once is within 2^-23 float32 spacings of the boundary
    with np.errstate(all='ignore'):
        t = (np.tan if fn == 'tan' else np.log)(arg.view(np.float32).astype(np.float64))
    assert np.all(oh.boundary_distance(t) < 2.0 ** -23)


def test_rescan_finds_exactly_the_entries():
    tool = _tool()
    tables = round_tables()
    jobs = []
    for fn, (arg, _) in tables.items():
        held = sorted(set((arg >> 24).tolist()))
        empty = [c for c in range(128) if c not in held][:3]
        jobs += [(fn, c << 24) for c in held + empty]
    ctx = multiprocessing.get_context('spawn')
    with ctx.Pool(min(8, os.cpu_count() or 1)) as pool:
        found = pool.map(tool.scan, jobs)
    for (fn, start), bits in zip(jobs, found):
        arg = tables[fn][0]
        want = arg[(arg >= start) & (arg < start + tool.CHUNK)]
        assert np.array_equal(bits, want), (fn, hex(start))

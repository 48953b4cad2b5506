"""CPU test: the solve kernel's phase-clock hook is declared in the header with the arity its binding uses."""
import os
import re

from lidar_snow_sim_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'lidar_snow_sim.h')


def test_debug_solve_phases_declared_with_its_arity():
    text = open(HEADER).read()
    m = re.search(r'lss_status\s+lss_debug_solve_phases\s*\(([^)]*)\)\s*;', text)
    assert m, 'lss_debug_solve_phases is not declared in include/lidar_snow_sim.h'
    params = [p.strip() for p in m.group(1).split(',')]
    assert params == ['lss_engine *e', 'int reset', 'uint64_t *h_out', 'int n']
    sig = {name: args for name, _, args in _lib.SIGNATURES}
    assert len(sig['lss_debug_solve_phases']) == len(params)
    words = re.search(r'#define\s+LSS_DEBUG_SOLVE_PHASE_WORDS\s+(\d+)', text)
    assert words and int(words.group(1)) == 7 + 2 + 128      # phases, tiles, warps, listed beams per work class

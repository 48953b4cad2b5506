"""
The oracle of estimation_method='poly' (tests/wet_poly_oracle.py) against tests/golden/wet_poly.npz, which the
unmodified reference wrote: on the fixture's plane, picks and post-plane NumPy state, the same rows, intensities and
final state, bit for bit; and the passthrough cases raise or return as the reference did, drawing nothing.
"""
import os
import warnings

import numpy as np
import pytest

import wet_poly_oracle
from wet_poly_cases import CASES, sha

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wet_poly.npz')


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_equals_fixture(name):
    g = np.load(GOLD)
    build, kw, seed = CASES[name]
    pc = build()
    code = int(g[f'{name}__code'])
    if 'plane_w' in [k.split('__')[1] for k in g.files if k.startswith(name + '__')]:
        np.random.set_state(('MT19937', g[f'{name}__state_key'], int(g[f'{name}__state_pos'])))
        plane = (g[f'{name}__plane_w'], float(g[f'{name}__plane_h']))
    else:
        np.random.seed(seed)
        plane = None
    picks = g[f'{name}__ymins'] if f'{name}__ymins' in g.files else 'first_min'
    before = np.random.get_state()
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        if code == 2:
            with pytest.raises(ValueError):
                wet_poly_oracle.ground_water_augmentation(pc, plane=plane, **kw)
        elif code == 3:
            with pytest.raises(TypeError):
                wet_poly_oracle.ground_water_augmentation(pc, plane=plane, least_populated=picks, **kw)
        else:
            out = wet_poly_oracle.ground_water_augmentation(pc, plane=plane, least_populated=picks, **kw)
    fin = np.random.get_state()
    if code in (2, 3):
        assert np.array_equal(fin[1], before[1]) and fin[2] == before[2]       # nothing drawn
        return
    if code == 1:
        assert out is pc
        return
    n_non = int(g[f'{name}__out_n_non'])
    assert tuple(out.shape) == tuple(g[f'{name}__out_shape'])
    assert sha(np.concatenate([out[:, [0, 1, 2, 4]].ravel(), out[:n_non, 3]])) == str(g[f'{name}__out_sha'])
    assert np.array_equal(out[n_non:, 3], g[f'{name}__out_i'])
    assert np.array_equal(fin[1], g[f'{name}__final_key']) and fin[2] == int(g[f'{name}__final_pos'])

"""
NumPy restatement of the robustness test sets' device side (csrc/pa_aug.cu): k_pa_fps_cluster / k_pa_fps over a whole
cloud (KITTI-S) and k_jit_rows (KITTI-J), and the fixture's cases (tests/golden/pa_robust.npz,
tools/make_golden_pa_robust.py).
"""
import contextlib
import io
import os

import numpy as np

import legacy_gauss_model as LG

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'pa_robust.npz')
CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']


def load():
    g = np.load(GOLDEN)
    return [{f[len(f'c{k}_'):]: g[f] for f in g.files if f.startswith(f'c{k}_')} for k in range(int(g['n_cases']))]


def names(boxes):
    return np.asarray([CLASS_NAMES[int(v) - 1] for v in boxes[:, -1]]) if boxes.shape[0] else np.zeros(0, '<U10')


def start_state(c):
    """NumPy's global state as the fixture's case started"""
    np.random.seed(int(c['seed']))
    if int(c['mode']) == 1:
        np.random.normal()
    elif int(c['mode']) == 624:
        st = np.random.get_state()
        np.random.set_state((st[0], st[1], 624, 0, 0.0))


def same_state(c):
    _, keys, pos, has, g = np.random.get_state()
    return (np.array_equal(keys, c['st_key']) and pos == int(c['st_pos']) and has == int(c['st_has_gauss'])
            and (not has or g == float(c['st_gauss'])))


def fps_index(xyz, K, start):
    """the picks of farthest_point_sampling on float32 or float64 xyz rows: float64 distances ((dx^2 + dy^2) + dz^2)
    from the widened pick, np.minimum's NaN, np.argmax's first NaN or first maximum"""
    p = xyz.astype(np.float64)

    def dist(q):
        return ((q[0] - p[:, 0]) ** 2 + (q[1] - p[:, 1]) ** 2) + (q[2] - p[:, 2]) ** 2
    idx = [int(start)]
    d = dist(p[start])
    for _ in range(1, K):
        k = int(np.argmax(d))
        idx.append(k)
        d = np.minimum(d, dist(p[k]))
    return np.array(idx, np.int64)


def jitter(rows, gauss, sigma):
    """k_jit_rows: x, y, z = float(double(x) + (0 + sigma g)) in the rows' dtype, g the cloud's Gaussians row-major"""
    out = rows.copy()
    n = 0.0 + sigma * gauss.reshape(-1, 3)
    out[:, :3] = (rows[:, :3].astype(np.float64) + n).astype(rows.dtype)
    return out


def captured(fn, *a, **k):
    """(result or exception, stdout) of fn(*a, **k)"""
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        try:
            r = fn(*a, **k)
        except Exception as ex:                                    # noqa: BLE001
            r = ex
    return r, buf.getvalue()

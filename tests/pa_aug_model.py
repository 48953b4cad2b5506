"""
NumPy restatement of the device side of PA-AUG, in the kernels' operation order: the partition test (k_pa_count /
k_pa_scatter of csrc/pa_aug.cu) and the execution of a plan from lidar_snow_sim_b200.pa_aug.plan (k_pa_emit, k_pa_fps).
Together with the planner it must reproduce the reference's rows bit for bit (tests/test_pa_aug_cpu.py).
"""
import numpy as np

from lidar_snow_sim_b200.pa_aug.plan import OP_ADD, OP_DIV, OP_JIT, OP_MUL, OP_ROT, OP_SUB, MAX_PARTS


def _inside(p, planes, dt):
    """rows of p (N, 3) float32 inside the polyhedron of planes (6, 4): sign = ((x n0 + y n1) + z n2) + d in dt,
    outside as soon as one sign >= 0 (a NaN sign is never >= 0)"""
    x, y, z = (p[:, k].astype(dt) for k in range(3))
    ins = np.ones(p.shape[0], bool)
    for n0, n1, n2, d in planes.astype(dt):
        s = ((x * n0 + y * n1) + z * n2) + d
        ins &= ~(s >= 0)
    return ins


def partition(points, planes, n_parts, boxes_f64):
    """-> members: list over boxes of lists over parts of row indices (row order), bg row indices"""
    dt = np.float64 if boxes_f64 else np.float32
    p = points[:, :3]
    any_box = np.zeros(p.shape[0], bool)
    members = []
    for i in range(planes.shape[0]):
        ib = _inside(p, planes[i, 0], dt)
        any_box |= ib
        members.append([np.nonzero(ib & _inside(p, planes[i, 1 + j], dt))[0] for j in range(n_parts[i])])
    return members, np.nonzero(~any_box)[0]


def counts_of(members):
    c = np.zeros((len(members), MAX_PARTS), np.int64)
    for i, m in enumerate(members):
        for j, r in enumerate(m):
            c[i, j] = len(r)
    return c


def _step(v, op, c64, s64, prm, normals, local):
    dt = np.float64 if c64 else np.float32
    a = v.astype(dt)
    q = np.asarray(prm, np.float64).astype(dt)
    if op == OP_JIT:
        nr = normals[int(prm[0]) + local]
        r = a + nr.astype(dt)
    else:
        r = a.copy()
        if op == OP_ROT:
            R = q.reshape(3, 3)
            for k in range(3):
                r[:, k] = (a[:, 0] * R[0, k] + a[:, 1] * R[1, k]) + a[:, 2] * R[2, k]
        else:
            f = {OP_SUB: np.subtract, OP_ADD: np.add, OP_MUL: np.multiply, OP_DIV: np.divide}[op]
            for k in range(3):
                r[:, k] = f(a[:, k], q[k])
    if not s64:
        r = r.astype(np.float32)
    return r.astype(np.float64)


def _segment(seg, points, members, bg, plan, fps_rows):
    kind, ref, n, steps = seg
    if kind == 'src':
        v = points[members[ref[0]][ref[1]], :4].astype(np.float64)
    elif kind == 'bg':
        v = points[bg, :4].astype(np.float64)
    elif kind == 'fps':
        v = fps_rows[ref]
    else:
        v = plan['noise'][ref:ref + n]
    assert v.shape[0] == n
    local = np.arange(n)
    for op, c64, s64, prm in steps:
        v = _step(v, op, c64, s64, prm, plan['normals'], local)
    return v


def fps(rows, K, start):
    """farthest_point_sampling on rows[:, :3]: float64 distances ((dx^2 + dy^2) + dz^2), np.argmax (first index of the
    maximum, a NaN first) and np.minimum (NaN propagates)"""
    p = rows[:, :3]

    def dist(q):
        return ((q[0] - p[:, 0]) ** 2 + (q[1] - p[:, 1]) ** 2) + (q[2] - p[:, 2]) ** 2
    idx = [start]
    d = dist(p[start])
    for _ in range(1, K):
        k = int(np.argmax(d))
        idx.append(k)
        d = np.minimum(d, dist(p[k]))
    return rows[idx]


def execute(plan, points, members, bg):
    """the cloud's output rows, float64 (N', 4)"""
    fps_rows = []
    for segs, n, K, start, _ in plan['fps']:
        rows = np.concatenate([_segment(s, points, members, bg, plan, None) for s in segs])
        assert rows.shape[0] == n
        fps_rows.append(fps(rows, K, start))
    out = [_segment(s, points, members, bg, plan, fps_rows) for segs in plan['parts'] for s in segs]
    out.append(_segment(plan['bg'], points, members, bg, plan, fps_rows))
    res = np.concatenate(out) if out else np.zeros((0, 4))
    assert res.shape[0] == plan['n_out']
    return res

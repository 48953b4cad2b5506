"""
Host side of PA-AUG (lib/pa_aug/part_aware_augmentation.py): the parameter parser, the box and part planes the
partition kernel tests against, and the planner.

Every random draw of the reference depends only on how many rows each (box, part) holds and on the boxes, never on
the rows' values.  So once the partition kernel's member counts are on the host, `plan_cloud` replays dropout ->
remove_empty_gt_boxes -> swap -> mix -> sparse -> jitter -> noise on counts alone, making NumPy's global RandomState
calls of the reference in its order and with its sizes, and writes down what the device must do to the rows:

  a part's content is an ordered list of segments; a segment is
    ('src', (box, part)) the part's original member rows, or ('bg', None) the rows in no box,
    ('fps', job)         the rows farthest-point sampling job `job` selected, or
    ('noise', offset)    rows the host generated (their arithmetic has no row input, so it is done here, in NumPy),
  plus the chain of steps the rows went through.  A step is (op, compute in float64, store in float64, 9 params):
  SUB / ADD / MUL / DIV by a box's 3-vector, ROT by rotation_3d_in_axis's matrix (out_k = (p0 R0k + p1 R1k) + p2 R2k),
  JIT (+ host-drawn normals, all four columns, params[0] = offset of the segment's first normal row).

A part array's dtype is followed as the reference changes it: np.zeros((0, 4)) after dropout is float64, np.concatenate
promotes, in-place += / -= / *= / /= keep it.  An in-place op computes in the promotion of the array's and the
operand's dtype and rounds to the array's dtype: that is each step's (compute, store) pair.
"""
import numpy as np

NUM_PARTITION = {'Car': 8, 'Pedestrian': 4, 'Cyclist': 4}
MAX_PARTS = 8
OP_SUB, OP_ADD, OP_MUL, OP_DIV, OP_ROT, OP_JIT = 1, 2, 3, 4, 5, 6

# the eight corners of every part, as keys of the box's corners and edge/face/diagonal midpoints
# (get_partition_corners; 'ab' is (corner a + corner b) / 2)
PARTITION_KEYS = {
    'Car': [['0', '01', '02', '03', '04', '05', '06', '07'], ['01', '1', '12', '02', '05', '15', '16', '06'],
            ['02', '12', '2', '23', '06', '16', '26', '27'], ['03', '02', '23', '3', '07', '06', '27', '37'],
            ['04', '05', '06', '07', '4', '45', '46', '47'], ['05', '15', '16', '06', '45', '5', '56', '46'],
            ['06', '16', '26', '27', '46', '56', '6', '67'], ['07', '06', '27', '37', '47', '46', '67', '7']],
    'Pedestrian': [['0', '01', '23', '3', '04', '05', '27', '37'], ['01', '1', '2', '23', '05', '15', '26', '27'],
                   ['05', '15', '26', '27', '45', '5', '6', '67'], ['04', '05', '27', '37', '4', '45', '67', '7']],
    'Cyclist': [['0', '01', '02', '03', '4', '45', '46', '47'], ['01', '1', '12', '02', '45', '5', '56', '46'],
                ['02', '12', '2', '23', '46', '56', '6', '67'], ['03', '02', '23', '3', '47', '46', '67', '7']],
}
MIDPOINTS = ['01', '02', '03', '04', '05', '06', '07', '12', '15', '16', '23', '26', '27', '37', '45', '46', '47', '56',
             '67']
# corner_to_surfaces_3d: the four corners of each of the six faces, normals pointing inwards
SURFACES = [[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]]


def interpret_pa_aug_param(pa_aug_param):
    """PartAwareAugmentation.interpret_pa_aug_param token for token: a method token in last place raises IndexError
    at param_list[i + 1], 'p' values of other than 2 or 3 digits are ignored, jitter<digits> is digits / 10 **
    (len - 1), distance<n> takes no probability, a method matches once (later tokens of it are ignored)."""
    d = {}
    method_list = ['dropout', 'sparse', 'noise', 'swap', 'mix', 'jitter', 'random', 'distance']
    for method in method_list:
        if method == 'distance':
            d[method] = 100
        elif method == 'random':
            d[method] = False
        else:
            d[method] = 0
            d[method + '_p'] = 0
    if pa_aug_param is None:
        return d
    tokens = pa_aug_param.split('_')
    for i, tok in enumerate(tokens):
        if tok.startswith('p'):
            continue
        for method in list(method_list):
            if not tok.startswith(method):
                continue
            if method == 'random':
                d[method] = True
                method_list.remove(method)
                break
            number = tok.replace(method, '')
            if len(number) == 0:
                d[method] = 0.1 if method == 'jitter' else 1
            else:
                d[method] = float(number) / 10 ** (len(number) - 1) if method == 'jitter' else int(number)
            if method == 'distance':
                method_list.remove(method)
                break
            d[method + '_p'] = 1.0
            nxt = tokens[i + 1]                                    # IndexError for a method token in last place
            if nxt.startswith('p'):
                number = nxt.replace('p', '')
                if len(number) == 2:
                    d[method + '_p'] = float(number) / 10.0
                elif len(number) == 3:
                    d[method + '_p'] = float(number) / 100.0
            method_list.remove(method)
            break
    return d


# ---------------------------------------------------------------------------------------------------------------- geometry
def _rot_mat_t(angles):
    """rotation_3d_in_axis's rot_mat_T for axis 2: (3, 3, n) in the angles' dtype"""
    s, c = np.sin(angles), np.cos(angles)
    one, zero = np.ones_like(c), np.zeros_like(c)
    return np.stack([[c, -s, zero], [s, c, zero], [zero, zero, one]])


def _rotate(points, angles):
    if points.ndim == 2:
        points = points[None]
    return np.einsum('aij,jka->aik', points, _rot_mat_t(angles))


def _corners(dims):
    """corners_nd(dims, origin=0.5) for 3-D boxes, in dims' dtype"""
    norm = np.stack(np.unravel_index(np.arange(8), [2] * 3), axis=1).astype(dims.dtype)[[0, 1, 3, 2, 4, 5, 7, 6]]
    norm = norm - np.array((0.5, 0.5, 0.5), dtype=dims.dtype)
    return dims.reshape([-1, 1, 3]) * norm.reshape([1, 8, 3])


def box_corners(gt_boxes):
    """center_to_corner_box3d(boxes[:, :3], boxes[:, 3:6], boxes[:, 6], origin=(0.5, 0.5, 0.5), axis=2)"""
    c = _rotate(_corners(gt_boxes[:, 3:6]), gt_boxes[:, 6])
    c += gt_boxes[:, :3].reshape([-1, 1, 3])
    return c


# the 27 points of augment_box_corners, in this order: the eight corners, then the midpoints
AUG_KEYS = [str(i) for i in range(8)] + MIDPOINTS
PART_INDEX = {name: np.array([[AUG_KEYS.index(k) for k in part] for part in parts])
              for name, parts in PARTITION_KEYS.items()}


def _augmented(corners):
    """augment_box_corners for (..., 8, 3) corners: (..., 27, 3), midpoint 'ab' = (corner a + corner b) / 2"""
    mids = [(corners[..., int(k[0]), :] + corners[..., int(k[1]), :]) / 2 for k in MIDPOINTS]
    return np.concatenate([corners] + [m[..., None, :] for m in mids], axis=-2)


def partition_corners(corners, name, j):
    """get_partition_corners: the (8, 3) corners of part j of a box with (8, 3) corners"""
    return _augmented(corners)[PART_INDEX[name][j]]


def _planes(corners):
    """corner_to_surfaces_3d + surface_equ_3d_jitv2 for (..., 8, 3) polyhedra: (..., 6, 4) = normal, d in their
    dtype, element by element in the reference's operation order"""
    s = corners[..., np.array(SURFACES), :]                       # (..., 6, 4, 3)
    sv0 = s[..., 0, :] - s[..., 1, :]
    sv1 = s[..., 1, :] - s[..., 2, :]
    n = np.stack([sv0[..., 1] * sv1[..., 2] - sv0[..., 2] * sv1[..., 1],
                  sv0[..., 2] * sv1[..., 0] - sv0[..., 0] * sv1[..., 2],
                  sv0[..., 0] * sv1[..., 1] - sv0[..., 1] * sv1[..., 0]], axis=-1)
    d = -s[..., 0, 0] * n[..., 0] - s[..., 0, 1] * n[..., 1] - s[..., 0, 2] * n[..., 2]
    return np.concatenate([n, d[..., None]], axis=-1)


def box_planes(gt_boxes, gt_names):
    """(M, 1 + MAX_PARTS, 6, 4) float64: each box's six face planes, then its parts' (zeros past its part count).
    Values are computed in the boxes' dtype, as the reference does; float64 holds float32 values exactly."""
    M = gt_boxes.shape[0]
    out = np.zeros((M, 1 + MAX_PARTS, 6, 4), np.float64)
    if M == 0:
        return out
    corners = box_corners(gt_boxes)
    out[:, 0] = _planes(corners)
    aug = _augmented(corners)
    names = np.asarray(gt_names)
    for name, idx in PART_INDEX.items():
        sel = names == name
        if sel.any():
            out[sel, 1:1 + idx.shape[0]] = _planes(aug[sel][:, idx])
    return out


# ----------------------------------------------------------------------------------------------------------------- planner
class _Part:
    """one entry of separated_box_points: segments [kind, ref, n, steps], the rows, the dtype (True: float64) and
    the columns (the cloud's F, or 4 for the np.zeros((0, 4)) of dropout)"""
    __slots__ = ('segs', 'n', 'f64', 'cols')

    def __init__(self, segs, n, f64, cols):
        self.segs, self.n, self.f64, self.cols = segs, n, f64, cols


def _concat_cols(a, b):
    if a != b:                                                     # np.concatenate / np.vstack of (., a) and (., b)
        raise ValueError(f'all the input array dimensions except for the concatenation axis must match exactly, '
                         f'but along dimension 1, the array at index 0 has size {a} and the array at index 1 has '
                         f'size {b}')
    return a


def _transformed(part, box_t, box_c, f64_boxes):
    """swap / mix: np.copy(target part), then -= centre_t, rotate by -angle_t, /= dim_t, *= dim_c, rotate by angle_c,
    += centre_c, each in place on the copy (columns 0..2)"""
    c64 = part.f64 or f64_boxes
    s64 = part.f64
    vec = lambda v: tuple(float(x) for x in v) + (0.0,) * 6   # noqa: E731
    rot = lambda a: tuple(float(x) for x in _rot_mat_t(a)[:, :, 0].reshape(-1))   # noqa: E731
    steps = [(OP_SUB, c64, s64, vec(box_t[:3])), (OP_ROT, c64, s64, rot(-box_t[6:7])),
             (OP_DIV, c64, s64, vec(box_t[3:6])), (OP_MUL, c64, s64, vec(box_c[3:6])),
             (OP_ROT, c64, s64, rot(box_c[6:7])), (OP_ADD, c64, s64, vec(box_c[:3]))]
    return _Part([[k, r, n, st + steps] for k, r, n, st in part.segs], part.n, part.f64, part.cols)


def _noise_rows(box, name, j, num):
    """generate_random_noise's rows for part j of `box`: four uniform draws, then rotated and shifted (float64)"""
    center = np.expand_dims(box[:3], axis=0)
    corners = np.squeeze(_corners(np.expand_dims(box[3:6], axis=0)), axis=0)
    pc = partition_corners(corners, name, j)
    lo, hi = pc.min(axis=0), pc.max(axis=0)
    g = np.zeros((1, num, 4))
    g[0, :, 0] = np.random.uniform(low=lo[0], high=hi[0], size=(num,))
    g[0, :, 1] = np.random.uniform(low=lo[1], high=hi[1], size=(num,))
    g[0, :, 2] = np.random.uniform(low=lo[2], high=hi[2], size=(num,))
    g[0, :, 3] = np.random.uniform(low=0.0, high=1.0, size=(num,))
    g[:, :, :3] = _rotate(g[:, :, :3], box[6:7])
    g[:, :, :3] += center.reshape([-1, 1, 3])
    return g[0]


def _pick_target(parts, i, gt_names, num_classes):
    """swap_partitions / mix_partitions: the target box (of the same class unless there is one class name) and a part
    non-empty in both, by the reference's draws; (-1, -1) when there is none"""
    idxes = list(range(len(gt_names)))
    if num_classes > 1:
        same = gt_names == gt_names[i]
        same[i] = False
        idxes = [k for k, m in zip(idxes, same) if m]
    else:
        idxes.remove(i)
    while len(idxes) > 0:
        t = np.random.choice(idxes, 1, replace=False)[0]
        cand = [k for k, p in enumerate(parts[i]) if p.n != 0]
        while len(cand) > 0:
            c = np.random.choice(cand, 1, replace=False)[0]
            if parts[t][c].n != 0:
                return t, c
            cand.remove(c)
        idxes.remove(t)
    return -1, -1


def plan_cloud(counts, n_bg, gt_boxes, gt_names, num_classes, param, n_features=4, points_f64=False):
    """
    Replay PartAwareAugmentation(points, gt_boxes, gt_names, class_names).augment(param) on member counts.
    counts: (M, MAX_PARTS) rows of every (box, part); n_bg: rows in no box.  Draws from NumPy's global RandomState.
    Returns dict(parts: output parts in order, each a list of segments [kind, ref, n, steps]; bg segment;
    fps: jobs [segments, n, K, start, f64]; noise (R, 4) float64; normals (Q, 4) float64; mask: list of bool;
    n_out).  The exceptions are the reference's (IndexError from the parser, ...), raised after the same draws.
    """
    p = interpret_pa_aug_param(param)
    gt_names = np.asarray(gt_names)
    f64_boxes = gt_boxes.dtype == np.float64
    M = gt_boxes.shape[0]
    F = n_features
    parts = [[_Part([['src', (i, j), int(counts[i][j]), []]], int(counts[i][j]), points_f64, F)
              for j in range(NUM_PARTITION[gt_names[i]])] for i in range(M)]
    mask = [True] * M
    boxes, names = gt_boxes, gt_names
    dist = p['distance']

    if p['dropout'] > 0:
        for i in range(M):
            if boxes[i][0] > dist or np.random.rand(1) > p['dropout_p']:
                continue
            for j in np.random.choice(range(NUM_PARTITION[names[i]]), p['dropout'], replace=False):
                parts[i][j] = _Part([], 0, True, 4)                # np.zeros((0, 4))
        for i in range(M):
            if all(q.n == 0 for q in parts[i]):
                mask[i] = False
        boxes, names = boxes[mask], names[mask]
        parts = [q for q, s in zip(parts, mask) if s]

    for method in ('swap', 'mix'):
        if p[method] <= 0:
            continue
        for i in range(len(boxes)):
            if boxes[i][0] > dist or np.random.rand(1) > p[method + '_p']:
                continue
            t, c = _pick_target(parts, i, names, num_classes)
            if c == -1:
                continue
            moved = _transformed(parts[t][c], boxes[t], boxes[i], f64_boxes)
            if method == 'swap':
                parts[i][c] = moved
            else:
                cur = parts[i][c]
                parts[i][c] = _Part(cur.segs + moved.segs, cur.n + moved.n, cur.f64 or moved.f64,
                                    _concat_cols(cur.cols, moved.cols))

    fps = []
    if p['sparse'] > 0:
        K = p['sparse']
        for i in range(len(boxes)):
            if boxes[i][0] > dist:
                continue
            for j in range(NUM_PARTITION[names[i]]):
                q = parts[i][j]
                if q.n > K:
                    if np.random.rand(1) > p['sparse_p']:
                        continue
                    start = np.random.randint(q.n)
                    fps.append([q.segs, q.n, K, int(start), q.f64])
                    parts[i][j] = _Part([['fps', len(fps) - 1, K, []]], K, q.f64, q.cols)

    normals = []
    n_normals = 0
    for i in range(len(boxes)):
        if boxes[i][0] > dist:
            continue
        for j in range(NUM_PARTITION[names[i]]):
            q = parts[i][j]
            if q.n <= 0 or np.random.rand(1) > p['jitter_p']:
                continue
            normals.append(np.random.normal(0, p['jitter'], size=(q.n, q.cols)))
            segs, off = [], n_normals
            for k, r, n, st in q.segs:
                segs.append([k, r, n, st + [(OP_JIT, True, q.f64, (float(off),) + (0.0,) * 8)]])
                off += n
            n_normals += q.n
            parts[i][j] = _Part(segs, q.n, q.f64, q.cols)

    noise = []
    n_noise = 0
    if p['noise'] > 0:
        num = p['noise']
        for i in range(len(boxes)):
            if boxes[i][0] > dist:
                continue
            for j in range(NUM_PARTITION[names[i]]):
                if np.random.rand(1) > p['noise_p']:
                    continue
                rows = _noise_rows(boxes[i], names[i], j, num)
                q = parts[i][j]
                _concat_cols(q.cols, 4)
                noise.append(rows)
                parts[i][j] = _Part(q.segs + [['noise', n_noise, num, []]], q.n + num, True, 4)
                n_noise += num

    for i in range(len(boxes)):                                    # stack_fg_points: np.vstack onto np.zeros((0, 4))
        for j in range(NUM_PARTITION[names[i]]):
            _concat_cols(4, parts[i][j].cols)
    _concat_cols(4, F)                                             # np.vstack((fg_points, bg_points))
    out_parts = [parts[i][j].segs for i in range(len(boxes)) for j in range(NUM_PARTITION[names[i]])]
    n_out = sum(parts[i][j].n for i in range(len(boxes)) for j in range(NUM_PARTITION[names[i]])) + int(n_bg)
    return dict(parts=out_parts, bg=['bg', None, int(n_bg), []], fps=fps,
                noise=np.concatenate(noise) if noise else np.zeros((0, 4)),
                normals=np.concatenate(normals) if normals else np.zeros((0, 4)), mask=mask, n_out=n_out)


# ------------------------------------------------------------------------------------------------ robustness test sets
def partition_corners_list(gt_boxes, gt_names):
    """the constructor's partition_corners: per box a float64 (parts, 8, 3) array, the parts' corners in the boxes'
    dtype (assign_box_points_partition)"""
    corners = box_corners(gt_boxes) if gt_boxes.shape[0] else np.zeros((0, 8, 3))
    out = []
    for i, name in enumerate(np.asarray(gt_names)):
        pc = np.zeros((NUM_PARTITION[name], 8, 3))
        for j in range(NUM_PARTITION[name]):
            pc[j] = partition_corners(corners[i], name, j)
        out.append(pc)
    return out


class RobustState:
    """The state create_robusteness_test_data('KITTI-D') reads and changes, on member counts: the boxes and names left,
    gt_boxes_mask, aug_flag and, per box left, its parts as [input box, part, rows, dropped]."""

    def __init__(self, gt_boxes, gt_names):
        self.gt_boxes = gt_boxes
        self.gt_names = np.asarray(gt_names)
        self.num_gt_boxes = gt_boxes.shape[0]
        self.gt_boxes_mask = [True] * self.num_gt_boxes
        self.aug_flag = np.zeros((self.num_gt_boxes, 8, 6), dtype=bool)
        self.parts = None

    def dropout_test(self, counts, n_features):
        """dropout_partitions(num_dropout_partition=1, p=1.0, robustness_test=True), stack_fg_points and the vstack with
        the background: per box within distance one rand(1) draw, the last fullest part dropped and its count printed,
        then remove_empty_gt_boxes.  Returns the output's member segments [(input box, part, rows)] before the
        background; raises the reference's ValueError for rows of other than four columns after the draws.
        counts: (M, MAX_PARTS) member counts of the constructor's boxes, read by the first call only."""
        if self.parts is None:
            self.parts = [[[i, j, int(counts[i][j]), False] for j in range(NUM_PARTITION[n])]
                          for i, n in enumerate(self.gt_names)]
        for i in range(self.num_gt_boxes):
            if self.gt_boxes[i][0] > 100:
                continue
            if np.random.rand(1) > 1.0:
                continue
            max_num_points = 0
            for j, q in enumerate(self.parts[i]):
                n = 0 if q[3] else q[2]
                if n >= max_num_points:
                    max_num_points = n
                    idx = j
            print(max_num_points)
            self.parts[i][idx][3] = True
            self.aug_flag[i, idx, 0] = True
        for i in range(self.num_gt_boxes):                        # remove_empty_gt_boxes, statement for statement
            if all(q[3] or q[2] == 0 for q in self.parts[i]):
                self.gt_boxes_mask[i] = False
        self.gt_boxes = self.gt_boxes[self.gt_boxes_mask]
        self.gt_names = self.gt_names[self.gt_boxes_mask]
        self.num_gt_boxes = self.gt_boxes.shape[0]
        self.parts = [d for d, s in zip(self.parts, self.gt_boxes_mask) if s]
        self.aug_flag = self.aug_flag[self.gt_boxes_mask]
        for box in self.parts:                                     # np.vstack onto np.zeros((0, 4))
            for q in box:
                if not q[3]:
                    _concat_cols(4, n_features)
        _concat_cols(4, n_features)                                # np.vstack((fg_points, bg_points))
        return [(q[0], q[1], q[2]) for box in self.parts for q in box if not q[3] and q[2] > 0]

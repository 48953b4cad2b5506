"""
SnowfallEngine -- thin host-side owner of one C-ABI engine (one GPU).  PyTorch is used only as the device container
(tensors, streams); all arithmetic happens in liblss_b200.so.

One process per GPU: create one engine per rank; clouds are independent, so a batch shards across ranks with no
data-path collective (see lidar_snow_sim_b200/distributed.py for the gather of the augmented batch).

Every public method checks all of its arguments (ValueError, like the library's LSS_ERR_INVALID_ARG) before it
allocates, touches the device or calls the library: a pointer reaches a kernel only from a tensor that was checked.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib
from .calib.hdl64e_s3 import sensor_arrays

DEFAULT_MAX_DIVERGENCE_RAD = 3e-3          # callers pass beam_divergence = degrees(3e-3) (precompute.py:104)
# sample_tables_device calls the sampler at most this often: the darts per plane start at 1.5x the expected table size
# (+4096) and double after each call that ends short of the occupancy; the last call's failure is raised
SAMPLER_ATTEMPTS = 4
LISA_SEED_STATE = np.random.RandomState(666).get_state()    # np.random.seed(666): LISA's fixed_seed (lisa.py:54-55)
MAX_CLOUDS = 65535                      # clouds per batch call: the kernels' grid y dimension (lss_batch_geometry)
_CPU = torch.device('cpu')


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        return ctypes.c_void_p(t.data_ptr())
    if isinstance(t, np.ndarray):
        return ctypes.c_void_p(t.ctypes.data)
    raise TypeError(type(t))


def _check_n_clouds(B):
    """Raise the library's ValueError for a batch of more than MAX_CLOUDS clouds here, before any workspace query: the
    queries of some entry points can only answer -1 for it."""
    if B > MAX_CLOUDS:
        raise ValueError(f'at most {MAX_CLOUDS} clouds per call, got {B}')


def _row_offsets(offsets, name):
    """(off, B, N): host row offsets as a contiguous int64 array of B + 1 entries, the number of groups and of rows.
    That they start at 0 and never decrease is checked by the library, which names the argument."""
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    if off.ndim != 1 or off.shape[0] == 0:
        raise ValueError(f'{name}: expected a 1-D array of B + 1 row offsets, got shape {off.shape}')
    return off, off.shape[0] - 1, int(off[-1])


def _cloud_offsets(offsets, name='cloud_offsets'):
    """_row_offsets of a batch of clouds: B is at most MAX_CLOUDS"""
    off, B, N = _row_offsets(offsets, name)
    _check_n_clouds(B)
    return off, B, N


def _f32_flags(f32_distance, B):
    """f32_distance (None, or one flag per cloud) as the int32 array of B flags the library reads"""
    if f32_distance is None:
        return None
    f32 = np.ascontiguousarray(f32_distance, dtype=np.int32).reshape(-1)
    if f32.shape[0] != B:
        raise ValueError(f'f32_distance: expected {B} flags, got {f32.shape[0]}')
    return f32


def _check_tensor(name, t, device, dtype, shape=None, min_cols=0, optional=False):
    """
    Raise ValueError unless `t` is a contiguous tensor of `dtype` (or of one of a tuple of dtypes) on `device` (None: on
    any CUDA device, for mappings of another rank's buffers) of shape `shape`, where None matches any size and dimension
    1 has at least min_cols entries.  None passes for an optional argument.
    """
    if t is None and optional:
        return
    dtypes = dtype if isinstance(dtype, tuple) else (dtype,)
    if (isinstance(t, torch.Tensor) and (t.is_cuda if device is None else t.device == device) and t.dtype in dtypes
            and t.is_contiguous()
            and (shape is None or t.shape == shape
                 or (t.dim() == len(shape) and all(w is None or s == w for s, w in zip(t.shape, shape))))
            and (not min_cols or t.shape[1] >= min_cols)):
        return
    dims = [] if shape is None else ['*' if w is None else str(w) for w in shape]
    if min_cols:
        dims[1] = f'n_features >= {min_cols}'
    want = (f'a contiguous {" or ".join(map(str, dtypes))} tensor on {device or "a CUDA device"}'
            + ('' if shape is None else f' of shape ({", ".join(dims)}{"," if len(dims) == 1 else ""})'))
    got = (f'a {"" if t.is_contiguous() else "non-contiguous "}{t.dtype} tensor of shape {tuple(t.shape)} on {t.device}'
           if isinstance(t, torch.Tensor) else type(t).__name__)
    raise ValueError(f'{name}: expected {want}, got {got}')


def _outputs(out, device, **spec):
    """`out` (None, or the dict a previous call returned, to reuse its buffers) with a buffer for every key of spec whose
    value (shape, dtype) is not false: the buffers out has are checked, then the missing ones allocated (pinned on the
    host)."""
    out = {} if out is None else out
    for k, v in spec.items():
        if v and k in out:
            _check_tensor(f"out['{k}']", out[k], device, v[1], v[0])
    for k, v in spec.items():
        if v and k not in out:
            t = torch.empty(v[0], dtype=v[1], device=device)
            out[k] = t.pin_memory() if device == _CPU else t
    return out


# the kind word [625] of a 630-word state record (gauss=True): no cached Gaussian; the cached Gaussian in the float64 at
# [626]; the cached Gaussian sqrt(-2 log r2 / r2) x1 of the float64s x1, r2 at [626], [628]; the start state's
_GAUSS_NONE, _GAUSS_VALUE, _GAUSS_X1_R2, _GAUSS_AS_START = 0, 1, 2, 3
MT_GAUSS_WORDS = 630


def _mt_words(state, name, gauss=False):
    """The 625 uint32 words the library reads of an np.random.get_state() tuple: the 624 key words, then pos.  Raises
    ValueError, naming the state `name`, for another generator or a pos outside [0, 624].  With `gauss`, the 630-word
    record of the entry points that draw Gaussians: then has_gauss (0 or 1) and the cached Gaussian as a float64 follow."""
    if state[0] != 'MT19937':
        raise ValueError(f'{name} is {state[0]}, not MT19937')
    if not 0 <= int(state[2]) <= 624:
        raise ValueError(f'{name}: expected an MT19937 np.random.get_state() tuple with pos in [0, 624], got pos '
                         f'{state[2]}')
    words = np.zeros(MT_GAUSS_WORDS if gauss else 625, np.uint32)
    words[:624] = np.asarray(state[1], dtype=np.uint32)
    words[624] = int(state[2])
    if gauss:
        if int(state[3]) not in (0, 1):
            raise ValueError(f'{name}: has_gauss must be 0 or 1, got {state[3]}')
        words[625] = int(state[3])
        words[626:628] = np.array([float(state[4])], np.float64).view(np.uint32)
    return words


def _mt_tuple(words, start):
    """The np.random.get_state() tuple of 625 words (key, pos), with the cached Gaussian (has_gauss, gauss) of the state
    `start`: the draws that led from start to the words take no Gaussian.  A 630-word record carries its own cached
    Gaussian (see _GAUSS_*); a device-drawn one is computed here as NumPy's legacy_gauss does, with C's libm."""
    if words.shape[0] < MT_GAUSS_WORDS:
        return ('MT19937', words[:624].copy(), int(words[624]), start[3], start[4])
    kind = int(words[625])
    v = np.ascontiguousarray(words[626:630]).view(np.float64)
    if kind == _GAUSS_AS_START:
        has, g = start[3], start[4]
    elif kind == _GAUSS_X1_R2:
        has, g = 1, math.sqrt(-2.0 * math.log(float(v[1])) / float(v[1])) * float(v[0])
    elif kind == _GAUSS_VALUE:
        has, g = 1, float(v[0])
    else:
        has, g = 0, 0.0
    return ('MT19937', words[:624].copy(), int(words[624]), has, g)


def _mt_state(gauss=False):
    """(words, state): NumPy's global RandomState as the words the library reads (_mt_words), and get_state()"""
    st = np.random.get_state()
    return _mt_words(st, "NumPy's global generator", gauss), st


def _set_mt_state(start, d_words):
    """set NumPy's global RandomState to the device's final words (one synchronising 2.5 KB copy), with the cached
    Gaussian of `start` or, for a 630-word record, its own"""
    np.random.set_state(_mt_tuple(d_words.cpu().numpy().view(np.uint32), start))


def _snowfall_flags(threshold_filter, camera_fov, device_prepass, assume_sorted=False):
    return ((_lib.FLAG_THRESHOLD_FILTER if threshold_filter else 0) | (_lib.FLAG_CAMERA_FOV if camera_fov else 0)
            | (_lib.FLAG_DEVICE_PREPASS if device_prepass else 0) | (_lib.FLAG_ASSUME_SORTED if assume_sorted else 0))


class SnowfallEngine:
    def __init__(self, device=0, sensor_table=None, camera=None):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError('SnowfallEngine needs a CUDA device (no CPU fallback)')
        self.device = torch.device('cuda', device)
        h = ctypes.c_void_p()
        _lib.check(self.lib.lss_create(device, ctypes.byref(h)))
        self.h = h
        fd, fs, mi, mx = sensor_arrays(sensor_table)
        self._sensor = [np.ascontiguousarray(a, dtype=np.float64) for a in (fd, fs, mi, mx)]
        _lib.check(self.lib.lss_set_sensor(self.h, len(fd), *[_ptr(a) for a in self._sensor]), self.h)
        if camera is None:
            from .calib.dense_camera import STF_HDL64_CAMERA as camera
        self.set_camera(camera)
        self._tables = {}
        self._scratch_ws = {}                   # name -> its cached workspace (_scratch)
        self._pa_part_bytes = None              # the partition pa_partition_batch left at the front of the 'pa' workspace

    # ------------------------------------------------------------------------------------------------------------------
    def close(self):
        if getattr(self, 'h', None):
            self.lib.lss_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, name, *args, check=True):
        """
        self.lib.<name>(handle, *args, current stream) on the engine's device.  Device tensors are passed as they are:
        their pointers are taken here, after the caller's checks.  Host arrays go through _ptr.  Raises the status
        through _lib.check unless check=False, and returns it.
        """
        with torch.cuda.device(self.device):
            st = getattr(self.lib, name)(self.h, *[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args],
                                         self._stream())
        if check:
            _lib.check(st, self.h)
        return st

    def _scratch(self, name, need, keep=0):
        """The cached uint8 workspace `name`, reallocated at 1.25x + 256 bytes with its first `keep` bytes copied when
        it holds fewer than `need` (a negative query answer counts as 0: the library then rejects the call).  The calls
        of one name share it in stream order: no caller runs them on several streams (snowfall_batch takes its own)."""
        need = max(int(need), 0)
        ws = self._scratch_ws.get(name)
        if ws is None or ws.numel() < need:
            grown = torch.empty(int(need * 1.25) + 256, dtype=torch.uint8, device=self.device)
            if keep:
                grown[:keep].copy_(ws[:keep])
            ws = self._scratch_ws[name] = grown
        return ws

    def set_camera(self, camera):
        P2 = np.ascontiguousarray(camera['P2'], dtype=np.float32).reshape(3, 4)
        R0 = np.ascontiguousarray(camera['R0'], dtype=np.float32).reshape(3, 3)
        V2C = np.ascontiguousarray(camera['V2C'], dtype=np.float32).reshape(3, 4)
        h, w = camera.get('img_shape', (1024, 1920))
        _lib.check(self.lib.lss_set_camera(self.h, _ptr(P2), _ptr(R0), _ptr(V2C), int(h), int(w)), self.h)

    # ------------------------------------------------------------------------------------------------------------------
    def upload_tables(self, tables, max_beam_divergence_rad=DEFAULT_MAX_DIVERGENCE_RAD, n_buckets=2048):
        """tables: sequence of float64 (Np_k, 3) arrays (x, y, r); plane index k <-> file '<prefix>_<k+1>.npy'."""
        off = np.zeros(len(tables) + 1, dtype=np.int64)
        for k, t in enumerate(tables):
            t = np.asarray(t)
            if t.ndim != 2 or t.shape[1] != 3:
                raise ValueError('particle table must be (N, 3)')
            off[k + 1] = off[k] + t.shape[0]
        xyr = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.float64) for t in tables], axis=0))
        return self._upload('lss_upload_particles', _ptr(xyr), off, max_beam_divergence_rad, n_buckets)

    def upload_tables_device(self, xyr, plane_offsets, max_beam_divergence_rad=DEFAULT_MAX_DIVERGENCE_RAD,
                             n_buckets=2048):
        """xyr: CUDA float64 tensor (sum Np, 3); plane_offsets: int64 host array (n_planes + 1)."""
        off, _, n_rows = _row_offsets(plane_offsets, 'plane_offsets')
        _check_tensor('xyr', xyr, self.device, torch.float64, (n_rows, 3))
        return self._upload('lss_upload_particles_device', xyr, off, max_beam_divergence_rad, n_buckets)

    def _upload(self, name, xyr, off, max_div, n_buckets):
        """lss_upload_particles[_device] of xyr (a host array's pointer or a checked device tensor)"""
        tid = ctypes.c_int(0)
        with torch.cuda.device(self.device):
            xyr = xyr.data_ptr() if isinstance(xyr, torch.Tensor) else xyr
            _lib.check(getattr(self.lib, name)(self.h, len(off) - 1, xyr, _ptr(off), float(max_div), int(n_buckets),
                                               self._stream(), ctypes.byref(tid)), self.h)
        self._tables[tid.value] = dict(n_planes=len(off) - 1, max_div=float(max_div))
        return tid.value

    def sample_tables_device(self, mode, snowfall_rate, terminal_velocity, seed=1000, R_0=80.0, n_planes=64,
                             upload=True, max_beam_divergence_rad=DEFAULT_MAX_DIVERGENCE_RAD, n_buckets=2048,
                             return_candidates=False):
        """
        Draw the n_planes snowflake tables of one (snowfall_rate, terminal_velocity) configuration ON THE DEVICE
        (greedy dart throwing, tools/snowfall/sampling.py:90-194, counter-based random stream) and, with `upload`,
        build the candidate index from them without a host round trip.  Returns the table id, or with upload=False
        (xyr (sum N, 3) CUDA float64 tensor, plane_offsets int64 array[, candidates]).
        """
        from .snowfall.sampling import compute_occupancy, snowfall_rate_to_rainfall_rate, _expected_capacity, _DIST
        if mode not in _DIST:
            raise NotImplementedError('Distribution model unknown.')
        occ = compute_occupancy(float(snowfall_rate), float(terminal_velocity))
        rr = float(snowfall_rate_to_rainfall_rate(float(snowfall_rate), float(terminal_velocity)))
        M = _expected_capacity(occ, rr, R_0, mode)
        for attempt in range(SAMPLER_ATTEMPTS):
            # the output holds M rows per plane, as many as there are darts, so only a target not reached with M
            # darts (the stream is keyed per dart: more darts extend it, they do not change it) can fail here
            ws = self._scratch('sampler', self.lib.lss_sample_particles_workspace_bytes(n_planes, M))
            out = torch.empty((n_planes, M, 3), dtype=torch.float64, device=self.device)
            counts = torch.empty((n_planes,), dtype=torch.int32, device=self.device)
            cand = torch.empty((n_planes, M, 3), dtype=torch.float64, device=self.device) if return_candidates else None
            st = self._call('lss_sample_particles', n_planes, occ, rr, float(R_0), _DIST[mode], int(seed), M, out, M,
                            counts, cand, ws, ws.numel(), check=False)
            if st != _lib.LSS_ERR_WORKSPACE or attempt == SAMPLER_ATTEMPTS - 1:
                break
            M *= 2
        _lib.check(st, self.h)
        cnt = counts.cpu().numpy().astype(np.int64)
        off = np.concatenate([[0], np.cumsum(cnt)])
        xyr = torch.cat([out[p, :cnt[p]] for p in range(n_planes)], dim=0).contiguous()
        if not upload:
            return (xyr, off, cand) if return_candidates else (xyr, off)
        return self.upload_tables_device(xyr, off, max_beam_divergence_rad, n_buckets)

    def free_tables(self, table_id):
        _lib.check(self.lib.lss_free_particles(self.h, int(table_id)), self.h)
        self._tables.pop(table_id, None)

    def table_info(self, table_id):
        a, b, c = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        _lib.check(self.lib.lss_table_info(self.h, int(table_id), ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)),
                   self.h)
        return dict(n_particles=a.value, n_entries=b.value, bytes=c.value)

    # ------------------------------------------------------------------------------------------------------------------
    def snowfall_batch(self, table_id, points, cloud_offsets, order, beam_divergence_deg, theta=None,
                       thresh_poly=None, plane=None, ymins=None, noise_floor=0.7, threshold_filter=True, camera_fov=False,
                       device_prepass=False, assume_sorted=False, want_full=False, want_perm=False, want_nocc=False,
                       out=None, workspace=None, counts=None):
        """
        Batched augment() on device-resident clouds (enqueued on torch's current stream, no synchronisation).

        points: CUDA float32 (N, 5); cloud_offsets: int64 host array (B + 1); order: int32 host (B, 64).
        counts: optional CUDA int32 (B,) valid rows per slot (slot-compacted input, lss_snowfall_batch_slots): cloud b
        is rows cloud_offsets[b] .. cloud_offsets[b] + counts[b], and the rows behind them are ignored.
        plane (B,4) / ymins (B,50): optional host arrays replayed by the device pre-pass (lss_noise_threshold_poly).
        workspace: optional CUDA uint8 tensor of at least lss_snowfall_workspace_bytes(N, B) bytes (default: the
        engine's), for calls in flight on several streams.
        Returns dict(points=(N,5) slot-compacted rows, counts=(B,), stats=(B,4) [, full, perm, nocc]).
        Call `check()` (synchronises) to surface asynchronous device errors.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, 5))
        _check_tensor('theta', theta, self.device, torch.float32, (N,), optional=True)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('workspace', workspace, self.device, torch.uint8, (None,), optional=True)
        order = np.ascontiguousarray(order, dtype=np.int32).reshape(B, 64)
        tp = None if thresh_poly is None else np.ascontiguousarray(thresh_poly, dtype=np.float64).reshape(B, 3)
        pl = None if plane is None else np.ascontiguousarray(plane, dtype=np.float64).reshape(B, 4)
        ym = None if ymins is None else np.ascontiguousarray(ymins, dtype=np.int32).reshape(B, 50)
        want_full = want_full or want_perm or want_nocc      # the debug views are produced together
        out = _outputs(out, self.device, points=((N, 5), torch.float32), counts=((B,), torch.int32),
                       stats=((B, 4), torch.float64), full=want_full and ((N, 5), torch.float32),
                       perm=want_perm and ((N,), torch.int32), nocc=want_nocc and ((N,), torch.int32))
        need = self.lib.lss_snowfall_workspace_bytes(N, B)
        if workspace is not None and workspace.numel() < need:
            raise ValueError(f'workspace: {workspace.numel()} bytes, the batch needs {need}')
        ws = self._scratch('snowfall', need) if workspace is None else workspace
        self._call('lss_snowfall_batch_slots', int(table_id), points, _ptr(off), counts, B, _ptr(order),
                   float(beam_divergence_deg), theta, _ptr(tp), _ptr(pl), _ptr(ym), float(noise_floor),
                   _snowfall_flags(threshold_filter, camera_fov, device_prepass, assume_sorted), out['points'],
                   out['counts'], out['stats'], out.get('full') if want_full else None,
                   out.get('perm') if want_perm else None, out.get('nocc') if want_nocc else None, ws, ws.numel())
        return out

    def snowfall_batch_host_submit(self, table_id, host_points, cloud_offsets, order, beam_divergence_deg,
                                   host_out=None, n_chunks=4, thresh_poly=None, noise_floor=0.7, threshold_filter=True,
                                   camera_fov=False, device_prepass=False):
        """
        Enqueue a host-to-host batched augment() (`lss_snowfall_batch_host_submit`) and return a ticket for
        `snowfall_batch_host_wait`.  `host_points`: CPU float32 (N, 5) tensor or numpy array (pinned memory gives full
        PCIe speed).  The batch is cut into `n_chunks` groups of whole clouds that flow through the engine's native
        pipeline (H2D copy, pre-pass, beam stage, D2H copy on separate streams).  Up to 3 batches may be in flight; with
        2-3 in flight (a prefetching loader) batch k+1's copy-in, batch k's kernels and batch k-1's copy-out overlap.
        The input and `host_out` buffers must not be touched until the ticket has been waited for.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        if isinstance(host_points, np.ndarray):
            host_points = torch.from_numpy(np.ascontiguousarray(host_points, dtype=np.float32))
        _check_tensor('host_points', host_points, _CPU, torch.float32, (N, 5))
        order = np.ascontiguousarray(order, dtype=np.int32).reshape(B, 64)
        tp = None if thresh_poly is None else np.ascontiguousarray(thresh_poly, dtype=np.float64).reshape(B, 3)
        host_out = _outputs(host_out, _CPU, points=((N, 5), torch.float32), counts=((B,), torch.int32),
                            stats=((B, 4), torch.float64))
        ticket = ctypes.c_int(-1)
        st = self.lib.lss_snowfall_batch_host_submit(
            self.h, int(table_id), _ptr(host_points), _ptr(off), B, _ptr(order), float(beam_divergence_deg), _ptr(tp),
            float(noise_floor), _snowfall_flags(threshold_filter, camera_fov, device_prepass), int(n_chunks),
            _ptr(host_out['points']), _ptr(host_out['counts']), _ptr(host_out['stats']), ctypes.byref(ticket))
        _lib.check(st, self.h)
        # the ticket keeps the buffers of the in-flight batch alive
        return dict(id=int(ticket.value), out=host_out, keep=(host_points, off, order, tp))

    def snowfall_batch_host_wait(self, ticket):
        """Block until the batch is in its host buffers; raises what the reference would have raised for it.
        Returns dict(points, counts, stats): pinned CPU tensors, slot-compacted layout of snowfall_batch."""
        _lib.check(self.lib.lss_snowfall_batch_host_wait(self.h, int(ticket['id'])), self.h)
        return ticket['out']

    def snowfall_batch_host(self, table_id, host_points, cloud_offsets, order, beam_divergence_deg, **kw):
        """Synchronous host-to-host batched augment(): submit + wait (see snowfall_batch_host_submit)."""
        return self.snowfall_batch_host_wait(
            self.snowfall_batch_host_submit(table_id, host_points, cloud_offsets, order, beam_divergence_deg, **kw))

    def host_pipeline_trace(self, max_chunks=64):
        """Device timeline (ms since call start) of the last snowfall_batch_host call: rows (n_chunks, 4) =
        rows landed, polynomial ready, beam stage done, results on host."""
        buf = np.zeros((max_chunks, 4), dtype=np.float32)
        n = self.lib.lss_host_pipe_trace(self.h, _ptr(buf), max_chunks)
        return buf[:n]

    def noise_threshold_poly(self, points, cloud_offsets, noise_floor=0.7, plane=None, ymins=None, want_fits=False):
        """Device pre-pass only: returns (poly (B,3) float64 tensor in np.polyfit order, plane (B,4) tensor)
        [, fits (B,8) float64, picks (B,50) int32 with want_fits].
        plane: optional host array (B,4) = (w0, w1, w2, h) to use instead of the RANSAC estimate;
        ymins: optional host int array (B,50), the reference host's np.argpartition picks (augmentation.py:236)."""
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, 5))
        pl = None if plane is None else np.ascontiguousarray(plane, dtype=np.float64).reshape(B, 4)
        ym = None if ymins is None else np.ascontiguousarray(ymins, dtype=np.int32).reshape(B, 50)
        ws = self._scratch('prepass', self.lib.lss_prepass_workspace_bytes(N, B))
        out = _outputs(None, self.device, poly=((B, 3), torch.float64), plane=((B, 4), torch.float64),
                       fits=want_fits and ((B, 8), torch.float64), picks=want_fits and ((B, 50), torch.int32))
        self._call('lss_noise_threshold_poly', points, _ptr(off), B, float(noise_floor), _ptr(pl), _ptr(ym), out['poly'],
                   out['plane'], out.get('fits'), out.get('picks'), ws, ws.numel())
        return tuple(out.values())                          # (poly, plane[, fits, picks])

    def wet_ground_batch(self, points, cloud_offsets, counts=None, water_height=0.001, pavement_depth=0.0012,
                         noise_floor=0.7, power_factor=15, flat_earth=False, delta=0.5, replace=True, plane=None,
                         want_intensity64=False, ymins=None, out=None, want_fits=False, estimation_method='linear'):
        """
        Batched ground_water_augmentation() on device-resident clouds (current stream, no synchronisation).
        counts: optional CUDA int32 (B,) valid rows per cloud slot (fused snow -> wet path).
        water_height: a number, or a (B,) array of one height per cloud (lss_wet_ground_batch_params; a degenerate I/cos
        range is then only reported as passthrough 2, and check() does not raise for it).
        Returns dict(points (N,5) float32 slot-compacted, counts (B,), passthrough (B,), plane (B,4) [, intensity64]
        [, fits (B,8) float64, picks (B,50) int32 with want_fits, laid out as in noise_threshold_poly]).
        passthrough: 0 augmented, 1 fewer than 1000 ground points, 2 degenerate I/cos range (check() raises ValueError).
        estimation_method='poly' (lss_wet_ground_batch_poly): the quadratic laser power and the RANSAC noise floor of
        augmentation.py:171-192,223-246, drawn on NumPy's global RandomState, whose state is then set as B sequential
        calls leave it (the call synchronises once to copy it back).  water_height is forwarded once per cloud, check()
        raises for no cloud, and passthrough adds 3: no minima point, where the reference raises TypeError.  want_fits
        adds poly_fits (B,8) float64: p0, p1, p2, pmin0, pmin1, pmin2, the chosen trial (-1: the full fit), m.
        """
        if estimation_method not in ('linear', 'poly'):
            raise ValueError(f"estimation_method: 'linear' or 'poly', got {estimation_method!r}")
        poly = estimation_method == 'poly'
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, 5))
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        pl = None if plane is None else np.ascontiguousarray(plane, dtype=np.float64).reshape(B, 4)
        ym = None if ymins is None else np.ascontiguousarray(ymins, dtype=np.int32).reshape(B, 50)
        per_cloud = np.ndim(water_height) > 0 or poly
        if per_cloud:
            heights = np.ascontiguousarray(np.broadcast_to(np.asarray(water_height, dtype=np.float64),
                                                           (B,) if np.ndim(water_height) == 0 else np.shape(water_height)))
            heights = heights.reshape(-1)
            if heights.shape[0] != B:
                raise ValueError(f'water_height: {heights.shape[0]} heights for {B} clouds')
        # (pass the returned dict back in as `out` to reuse the buffers)
        out = _outputs(out, self.device, points=((N, 5), torch.float32), counts=((B,), torch.int32),
                       passthrough=((B,), torch.int32), plane=((B, 4), torch.float64),
                       intensity64=want_intensity64 and ((N,), torch.float64), fits=want_fits and ((B, 8), torch.float64),
                       picks=want_fits and ((B, 50), torch.int32),
                       poly_fits=poly and want_fits and ((B, 8), torch.float64), state=poly and ((625,), torch.int32))
        if poly:
            words, start = _mt_state()
            ws = self._scratch('wet', self.lib.lss_wet_ground_poly_workspace_bytes(N, B))
            self._call('lss_wet_ground_batch_poly', points, _ptr(off), counts, B, _ptr(heights), float(pavement_depth),
                       float(noise_floor), float(power_factor), 1 if flat_earth else 0, float(delta), 1 if replace else 0,
                       _ptr(pl), _ptr(ym), _ptr(words), out['points'], out.get('intensity64') if want_intensity64 else None,
                       out['counts'], out['passthrough'], out['plane'], out.get('fits') if want_fits else None,
                       out.get('picks') if want_fits else None, out['state'], out.get('poly_fits'), ws, ws.numel())
            _set_mt_state(start, out.pop('state'))
            return out
        ws = self._scratch('wet', self.lib.lss_wet_ground_workspace_bytes(N, B))
        self._call('lss_wet_ground_batch_params' if per_cloud else 'lss_wet_ground_batch', points, _ptr(off), counts, B,
                   _ptr(heights) if per_cloud else float(water_height), float(pavement_depth), float(noise_floor),
                   float(power_factor), 1 if flat_earth else 0, float(delta), 1 if replace else 0, _ptr(pl), _ptr(ym),
                   out['points'], out.get('intensity64') if want_intensity64 else None, out['counts'],
                   out['passthrough'], out['plane'], out.get('fits') if want_fits else None,
                   out.get('picks') if want_fits else None, ws, ws.numel())
        return out

    def fog_batch(self, points, cloud_offsets, lut, alpha, beta, beta_0, hard=True, soft=True, gain=False, noise=0,
                  noise_variant=1, rng_states=None, ext_noise=None, want_rank=False):
        """
        Batched simulate_fog() (lib/LiDAR_fog_sim/fog_simulation.py:299-316) on device-resident clouds (current stream,
        no synchronisation).  points: CUDA float32 (N, F), F >= 4; lut: CUDA float64 (2001, 2) integral look-up table;
        rng_states: host uint64 (B, 4) PCG64 states (variants 1-3) or ext_noise: CUDA float64 (N,) values by rank.
        Returns dict(points float64 (N, F), fog_mask uint8 (N,), info float64 (B, 3) [, rank int32 (N,)]); info[b] =
        (min response, max response, count), count -1 - (2 * fog points before the row + kind) for a cloud where the
        reference raises (kind 0: a NaN range, KeyError; 1: v1 noise at an infinite range, OverflowError).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('lut', lut, self.device, torch.float64, (2001, 2), optional=True)
        return self._fog('lss_fog_batch', 'lss_fog_workspace_bytes', (float(alpha), float(beta), float(beta_0), lut),
                         points, off, B, N, hard, soft, gain, noise, noise_variant, rng_states, ext_noise, want_rank)

    def fog_batch_params(self, points, cloud_offsets, luts, alpha, beta, beta_0, table_index=None, hard=True, soft=True,
                         gain=False, noise=0, noise_variant=1, rng_states=None, ext_noise=None, want_rank=False):
        """
        fog_batch with the fog parameters chosen per cloud (lss_fog_batch_params): alpha, beta, beta_0 and table_index
        are length-B host sequences; luts: CUDA float64 (T, 2001, 2) stack of integral tables (e.g. fog_integral_tables);
        cloud b uses luts[table_index[b]].  A cloud's results are bit-identical to fog_batch with its own parameters.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('luts', luts, self.device, torch.float64, (None, 2001, 2), optional=True)
        per = [np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (B,))) for v in (alpha, beta, beta_0)]
        ti = None if table_index is None else np.ascontiguousarray(table_index, dtype=np.int32).reshape(B)
        params = (*[_ptr(v) for v in per], _ptr(ti), luts, 0 if luts is None else int(luts.shape[0]))
        return self._fog('lss_fog_batch_params', 'lss_fog_batch_params_workspace_bytes', params, points, off, B, N, hard,
                         soft, gain, noise, noise_variant, rng_states, ext_noise, want_rank)

    def _fog(self, name, ws_name, params, points, off, B, N, hard, soft, gain, noise, noise_variant, rng_states,
             ext_noise, want_rank):
        """fog_batch and fog_batch_params, which differ in the entry point and its fog parameter block `params`"""
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=4)
        _check_tensor('ext_noise', ext_noise, self.device, torch.float64, optional=True)
        if ext_noise is not None and ext_noise.numel() < N:
            raise ValueError(f'ext_noise: {ext_noise.numel()} values for {N} rows')
        rs = None if rng_states is None else np.ascontiguousarray(rng_states, dtype=np.uint64).reshape(B, 4)
        flags = (_lib.FOG_HARD if hard else 0) | (_lib.FOG_SOFT if soft else 0) | (_lib.FOG_GAIN if gain else 0)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((N, F), torch.float64), fog_mask=((N,), torch.uint8),
                       info=((B, 3), torch.float64), rank=want_rank and ((N,), torch.int32))
        ws = self._scratch('fog', getattr(self.lib, ws_name)(N, B))
        self._call(name, points, F, _ptr(off), B, *params, flags, int(noise), int(noise_variant), _ptr(rs), ext_noise,
                   out['points'], out['fog_mask'], out.get('rank'), out['info'], ws, ws.numel())
        return out

    def fog_integral_tables(self, params, shift=False, n=2000, r_range=200, r_0_max=200, granularity=None):
        """
        The fog integral look-up tables of `params` (a sequence of fog ParameterSets, or one), generated on the device
        (lss_fog_integral_tables, current stream, no synchronisation): the reference generator's table for each
        parameter set (generate_integral_lookup_table.py), row k = (fog_distance, fog_integral) at r_0 =
        round(k * granularity, 2).  The defaults are the shipped grid (n_steps = 2000 over 200 m, 2001 rows; the
        generator sets n = n_steps and r_range = r_0_max).  Returns a CUDA float64 tensor (T, rows, 2).
        """
        if not isinstance(params, (list, tuple)):
            params = [params]
        granularity = r_0_max / n if granularity is None else granularity
        T = len(params)
        arr = (_lib.FogTableParams * max(T, 1))()
        for t, p in enumerate(params):
            q = arr[t]
            for f in ('alpha', 'tau_h', 'r_1', 'r_2', 'D', 'ROH_T', 'ROH_R', 'GAMMA_T', 'GAMMA_R', 'c_a', 'p_0', 'beta'):
                setattr(q, f, float(getattr(p, f)))
            q.r_range, q.r_0_max, q.granularity = float(r_range), float(r_0_max), float(granularity)
            q.n, q.linear_xsi, q.shift = int(n), 1 if p.linear_xsi else 0, 1 if shift else 0
        steps = float(r_0_max) / float(granularity)
        rows = int(steps) + 1 if np.isfinite(steps) and 0 <= steps < 2 ** 24 else 0
        out = torch.empty((T, rows, 2), dtype=torch.float64, device=self.device)
        ws = self._scratch('fog_tables', self.lib.lss_fog_integral_tables_workspace_bytes(int(n), T))
        self._call('lss_fog_integral_tables', ctypes.cast(arr, ctypes.c_void_p), T, out, ws, ws.numel())
        return out

    def mie_tables(self, refractive_indices, wavelengths_nm, diameters_nm=None):
        """
        LISA's Mie efficiency tables generated on the device (lss_mie_tables, current stream, no synchronisation): for
        each (real refractive index, wavelength [nm]) pair, (qext, qback) at every diameter of `diameters_nm` [nm], as
        PyMieScatt.MieQ_withDiameterRange computes them for lisa.py:446-465.  diameters_nm defaults to its logD grid of
        2000 diameters from 1 nm to 1 cm.  Returns a CUDA float64 tensor (T, n_diameters, 2).
        """
        m = np.ascontiguousarray(np.atleast_1d(np.asarray(refractive_indices, dtype=np.float64)))
        wl = np.ascontiguousarray(np.atleast_1d(np.asarray(wavelengths_nm, dtype=np.float64)))
        if m.ndim != 1 or m.shape != wl.shape:
            raise ValueError('need one wavelength per refractive index')
        if diameters_nm is None:
            diameters_nm = np.logspace(0, 7, 2000)
        d = np.ascontiguousarray(np.asarray(diameters_nm, dtype=np.float64).reshape(-1))
        T, nd = int(m.shape[0]), int(d.shape[0])
        ws = self._scratch('mie', self.lib.lss_mie_tables_workspace_bytes(_ptr(m), _ptr(wl), T, _ptr(d), nd))
        out = torch.empty((T, nd, 2), dtype=torch.float64, device=self.device)
        self._call('lss_mie_tables', _ptr(m), _ptr(wl), T, _ptr(d), nd, out, ws, ws.numel())
        return out

    def voxelize_batch(self, points, cloud_offsets, point_cloud_range, voxel_size, max_points_per_voxel, max_voxels,
                       counts=None, mask_xy_range=True):
        """
        Batched point-range mask + voxelisation (DataProcessor.mask_points_and_boxes_outside_range +
        transform_points_to_voxels, lib/OpenPCDet/pcdet/datasets/processor/data_processor.py:78-91,115-143) on
        device-resident clouds (current stream, no synchronisation).  points: CUDA float32 (N, F); counts: optional CUDA
        int32 (B,) valid rows per cloud slot.  Returns dict(voxels (B, max_voxels, max_points, F) float32, coords
        (B, max_voxels, 4) int32 = (cloud, z, y, x), num_points (B, max_voxels) int32, n_voxels (B,) int32).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        F = points.shape[1]
        rng = np.ascontiguousarray(point_cloud_range, dtype=np.float32).reshape(6)
        vs = np.ascontiguousarray(voxel_size, dtype=np.float32).reshape(3)
        T, MV = int(max_points_per_voxel), int(max_voxels)
        out = _outputs(None, self.device, voxels=((B, MV, T, F), torch.float32), coords=((B, MV, 4), torch.int32),
                       num_points=((B, MV), torch.int32), n_voxels=((B,), torch.int32))
        ws = self._scratch('voxelize', self.lib.lss_voxelize_workspace_bytes(N, B, T, MV))
        self._call('lss_voxelize_batch', points, F, _ptr(off), counts, B, _ptr(rng), _ptr(vs), T, MV,
                   1 if mask_xy_range else 0, out['voxels'], out['coords'], out['num_points'], out['n_voxels'], ws,
                   ws.numel())
        return out

    def processor_batch(self, points, cloud_offsets, columns, point_cloud_range, counts=None, mask_points=True,
                        shuffle=True, voxel_size=None, max_points_per_voxel=0, max_voxels=0):
        """
        The DataProcessor tail of prepare_data (lss_processor_batch, current stream): feature encoding through the
        column map `columns` (x, y, z first), mask_points_by_range when mask_points, shuffle_points on NumPy's global
        RandomState when shuffle (cloud after cloud, exactly np.random.permutation), and with voxel_size the voxels of
        voxelize_batch.  points: CUDA float32 (N, F); counts: optional CUDA int32 (B,) valid rows per slot.  Returns
        dict(points (N, len(columns)) float32 rows at the front of each slot, counts (B,) int32 CUDA [, voxels, coords,
        num_points, n_voxels as voxelize_batch]).  With shuffle, the call synchronises once: it copies the generator's
        final 625 words back and sets NumPy's state to them.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        cols = np.ascontiguousarray(columns, dtype=np.int32).reshape(-1)
        F, Fo = points.shape[1], cols.shape[0]
        if not 3 <= Fo <= 16 or list(cols[:3]) != [0, 1, 2] or cols.min() < 0 or cols.max() >= F:
            raise ValueError(f'columns: x, y, z (0, 1, 2) first, then at most 13 of the {F} input columns, got {cols}')
        rng = np.ascontiguousarray(point_cloud_range, dtype=np.float64).reshape(6)
        voxels = voxel_size is not None
        T, MV = (int(max_points_per_voxel), int(max_voxels)) if voxels else (0, 0)
        if voxels and (T <= 0 or MV <= 0):
            raise ValueError('max_points_per_voxel > 0 and max_voxels > 0 required')
        vs = np.ascontiguousarray(voxel_size, dtype=np.float32).reshape(3) if voxels else None
        words, start = _mt_state() if shuffle else (None, None)
        out = _outputs(None, self.device, points=((N, Fo), torch.float32), counts=((B,), torch.int32),
                       state=shuffle and ((625,), torch.int32), voxels=voxels and ((B, MV, T, Fo), torch.float32),
                       coords=voxels and ((B, MV, 4), torch.int32), num_points=voxels and ((B, MV), torch.int32),
                       n_voxels=voxels and ((B,), torch.int32))
        ws = self._scratch('processor', self.lib.lss_processor_workspace_bytes(N, B, Fo, T, MV))
        self._call('lss_processor_batch', points, F, _ptr(off), counts, B, _ptr(cols), Fo, _ptr(rng),
                   1 if mask_points else 0, _ptr(words), out.get('state'), _ptr(vs), T, MV, out['points'],
                   out['counts'], out.get('voxels'), out.get('coords'), out.get('num_points'), out.get('n_voxels'), ws,
                   ws.numel())
        if shuffle:
            _set_mt_state(start, out.pop('state'))
        return out

    def mt19937_permutations(self, cloud_offsets, counts=None):
        """
        np.random.permutation(n_b) for the clouds in turn, drawn on the device from NumPy's global RandomState
        (lss_mt19937_permutations), whose state is then set as B sequential calls leave it.  n_b = counts[b] (CUDA int32
        (B,)) or the slot's length.  Returns a CUDA int32 (N,) tensor: cloud b's permutation at rows cloud_offsets[b]..
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        words, start = _mt_state()
        out = _outputs(None, self.device, perm=((N,), torch.int32), state=((625,), torch.int32))
        ws = self._scratch('processor', self.lib.lss_processor_workspace_bytes(N, B, 0, 0, 0))
        self._call('lss_mt19937_permutations', _ptr(off), counts, B, _ptr(words), out['perm'], out['state'], ws,
                   ws.numel())
        _set_mt_state(start, out['state'])
        return out['perm']

    def sample_points_batch(self, points, cloud_offsets, num_points, counts=None, shuffle=False, run_starts=None,
                            run_states=None, f32_distance=None):
        """
        DataProcessor.sample_points (data_processor.py:145-175) with NUM_POINTS = num_points (>= 0) on NumPy's legacy
        RandomState for every cloud, followed by shuffle_points' np.random.permutation when shuffle (lss_sample_points_batch,
        current stream).  points: CUDA float32 or float64 (N, F >= 3); counts: optional CUDA int32 (B,) valid rows per
        slot.  The clouds draw in batch order from NumPy's global state, or in runs: run_starts (R,) the first cloud of each
        run (0 first, increasing) and run_states R np.random.get_state() tuples, each run continuing from its own state.
        f32_distance: optional host bool (B,), with float64 rows: the clouds whose near / far test is taken in float32 (rows
        holding float32 values).  Returns dict(points (B * num_points, F) of points' dtype, offsets num_points *
        arange(B + 1) host int64, counts (B,) int32 CUDA, states (R, 625) uint32 host: each run's final key and pos).
        The call synchronises once, for the copy of the final states and the status; NumPy's global state is then the last
        run's (the cached Gaussian as that run's start state has it).  Where the reference raises ValueError (a cloud with
        no rows and num_points > 0, or more than twice its rows), this raises it for the first such cloud, with NumPy's
        state as it was before that cloud's draws.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, (torch.float32, torch.float64), (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        k = int(num_points)
        if not 0 <= k < 2 ** 30:
            raise ValueError(f'num_points must be in [0, 2^30), got {k}')
        if run_starts is None:
            starts = np.zeros(1, np.int64)
            run_states = [np.random.get_state()] if run_states is None else list(run_states)
        else:
            starts = np.ascontiguousarray(run_starts, dtype=np.int64).reshape(-1)
            run_states = list(run_states or [])
        R = starts.shape[0]
        if (len(run_states) != R or starts[0] != 0 or np.any(np.diff(starts) <= 0) or starts[-1] >= max(B, 1)):
            raise ValueError('run_starts: 0 first, increasing, below the number of clouds, one state per run')
        words = np.stack([_mt_words(st, f'run_states[{r}]') for r, st in enumerate(run_states)])
        run_off = np.append(starts, B).astype(np.int32)
        f32 = _f32_flags(f32_distance, B)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((B * k, F), points.dtype))
        tail = torch.empty(R * 627, dtype=torch.int32, device=self.device)     # states then status: one copy back
        ws = self._scratch('sample_points', self.lib.lss_sample_points_workspace_bytes(N, B, k, R))
        self._call('lss_sample_points_batch', points, 1 if points.dtype == torch.float64 else 0, F, _ptr(off), counts, B,
                   _ptr(f32), k, 1 if shuffle else 0, _ptr(run_off), R, _ptr(words), out['points'], tail[:R * 625],
                   tail[R * 625:], ws, ws.numel())
        h = tail.cpu().numpy()
        states = h[:R * 625].view(np.uint32).reshape(R, 625)
        status = h[R * 625:].reshape(R, 2)
        failed = [r for r in range(R) if status[r, 0] >= 0]
        last = min(failed, key=lambda r: status[r, 0]) if failed else R - 1
        np.random.set_state(_mt_tuple(states[last], run_states[last]))
        if failed:
            raise ValueError("'a' cannot be empty unless no samples are taken" if status[last, 1] == 1 else
                             "Cannot take a larger sample than population when 'replace=False'")
        return {'points': out['points'], 'offsets': np.arange(B + 1, dtype=np.int64) * k,
                'counts': torch.full((B,), k, dtype=torch.int32, device=self.device), 'states': states}

    def farthest_distance_batch(self, points, cloud_offsets, counts=None, f32_distance=None):
        """
        max(np.linalg.norm(points[:, 0:3], axis=1)) of every cloud with Python's builtin max, as FILTER_OUT_OF_MOR_BOXES
        takes it (dense_dataset.py:930; lss_farthest_distance_batch, current stream): NaN when row 0's distance is NaN,
        else the largest non-NaN distance; -1 for an empty cloud.  points, counts, f32_distance as sample_points_batch.
        Returns a CUDA float64 (B,) tensor; float32 distances are exact in it.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, (torch.float32, torch.float64), (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        f32 = _f32_flags(f32_distance, B)
        out = torch.empty(B, dtype=torch.float64, device=self.device)
        ws = self._scratch('farthest', self.lib.lss_farthest_distance_workspace_bytes(B))
        self._call('lss_farthest_distance_batch', points, 1 if points.dtype == torch.float64 else 0, points.shape[1],
                   _ptr(off), counts, B, _ptr(f32), out, ws, ws.numel())
        return out

    def haze_batch(self, points, cloud_offsets, beta, fourier, noise_level=0.04, gain=0.45, dmin=2.0,
                   fraction_random=0.05, counts=None, state=None, angle=None, out_dtype=torch.float32, label=False):
        """
        DENSE fog: haze_point_cloud with BetaRadomization's beta field (lss_haze_batch, current stream) for every cloud,
        each drawing from the same MT19937 start state `state` (an np.random.get_state() tuple; None: NumPy's global
        state), as the dataset's per-sample BetaRadomization(seed=0) makes them.  points: CUDA float32 (N, F), F >= 4;
        counts: optional CUDA int32 (B,) valid rows per slot; beta: (B,) float64 >= 0, 0 = the reference's tuple
        branch; fourier: (n_components, 6) float64 rows (fa, fh, oa, oh, ih, ia) after propagate_in_time; noise_level,
        gain, dmin: the sensor's n, g, dmin; fraction_random in [0, 0.05]; angle: optional CUDA float32 (N,) tangent
        per row to use instead of the device's correctly rounded one.  Returns dict(points (M, F + label) out_dtype with
        cloud b's rows at offsets[b] (M = offsets[B], slots of n_b + n_b // 20 + 1 rows), offsets int64 numpy (B + 1,),
        counts int32 CUDA (B,), states uint32 numpy (B, 625) each cloud's final key and pos).  The one synchronisation
        is the copy of the states and counts; NumPy's global state is then set to the last cloud's (the cached Gaussian
        as `state` has it, as no Gaussian is drawn).  Where the reference raises OverflowError('Range exceeds valid
        bounds') -- a random scatter candidate whose min(d_max, d) is NaN or infinite, e.g. from a NaN intensity, I = -g
        or a non-finite y / x or z -- this raises it for the first such cloud, with NumPy's global state set to that
        cloud's (after its lost draws).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=4)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('angle', angle, self.device, torch.float32, (N,), optional=True)
        if out_dtype not in (torch.float32, torch.float64):
            raise ValueError(f'out_dtype: expected torch.float32 or torch.float64, got {out_dtype}')
        betas = np.ascontiguousarray(beta, dtype=np.float64).reshape(-1)
        if betas.shape[0] != B or not np.all(np.isfinite(betas) & (betas >= 0)):
            raise ValueError(f'beta: expected {B} finite values >= 0, got {betas}')
        four = np.ascontiguousarray(fourier, dtype=np.float64)
        if four.ndim != 2 or four.shape[1] != 6 or four.shape[0] > 16:
            raise ValueError(f'fourier: expected an (n_components <= 16, 6) array, got shape {four.shape}')
        if not 0.0 <= fraction_random <= 0.05:
            raise ValueError(f'fraction_random must be in [0, 0.05], got {fraction_random}')
        words, state = _mt_state() if state is None else (_mt_words(state, 'state'), state)
        F = points.shape[1]
        Fo = F + (1 if label else 0)
        n = np.diff(off)
        out_off = np.zeros(B + 1, np.int64)
        np.cumsum(n + n // 20 + 1, out=out_off[1:])
        out = _outputs(None, self.device, points=((int(out_off[-1]), Fo), out_dtype))
        tail = torch.empty(B * 626, dtype=torch.int32, device=self.device)     # states then counts: one copy back
        out['states'], out['counts'] = tail[:B * 625].view(B, 625), tail[B * 625:]
        ws = self._scratch('haze', self.lib.lss_haze_workspace_bytes(N, B))
        self._call('lss_haze_batch', points, F, _ptr(off), counts, B, _ptr(betas), _ptr(four), four.shape[0],
                   float(noise_level), float(gain), float(dmin), float(fraction_random), _ptr(words), angle,
                   1 if out_dtype == torch.float64 else 0, 1 if label else 0, out['points'], out['counts'],
                   out['states'], ws, ws.numel())
        h = tail.cpu().numpy()
        states = h[:B * 625].view(np.uint32).reshape(B, 625)
        bad = np.flatnonzero(h[B * 625:] < 0)
        if B > 0:
            np.random.set_state(_mt_tuple(states[int(bad[0]) if bad.size else B - 1], state))
        if bad.size:
            # the reference's np.random.uniform(high=scatter_max[...]) on a NaN or infinite bound, after the lost draws
            raise OverflowError('Range exceeds valid bounds')
        return {'points': out['points'], 'offsets': out_off, 'counts': out['counts'], 'states': states}

    def dror_batch(self, points, cloud_offsets, alpha=0.16, beta=3.0, k_min=3, sr_min=0.04, counts=None, crop=False,
                   want_points=True, work_stats=False, out=None):
        """
        Batched DROR snow removal (dynamic_radius_outlier_filter, lib/cadc_devkit/other/dror.py:288-334) on
        device-resident clouds (current stream, no synchronisation).  points: CUDA float32 (N, F), F >= 3; counts:
        optional CUDA int32 (B,) valid rows per cloud slot (e.g. the output of snowfall_batch); crop: only rows inside
        get_cube_mask's box take part (dror.py:73-84).  Returns dict(keep uint8 (N,) = 1 keep / 0 snow / 2 outside the
        cube, counts int32 (B,) kept rows, n_snow int32 (B,) [, points (N, F) kept rows slot-compacted in input order]
        [, work: uint64 CUDA tensor (4,) = queries, cells visited, candidates tested, early exits]).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        F = points.shape[1]
        flags = (_lib.DROR_CUBE if crop else 0) | (_lib.DROR_WORK_STATS if work_stats else 0)
        out = _outputs(out, self.device, keep=((N,), torch.uint8), counts=((B,), torch.int32),
                       n_snow=((B,), torch.int32), points=want_points and ((N, F), torch.float32))
        need = self.lib.lss_dror_workspace_bytes(N, B)
        if need < 0:
            raise RuntimeError('lss_dror_workspace_bytes failed (2^31 rows or more, or no usable CUDA device?)')
        ws = self._scratch('dror', need)
        self._call('lss_dror_batch', points, F, _ptr(off), counts, B, float(alpha), float(beta), int(k_min),
                   float(sr_min), flags, out['keep'], out['points'] if want_points else None, out['counts'],
                   out['n_snow'], ws, ws.numel())
        if work_stats:
            out['work'] = ws[:32].view(torch.int64).clone()
        return out

    def strongest_last_batch(self, last, last_offsets, strongest, strongest_offsets, min_dist=3.0, last_counts=None,
                             strongest_counts=None, want_mask=False):
        """
        The dataset's STRONGEST_LAST_FILTER (compare_points, dense_dataset.py:519-562, then pc_master[mask]) on a batch
        of device-resident echo pairs (lss_strongest_last_batch, current stream, no synchronisation).  last / strongest:
        CUDA float32 (N_l, F) / (N_s, F), F >= 3, cloud b at rows *_offsets[b]:*_offsets[b+1] (the first *_counts[b] with
        counts).  Cloud b's output slot has max(slot_l, slot_s) rows.  Returns dict(points (N_out, F) float32, each
        cloud's kept master rows at the front of its slot; offsets int64 host array (B + 1) of those slots; counts (B,)
        int32; master_is_strongest (B,) uint8 [, mask (N_out,) uint8: compare_points' mask on each slot's master rows]).
        """
        off_l, B, N_l = _cloud_offsets(last_offsets, 'last_offsets')
        off_s, B_s, N_s = _cloud_offsets(strongest_offsets, 'strongest_offsets')
        if B_s != B:
            raise ValueError('last and strongest need the same number of clouds')
        for off in (off_l, off_s):
            if off[0] != 0 or (np.diff(off) < 0).any():              # (the workspace query cannot say why it fails)
                raise ValueError('cloud_offsets must start at 0 and be non-decreasing')
        _check_tensor('last', last, self.device, torch.float32, (N_l, None), min_cols=3)
        _check_tensor('strongest', strongest, self.device, torch.float32, (N_s, None), min_cols=3)
        if last.shape[1] != strongest.shape[1]:
            raise ValueError('last and strongest need the same number of columns')
        _check_tensor('last_counts', last_counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('strongest_counts', strongest_counts, self.device, torch.int32, (B,), optional=True)
        F = last.shape[1]
        off_o = np.concatenate([[0], np.cumsum(np.maximum(np.diff(off_l), np.diff(off_s)))]).astype(np.int64)
        N = int(off_o[-1])
        out = dict(points=torch.empty((N, F), dtype=torch.float32, device=self.device), offsets=off_o,
                   counts=torch.empty((B,), dtype=torch.int32, device=self.device),
                   master_is_strongest=torch.empty((B,), dtype=torch.uint8, device=self.device))
        if want_mask:
            out['mask'] = torch.zeros((N,), dtype=torch.uint8, device=self.device)
        need = self.lib.lss_strongest_last_batch_workspace_bytes(_ptr(off_l), _ptr(off_s), B)
        if need < 0:
            raise RuntimeError('lss_strongest_last_batch_workspace_bytes failed (bad offsets or no CUDA device?)')
        ws = self._scratch('strongest_last', need)
        self._call('lss_strongest_last_batch', last, _ptr(off_l), last_counts, strongest, _ptr(off_s), strongest_counts,
                   F, B, float(min_dist), out['points'], out['counts'], out['master_is_strongest'], out.get('mask'), ws,
                   ws.numel())
        return out

    def camera_fov_batch(self, points, cloud_offsets, counts=None, img_shapes=None, want_mask=False):
        """
        The dataset's FOV_POINTS_ONLY (calib.lidar_to_rect + get_fov_flag, dense_dataset.py:36-44,689-711) on a batch of
        device-resident clouds with this engine's camera (set_camera; lss_camera_fov_batch, current stream, no
        synchronisation).  points: CUDA float32 (N, F), F >= 3; counts: optional CUDA int32 (B,) valid rows per slot;
        img_shapes: optional (B, 2) host (img_h, img_w) per cloud, default the camera's.  Returns dict(points (N, F)
        float32, each cloud's rows inside the image at the front of its slot; counts (B,) int32 -- 0 where the dataset
        would draw another sample [, mask (N,) uint8 flag of every valid row]).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        F = points.shape[1]
        shp = None if img_shapes is None else np.ascontiguousarray(
            np.broadcast_to(np.asarray(img_shapes, dtype=np.int32).reshape(-1, 2), (B, 2)))
        out = _outputs(None, self.device, points=((N, F), torch.float32), counts=((B,), torch.int32))
        if want_mask:
            out['mask'] = torch.zeros((N,), dtype=torch.uint8, device=self.device)
        ws = self._scratch('camera_fov', self.lib.lss_camera_fov_batch_workspace_bytes(N, B))
        self._call('lss_camera_fov_batch', points, F, _ptr(off), counts, B, _ptr(shp), out['points'], out['counts'],
                   out.get('mask'), ws, ws.numel())
        return out

    def lisa_batch(self, points, rain_rate, alpha, seed, mode, r_min=0.9, r_max=120.0, beam_divergence=3e-3,
                   min_diameter=0.05, range_accuracy=0.09, signal_last=False, draw_table=None):
        """LISA.monte_carlo_augment (lib/LISA/python/lisa.py:293-341) on one device-resident cloud (lss_lisa_batch,
        current stream, no synchronisation).  points: CUDA float64 (n, F), F >= 4, intensity in [0, 1]; seed: the
        counter-based generator's key, or draw_table: CUDA float64 fixed-seed draw sequence (too short: raised at
        check()); the other arguments as lisa_cloud_batch's.  Returns CUDA float64 (n, F + 2): x, y, z, intensity,
        label, intensity_diff, zeros."""
        _check_tensor('points', points, self.device, torch.float64, (None, None), min_cols=4)
        _check_tensor('draw_table', draw_table, self.device, torch.float64, optional=True)
        n, F = points.shape
        out = torch.empty((n, F + 2), dtype=torch.float64, device=self.device)
        self._call('lss_lisa_batch', points, F, n, float(rain_rate), int(mode), float(alpha), float(r_min),
                   float(r_max), float(beam_divergence), float(min_diameter), float(range_accuracy),
                   1 if signal_last else 0, draw_table, 0 if draw_table is None else draw_table.numel(), int(seed), out)
        return out

    def lisa_cloud_batch(self, points, cloud_offsets, rain_rate, alpha, seed, mode, r_min=0.9, r_max=120.0,
                         beam_divergence=3e-3, min_diameter=0.05, range_accuracy=0.09, signal_last=False, counts=None,
                         apply=None, draw_table=None):
        """
        The dataset's LISA block (dense_dataset.py:732-746) on a batch of device-resident clouds (lss_lisa_cloud_batch,
        current stream, no synchronisation).  points: CUDA float32 (N, F), F >= 5, intensity in [0, 255]; rain_rate,
        alpha, seed: length-B host sequences (seed may be None with a draw table); mode 0 'rain', 1 'gunn', 2 'sekhon';
        counts: optional CUDA int32 (B,) valid rows per slot; apply: optional length-B booleans (clouds with False are
        copied through); draw_table: CUDA float64 fixed-seed draw sequence or None.  Returns dict(points (N, F) float32:
        each cloud's kept rows at the front of its slot, label in column 4; counts (B,) int32; n_lost (B,) int32).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=5)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('draw_table', draw_table, self.device, torch.float64, optional=True)
        F = points.shape[1]
        rr, al = [np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (B,))) for v in (rain_rate, alpha)]
        sd = None if seed is None else np.ascontiguousarray(np.broadcast_to(np.asarray(seed, dtype=np.uint64), (B,)))
        ap = None if apply is None else np.ascontiguousarray(np.asarray(apply, dtype=bool).reshape(B), dtype=np.uint8)
        out = _outputs(None, self.device, points=((N, F), torch.float32), counts=((B,), torch.int32),
                       n_lost=((B,), torch.int32))
        ws = self._scratch('lisa', self.lib.lss_lisa_cloud_batch_workspace_bytes(N, B))
        self._call('lss_lisa_cloud_batch', points, F, _ptr(off), counts, B, _ptr(rr), _ptr(al), _ptr(sd), _ptr(ap),
                   int(mode), float(r_min), float(r_max), float(beam_divergence), float(min_diameter),
                   float(range_accuracy), 1 if signal_last else 0, draw_table,
                   0 if draw_table is None else draw_table.numel(), out['points'], out['counts'], out['n_lost'], ws,
                   ws.numel())
        return out

    def pylisa_qext(self, x, m):
        """
        The reference pylisa's calc_qext(x, m) for every size parameter of `x` and one complex refractive index m
        (lss_pylisa_qext, current stream, no synchronisation).  Returns a CUDA float64 tensor of len(x).  The workspace
        (about 200 MB for the 2000 diameters of a MiniLisa at 0.903 um) is allocated for the call only.
        """
        x = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1))
        m = complex(m)
        n = int(x.shape[0])
        need = self.lib.lss_pylisa_qext_workspace_bytes(_ptr(x), n, m.real, m.imag)
        ws = torch.empty(max(int(need), 0), dtype=torch.uint8, device=self.device)
        out = torch.empty((n,), dtype=torch.float64, device=self.device)
        self._call('lss_pylisa_qext', _ptr(x), n, m.real, m.imag, out, ws, ws.numel())
        return out

    def pylisa_batch(self, points, cloud_offsets, rain_rate, aug_key, aug_call, dist_key=None, dist_call=None,
                     mini=False, alpha=None, qext_table=None, ran_uncer=0.06, min_range=1.5, max_range=200.0,
                     b_div=0.5e-3, ref_r=0.0, counts=None, want_record=False):
        """
        The reference pylisa's Lisa.augment(pc, Rr) (mini=False, 5 columns) or MiniLisa.augment(pc, Rr) (4 columns) as
        one call per cloud on a batch of device-resident clouds (lss_pylisa_batch, current stream, no synchronisation).
        points: CUDA float64 (N, F), F >= 4; rain_rate, aug_key, aug_call, dist_key, dist_call, alpha: length-B host
        sequences (or scalars); alpha None: each cloud's MiniLisa.calc_alpha with the Marshall-Palmer law over
        qext_table, a CUDA float64 (n_d, 2) of (d [mm], qext).  counts: optional CUDA int32 (B,) valid rows per slot.
        Returns dict(points (N, 5 or 4) float64, alpha (B,) float64, status (B,) int32: 1 NaN particle count, 2 infinite;
        record (N, 3) int32 with want_record: ranges drawn, kept, Gaussian pairs rejected).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float64, (N, None), min_cols=4)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('qext_table', qext_table, self.device, torch.float64, (None, 2), optional=True)
        if alpha is None and qext_table is None:
            raise ValueError('alpha: give alpha per cloud or a qext_table')

        def per_cloud(v, dtype):
            return None if v is None else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=dtype), (B,)))
        rr, al = per_cloud(rain_rate, np.float64), per_cloud(alpha, np.float64)
        ak, ac, dk, dc = [per_cloud(v, np.uint64) for v in (aug_key, aug_call, dist_key, dist_call)]
        if not mini and (dk is None or dc is None):
            raise ValueError('dist_key and dist_call are required for Lisa (mini=False)')
        out = _outputs(None, self.device, points=((N, 4 if mini else 5), torch.float64), alpha=((B,), torch.float64),
                       status=((B,), torch.int32), record=want_record and ((N, 3), torch.int32))
        ws = self._scratch('pylisa', self.lib.lss_pylisa_batch_workspace_bytes(B))
        n_d = 0 if qext_table is None else int(qext_table.shape[0])
        self._call('lss_pylisa_batch', points, points.shape[1], _ptr(off), counts, B,
                   _lib.PYLISA_MINI if mini else 0, _ptr(rr), _ptr(al), qext_table, n_d, _ptr(ak), _ptr(ac), _ptr(dk),
                   _ptr(dc), float(ran_uncer), float(min_range), float(max_range), float(b_div), float(ref_r),
                   out['points'], out['alpha'], out['status'], out.get('record'), ws, ws.numel())
        return out

    def _lisa_average_params(self, B, model, alpha, range_scale, fixed_seed):
        """(alpha, range_scale, start state, its 630 words) of lisa_average_batch / lisa_average_cloud_batch, checked"""
        if model not in (0, 1):
            raise ValueError(f'model: expected 0 (average_augment) or 1 (goodin_augment), got {model}')
        al = np.ascontiguousarray(np.broadcast_to(np.asarray(alpha, dtype=np.float64), (B,)))
        sc = None
        if model == 1:
            if range_scale is None:
                raise ValueError('range_scale: Goodin needs (1 - exp(-Rr))**2 per cloud')
            sc = np.ascontiguousarray(np.broadcast_to(np.asarray(range_scale, dtype=np.float64), (B,)))
        start = LISA_SEED_STATE if fixed_seed else np.random.get_state()
        return al, sc, start, _mt_words(start, 'fixed_seed state' if fixed_seed else "NumPy's global generator", True)

    def lisa_average_batch(self, points, cloud_offsets, model, alpha, p_min, r_min=0.9, range_accuracy=0.09,
                           range_scale=None, fixed_seed=False):
        """
        LISA.average_augment (model 0: the fog, haze and spray modes, lisa.py:340-388) or LISA.goodin_augment (model 1,
        :391-443) on a batch of device-resident float64 clouds (lss_lisa_average_batch, current stream).  points: CUDA
        float64 (N, F), F >= 4, intensity in [0, 1]; alpha: per cloud (or one for all), LISA.alpha(LISA.Nd(D, Rr));
        p_min: 0.9 r_max^-2 (average) or that / pi (Goodin); range_scale: Goodin's (1 - exp(-Rr))**2 per cloud.  The
        detected rows draw NumPy's legacy Gaussians: without fixed_seed from the global generator, cloud after cloud (B
        augment calls in turn); with it, every cloud from np.random.seed(666).  The call synchronises once, for the copy
        of the final state, and sets NumPy's global state to it (as the last augment call leaves it).  Returns CUDA
        float64 (N, F + 2), the reference's pc_new of every cloud at its rows.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float64, (N, None), min_cols=4)
        al, sc, start, words = self._lisa_average_params(B, model, alpha, range_scale, fixed_seed)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((N, F + 2), torch.float64), state=((MT_GAUSS_WORDS,), torch.int32))
        ws = self._scratch('lisa_average', self.lib.lss_lisa_average_batch_workspace_bytes(N, B))
        self._call('lss_lisa_average_batch', points, F, _ptr(off), B, int(model), _ptr(al), _ptr(sc), float(p_min),
                   float(r_min), float(range_accuracy), 1 if fixed_seed else 0, _ptr(words), out['points'],
                   out['state'], ws, ws.numel())
        if B > 0:
            _set_mt_state(start, out['state'])
        return out['points']

    def lisa_average_cloud_batch(self, points, cloud_offsets, model, alpha, p_min, r_min=0.9, range_accuracy=0.09,
                                 range_scale=None, counts=None, apply=None, fixed_seed=False):
        """
        The dataset's LISA block (dense_dataset.py:713-746) with average_augment or goodin_augment on a batch of
        device-resident float32 clouds (lss_lisa_average_cloud_batch, current stream): lisa_cloud_batch's conversions and
        layout, lisa_average_batch's models and Gaussians.  points: CUDA float32 (N, F), F >= 5, intensity in [0, 255];
        counts: optional CUDA int32 (B,) valid rows per slot; apply: optional length-B booleans (clouds with False are
        copied through and draw nothing).  Synchronises once and sets NumPy's global state as B augment calls on the
        applied clouds leave it.  Returns dict(points (N, F) float32: each cloud's detected rows at the front of its slot,
        label 2 in column 4; counts (B,) int32; n_lost (B,) int32).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=5)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        al, sc, start, words = self._lisa_average_params(B, model, alpha, range_scale, fixed_seed)
        ap = None if apply is None else np.ascontiguousarray(np.asarray(apply, dtype=bool).reshape(B), dtype=np.uint8)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((N, F), torch.float32), counts=((B,), torch.int32),
                       n_lost=((B,), torch.int32), state=((MT_GAUSS_WORDS,), torch.int32))
        ws = self._scratch('lisa_average', self.lib.lss_lisa_average_cloud_batch_workspace_bytes(N, B))
        self._call('lss_lisa_average_cloud_batch', points, F, _ptr(off), counts, B, _ptr(ap), int(model), _ptr(al),
                   _ptr(sc), float(p_min), float(r_min), float(range_accuracy), 1 if fixed_seed else 0, _ptr(words),
                   out['points'], out['counts'], out['n_lost'], out['state'], ws, ws.numel())
        state = out.pop('state')
        if B > 0 and (ap is None or ap.any()):
            _set_mt_state(start, state)
        return out

    def lisa_average_block_batch(self, points, cloud_offsets, model, alpha, p_min, choices, rate_candidate=None,
                                 r_min=0.9, range_accuracy=0.09, range_scale=None, counts=None):
        """
        The dataset's whole LISA block (dense_dataset.py:713-746) with average_augment or goodin_augment on a batch of
        device-resident float32 clouds, its per-sample draws included (lss_lisa_average_block_batch, current stream):
        each cloud draws its coin flip np.random.choice(choices), then, when applied and rate_candidate is given, the
        rain rate np.random.choice(rainfall_rates), then its detected rows' Gaussians, all from NumPy's global
        generator in batch order.  alpha (and Goodin's range_scale): one value per candidate rate (at most 64);
        rate_candidate: for each entry of the rate list the candidate its value maps to (None: no rate is drawn, the
        dataset's sampling other than 'uniform', and every applied cloud takes candidate 0).  points, counts, r_min,
        range_accuracy and p_min as lisa_average_cloud_batch.  Synchronises once and sets NumPy's global state as B
        calls of the block leave it.  Returns dict(points (N, F) float32: each cloud's kept rows at the front of its
        slot; counts (B,) int32; n_lost (B,) int32; draws: host int64 (B, 4), per cloud the rate index drawn (-1 not
        applied, 0 without a rate draw), the raw word its Gaussians start at (from word 0 of the start key), whether
        a cached Gaussian waited there, and the Gaussians it took).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=5)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        ch = np.ascontiguousarray(np.asarray(choices).reshape(-1) != 0, dtype=np.uint8)
        if not 1 <= ch.shape[0] <= 64:
            raise ValueError(f'choices: expected 1 to 64 entries, got {ch.shape[0]}')
        K = np.asarray(alpha).size
        if not 1 <= K <= 64:
            raise ValueError(f'alpha: expected 1 to 64 candidate rates, got {K}')
        rc = None if rate_candidate is None else np.ascontiguousarray(rate_candidate, dtype=np.int32).reshape(-1)
        if rc is not None and (rc.shape[0] == 0 or rc.min() < 0 or rc.max() >= K):
            raise ValueError(f'rate_candidate: expected a non-empty list of candidates in [0, {K})')
        al, sc, start, words = self._lisa_average_params(K, model, alpha, range_scale, False)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((N, F), torch.float32), counts=((B,), torch.int32),
                       n_lost=((B,), torch.int32))
        host = torch.empty(MT_GAUSS_WORDS // 2 + 4 * B, dtype=torch.int64, device=self.device)   # state, then draws
        n_rates = 0 if rc is None else rc.shape[0]
        ws = self._scratch('lisa_block', self.lib.lss_lisa_average_block_batch_workspace_bytes(N, B, K, n_rates))
        self._call('lss_lisa_average_block_batch', points, F, _ptr(off), counts, B, _ptr(ch), ch.shape[0], _ptr(rc),
                   n_rates, int(model), _ptr(al), _ptr(sc), K, float(p_min), float(r_min), float(range_accuracy),
                   _ptr(words), out['points'], out['counts'], out['n_lost'], host[MT_GAUSS_WORDS // 2:],
                   host[:MT_GAUSS_WORDS // 2], ws, ws.numel())
        draws = np.zeros((0, 4), np.int64)
        if B > 0:
            host = host.cpu()                                      # the one synchronisation: state and draws
            _set_mt_state(start, host[:MT_GAUSS_WORDS // 2].view(torch.int32))
            draws = host[MT_GAUSS_WORDS // 2:].numpy().reshape(B, 4)
        out['draws'] = draws
        return out

    def _pa_args(self, points, cloud_offsets, planes, nparts, box_offsets, counts):
        """(off, B, boff, M) of the arguments pa_partition_batch and pa_apply_batch share, checked"""
        off, B, N = _cloud_offsets(cloud_offsets)
        boff, B_boxes, M = _cloud_offsets(box_offsets, 'box_offsets')
        if B_boxes != B:
            raise ValueError(f'box_offsets: {B_boxes + 1} entries for {B} clouds')
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        _check_tensor('planes', planes, self.device, torch.float64, (M, 9, 6, 4))
        _check_tensor('nparts', nparts, self.device, torch.int32, (M,))
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        return off, B, boff, M

    def pa_partition_batch(self, points, cloud_offsets, planes, nparts, box_offsets, boxes_f64, counts=None):
        """
        PA-AUG's partition (lss_pa_partition_batch, current stream, no synchronisation): which rows of every cloud lie
        in which (box, part).  points: CUDA float32 (N, F), F >= 3; planes: CUDA float64 (M, 9, 6, 4) and nparts CUDA
        int32 (M,) from pa_aug.plan.box_planes; box_offsets: (B + 1) host int64.  Returns the CUDA int32
        (8 * M + B,) class totals (cloud b's classes at 8 * box_offsets[b] + b: 8 per box, then its background).
        The partition stays in this engine's PA-AUG workspace for pa_apply_batch.
        """
        off, B, boff, M = self._pa_args(points, cloud_offsets, planes, nparts, box_offsets, counts)
        need = self.lib.lss_pa_partition_workspace_bytes(_ptr(off), _ptr(boff), B)
        if need < 0:
            raise ValueError('bad cloud_offsets / box_offsets (at most 256 boxes per cloud)')
        totals = torch.empty((8 * M + B,), dtype=torch.int32, device=self.device)
        ws = self._scratch('pa', need)
        self._pa_part_bytes = int(need)
        self._call('lss_pa_partition_batch', points, points.shape[1], _ptr(off), counts, B, planes, nparts, _ptr(boff),
                   1 if boxes_f64 else 0, totals, ws, ws.numel())
        return totals

    def pa_apply_batch(self, points, cloud_offsets, planes, nparts, box_offsets, boxes_f64, class_start, n_members,
                       fps_segs, n_fps_rows, fps_jobs, n_fps_out, segs, steps, noise, normals, n_out, out_dtype,
                       counts=None):
        """
        PA-AUG's row work after the plan (lss_pa_apply_batch, current stream, no synchronisation), on the partition the
        last pa_partition_batch of this engine left: member lists, the FPS of the thinned parts, the output rows.
        Plan tables: CUDA tensors as include/lidar_snow_sim.h describes them.  Returns CUDA (n_out, 4) out_dtype
        (torch.float32 or torch.float64).
        """
        off, B, boff, M = self._pa_args(points, cloud_offsets, planes, nparts, box_offsets, counts)
        if out_dtype not in (torch.float32, torch.float64):
            raise ValueError(f'out_dtype: expected torch.float32 or torch.float64, got {out_dtype}')
        _check_tensor('class_start', class_start, self.device, torch.int64, (8 * M + B,))
        for name, t, cols in (('fps_segs', fps_segs, 6), ('fps_jobs', fps_jobs, 5), ('segs', segs, 6)):
            _check_tensor(name, t, self.device, torch.int64, (None, cols))
        for name, t, cols in (('steps', steps, 12), ('noise', noise, 4), ('normals', normals, 4)):
            _check_tensor(name, t, self.device, torch.float64, (None, cols))
        if self._pa_part_bytes is None:
            raise RuntimeError('pa_apply_batch needs the partition of a pa_partition_batch call on this engine first')
        need = self.lib.lss_pa_apply_workspace_bytes(_ptr(off), _ptr(boff), B, int(n_members), int(n_fps_rows),
                                                     int(n_fps_out))
        if need < 0:
            raise ValueError('bad PA-AUG plan sizes')
        ws = self._scratch('pa', need, keep=self._pa_part_bytes)     # the partition lives at the front
        out =torch.empty((int(n_out), 4), dtype=out_dtype, device=self.device)
        self._call('lss_pa_apply_batch', points, points.shape[1], _ptr(off), counts, B, planes, nparts, _ptr(boff),
                   1 if boxes_f64 else 0, class_start, int(n_members), fps_segs, fps_segs.shape[0], int(n_fps_rows),
                   fps_jobs, fps_jobs.shape[0], int(n_fps_out), segs, segs.shape[0], steps, noise, normals, int(n_out),
                   out, 1 if out_dtype == torch.float64 else 0, ws, ws.numel())
        return out

    def pa_fps_cloud_config(self, n_rows):
        """(cluster size, capacity) of lss_pa_fps_cloud_config on this engine's device: the cluster size a call whose
        largest on-chip cloud has n_rows rows uses (0 above the capacity), and the most rows an on-chip cloud may have"""
        cs, cap = ctypes.c_int(), ctypes.c_int64()
        _lib.check(self.lib.lss_pa_fps_cloud_config(self.device.index, int(n_rows), ctypes.byref(cs), ctypes.byref(cap)))
        return cs.value, cap.value

    def pa_fps_cloud_batch(self, points, cloud_offsets, k, start, counts=None):
        """
        farthest_point_sampling (part_aware_augmentation.py:197-209) over every whole cloud (lss_pa_fps_cloud_batch,
        current stream, no synchronisation).  points: CUDA float32 or float64 (N, F >= 3); counts: optional HOST int32
        (B,) rows per slot; k, start: host (B,) picks and first picks (the caller's np.random.randint(n_b)).  Returns
        dict(points (sum k, F) of points' dtype, cloud b's picked rows at the exclusive prefix of k; index CUDA int32
        (sum k,) the picks inside each cloud).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, (torch.float32, torch.float64), (N, None), min_cols=3)
        cnt = None if counts is None else np.ascontiguousarray(counts, dtype=np.int32).reshape(-1)
        kk = np.ascontiguousarray(k, dtype=np.int32).reshape(-1)
        s0 = np.ascontiguousarray(start, dtype=np.int32).reshape(-1)
        for name, a in (('counts', cnt), ('k', kk), ('start', s0)):
            if a is not None and a.shape[0] != B:
                raise ValueError(f'{name}: expected {B} entries, got {a.shape[0]}')
        f64 = 1 if points.dtype == torch.float64 else 0
        F = points.shape[1]
        K = int(kk.astype(np.int64).sum())
        out = _outputs(None, self.device, points=((K, F), points.dtype), index=((K,), torch.int32))
        with torch.cuda.device(self.device):
            need = self.lib.lss_pa_fps_cloud_workspace_bytes(_ptr(off), _ptr(cnt), _ptr(kk), B, f64)
        if need < 0:
            raise ValueError('bad cloud_offsets / counts / k (counts within the slots, k >= 1 for a cloud with rows)')
        ws = self._scratch('pa_fps', need)
        self._call('lss_pa_fps_cloud_batch', points, f64, F, _ptr(off), _ptr(cnt), B, _ptr(kk), _ptr(s0), out['points'],
                   out['index'], ws, ws.numel())
        return out

    def pa_noise_test_batch(self, points, cloud_offsets, k, n_draw_clouds=None, counts=None):
        """
        generate_noise_robustness_test (part_aware_augmentation.py:749-767) on B clouds in turn
        (lss_pa_noise_test_batch, current stream): per cloud np.random.choice(range(n_b), k_b, replace=False) and 4 k_b
        uniforms on NumPy's global RandomState, the kept rows in order then the noise rows.  points: CUDA float32 or
        float64 (N, F >= 4); counts: optional HOST int32 (B,) rows per slot; k: host (B,); only the first n_draw_clouds
        clouds (default B) draw.  Synchronises once and sets NumPy's global state (the cached Gaussian kept) as the
        draws leave it.  Returns dict(points CUDA float64 (sum n_b, 4), cloud b at the exclusive prefix of n_b;
        columns host int32 (B,): 4, or the first column whose range is not finite, after which nothing was drawn).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, (torch.float32, torch.float64), (N, None), min_cols=4)
        cnt = None if counts is None else np.ascontiguousarray(counts, dtype=np.int32).reshape(-1)
        kk = np.ascontiguousarray(k, dtype=np.int32).reshape(-1)
        for name, a in (('counts', cnt), ('k', kk)):
            if a is not None and a.shape[0] != B:
                raise ValueError(f'{name}: expected {B} entries, got {a.shape[0]}')
        D = B if n_draw_clouds is None else int(n_draw_clouds)
        n = np.diff(off) if cnt is None else cnt.astype(np.int64)
        words, start = _mt_state()
        tail = torch.empty(625 + B, dtype=torch.int32, device=self.device)      # state, columns: one copy back
        out = torch.empty((int(n.sum()), 4), dtype=torch.float64, device=self.device)
        need = self.lib.lss_pa_noise_test_workspace_bytes(_ptr(off), _ptr(cnt), _ptr(kk), B)
        if need < 0:
            raise ValueError('bad cloud_offsets / counts / k (counts within the slots, k in [0, count])')
        ws = self._scratch('pa_noise', need)
        self._call('lss_pa_noise_test_batch', points, 1 if points.dtype == torch.float64 else 0, points.shape[1],
                   _ptr(off), _ptr(cnt), B, _ptr(kk), D, _ptr(words), out, tail[625:], tail[:625], ws, ws.numel())
        h = tail.cpu().numpy()
        if B > 0:
            np.random.set_state(_mt_tuple(h[:625].view(np.uint32), start))
        return {'points': out, 'columns': h[625:].copy()}

    def pa_jitter_test_batch(self, points, cloud_offsets, out_offsets, sigma, counts=None):
        """
        jitter_robustness_test (part_aware_augmentation.py:775-778) on B clouds in turn (lss_pa_jitter_test_batch,
        current stream): np.random.normal(0, sigma, (n_b, 3)) from NumPy's global RandomState, cloud after cloud, added
        to x, y, z in float64 and stored in the rows' dtype.  points: CUDA float32 or float64 (N, F >= 3); counts:
        optional CUDA int32 (B,); out_offsets: host (B + 1) exact-size slots of n_b rows.  Synchronises once, for the
        final state, and sets NumPy's global state to it.  Returns (out_offsets[-1], F) of points' dtype.
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, (torch.float32, torch.float64), (N, None), min_cols=3)
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        ooff, B_out, n_out = _row_offsets(out_offsets, 'out_offsets')
        if B_out != B:
            raise ValueError(f'out_offsets: {B_out + 1} entries for {B} clouds')
        words, start = _mt_state(gauss=True)
        F = points.shape[1]
        out = _outputs(None, self.device, points=((n_out, F), points.dtype), state=((MT_GAUSS_WORDS,), torch.int32))
        ws = self._scratch('pa_jitter', self.lib.lss_pa_jitter_test_workspace_bytes(N, B))
        self._call('lss_pa_jitter_test_batch', points, 1 if points.dtype == torch.float64 else 0, F, _ptr(off), counts, B,
                   _ptr(ooff), float(sigma), _ptr(words), out['points'], out['state'], ws, ws.numel())
        if B > 0:
            _set_mt_state(start, out['state'])
        return out['points']

    def gt_collide_batch(self, boxes, box_offsets, n_gt, class_offsets, bits_offsets, max_pairs, n_pairs, n_classes):
        """
        GT sampling's collision test (lss_gt_collide_batch, current stream, no synchronisation).  boxes: CUDA float32
        (M, 11); box_offsets (B + 1,) / bits_offsets (B,) CUDA int64; n_gt (B,) / class_offsets (B, 9) CUDA int32.
        Returns (valid, bits): CUDA uint8 (M,) and (n_pairs,).
        """
        _check_tensor('n_gt', n_gt, self.device, torch.int32, (None,))
        B = n_gt.shape[0]
        _check_n_clouds(B)
        _check_tensor('boxes', boxes, self.device, torch.float32, (None, 11))
        _check_tensor('box_offsets', box_offsets, self.device, torch.int64, (B + 1,))
        _check_tensor('class_offsets', class_offsets, self.device, torch.int32, (B, 9))
        _check_tensor('bits_offsets', bits_offsets, self.device, torch.int64, (B,))
        valid = torch.empty((boxes.shape[0],), dtype=torch.uint8, device=self.device)
        bits = torch.empty((max(int(n_pairs), 1),), dtype=torch.uint8, device=self.device)
        self._call('lss_gt_collide_batch', B, int(n_classes), boxes, box_offsets, n_gt, class_offsets, bits_offsets,
                   int(max_pairs), bits, valid)
        return valid, bits[:int(n_pairs)]

    def gt_paste_batch(self, points, cloud_offsets, rm_boxes, rm_offsets, max_rm, ops, db, objects, object_shift,
                       n_object_rows, out_offsets, object_rows, n_out, counts=None):
        """
        GT sampling's row work, with the world flip / rotation / scaling (lss_gt_paste_batch, current stream, no
        synchronisation).  points: CUDA float32 (N, F); cloud_offsets (B + 1) host int64; the tables are CUDA tensors
        laid out as include/lidar_snow_sim.h describes them.  Returns (rows, counts): CUDA float32 (n_out, F) in the
        slots out_offsets, and CUDA int32 (B,).
        """
        off, B, N = _cloud_offsets(cloud_offsets)
        _check_tensor('points', points, self.device, torch.float32, (N, None), min_cols=3)
        F = points.shape[1]
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        _check_tensor('rm_boxes', rm_boxes, self.device, torch.float32)              # rows of 9, flat
        _check_tensor('rm_offsets', rm_offsets, self.device, torch.int64, (B + 1,))
        _check_tensor('ops', ops, self.device, torch.float32, (B, None, 3))
        _check_tensor('db', db, self.device, torch.float32, (None, F))
        _check_tensor('objects', objects, self.device, torch.int64, (None, 4))
        _check_tensor('object_shift', object_shift, self.device, torch.float64, (objects.shape[0], 4))
        _check_tensor('out_offsets', out_offsets, self.device, torch.int64, (B + 1,))
        _check_tensor('object_rows', object_rows, self.device, torch.int32, (B,))
        need = self.lib.lss_gt_paste_workspace_bytes(_ptr(off), B)
        if need < 0:
            raise ValueError('bad cloud_offsets')
        ws = self._scratch('gt_paste', need)
        out = torch.empty((int(n_out), F), dtype=torch.float32, device=self.device)
        out_counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        self._call('lss_gt_paste_batch', points, F, _ptr(off), counts, B, rm_boxes, rm_offsets, int(max_rm), ops,
                   ops.shape[1], db, objects, object_shift, objects.shape[0], int(n_object_rows), out_offsets,
                   object_rows, out, out_counts, ws, ws.numel())
        return out, out_counts

    def gather_push(self, points, counts, d_cloud_offsets, n_rows, world, rank, peer_points, peer_counts, mc_points=0,
                    mc_counts=0, blocks=0):
        """lss_gather_push on the current stream: write the kept rows of this rank's slot-compacted batch (+ counts) into
        every rank's gathered buffers (SURVEY.md 8e).  peer_points / peer_counts: per rank, a CUDA tensor mapping that
        rank's gathered buffer (world * n_rows, 5) float32 / (world * n_clouds,) int32 into this process (see
        distributed.BatchGather, which owns the symmetric allocations and the side stream)."""
        _check_tensor('d_cloud_offsets', d_cloud_offsets, self.device, torch.int64, (None,))
        B = d_cloud_offsets.shape[0] - 1
        _check_tensor('points', points, self.device, torch.float32, (None, 5))
        _check_tensor('counts', counts, self.device, torch.int32, (B,), optional=True)
        peer_points, peer_counts, world = list(peer_points), list(peer_counts), int(world)
        if len(peer_points) != world or len(peer_counts) != world:
            raise ValueError(f'peer_points / peer_counts: {len(peer_points)} / {len(peer_counts)} buffers for {world} ranks')
        for r in range(world):                  # mappings of the other ranks' buffers: any device
            _check_tensor(f'peer_points[{r}]', peer_points[r], None, torch.float32, (world * int(n_rows), 5))
            _check_tensor(f'peer_counts[{r}]', peer_counts[r], None, torch.int32, (world * B,))
        P = ctypes.c_void_p * world
        self._call('lss_gather_push', points, counts, d_cloud_offsets, B, int(n_rows), world, int(rank),
                   P(*[t.data_ptr() for t in peer_points]), P(*[t.data_ptr() for t in peer_counts]), mc_points or None,
                   mc_counts or None, int(blocks))

    def check(self):
        """Synchronise the current stream and raise the exception type the reference would have raised."""
        self._call('lss_check_async')

    def launch_count(self):
        return int(self.lib.lss_launch_count(self.h))

    def set_profiling(self, enable=True):
        _lib.check(self.lib.lss_set_profiling(self.h, 1 if enable else 0), self.h)

    def kernel_times(self, reset=True):
        """{kernel name: (total ms, launches)} measured with CUDA events on the launching stream (synchronises)."""
        torch.cuda.synchronize(self.device)
        n = 16                                        # every id the library can have; unused ids have no name
        ms = np.zeros(n, dtype=np.float64)
        calls = np.zeros(n, dtype=np.int64)
        _lib.check(self.lib.lss_kernel_times(self.h, 1 if reset else 0, _ptr(ms), _ptr(calls), n), self.h)
        names = [self.lib.lss_kernel_name(k).decode() for k in range(n)]
        return {names[k]: (float(ms[k]), int(calls[k])) for k in range(n) if names[k]}


_default_engines = {}


def default_engine(device=None):
    """Process-wide engine per device, created on first use (used by the reference-signature wrappers)."""
    if device is None:
        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    if device not in _default_engines:
        _default_engines[device] = SnowfallEngine(device)
    return _default_engines[device]

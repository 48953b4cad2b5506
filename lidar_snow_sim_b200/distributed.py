"""
Multi-GPU use of the engine: one process per GPU (torch.distributed, NCCL over NVLink/NVSwitch on the GPU box, gloo
in the CPU tests).  Clouds are independent (SURVEY.md 8e), so a batch is sharded over ranks by cloud with NO
data-path collective; the only exchange is the final all-gather that reassembles the augmented batch on every rank
(BASELINE.json configs[3]) -- and a consumer that lives on the same rank (a per-rank DataLoader) can skip even that.

Layout of the gathered batch: fixed stride per rank.  Every rank contributes a (slot_rows, 5) float32 buffer in which
cloud b occupies rows local_offsets[b] .. local_offsets[b] + counts[b] (the slot-compacted output of
SnowfallEngine.snowfall_batch), padded to the largest rank's row count, plus its per-cloud counts and stats padded to
the largest rank's cloud count.
"""
import numpy as np
import torch
import torch.distributed as dist


def bind_host_to_gpu(device: int = 0):
    """Pin this process to the CPUs of the NUMA node the GPU hangs off (first-touch then places pinned host buffers
    there), so that one rank's PCIe traffic does not cross the socket interconnect.  Call before allocating host
    buffers.  Returns the cpu list used, or None when the topology cannot be read (no-op)."""
    import os
    try:
        bus = torch.cuda.get_device_properties(device)
        pci = f'{bus.pci_domain_id:04x}:{bus.pci_bus_id:02x}:{bus.pci_device_id:02x}.0'
        with open(f'/sys/bus/pci/devices/{pci}/local_cpulist') as f:
            txt = f.read().strip()
        cpus = set()
        for part in txt.split(','):
            if '-' in part:
                lo, hi = part.split('-')
                cpus.update(range(int(lo), int(hi) + 1))
            elif part:
                cpus.add(int(part))
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return sorted(cpus)
    except Exception:
        return None


def shard_range(n_clouds: int, rank: int, world: int):
    """Contiguous block partition of cloud indices: rank r owns [start, stop)."""
    base, rem = divmod(n_clouds, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def all_gather_augmented(points, local_offsets, counts, stats, group=None):
    """
    points: (N_local, 5) float32 slot-compacted rows; local_offsets: host int64 (B_local + 1); counts: (B_local,) int32;
    stats: (B_local, 4) float64.  Works for ragged shards (different N_local / B_local per rank).
    Returns dict(points (world, N_max, 5), counts (world, B_max), stats (world, B_max, 4), offsets list per rank,
                 n_clouds list per rank); `cloud(r, b)` slices are `points[r, offsets[r][b] : offsets[r][b] + counts[r, b]]`.
    One all-gather for the rows (the only large message), two small ones for counts / stats, one for the shapes.
    """
    world = dist.get_world_size(group)
    dev = points.device
    local_offsets = np.ascontiguousarray(local_offsets, dtype=np.int64)
    b_local = local_offsets.shape[0] - 1
    n_local = int(local_offsets[-1])
    meta = torch.tensor([n_local, b_local], dtype=torch.int64, device=dev)
    metas = torch.empty((world * 2,), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(metas, meta, group=group)
    metas_h = metas.cpu().numpy().reshape(world, 2)
    n_max, b_max = int(metas_h[:, 0].max()), int(metas_h[:, 1].max())

    def padded(t, rows, tail_shape, dtype):
        if t.shape[0] == rows:
            return t.contiguous()
        buf = torch.zeros((rows,) + tail_shape, dtype=dtype, device=dev)
        buf[:t.shape[0]] = t
        return buf

    p = padded(points, n_max, (5,), torch.float32)
    c = padded(counts, b_max, (), torch.int32)
    s = padded(stats, b_max, (4,), torch.float64)
    o = padded(torch.from_numpy(local_offsets[:-1].copy()).to(dev), b_max, (), torch.int64)
    # outputs are the concatenation along dim 0 (the layout every backend accepts), viewed per rank afterwards
    g_p = torch.empty((world * n_max, 5), dtype=torch.float32, device=dev)
    g_c = torch.empty((world * b_max,), dtype=torch.int32, device=dev)
    g_s = torch.empty((world * b_max, 4), dtype=torch.float64, device=dev)
    g_o = torch.empty((world * b_max,), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(g_p, p, group=group)
    dist.all_gather_into_tensor(g_c, c, group=group)
    dist.all_gather_into_tensor(g_s, s, group=group)
    dist.all_gather_into_tensor(g_o, o, group=group)
    g_p = g_p.view(world, n_max, 5)
    g_c = g_c.view(world, b_max)
    g_s = g_s.view(world, b_max, 4)
    g_o_h = g_o.cpu().numpy().reshape(world, b_max)
    return dict(points=g_p, counts=g_c, stats=g_s, offsets=[g_o_h[r, :metas_h[r, 1]] for r in range(world)],
                n_clouds=[int(v) for v in metas_h[:, 1]])


def unpack_clouds(gathered):
    """Host-side view of a gathered batch as a flat list of per-cloud (count, 5) tensors in global cloud order."""
    out = []
    counts = gathered['counts'].cpu().numpy()
    for r, nb in enumerate(gathered['n_clouds']):
        for b in range(nb):
            o = int(gathered['offsets'][r][b])
            out.append(gathered['points'][r, o:o + int(counts[r, b])])
    return out


class ShardedAugmenter:
    """
    Batch-level driver: every rank augments its contiguous block of the global batch on its own GPU and (optionally)
    all ranks exchange the results.  `augment_fn(points, offsets, orders) -> dict(points, counts, stats)` is
    SnowfallEngine.snowfall_batch bound to a table set (tests pass a CPU stand-in to exercise the plumbing on gloo).
    """

    def __init__(self, augment_fn, group=None):
        self.augment_fn = augment_fn
        self.group = group

    def run(self, clouds, orders, device, gather=True):
        world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        lo, hi = shard_range(len(clouds), rank, world)
        mine = clouds[lo:hi]
        off = np.concatenate([[0], np.cumsum([c.shape[0] for c in mine])]).astype(np.int64)
        if len(mine):
            pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(mine), dtype=np.float32)).to(device)
        else:
            pts = torch.zeros((0, 5), dtype=torch.float32, device=device)
        res = self.augment_fn(pts, off, np.asarray(orders[lo:hi], dtype=np.int32).reshape(-1, 64))
        if not gather:
            return res, (lo, hi)
        return all_gather_augmented(res['points'], off, res['counts'], res['stats'], group=self.group), (lo, hi)


class BatchGather:
    """
    The all-gather of BASELINE.json configs[3] for a stream of steps: every rank contributes its fixed-stride
    augmented batch ((n_rows, 5) float32, slot-compacted) + per-cloud counts, double-buffered so that the exchange of
    step k overlaps the kernels of step k + 1.

    kind 'push' (default with an engine and usable symmetric memory): the gathered buffers are symmetric allocations; each
                rank writes the KEPT rows of its batch into every rank's buffer with the engine's own kernel
                (lss_gather_push, csrc/gather.cu: peer-to-peer stores over NVLink, or one multicast store per 16 bytes
                when the allocation has an NVLS mapping) on a high-priority side stream.  Needs `cloud_offsets`.
    kind 'ce'   the same buffers, whole slots pushed with peer-to-peer device copies (copy engines, no SM).
    kind 'nccl' dist.all_gather_into_tensor(async_op=True) on NCCL's stream (also what the gloo CPU tests exercise); its
                SM-resident channels compete with the latency-bound beam kernels.

    Completion: `wait(j)` makes the caller's stream wait for THIS rank's outgoing copies of buffer j; a consumer that
    reads a gathered buffer needs a barrier across ranks first (bench.py brackets end with one).  LSS_GATHER=nccl|ce
    overrides the choice.
    """

    def __init__(self, n_rows, n_clouds, device, depth=2, group=None, kind=None, engine=None, cloud_offsets=None):
        import os
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.n_rows, self.n_clouds, self.depth = int(n_rows), int(n_clouds), depth
        self.device = device
        on_gpu = getattr(device, 'type', 'cpu') == 'cuda'
        can_push = on_gpu and engine is not None and cloud_offsets is not None
        kind = kind or os.environ.get('LSS_GATHER') or ('push' if can_push else ('ce' if on_gpu else 'nccl'))
        if kind == 'push' and not can_push:
            kind = 'ce'
        self.pending = [None] * depth
        self.kind = 'nccl'
        self.points = self.counts = None
        self.engine = engine
        self.fallback_reason = None
        self.multicast = False
        if kind in ('ce', 'push'):
            try:
                self._init_ce()
                self.kind = kind
                if kind == 'push':
                    self._init_push(cloud_offsets)
            except Exception as exc:                      # symmetric memory unavailable: fall back, say so
                self.fallback_reason = f'{type(exc).__name__}: {exc}'
                self.kind = 'nccl'
        if self.kind == 'nccl':
            self.points = [torch.empty((self.world * self.n_rows, 5), dtype=torch.float32, device=device)
                           for _ in range(depth)]
            self.counts = [torch.empty((self.world * self.n_clouds,), dtype=torch.int32, device=device)
                           for _ in range(depth)]

    def _init_ce(self):
        import torch.distributed._symmetric_memory as symm_mem
        grp = self.group if self.group is not None else dist.group.WORLD
        self.points, self.counts, self._peer_pts, self._peer_cnt, self._mc = [], [], [], [], []
        for _ in range(self.depth):
            p = symm_mem.empty((self.world * self.n_rows, 5), dtype=torch.float32, device=self.device)
            c = symm_mem.empty((self.world * self.n_clouds,), dtype=torch.int32, device=self.device)
            hp = symm_mem.rendezvous(p, grp)
            hc = symm_mem.rendezvous(c, grp)
            self.points.append(p)
            self.counts.append(c)
            self._peer_pts.append([hp.get_buffer(r, (self.world * self.n_rows, 5), torch.float32)
                                   for r in range(self.world)])
            self._peer_cnt.append([hc.get_buffer(r, (self.world * self.n_clouds,), torch.int32)
                                   for r in range(self.world)])
            self._mc.append((int(getattr(hp, 'multicast_ptr', 0) or 0), int(getattr(hc, 'multicast_ptr', 0) or 0)))
        # one side stream per peer: the world - 1 pushes of a step run on different copy engines at the same time (one
        # stream would serialise them)
        self._side = [torch.cuda.Stream(device=self.device) for _ in range(max(1, self.world))]
        self._done = [[torch.cuda.Event() for _ in range(max(1, self.world))] for _ in range(self.depth)]
        self._ready = torch.cuda.Event()

    def _init_push(self, cloud_offsets):
        import ctypes
        import os
        import numpy as np
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        assert off.shape[0] == self.n_clouds + 1 and int(off[-1]) == self.n_rows
        self._d_off = torch.from_numpy(off).to(self.device)
        P = ctypes.c_void_p * self.world
        self._pp = [P(*[t.data_ptr() for t in self._peer_pts[j]]) for j in range(self.depth)]
        self._pc = [P(*[t.data_ptr() for t in self._peer_cnt[j]]) for j in range(self.depth)]
        use_mc = os.environ.get('LSS_GATHER_MULTICAST', '1') != '0'
        self.multicast = bool(use_mc and all(m[0] and m[1] for m in self._mc))
        self.blocks = int(os.environ.get('LSS_GATHER_BLOCKS', '0'))
        try:
            hi = torch.cuda.Stream.priority_range()[1]     # (least, greatest) = (0, -1) on current GPUs
        except Exception:
            hi = -1
        self._push_stream = torch.cuda.Stream(device=self.device, priority=hi)
        self._push_done = [torch.cuda.Event() for _ in range(self.depth)]

    def _start_push(self, j, points, counts):
        from . import _lib
        eng = self.engine
        cur = torch.cuda.current_stream(self.device)
        self._ready.record(cur)
        st = self._push_stream
        mcp, mcc = self._mc[j] if self.multicast else (0, 0)
        with torch.cuda.stream(st):
            st.wait_event(self._ready)
            rc = eng.lib.lss_gather_push(eng.h, points.data_ptr(), counts.data_ptr(), self._d_off.data_ptr(), self.n_clouds,
                                         self.n_rows, self.world, self.rank, self._pp[j], self._pc[j], mcp or None, mcc or None,
                                         self.blocks, st.cuda_stream)
            _lib.check(rc, eng.h)
            self._push_done[j].record(st)
        self.pending[j] = (points, counts)                 # the kernel reads them: keep them alive until wait(j)

    def start(self, j, points, counts):
        """Enqueue the exchange of this rank's (points, counts) into buffer j of every rank."""
        if self.kind == 'push':
            return self._start_push(j, points, counts)
        if self.kind == 'nccl':
            self.pending[j] = [dist.all_gather_into_tensor(self.points[j], points, group=self.group, async_op=True),
                               dist.all_gather_into_tensor(self.counts[j], counts, group=self.group, async_op=True)]
            return
        cur = torch.cuda.current_stream(self.device)
        self._ready.record(cur)
        r0, r1 = self.rank * self.n_rows, (self.rank + 1) * self.n_rows
        c0, c1 = self.rank * self.n_clouds, (self.rank + 1) * self.n_clouds
        for k in range(self.world):                        # start with the right-hand neighbour: spreads the NVSwitch load
            r = (self.rank + 1 + k) % self.world
            st = self._side[k]
            with torch.cuda.stream(st):
                st.wait_event(self._ready)
                self._peer_pts[j][r][r0:r1].copy_(points, non_blocking=True)
                self._peer_cnt[j][r][c0:c1].copy_(counts, non_blocking=True)
                self._done[j][k].record(st)
        self.pending[j] = True

    def wait(self, j):
        if self.pending[j] is None:
            return
        if self.kind == 'nccl':
            for wk in self.pending[j]:
                wk.wait()
        elif self.kind == 'push':
            torch.cuda.current_stream(self.device).wait_event(self._push_done[j])
        else:
            cur = torch.cuda.current_stream(self.device)
            for ev in self._done[j]:
                cur.wait_event(ev)
        self.pending[j] = None

    def wait_all(self):
        for j in range(self.depth):
            self.wait(j)

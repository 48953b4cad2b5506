"""What the benchmark scripts under tools/ share: the card a number was measured on, per-call times, per-kernel times,
registers and spills from ptxas, and the rank setup of the torchrun tools.  Every helper that reads or times the GPU
raises when there is no CUDA device: a measurement path that finds no GPU fails, it does not fall back."""
import contextlib
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
from lidar_snow_sim_b200 import build                                           # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: this measurement needs a GPU')


def card(index=0):
    """The card's name and power limit in W, read now: they belong beside every absolute number measured on it."""
    _need_gpu()
    return dict(name=torch.cuda.get_device_name(index), power_limit_w=bench.power_limit_w(index))


def time_calls(fn, runs, warmup):
    """Milliseconds of each of `runs` calls of fn() after `warmup` untimed ones: a host clock around fn() and the device
    synchronise that follows it, so each time includes the call's work on the device."""
    _need_gpu()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return ms


def median_min_max(ms):
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def _kernel_name(name):
    name = re.sub(r'\(.*', '', name.replace('(anonymous namespace)::', ''))
    return name.removeprefix('void ').strip()[:60]


def kernel_ms(fn):
    """{kernel name: ms} of the device activities of one fn() under torch.profiler (launches of one name summed).  Run
    it apart from the timed calls: tracing slows the host."""
    _need_gpu()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = _kernel_name(e.key)
            out[name] = round(out.get(name, 0.0) + e.device_time_total / 1e3, 4)
    return out


def ptxas(cu_name, kernels):
    """{kernel: {registers, spill_bytes}} of the kernels of csrc/<cu_name> whose names start with one of `kernels`, from
    `-Xptxas -v` with the library's own flags for sm_90a (compiled into a temporary directory; needs no GPU)."""
    nvcc = build.find_nvcc()
    flags = [f for f in build.NVCC_FLAGS if f != '--shared']
    with tempfile.TemporaryDirectory() as tmp:
        log = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', '-o', os.path.join(tmp, 'k.o'),
                                               os.path.join(build.CSRC, cu_name)],
                             capture_output=True, text=True, check=True).stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    names = subprocess.run(['c++filt'], input='\n'.join(entries), capture_output=True, text=True,
                           check=True).stdout.splitlines()           # demangled as torch.profiler names them
    names = dict(zip(entries, map(_kernel_name, names)))
    res, name, spill = {}, None, 0
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = names[m.group(1)]
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and name:
            spill = int(m.group(1)) + int(m.group(2))
        m = re.search(r'Used (\d+) registers', line)
        if m and name:
            if name.startswith(tuple(kernels)):
                res[name] = {'registers': int(m.group(1)), 'spill_bytes': spill}
            name = None                   # a spill line after this one belongs to a called function
    return res


def init_ranks():
    """(world, rank, local_rank, device) of this process; under torchrun it also joins the NCCL process group."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if 'WORLD_SIZE' in os.environ:
        import torch.distributed as dist
        dist.init_process_group('nccl', device_id=dev)
    return world, rank, local, dev


@contextlib.contextmanager
def env(**vars):
    """Set these environment variables inside the block and restore the previous values after it."""
    old = {k: os.environ.get(k) for k in vars}
    os.environ.update(vars)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v

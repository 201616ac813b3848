"""What the measurement scripts share: the card line every number goes out with, the two timers, the distributed
barrier, and random pair predictions synthesised directly in device memory."""
import subprocess
import time

import numpy as np
import torch
import torch.distributed as dist


def card(device=None):
    """'name, power limit, SM clock, max SM clock' of the GPU being measured (`device`, default the current one), from one
    read-only nvidia-smi query; the device name and 'power limit unknown' when the query fails."""
    index = torch.device(device).index if device is not None else None
    if index is None:
        index = torch.cuda.current_device()
    p = torch.cuda.get_device_properties(index)
    # selected by PCI address: CUDA_VISIBLE_DEVICES renumbers torch's devices but not nvidia-smi's
    bus = f'{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0'
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                            '-i', bus], capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pass
    return f'{torch.cuda.get_device_name(index)}, power limit unknown'


def events_ms(fn, iters, warmup):
    """ms per call of `fn`: CUDA events on the current stream around `iters` calls, after `warmup` calls and a synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def wall_ms(fn, iters, warmup):
    """ms per call of `fn`: the host clock around `iters` calls and the device synchronise that ends them, after `warmup`
    calls and a synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / iters


def barrier_sync():
    """Waits for this rank's device work, then for every rank when a process group is initialised."""
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()


def synth_on_device(n, edges, H, W, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    E = len(edges)
    off = torch.tensor([0.0, 0.0, 3.0], device=dev)
    ts = torch.from_numpy(np.int32([[H, W]] * E))
    mk = lambda: torch.randn((E, H, W, 3), generator=g, device=dev) + off
    cf = lambda: 1 + 5 * torch.rand((E, H, W), generator=g, device=dev)
    return dict(view1=dict(idx=[int(i) for i, j in edges], instance=[str(i) for i, j in edges], true_shape=ts),
                view2=dict(idx=[int(j) for i, j in edges], instance=[str(j) for i, j in edges], true_shape=ts),
                pred1=dict(pts3d=mk(), conf=cf()), pred2=dict(pts3d_in_other_view=mk(), conf=cf()), loss=None)

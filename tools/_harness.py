"""What every tools/bench_*.py shares: the record of the card a run measured on, and the timers.

A number is only worth something beside the card it was measured on, so card() is read in the same run.  Each timer
refuses to run without CUDA rather than time something else.
"""
import statistics
import subprocess
import time

import torch


def card(device=None):
    """{"name", "power_limit", "sm_clock", "max_sm_clock"} of the GPU this process measures on (the current device by
    default), as nvidia-smi reports them.  The card is selected by its UUID: nvidia-smi's indices ignore
    CUDA_VISIBLE_DEVICES, so on a multi-GPU host an index can name a card the run did not use.  A read-only query; on
    any failure the record holds the torch device name and an "error" instead of raising."""
    props = torch.cuda.get_device_properties(torch.cuda.current_device() if device is None else device)
    try:
        out = subprocess.run(["nvidia-smi", f"--id=GPU-{props.uuid}",
                              "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30, check=True).stdout
        name, power, sm, max_sm = (f.strip() for f in out.strip().split(","))
        return {"name": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": max_sm}
    except (OSError, subprocess.SubprocessError, ValueError) as e:
        return {"name": props.name, "error": f"nvidia-smi: {type(e).__name__}: {e}"}


def _need_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("the benchmark timers measure on a CUDA device; none is visible")


def events_ms(fn, reps, warmup, sync=False):
    """Mean milliseconds per fn() call: warmup calls, then one CUDA event pair around reps calls.  With sync, a device
    synchronise between the two opens the window on an idle device; without, the window opens once the warm-up calls
    have run, so launches shorter than their enqueue still find work queued."""
    _need_cuda()
    for _ in range(warmup):
        fn()
    if sync:
        torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def median_events_s(fn, reps, warmup=1):
    """Median seconds of one fn() call over reps calls, each between its own CUDA event pair, after warmup calls."""
    _need_cuda()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return statistics.median(ts)


def median_wall_s(fn, reps, calls=1, warmup=1, samples=None):
    """Median over reps windows of the host seconds per fn() call, each window `calls` calls closed by a device
    synchronise, after warmup calls and a synchronise.  samples, a list, also receives every window's value."""
    _need_cuda()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) / calls)
    if samples is not None:
        samples.extend(ts)
    return statistics.median(ts)


def graph_us(fn, reps, replays):
    """Device microseconds per fn() call: after one eager call, reps calls captured in one CUDA graph, replayed once,
    then timed by one event pair over `replays` replays (launch gaps included, Python's enqueue cost not)."""
    _need_cuda()
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        keep = [fn() for _ in range(reps)]   # noqa: F841  every call's outputs stay allocated for the whole graph
    return 1e3 * events_ms(g.replay, replays, 1, sync=True) / reps

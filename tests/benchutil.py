"""Timing and device helpers shared by the bench scripts (not a pytest file)."""
import subprocess
import warnings

import torch


def card():
    """the GPU's name, power limit and maximum SM clock, as nvidia-smi reports them"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                                     # the numbers still stand; say what is missing
        return dict(gpu=torch.cuda.get_device_name(), power_limit=f'not read ({e})')


def device_line():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        q = f'nvidia-smi unavailable ({e!r})'
    return f'device: {q}'


def timed(fn, steps, warmup):
    """ms per call of fn over `steps` calls after `warmup`, by CUDA events"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def time_call(fn, min_ms):
    """ms per call: CUDA events over a window of at least min_ms, after warm-up"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    n = max(3, int(min_ms / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def count_syncs(fn):
    """host synchronisations fn makes, as torch's sync debug mode reports them"""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum('synchroniz' in str(m.message) for m in w)

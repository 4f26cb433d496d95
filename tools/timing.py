"""The timer and the card line the timing scripts share."""
import subprocess

import numpy as np
import torch

_l2_flush = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2


def timeit(fn, warm=3, it=10, flush=True):
    """(median, minimum) in ms of `it` calls of fn after `warm` untimed ones, from CUDA events around each call.  With
    flush, the L2 is cleared before every timed call by overwriting a 256 MB buffer outside the timed window."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(it):
        if flush:
            _l2_flush.add_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def card():
    """The card's name, power limit, maximum and current SM clock, from a read-only nvidia-smi query."""
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()

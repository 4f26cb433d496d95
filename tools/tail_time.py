"""Where the k = 1 sweep's tail goes on C3 (fused Chamfer + Hausdorff of two 10^6-point fp32 clouds, bench.py's seeds).

Prints, after the card's name and power limit:
  * the C3 step time the way bench.py times it (L2 flushed before every step, CUDA events around the call);
  * the library's per-stage CUDA-event times (`search` = nn1_kernel, `search_far` = nn1_far_kernel + nn1_vfar_kernel);
  * from a torch.profiler trace of a few steps: the durations of nn1_kernel, nn1_far_kernel and nn1_vfar_kernel and
    the gap from the end of nn1_kernel to the end of the step's last kernel (the tail);
  * n_far of both directions: the queries the main pass's 3 x 3 x 3 cells could not settle.

`python tools/tail_time.py [out_dir] [steps]`: the Chrome trace goes to <out_dir>/tail_trace.json (default: a new
temporary directory, so that nothing is written into the repository)."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from timing import card
import pcu_b200 as pcu

out_dir = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp(prefix="pcu_tail_")
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 200
os.makedirs(out_dir, exist_ok=True)
print(card(), flush=True)

rng = np.random.default_rng(1000)   # bench.py's C3 clouds (rank 0)
x = torch.from_numpy(rng.random((1000000, 3), dtype=np.float32)).cuda()
y = torch.from_numpy(rng.random((1000000, 3), dtype=np.float32)).cuda()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
stream = torch.cuda.current_stream().cuda_stream
dev = torch.cuda.current_device()

for s in range(5):
    flush.fill_(1)
    pcu.chamfer_distance(x, y)
torch.cuda.synchronize()
a = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
b = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
for s in range(steps):
    flush.fill_(s & 0xff)
    a[s].record(); pcu.chamfer_distance(x, y); b[s].record()
torch.cuda.synchronize()
ms = np.array([p.elapsed_time(q) for p, q in zip(a, b)])
print("C3 step: mean %.4f ms  median %.4f  min %.4f  (%d steps)" % (ms.mean(), np.median(ms), ms.min(), steps), flush=True)

internal = pcu._pcu_internal
internal._set_profiling(dev, stream, True)
stage = {}
reps = 30
for s in range(reps):
    flush.fill_(s & 0xff)
    pcu.chamfer_distance(x, y)
    torch.cuda.synchronize()
    for key, val in internal._last_profile(dev, stream).items():
        stage[key] = stage.get(key, 0.0) + val / reps
internal._set_profiling(dev, stream, False)
print("stage_ms:", json.dumps({k: round(v, 5) for k, v in stage.items()}), flush=True)

trace = os.path.join(out_dir, "tail_trace.json")
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for s in range(20):
        flush.fill_(s & 0xff)
        pcu.chamfer_distance(x, y)
    torch.cuda.synchronize()
prof.export_chrome_trace(trace)
with open(trace) as f:
    kernels = sorted((e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
names = ("nn1_kernel", "nn1_far_kernel", "nn1_vfar_kernel")
per = {k: [] for k in names}
gaps = []
for i, e in enumerate(kernels):
    if "nn1_kernel" not in e["name"]:
        continue
    step_end = e["ts"] + e["dur"]
    for f in kernels[i + 1:]:
        if "at::native" in f["name"] or "nn1_kernel" in f["name"]:
            break   # the next step's L2 flush
        step_end = f["ts"] + f["dur"]
        for k in names[1:]:
            if k in f["name"]:
                per[k].append(f["dur"])
    per["nn1_kernel"].append(e["dur"])
    gaps.append(step_end - (e["ts"] + e["dur"]))
for k in names:
    print("%-16s median %.2f us  min %.2f  (%d)" % (k, np.median(per[k]), np.min(per[k]), len(per[k])))
print("tail (end of nn1_kernel -> end of step): median %.2f us  min %.2f  max %.2f" % (np.median(gaps), np.min(gaps), np.max(gaps)))
print("trace:", trace)

buf, _ = pcu._stats_device(x, y, True, 10)
for which, name in ((0, "x->y"), (1, "y->x")):
    st = pcu._stats_from_tensor(buf, which)
    print("%s n_far %d  argmax_query %d argmax_data %d witness_tied %d" % (name, st["n_far"], st["argmax_query"],
                                                                         st["argmax_data"], st["witness_tied"]), flush=True)

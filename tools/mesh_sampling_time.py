"""Mesh sampling: time per call (CUDA events, device-resident inputs, warm-up, L2 flushed before every timed call).

  sample_mesh_random   10^7 samples on a jittered icosphere of 1 310 720 faces, fp32 and fp64 vertices, int32 faces:
                       the device call alone, and its face-weight + CDF stage alone (pcu_b200_mesh_area_*); the
                       bytes a sample must write (fidx + bc: 16 B fp32, 28 B fp64) over the time, against 3.35 TB/s
  sample_mesh_poisson_disk  num_samples = 10^5 and 10^6 (4 * 10^6 and 4 * 10^7 dense samples), the public function

`python tools/mesh_sampling_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import subprocess
import numpy as np
import torch
import pcu_b200 as pcu

I = pcu._pcu_internal
flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2


def icosphere(subdivisions, jitter, seed):
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    for _ in range(subdivisions):
        edges = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(edges, axis=0, return_inverse=True)
        mid = len(v) + inv.reshape(3, -1).T
        v = np.concatenate([v, 0.5 * (v[uniq[:, 0]] + v[uniq[:, 1]])])
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        f = np.concatenate([np.stack([a, mid[:, 0], mid[:, 2]], 1), np.stack([b, mid[:, 1], mid[:, 0]], 1),
                            np.stack([c, mid[:, 2], mid[:, 1]], 1), mid])
    v = v / np.linalg.norm(v, axis=1, keepdims=True)
    v = v + jitter * np.random.default_rng(seed).standard_normal(v.shape) * 2.0 ** -subdivisions
    return v, f.astype(np.int32)


def timeit(fn, warm=3, it=10):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(it):
        flush_buf.add_(1)
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip(), flush=True)
sub = int(sys.argv[1]) if len(sys.argv) > 1 else 8
v64, f = icosphere(sub, 0.2, 1)
ft = torch.from_numpy(f).cuda()
stream = torch.cuda.current_stream().cuda_stream
n = 10 ** 7
print("mesh: %d vertices, %d faces" % (len(v64), len(f)), flush=True)
for dt in (torch.float32, torch.float64):
    vt = torch.from_numpy(v64).to(dt).cuda()
    is64 = dt == torch.float64
    fidx = torch.empty(n, dtype=torch.int32, device="cuda")
    bc = torch.empty((n, 3), dtype=dt, device="cuda")
    area = torch.empty(3, dtype=torch.int64, device="cuda")
    call = lambda: I._sample_mesh_random_device(is64, vt.data_ptr(), len(v64), ft.data_ptr(), len(f), 0, n, 7, fidx.data_ptr(),
                                                bc.data_ptr(), area.data_ptr(), 0, stream)
    cdf = lambda: I._mesh_area_device(is64, vt.data_ptr(), len(v64), ft.data_ptr(), len(f), 0, area.data_ptr(), 0, stream)
    med, mn = timeit(call)
    cmed, cmn = timeit(cdf)
    out_bytes = n * (4 + 3 * vt.element_size())
    print("random %s: %d samples  call median %.3f ms min %.3f ms | weights+CDF alone median %.3f ms min %.3f ms"
          % (str(dt)[6:], n, med, mn, cmed, cmn), flush=True)
    print("    %d B/sample written: %.1f MB, %.1f us at 3.35 TB/s; call %.2f TB/s (%.1f %% of that)"
          % (out_bytes // n, out_bytes / 1e6, out_bytes / 3.35e12 * 1e6, out_bytes / (mn * 1e-3) / 1e12,
             100.0 * out_bytes / 3.35e12 / (mn * 1e-3)), flush=True)
    del fidx, bc
    for ns in (10 ** 5, 10 ** 6):
        med, mn = timeit(lambda: pcu.sample_mesh_poisson_disk(vt, ft, ns, random_seed=7), warm=1, it=3)
        got = pcu.sample_mesh_poisson_disk(vt, ft, ns, random_seed=7)
        print("poisson %s: num_samples %d (dense %d) -> %d samples: median %.1f ms min %.1f ms"
              % (str(dt)[6:], ns, 40 * ns, got[0].shape[0], med, mn), flush=True)

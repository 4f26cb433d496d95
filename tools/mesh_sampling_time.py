"""Mesh sampling: time per call (CUDA events, device-resident inputs, warm-up, L2 flushed before every timed call).

  sample_mesh_random   10^7 samples on a jittered icosphere of 1 310 720 faces, fp32 and fp64 vertices, int32 faces:
                       the device call alone, and its face-weight + CDF stage alone (pcu_b200_mesh_area_*); the
                       bytes a sample must write (fidx + bc: 16 B fp32, 28 B fp64) over the time, against 3.35 TB/s
  sample_mesh_poisson_disk  num_samples = 10^5 and 10^6 (4 * 10^6 and 4 * 10^7 dense samples), the public function

`python tools/mesh_sampling_time.py [subdivisions]` (default 8).  The card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
import torch
from meshes import icosphere
from timing import card, timeit
import pcu_b200 as pcu

I = pcu._pcu_internal


print(card(), flush=True)
sub = int(sys.argv[1]) if len(sys.argv) > 1 else 8
v64, f = icosphere(sub, 0.2 * 2.0 ** -sub, 1)
f = f.astype(np.int32)
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

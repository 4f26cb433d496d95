"""sample_mesh_lloyd and one evaluation of its restricted Voronoi cells: time per call (warm-up, L2 flushed before every
timed call, median and minimum of 10; host clock around the call, which ends by synchronising the device).

  sphere 1e4 / 1e5    sample_mesh_lloyd on a jittered icosphere of 1 310 720 faces with the defaults (10 Lloyd steps,
                      at most 10 Newton steps), 10^4 and 10^5 samples
  square 1e6          the two-triangle unit square, 10^6 samples: every seed pairs with both faces
  sphere 1e3          the icosphere with 10^3 samples: about 1 300 faces per seed
  cells ...           one evaluation of the cells of each workload's initial sample (_restricted_cell_moments: its
                      upload and download included)
The (face, seed) pairs each pass handled are printed beside every time (summed over the call's evaluations).  The
reference's time cannot be taken: geogram is not part of it as checked out.
`python tools/sample_mesh_lloyd_time.py [repeats]`; the card's name and power limit are printed first."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import time
import numpy as np
import torch
from meshes import icosphere
from timing import card
import pcu_b200 as pcu

flush_buf = torch.empty(64 << 20, dtype=torch.int32, device="cuda")   # 256 MB, several times the 50 MB L2
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush_buf.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return np.median(ts) * 1e3, min(ts) * 1e3


print(card())
vs, fs = icosphere(8, 0.1 * 2.0 ** -8, 1)
fs = fs.astype(np.int32)
sq_v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], dtype=np.float64)
sq_f = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
sphere = (torch.from_numpy(vs).cuda(), torch.from_numpy(fs).cuda())
square = (torch.from_numpy(sq_v).cuda(), torch.from_numpy(sq_f).cuda())
cases = (("sphere 1e4", sphere, 10_000), ("sphere 1e5", sphere, 100_000), ("square 1e6", square, 1_000_000),
         ("sphere 1e3", sphere, 1_000))
for name, (v, f), n in cases:
    np.random.seed(0)
    x0 = pcu.sample_mesh_lloyd(v, f, n, 0, 0).cpu().numpy()
    hv, hf = v.cpu().numpy(), f.cpu().numpy()
    med, lo = timed(lambda: pcu._lloyd._restricted_cell_moments(x0, hv, hf), reps)
    print("%-24s median %9.2f ms  min %9.2f ms  pairs per pass %s" % ("cells " + name, med, lo, pcu._lloyd.last_pass_counts),
          flush=True)

    def run():
        np.random.seed(0)
        pcu.sample_mesh_lloyd(v, f, n)

    med, lo = timed(run, reps)
    print("%-24s median %9.2f ms  min %9.2f ms  pairs per pass %s  Newton steps %d" % (
        "lloyd " + name, med, lo, pcu._lloyd.last_pass_counts, len(pcu._lloyd.last_newton_energies) - 1), flush=True)

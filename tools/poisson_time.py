"""Poisson-disk downsampling: time per call (CUDA events, device-resident inputs, L2 flushed before every timed call)
and selection rounds per call, for uniform and sphere-surface fp32 clouds at radii that keep about 1 % and 10 % of
the points, a tight cluster, and a target-count call.  `python tools/poisson_time.py [n ...]` (default 10^6 10^7)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from timing import card, timeit
import pcu_b200 as pcu

I = pcu._pcu_internal


def one_call(x, radius, rounds, count, idx):
    I._poisson_disk_device(x.dtype == torch.float64, x.data_ptr(), x.shape[0], float(radius), 12345, idx.data_ptr(),
                           count.data_ptr(), rounds.data_ptr(), x.device.index or 0, torch.cuda.current_stream().cuda_stream)


def radius_for(x, keep, idx, count, rounds):
    """Bisect the radius whose sample keeps about `keep` of the points (not timed)."""
    lo, hi = 1e-6, 1.0
    for _ in range(30):
        mid = (lo * hi) ** 0.5
        one_call(x, mid, rounds, count, idx)
        frac = int(count.item()) / x.shape[0]
        if abs(frac / keep - 1.0) < 0.05: return mid
        lo, hi = (mid, hi) if frac > keep else (lo, mid)
    return mid


print(card(), flush=True)
sizes = [int(float(a)) for a in sys.argv[1:]] or [1000000, 10000000]
g = torch.Generator(device="cuda").manual_seed(0)
for n in sizes:
    idx = torch.empty(n, dtype=torch.int32, device="cuda")
    count = torch.empty(1, dtype=torch.int64, device="cuda")
    rounds = torch.zeros(1, dtype=torch.int32, device="cuda")
    clouds = {"uniform": torch.rand((n, 3), generator=g, device="cuda")}
    s = torch.randn((n, 3), generator=g, device="cuda")
    clouds["sphere"] = (s / s.norm(dim=1, keepdim=True)).contiguous()
    for name, x in clouds.items():
        for keep in (0.01, 0.10):
            r = radius_for(x, keep, idx, count, rounds)
            med, mn = timeit(lambda: one_call(x, r, rounds, count, idx), warm=2, it=7)
            print("%-7s n=%8d r=%.5f kept %5.2f %%: median %8.3f ms  min %8.3f ms  rounds %d"
                  % (name, n, r, 100.0 * int(count.item()) / n, med, mn, int(rounds.item())), flush=True)
    del clouds, s
    # a tight cluster: every point in a 1e-4 cube, radius a tenth of the cube
    x = 0.5 + 1e-4 * torch.rand((min(n, 200000), 3), generator=g, device="cuda")
    med, mn = timeit(lambda: one_call(x, 1e-5, rounds, count, idx), warm=1, it=3)
    print("cluster n=%8d r=1e-5 kept %d: median %8.3f ms  min %8.3f ms  rounds %d"
          % (x.shape[0], int(count.item()), med, mn, int(rounds.item())), flush=True)
    # target mode through the public function (synchronises once per radius tried)
    x = torch.rand((n, 3), generator=g, device="cuda")
    med, mn = timeit(lambda: pcu.downsample_point_cloud_poisson_disk(x, 0.0, target_num_samples=n // 20, random_seed=7),
                     warm=1, it=3)
    got = pcu.downsample_point_cloud_poisson_disk(x, 0.0, target_num_samples=n // 20, random_seed=7)
    print("target  n=%8d target %d -> %d: median %8.3f ms  min %8.3f ms" % (n, n // 20, got.shape[0], med, mn), flush=True)
    del x, idx

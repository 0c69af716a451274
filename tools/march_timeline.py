"""Debug aid: per-block timeline of the ray-march kernel (which SM, when, how many steps) for one tick of
the benchmark workload.  python tools/march_timeline.py [variant]   (needs a GPU)"""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import f1tenth_gym_b200 as f110  # noqa: E402
from f1tenth_gym_b200 import _native as nat  # noqa: E402

dev = torch.device('cuda:0')
N, A, B = 4096, 1, 1080
sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, A, 12345, num_envs=N, device=dev)
sim.set_map(f110.maps.resolve_map_path('example_map'), '.png')
wp_np = f110.maps.load_waypoints()
wp = torch.from_numpy(wp_np).to(dev)
rng = np.random.default_rng(0)
ks = rng.integers(0, wp_np.shape[0], N)
sim.env_reset(wp_np[ks][:, None, :])
gen = torch.Generator(device=dev); gen.manual_seed(1)
def act():
    u = torch.rand((N * A, 2), generator=gen, device=dev, dtype=torch.float64)
    u[:, 0] = -0.4189 + 0.8378 * u[:, 0]; u[:, 1] = 8.0 * u[:, 1]
    return u.view(N, A, 2)
for t in range(150):
    sim.step(act()); sim.env_post_step(); sim.autoreset(wp, 23, 1)
torch.cuda.synchronize()
L = nat.lib()
L.f110_debug_set_trace.argtypes = [C.c_void_p]
nblocks = N * A * 34 + 64
buf = torch.zeros((nblocks, 4), dtype=torch.int64, device=dev)
L.f110_debug_set_trace(buf.data_ptr())
sim.step(act())
torch.cuda.synchronize()
L.f110_debug_set_trace(None)
tr = buf.cpu().numpy()
tr = tr[tr[:, 2] > 0]
t0 = tr[:, 1].min()
start = (tr[:, 1] - t0) / 1e3; end = (tr[:, 2] - t0) / 1e3
print('blocks traced', tr.shape[0], 'kernel span %.1f us' % end.max())
dur = end - start
print('block duration us: mean %.2f p50 %.2f p90 %.2f p99 %.2f max %.2f' % (dur.mean(), *np.percentile(dur, [50, 90, 99]), dur.max()))
print('steps(max of warp0): mean %.1f p99 %d max %d' % (tr[:, 3].mean(), np.percentile(tr[:, 3], 99), tr[:, 3].max()))
print('last block START at %.1f us' % start.max())
nsm = torch.cuda.get_device_properties(0).multi_processor_count
sm_end = np.zeros(nsm); sm_busy = np.zeros(nsm)
for s in range(nsm):
    m = tr[:, 0] == s
    if m.any():
        sm_end[s] = end[m].max()
print('per-SM finish time us: min %.1f mean %.1f max %.1f' % (sm_end.min(), sm_end.mean(), sm_end.max()))
for q in (50, 75, 90, 95, 99, 99.9):
    print('  %5.1f%% of blocks finished by %.1f us' % (q, np.percentile(end, q)))
late = np.argsort(end)[-12:]
for j in late:
    print('  late block: start %.1f end %.1f dur %.1f steps %d sm %d' % (start[j], end[j], dur[j], tr[j, 3], tr[j, 0]))
# concurrency over time
ts = np.linspace(0, end.max(), 21)
for t in ts:
    print('  t=%6.1f us running blocks %6d  not-yet-started %6d' % (t, int(((start <= t) & (end > t)).sum()), int((start > t).sum())))

"""f1tenth_gym_b200 — batched F1TENTH simulator hot path for the H100.

Drop-in for the per-tick path of f1tenth/f1tenth_gym (Simulator.step: pid + RK4 single-track dynamics,
1080-beam lidar ray-march on the distance-transform grid, iTTC, opponent ray-cast, GJK collision)
behind the reference's own Python surface (F110Env / Simulator / ScanSimulator2D and the @njit kernel
names).  Compute happens only in libf110_b200.so (hand-written sm_90a CUDA behind a C ABI).
"""
from .simulator import Integrator, Simulator, DeviceMap, DeviceBeams   # noqa: F401
from .env import F110Env                                              # noqa: F401
from . import kernels, maps, trackgen                                 # noqa: F401
from .obstacles import obstacle_candidates                            # noqa: F401
from .kernels import ScanSimulator2D                                  # noqa: F401
from .planner import PurePursuitPlanner                               # noqa: F401
from .mppi import MPPIPlanner                                         # noqa: F401

__all__ = ['F110Env', 'Simulator', 'Integrator', 'ScanSimulator2D', 'PurePursuitPlanner', 'MPPIPlanner', 'DeviceMap', 'DeviceBeams', 'kernels', 'maps',
           'trackgen']

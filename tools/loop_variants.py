"""C2 step time (100 k points x 50 fixed iterations) and the per-iteration device times the log records."""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dcreg_b200 import Context, default_params
from dcreg_b200.scenes import make_cylinder, g2_initial_pose

pts = make_cylinder(100_000, seed=42)
T0 = g2_initial_pose()
prm = default_params(search_radius=1.0, max_iterations=50, fixed_iterations=1, kappa_target=10.0)
with Context(0) as ctx:
    ctx.set_target(pts, float(os.environ.get("ICP_CELL", "1.0")))
    ctx.set_source(pts)
    for _ in range(3):
        res = ctx.icp_run(prm, T0, want_log=False)
    stream = torch.cuda.ExternalStream(ctx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = ctx.launch_count
    t0 = time.perf_counter()
    e0.record(stream)
    for _ in range(20):
        res = ctx.icp_run(prm, T0, want_log=False)
    e1.record(stream)
    e1.synchronize()
    wall = time.perf_counter() - t0
    ms = e0.elapsed_time(e1) / 20
    print(f"{ms * 1e3 / 50:7.2f} us/iteration device, {wall / 20 * 1e6 / 50:7.2f} us/iteration wall, "
          f"launches/step {(ctx.launch_count - l0) / 20:.0f}")
    res = ctx.icp_run(prm, T0, want_log=True)
    t = np.array([L.iter_time_ms for L in res.logs]) * 1e3
    print("  iter_time_us:", " ".join(f"{x:.0f}" for x in t), f"| sum {t.sum():.0f}")
    ctx.iteration_counters(True)
    prev = (0, 0)
    rows = []
    for k in range(1, 51):
        ctx.icp_run(default_params(search_radius=1.0, max_iterations=k, fixed_iterations=1, kappa_target=10.0), T0, want_log=False)
        s_, f_ = ctx.iteration_counters(True)
        rows.append((s_ - prev[0], f_ - prev[1]))
        prev = (s_, f_)
    ctx.iteration_counters(False)
    print("  searched per iteration:", " ".join(str(r[0]) for r in rows))
    print("  refitted per iteration:", " ".join(str(r[1]) for r in rows))
    dx = [max(abs(x) for x in L.dx[3:]) for L in res.logs]
    print("  max |dx_t| per iteration (m):", " ".join(f"{x:.1e}" for x in dx))

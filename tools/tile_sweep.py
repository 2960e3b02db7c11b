"""Loop time against the tile size (source slots per block) of the iteration kernel: DCREG_TILE sweep.
C2 (100 k points, 50 fixed iterations) and the shipped 7 562-point cloud (30 fixed iterations).  A tile that would need
more blocks than a single run may keep resident (loop_plan.hpp: 3 per SM) is ignored by plan_tiles, so it is skipped."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dcreg_b200 import Context, default_params
from dcreg_b200.scenes import make_cylinder, g2_initial_pose, load_pcd_xyz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sweep(name, pts, iters, tiles, reps=20):
    T0 = g2_initial_pose()
    prm = default_params(search_radius=1.0, max_iterations=iters, fixed_iterations=1, kappa_target=10.0)
    with Context(0) as ctx:
        ctx.set_target(pts, 1.0)
        ctx.set_source(pts)
        stream = torch.cuda.ExternalStream(ctx.stream)
        ref = None
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        for t in tiles:
            if t and -(-len(pts) // t) > 3 * sms:
                print(f"{name}: tile {t:>7}  skipped: {-(-len(pts) // t)} blocks > 3 x {sms} SMs, plan_tiles would keep 256", flush=True)
                continue
            if t:
                os.environ["DCREG_TILE"] = str(t)
            else:
                os.environ.pop("DCREG_TILE", None)
            for _ in range(3):
                res = ctx.icp_run(prm, T0, want_log=False)
            best = 1e9
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(reps):
                    res = ctx.icp_run(prm, T0, want_log=False)
                e1.record(stream)
                e1.synchronize()
                best = min(best, e0.elapsed_time(e1) / reps)
            if ref is None:
                ref = res.T.copy()
            print(f"{name}: tile {t or 'default':>7}  {best * 1e3 / iters:7.2f} us/iteration   |T - T(first)| {np.abs(res.T - ref).max():.1e}", flush=True)


if __name__ == "__main__":
    sweep("C2 100k", make_cylinder(100_000, seed=42), 50, [0, 256, 240, 232, 226, 200, 170])
    sweep("shipped 7562", load_pcd_xyz(os.path.join(ROOT, "tests", "golden", "cylinder_7562.pcd")), 30, [0, 256, 128, 64, 52, 32])
    sweep("50k", make_cylinder(50_000, seed=42), 50, [0, 256, 170, 128])

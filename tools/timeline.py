"""Where one loop iteration spends its time: per-block phase stamps of the iteration kernel + the solve step (C2 scene).

A single folded run has a solver block (block 0, DCREG_NO_SOLVER_BLOCK=1 selects the ticket path instead): its row
shows when its warm-up step ended, when the last tile row landed and when the streamed sum was complete."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcreg_b200 import Context, default_params
from dcreg_b200.scenes import make_cylinder, g2_initial_pose

pts = make_cylinder(int(os.environ.get("ICP_POINTS", 100_000)), seed=42)
T0 = g2_initial_pose()
prm = default_params(kappa_target=10.0)
names = ["start", "cert", "search", "fitlist", "fits", "gram", "reduced", "sums", "solved"]
with Context(0) as ctx:
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    for iters in (1, 3, 8, 14, 25, 40):
        blocks, solve = ctx.iteration_timeline(prm, T0, iters)
        solver = solve[14] == 1
        sb = blocks[0]
        if solver:
            blocks = blocks[1:]                                   # tile blocks only
        t0 = blocks[:, 0].min()
        last = int(solve[15])
        print(f"iteration {iters - 1}: {len(blocks)} tile blocks{' + solver block' if solver else ''}; block starts span {(blocks[:, 0].max() - t0) / 1e3:.1f} us")
        for k in range(1, 6):
            col = blocks[:, k] - t0
            print(f"   {names[k]:8s} done: min {col.min() / 1e3:6.1f}  median {np.median(col) / 1e3:6.1f}  max {col.max() / 1e3:6.1f} us after the first block start")
        d = np.diff(blocks[:, :6], axis=1)
        print("   per-phase duration, median / max over blocks (us):", "  ".join(f"{names[k + 1]} {np.median(d[:, k]) / 1e3:.1f}/{d[:, k].max() / 1e3:.1f}" for k in range(5)))
        ws = blocks[:, 9:14].sum(axis=0).astype(float)
        if ws[3] > 0:
            print(f"   warp search (warp 0 of every block, {int(ws[3])} searches): set-up {ws[0] / ws[3]:.0f}  scan {ws[1] / ws[3]:.0f}  select {ws[2] / ws[3]:.0f} cycles, {ws[4] / ws[3]:.0f} candidates per search")
        gram_max = blocks[:, 5].max()
        if solver:
            landed = blocks[:, 6].max()
            warm = f"{(sb[1] - t0) / 1e3:.1f}" if sb[1] else "off"
            print(f"   solver block: start {(sb[0] - t0) / 1e3:.1f}, warm-up done {warm}, last row landed {(landed - t0) / 1e3:.1f}, "
                  f"sum complete {(sb[6] - t0) / 1e3:.1f} (+{(sb[6] - landed) / 1e3:.2f}), sums {(sb[7] - t0) / 1e3:.1f}, solved {(sb[8] - t0) / 1e3:.1f} us")
            end = sb[8]
        else:
            lb = blocks[last]
            print(f"   last block {last}: gram done at {(lb[5] - t0) / 1e3:.1f}, reduced {(lb[6] - t0) / 1e3:.1f}, sums {(lb[7] - t0) / 1e3:.1f}, solved {(lb[8] - t0) / 1e3:.1f} us")
            end = lb[8]
        print(f"   tail: slowest tile block's gram -> end of the solve {(end - gram_max) / 1e3:.2f} us")
        print("   solve step (us): " + "  ".join(f"{n} {(solve[k + 1] - solve[k]) / 1e3:.2f}" for k, n in enumerate(["inverses", "schur+jacobi", "precond", "pcg", "update"])),
              f" total {(solve[5] - solve[0]) / 1e3:.2f}")

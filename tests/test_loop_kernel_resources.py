"""Resource ceilings of the loop kernel, read from the ptxas report the build writes (dcreg_b200/build.log, `-Xptxas -v`).

Every phase of a loop iteration is a latency chain, and local-memory traffic in the tile loop lies on it (DESIGN.md §3,
"Tile loop state off the registers").  These ceilings are the figures the kernel reaches, so a change that spills more in
any `icp_iter2_kernel` instantiation, or needs more than 80 registers (3 blocks of 256 threads per SM), fails here
instead of quietly costing time on the GPU."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "dcreg_b200", "build.log")

MAX_REGS = 80
# <kUseWd, kGrids, kSeq, kPlanes, kSparse> (kUseWd gives the same figures): stack frame, spill stores, spill loads
# in bytes.  The stack frame is shared with the solve step the kernel's last block runs (its QR's arrays).
CEILINGS = {
    (0, 0, 0, 0): (848, 226, 208),
    (0, 0, 0, 1): (848, 230, 212),
    (0, 0, 1, 0): (848, 226, 208),
    (0, 0, 1, 1): (848, 230, 212),
    (0, 1, 0, 0): (848, 218, 212),
    (0, 1, 0, 1): (848, 222, 216),
    (1, 0, 0, 0): (848, 274, 480),
    (1, 0, 0, 1): (864, 274, 480),
    (1, 1, 0, 0): (848, 246, 256),
    (1, 1, 0, 1): (848, 246, 256),
}


def _report():
    if not os.path.exists(LOG):
        from dcreg_b200 import build
        build.build(force=True)
    kernels = {}
    cur = props = None
    with open(LOG) as f:
        for line in f:
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m:
                cur = m.group(1)
                continue
            m = re.search(r"Function properties for (\S+)", line)
            if m:
                props = m.group(1)
                continue
            if cur is None or "icp_iter2_kernel" not in cur:
                continue
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and props == cur:
                kernels.setdefault(cur, {}).update(stack=int(m[1]), stores=int(m[2]), loads=int(m[3]))
            m = re.search(r"Used (\d+) registers", line)
            if m:
                kernels.setdefault(cur, {})["regs"] = int(m[1])
    return kernels


def _flags(mangled):
    """<kUseWd, kGrids, kSeq, kPlanes, kSparse> from the mangled name (template arguments `Lb0E` / `Lb1E`)."""
    m = re.search(r"icp_iter2_kernelI((?:Lb[01]E){5})", mangled)
    return tuple(int(v) for v in re.findall(r"Lb([01])E", m.group(1)))


def test_every_loop_kernel_instantiation_stays_within_its_ceilings():
    kernels = _report()
    assert len(kernels) == 18, sorted(kernels)
    over = []
    for mangled, r in kernels.items():
        flags = _flags(mangled)
        stack, stores, loads = CEILINGS[flags[1:]]
        if r["regs"] > MAX_REGS or r["stack"] > stack or r["stores"] > stores or r["loads"] > loads:
            over.append((flags, r, (MAX_REGS, stack, stores, loads)))
    assert not over, over

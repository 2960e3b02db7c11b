"""What the record-checking GPU tests share: one loop record, or the picked records of a run, against the slot-level
reference oracle/dcreg_oracle_rows.py, and the per-label statistics each test prints.

A record is recomputed from the pose its iteration ran at (the previous record's T; T_init, or T_prior for sequences
and odometry, for iteration 0) and must match: H27, the objective (1/2 sum b^2) and the rmse (sqrt(sum r^2 / N_eff))
within the reference's allowance; N_pt exactly up to slots whose q is in band; N_eff_clear <= N_eff <= N_eff_clear +
N_band; gradient == -H27[21:] byte for byte; fitness == N_pt / N_total exactly."""
import numpy as np
from scipy.spatial import cKDTree

import dcreg_oracle_rows as rows

STATS = {}             # label -> [records, slots, band counts {reason: n}, worst error / allowance]


def check_record(label, rec, src, tgt, tree, T, prm, n_total=None, lattice=False, radius=None):
    """radius: the search radius the record's run used (default prm.search_radius; an odometry frame under the
    adaptive threshold registers at its own)"""
    radius = prm.search_radius if radius is None else radius
    ref = rows.iteration_reference(src, tgt, tree, T, radius, bool(prm.use_weight_derivative),
                                   slope=prm.weight_slope, gate=prm.weight_gate, min_norm=prm.min_normal_norm,
                                   thickness=prm.plane_thickness)
    n_total = len(src) if n_total is None else n_total
    H27 = np.array(rec.H27)
    n_eff = rec.n_effective
    sum_b2 = 2.0 * rec.objective
    sum_r2 = rec.rmse * rec.rmse * n_eff
    ref.allow[28] += 8 * rows.EPS * ref.sum_r2              # the rmse's square root and division
    ratio = ref.check(H27, sum_b2, sum_r2)
    where = (label, rec.iter)
    assert abs(rec.n_corr_pt - ref.n_pt) <= ref.n_pt_band, where + (rec.n_corr_pt, ref.n_pt, ref.n_pt_band)
    assert ref.n_eff_clear <= n_eff <= ref.n_eff_clear + ref.n_band, where + (n_eff, ref.n_eff_clear, ref.n_band)
    assert np.array(rec.gradient).tobytes() == (-H27[21:]).tobytes(), where
    assert rec.fitness == rec.n_corr_pt / n_total, where
    worst = float(ratio.max())
    assert worst <= 1.0, where + (int(ratio.argmax()), worst, ref.band_counts())
    if not lattice:
        assert ref.n_band <= 1e-3 * max(ref.n_slots, 1) + 1, where + (ref.band_counts(),)
    st = STATS.setdefault(label, [0, 0, {}, 0.0])
    st[0] += 1
    st[1] += ref.n_slots
    for k, v in ref.band_counts().items():
        st[2][k] = st[2].get(k, 0) + v
    st[3] = max(st[3], worst)
    return ref


def report(label):
    n, slots, band, worst = STATS[label]
    print(f"{label}: {n} records, {slots} slots, band {band or 'none'}, worst |error| / allowance {worst:.3g}")


def poses_of(res, T0):
    """the pose each record's iteration ran at"""
    return [np.asarray(T0, np.float64)] + [np.array(r.T).reshape(4, 4) for r in res.logs[:-1]]


def check_run(label, res, src, tgt, T0, prm, pick=None, tree=None, n_total=None, lattice=False, radius=None):
    tree = cKDTree(np.asarray(tgt, np.float64)) if tree is None else tree
    poses = poses_of(res, T0)
    done = 0
    for i, rec in enumerate(res.logs):
        if rec.status != 0 or (pick is not None and i not in pick):
            continue
        check_record(label, rec, src, tgt, tree, poses[i], prm, n_total=n_total, lattice=lattice, radius=radius)
        done += 1
    return done

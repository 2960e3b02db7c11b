"""ctypes host binding of include/dcreg_b200.h.

Mirrors the reference's operator interface for the hot path (names, argument meaning, error
behaviour) so the parity tests read like the reference's own call sites:

  reference (C++)                                            here
  ---------------------------------------------------------  ----------------------------------
  ICPContext::setTargetCloud          utils.hpp:393-424       Context.set_target
  TestRunner::Point2PlaneICP_SO3_OpenMP  icp_test_runner.h:92  Context.Point2PlaneICP_SO3 / icp_run
  DCReg::analyzeDegeneracy + solveDegenerateSystem
                                      dcreg.hpp:45-264        Context.analyze_and_solve
  DCReg::solvePCG                     dcreg.hpp:279-283       Context.solve_pcg
  SymmetricHessianComputer            hessian_computer.h:62   Context.reduce_normal_equations

There is NO CPU fallback: if the CUDA library is missing or no GPU is visible the calls raise.
"""
from __future__ import annotations

import bisect
import contextlib
import ctypes as C
import math
import operator
import os
import types

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libdcreg_b200.so")

# ---- enums (DCReg/include/utils.hpp:106-121) ----
DET = {"NONE_DETE": 0, "SCHUR_CONDITION_NUMBER": 1, "FULL_EVD_MIN_EIGENVALUE": 2,
       "EVD_SUB_CONDITION": 3, "FULL_SVD_CONDITION": 4}
HAND = {"NONE_HAND": 0, "STANDARD_REGULARIZATION": 1, "ADAPTIVE_REGULARIZATION": 2,
        "PRECONDITIONED_CG": 3, "SOLUTION_REMAPPING": 4, "TRUNCATED_SVD": 5}
STATUS = {0: "OK", 1: "NOT_ENOUGH_POINTS", 2: "NONFINITE_UPDATE", 3: "SINGULAR_BLOCK", 4: "CUDA_ERROR",
          5: "NCCL_ERROR", 6: "BAD_ARG", 7: "NO_DEVICE"}
OK, NOT_ENOUGH_POINTS, NONFINITE_UPDATE, SINGULAR_BLOCK, CUDA_ERROR, NCCL_ERROR, BAD_ARG, NO_DEVICE = range(8)
LOOP_VARIANTS = 18          # instantiations of the iteration kernel (loop_plan.hpp kVariants)


class IcpParams(C.Structure):
    _fields_ = [
        ("search_radius", C.c_double), ("max_iterations", C.c_int32), ("detection", C.c_int32),
        ("handling", C.c_int32), ("use_weight_derivative", C.c_int32),
        ("conv_thresh_rot", C.c_double), ("conv_thresh_trans", C.c_double),
        ("cond_thresh", C.c_double), ("eig_thresh", C.c_double), ("kappa_target", C.c_double),
        ("pcg_tol", C.c_double), ("pcg_max_iter", C.c_int32), ("reserved0", C.c_int32),
        ("std_reg_gamma", C.c_double), ("plane_thickness", C.c_double), ("weight_slope", C.c_double),
        ("weight_gate", C.c_double), ("min_normal_norm", C.c_double),
        ("min_effective_points", C.c_int32), ("fixed_iterations", C.c_int32),
    ]


class Analysis(C.Structure):
    _fields_ = [
        ("is_degenerate", C.c_int32), ("degenerate_mask", C.c_int32 * 6), ("pcg_iterations", C.c_int32),
        ("cond_schur_rot", C.c_double), ("cond_schur_trans", C.c_double),
        ("cond_diag_rot", C.c_double), ("cond_diag_trans", C.c_double), ("cond_full", C.c_double),
        ("cond_full_sub_rot", C.c_double), ("cond_full_sub_trans", C.c_double),
        ("eigenvalues_full", C.c_double * 6), ("singular_values", C.c_double * 6),
        ("lambda_schur_rot", C.c_double * 3), ("lambda_schur_trans", C.c_double * 3),
        ("lambda_sub_rot", C.c_double * 3), ("lambda_sub_trans", C.c_double * 3),
        ("schur_V_rot", C.c_double * 9), ("schur_V_trans", C.c_double * 9),
        ("aligned_V_rot", C.c_double * 9), ("aligned_V_trans", C.c_double * 9),
        ("rot_indices", C.c_int32 * 3), ("trans_indices", C.c_int32 * 3), ("schur_singular", C.c_int32),
        ("reserved1", C.c_int32), ("P_preconditioner", C.c_double * 36), ("W_adaptive", C.c_double * 36),
        ("pcg_residual", C.c_double),
    ]

    def np(self, name):
        return np.array(getattr(self, name))


class IterLog(C.Structure):
    _fields_ = [
        ("iter", C.c_int32), ("status", C.c_int32), ("n_effective", C.c_int32), ("n_corr_pt", C.c_int32),
        ("rmse", C.c_double), ("fitness", C.c_double), ("objective", C.c_double), ("iter_time_ms", C.c_double),
        ("gradient", C.c_double * 6), ("H27", C.c_double * 27), ("dx", C.c_double * 6), ("T", C.c_double * 16),
        ("analysis", Analysis),
    ]


PLANE_CALLBACK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double),
                             C.POINTER(C.c_int64))

class AdaptiveThreshold(C.Structure):
    """dcreg_adaptive_threshold: the settings of odometry's adaptive search radius (KISS-ICP's defaults)"""
    _fields_ = [("initial_threshold", C.c_double), ("min_motion", C.c_double), ("max_range", C.c_double)]

    def __init__(self, initial_threshold=2.0, min_motion=0.1, max_range=100.0):
        super().__init__(float(initial_threshold), float(min_motion), float(max_range))


class Gyro(C.Structure):
    """dcreg_gyro: R_sensor_imu (3, 3) maps IMU-frame rates into the LiDAR frame, bias (3,) rad/s is subtracted first"""
    _fields_ = [("R_sensor_imu", C.c_double * 9), ("bias", C.c_double * 3)]

    def __init__(self, R_sensor_imu=None, bias=(0.0, 0.0, 0.0)):
        super().__init__()
        R = np.eye(3) if R_sensor_imu is None else np.asarray(R_sensor_imu, dtype=np.float64).reshape(3, 3)
        self.R_sensor_imu[:] = [float(x) for x in R.reshape(-1)]
        self.bias[:] = [float(x) for x in np.asarray(bias, dtype=np.float64).reshape(3)]

    @property
    def R(self):
        return np.array(self.R_sensor_imu[:]).reshape(3, 3)

    @property
    def b(self):
        return np.array(self.bias[:])


class Imu(C.Structure):
    """dcreg_imu: R_sensor_imu (3, 3) maps IMU-frame vectors into the LiDAR frame, gyro_bias (3,) rad/s and accel_bias
    (3,) m/s^2 are subtracted first, gravity (3,) m/s^2 is the world-frame (T_init's frame) gravity vector"""
    _fields_ = [("R_sensor_imu", C.c_double * 9), ("gyro_bias", C.c_double * 3), ("accel_bias", C.c_double * 3),
                ("gravity", C.c_double * 3)]

    def __init__(self, R_sensor_imu=None, gyro_bias=(0.0, 0.0, 0.0), accel_bias=(0.0, 0.0, 0.0),
                 gravity=(0.0, 0.0, -9.80665)):
        super().__init__()
        R = np.eye(3) if R_sensor_imu is None else np.asarray(R_sensor_imu, dtype=np.float64).reshape(3, 3)
        self.R_sensor_imu[:] = [float(x) for x in R.reshape(-1)]
        self.gyro_bias[:] = [float(x) for x in np.asarray(gyro_bias, dtype=np.float64).reshape(3)]
        self.accel_bias[:] = [float(x) for x in np.asarray(accel_bias, dtype=np.float64).reshape(3)]
        self.gravity[:] = [float(x) for x in np.asarray(gravity, dtype=np.float64).reshape(3)]

    @property
    def R(self):
        return np.array(self.R_sensor_imu[:]).reshape(3, 3)

    @property
    def bg(self):
        return np.array(self.gyro_bias[:])

    @property
    def ba(self):
        return np.array(self.accel_bias[:])

    @property
    def g(self):
        return np.array(self.gravity[:])


_lib = None

# every symbol include/dcreg_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "dcreg_abi_version", "dcreg_create", "dcreg_destroy", "dcreg_last_error", "dcreg_default_params",
    "dcreg_stream", "dcreg_set_source", "dcreg_set_target", "dcreg_set_target_sparse", "dcreg_set_sparse_maps",
    "dcreg_set_lane_params", "dcreg_set_map_spacing", "dcreg_set_map_input_voxel",
    "dcreg_set_prior_map",
    "dcreg_find_planes",
    "dcreg_reduce_normal_equations", "dcreg_reduce_normal_equations_f64plane",
    "dcreg_reduce_normal_equations_host", "dcreg_analyze_and_solve", "dcreg_solve_pcg", "dcreg_icp_run",
    "dcreg_icp_run_batch", "dcreg_icp_run_scans", "dcreg_icp_run_pairs", "dcreg_icp_run_sequences", "dcreg_icp_run_odometry", "dcreg_icp_run_odometry_voxel", "dcreg_icp_run_odometry_voxel_n", "dcreg_icp_run_odometry_deskew", "dcreg_icp_run_odometry_map", "dcreg_odometry_open", "dcreg_odometry_open_map", "dcreg_odometry_push", "dcreg_odometry_push_deskew", "dcreg_odometry_local_map", "dcreg_odometry_close", "dcreg_icp_run_odometry_adaptive", "dcreg_odometry_open_adaptive", "dcreg_odometry_push_adaptive", "dcreg_icp_run_odometry_gyro", "dcreg_odometry_open_gyro", "dcreg_odometry_push_gyro", "dcreg_icp_run_odometry_imu", "dcreg_odometry_open_imu", "dcreg_odometry_push_imu", "dcreg_voxel_downsample", "dcreg_voxel_downsample_n", "dcreg_voxel_downsample_spaced", "dcreg_icp_enqueue", "dcreg_icp_fetch", "dcreg_icp_run_host_planes", "dcreg_comm_mode", "dcreg_last_covariance", "dcreg_point_to_point_metrics", "dcreg_comm_unique_id", "dcreg_comm_init",
    "dcreg_comm_destroy", "dcreg_set_global_source_count", "dcreg_launch_count", "dcreg_loop_variant_launches",
    "dcreg_device_source",
    "dcreg_device_planes_f64", "dcreg_device_planes_f32", "dcreg_freeze_planes_f32", "dcreg_time_reduce", "dcreg_time_iteration", "dcreg_iteration_counters", "dcreg_iteration_timeline",
]


def load_library():
    """dlopen the in-tree CUDA library.  Raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m dcreg_b200.build` "
            "(__graft_entry__.build()).  dcreg_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    dp, vp, i64, ci = C.POINTER(C.c_double), C.c_void_p, C.c_int64, C.c_int
    lib.dcreg_abi_version.restype = ci
    lib.dcreg_create.argtypes = [ci, C.POINTER(vp)]
    lib.dcreg_destroy.argtypes = [vp]
    lib.dcreg_last_error.argtypes = [vp]; lib.dcreg_last_error.restype = C.c_char_p
    lib.dcreg_default_params.argtypes = [C.POINTER(IcpParams)]; lib.dcreg_default_params.restype = None
    lib.dcreg_stream.argtypes = [vp]; lib.dcreg_stream.restype = vp
    lib.dcreg_set_source.argtypes = [vp, C.POINTER(C.c_float), i64, ci]
    lib.dcreg_set_target.argtypes = [vp, C.POINTER(C.c_float), i64, ci, C.c_double]
    lib.dcreg_set_target_sparse.argtypes = [vp, C.POINTER(C.c_float), i64, ci, C.c_double]
    lib.dcreg_set_sparse_maps.argtypes = [vp, ci]
    lib.dcreg_set_lane_params.argtypes = [vp, ci]
    lib.dcreg_set_map_spacing.argtypes = [vp, C.c_double]
    lib.dcreg_set_map_input_voxel.argtypes = [vp, C.c_double]
    lib.dcreg_set_prior_map.argtypes = [vp, ci]
    lib.dcreg_find_planes.argtypes = [vp, dp, C.c_double, dp, C.POINTER(i64)]
    lib.dcreg_reduce_normal_equations.argtypes = [vp, vp, vp, i64, dp, ci, dp, dp]
    lib.dcreg_reduce_normal_equations_f64plane.argtypes = [vp, vp, vp, i64, dp, ci, dp, dp]
    lib.dcreg_reduce_normal_equations_host.argtypes = [vp, C.POINTER(C.c_float), vp, ci, i64, dp, ci, dp, dp]
    lib.dcreg_analyze_and_solve.argtypes = [vp, dp, C.POINTER(IcpParams), C.POINTER(Analysis), dp]
    lib.dcreg_solve_pcg.argtypes = [vp, dp, dp, dp, ci, C.c_double, dp, C.POINTER(ci)]
    lib.dcreg_icp_run.argtypes = [vp, C.POINTER(IcpParams), dp, dp, C.POINTER(IterLog), ci, C.POINTER(ci),
                                  C.POINTER(ci)]
    lib.dcreg_icp_run_batch.argtypes = [vp, C.POINTER(IcpParams), ci, dp, dp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci),
                                        C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_scans.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp, dp,
                                        C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_pairs.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(C.c_float), C.POINTER(i64),
                                        C.POINTER(C.c_float), C.POINTER(i64), ci, C.c_double, dp, dp, C.POINTER(ci),
                                        C.POINTER(ci), C.POINTER(ci), dp, C.c_double, dp, C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_sequences.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                            C.POINTER(i64), ci, dp, dp, dp, dp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci),
                                            dp, C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_odometry.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                           C.POINTER(i64), ci, C.c_double, ci, ci, dp, dp, dp, dp, C.POINTER(ci),
                                           C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_odometry_voxel.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                                 C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, dp, dp,
                                                 C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp,
                                                 C.POINTER(IterLog), ci]
    lib.dcreg_voxel_downsample.argtypes = [vp, ci, C.POINTER(C.c_float), C.POINTER(i64), ci, C.c_double,
                                           C.POINTER(C.c_float), C.POINTER(i64), C.POINTER(i64)]
    lib.dcreg_icp_run_odometry_voxel_n.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                                   C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                                   dp, dp, C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci),
                                                   C.POINTER(ci), dp, C.POINTER(IterLog), ci]
    lib.dcreg_voxel_downsample_n.argtypes = [vp, ci, C.POINTER(C.c_float), C.POINTER(i64), ci, C.c_double, ci,
                                             C.POINTER(C.c_float), C.POINTER(i64), C.POINTER(i64)]
    lib.dcreg_voxel_downsample_spaced.argtypes = [vp, ci, C.POINTER(C.c_float), C.POINTER(i64), ci, C.c_double, ci,
                                                  C.c_double, C.POINTER(C.c_float), C.POINTER(i64), C.POINTER(i64)]
    lib.dcreg_odometry_open.argtypes = [vp, C.POINTER(IcpParams), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                        dp]
    lib.dcreg_odometry_push.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp,
                                        C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp,
                                        C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_odometry_deskew.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                                  C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                                  dp, dp, C.POINTER(C.c_float), C.POINTER(i64), dp, dp, C.POINTER(ci),
                                                  C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float), C.POINTER(IterLog),
                                                  ci]
    lib.dcreg_odometry_push_deskew.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp,
                                               C.POINTER(C.c_float), C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci),
                                               C.POINTER(ci), dp, C.POINTER(C.c_float), C.POINTER(IterLog), ci]
    lib.dcreg_odometry_close.argtypes = [vp]
    lib.dcreg_icp_run_odometry_map.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                               C.POINTER(i64), ci, C.c_double, ci, C.c_double, C.c_double, ci, ci,
                                               C.c_double, dp, dp, C.POINTER(C.c_float), C.POINTER(i64), dp, dp,
                                               C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float),
                                               C.POINTER(IterLog), ci]
    lib.dcreg_odometry_open_map.argtypes = [vp, C.POINTER(IcpParams), ci, C.c_double, ci, C.c_double, C.c_double, ci, ci,
                                            C.c_double, dp]
    lib.dcreg_odometry_local_map.argtypes = [vp, ci, C.POINTER(C.c_float), i64, C.POINTER(i64)]
    lib.dcreg_icp_run_odometry_adaptive.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                                    C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                                    C.c_double, C.POINTER(AdaptiveThreshold), dp, dp, C.POINTER(C.c_float),
                                                    C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp,
                                                    C.POINTER(C.c_float), dp, C.POINTER(IterLog), ci]
    lib.dcreg_odometry_open_adaptive.argtypes = [vp, C.POINTER(IcpParams), ci, C.c_double, ci, ci, C.c_double, C.c_double,
                                                 ci, ci, C.c_double, C.POINTER(AdaptiveThreshold), dp]
    lib.dcreg_odometry_push_adaptive.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp,
                                                 C.POINTER(C.c_float), C.POINTER(i64), dp, dp, C.POINTER(ci), C.POINTER(ci),
                                                 C.POINTER(ci), dp, C.POINTER(C.c_float), dp, C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_odometry_gyro.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                                C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                                C.c_double, C.POINTER(AdaptiveThreshold), C.POINTER(Gyro), dp, dp,
                                                C.POINTER(C.c_float), dp, dp, C.POINTER(i64), C.POINTER(i64), dp, dp,
                                                C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float), dp,
                                                C.POINTER(IterLog), ci]
    lib.dcreg_odometry_open_gyro.argtypes = [vp, C.POINTER(IcpParams), ci, C.c_double, ci, ci, C.c_double, C.c_double,
                                             ci, ci, C.c_double, C.POINTER(AdaptiveThreshold), C.POINTER(Gyro), dp]
    lib.dcreg_odometry_push_gyro.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp,
                                             C.POINTER(C.c_float), dp, dp, C.POINTER(i64), C.POINTER(i64), dp, dp,
                                             C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float), dp,
                                             C.POINTER(IterLog), ci]
    lib.dcreg_icp_run_odometry_imu.argtypes = [vp, C.POINTER(IcpParams), ci, C.POINTER(ci), ci, C.POINTER(C.c_float),
                                               C.POINTER(i64), ci, C.c_double, ci, ci, C.c_double, C.c_double, ci, ci,
                                               C.c_double, C.POINTER(AdaptiveThreshold), C.POINTER(Imu), dp, dp, dp,
                                               C.POINTER(C.c_float), dp, dp, C.POINTER(i64), C.POINTER(i64), dp, dp,
                                               C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float), dp,
                                               dp, C.POINTER(IterLog), ci]
    lib.dcreg_odometry_open_imu.argtypes = [vp, C.POINTER(IcpParams), ci, C.c_double, ci, ci, C.c_double, C.c_double,
                                            ci, ci, C.c_double, C.POINTER(AdaptiveThreshold), C.POINTER(Imu), dp, dp]
    lib.dcreg_odometry_push_imu.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(C.c_float), C.POINTER(i64), ci, dp,
                                            C.POINTER(C.c_float), dp, dp, C.POINTER(i64), C.POINTER(i64), dp, dp,
                                            C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), dp, C.POINTER(C.c_float), dp, dp,
                                            C.POINTER(IterLog), ci]
    lib.dcreg_comm_mode.argtypes = [vp]
    lib.dcreg_icp_enqueue.argtypes = [vp, C.POINTER(IcpParams), dp]
    lib.dcreg_icp_fetch.argtypes = [vp, dp, C.POINTER(ci), C.POINTER(ci)]
    lib.dcreg_icp_run_host_planes.argtypes = [vp, C.POINTER(IcpParams), dp, PLANE_CALLBACK, vp, dp,
                                              C.POINTER(IterLog), ci, C.POINTER(ci), C.POINTER(ci)]
    lib.dcreg_last_covariance.argtypes = [vp, dp]
    lib.dcreg_point_to_point_metrics.argtypes = [vp, dp, C.c_double, dp]
    lib.dcreg_comm_unique_id.argtypes = [vp, C.POINTER(C.c_uint8)]
    lib.dcreg_comm_init.argtypes = [vp, C.POINTER(C.c_uint8), ci, ci]
    lib.dcreg_comm_destroy.argtypes = [vp]
    lib.dcreg_set_global_source_count.argtypes = [vp, i64]
    lib.dcreg_launch_count.argtypes = [vp]; lib.dcreg_launch_count.restype = i64
    lib.dcreg_loop_variant_launches.argtypes = [vp, C.POINTER(i64)]
    for nm in ("dcreg_device_source", "dcreg_device_planes_f64", "dcreg_device_planes_f32"):
        getattr(lib, nm).argtypes = [vp]; getattr(lib, nm).restype = vp
    lib.dcreg_freeze_planes_f32.argtypes = [vp]
    lib.dcreg_time_reduce.argtypes = [vp, ci, dp, ci, ci, ci, C.POINTER(C.c_float)]
    lib.dcreg_time_iteration.argtypes = [vp, C.POINTER(IcpParams), dp, ci, ci, C.POINTER(C.c_float)]
    lib.dcreg_iteration_counters.argtypes = [vp, ci, C.POINTER(C.c_uint64)]
    lib.dcreg_iteration_timeline.argtypes = [vp, C.POINTER(IcpParams), dp, ci, C.POINTER(C.c_uint64), ci, C.POINTER(ci)]
    _lib = lib
    return lib


def default_params(**overrides) -> IcpParams:
    p = IcpParams()
    load_library().dcreg_default_params(C.byref(p))
    for k, v in overrides.items():
        if k == "detection" and isinstance(v, str):
            v = DET[v]
        if k == "handling" and isinstance(v, str):
            v = HAND[v]
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class DcregError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"dcreg status {status} ({STATUS.get(status, '?')}): {msg}")
        self.status = status


def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _as_points(xyz):
    a = np.ascontiguousarray(xyz, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] < 3:
        raise ValueError("points must be (N, >=3)")
    return a


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _iptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64)) if a is not None else None


def _optr(a):
    return _dptr(a) if a is not None else None


def _pack(clouds):
    """The clouds (a list of (N_b, >=3) arrays) as one contiguous (sum N_b, 3) float32 array and their int64 offsets
    [len + 1]; (None, None) for no clouds."""
    pts = [_as_points(c)[:, :3] for c in clouds]
    if not pts:
        return None, None
    off = np.zeros(len(pts) + 1, dtype=np.int64)
    off[1:] = np.cumsum([p.shape[0] for p in pts])
    return np.ascontiguousarray(np.concatenate(pts, axis=0)), off


def _pack_sequences(sequences):
    """The int32 sequence table [len + 1] of a list of lists of frames, and _pack of all frames in order."""
    seq_off = np.zeros(len(sequences) + 1, dtype=np.int32)
    seq_off[1:] = np.cumsum([len(s) for s in sequences])
    return (seq_off,) + _pack([f for s in sequences for f in s])


def _pack_timestamps(timestamps, off, name):
    """Per-frame timestamp arrays (nested like the frames) as one contiguous float32 array matching the packed points
    with offsets off, or None"""
    if timestamps is None:
        return None
    ts = [np.asarray(t, dtype=np.float32).reshape(-1) for t in timestamps]
    if len(ts) != len(off) - 1 or any(t.shape[0] != b - a for t, a, b in zip(ts, off[:-1], off[1:])):
        raise ValueError(f"{name}: timestamps must hold one value per point of every frame")
    return np.ascontiguousarray(np.concatenate(ts) if ts else np.zeros(0, np.float32))


def _pack_gyro(name, gyro, frame_times, gyro_samples, n_frames, n_seqs, cols=4):
    """(frame_times (n_frames, 2), samples (rows, cols), sample_offsets int64 [n_seqs + 1]) as contiguous arrays, or
    Nones without gyro input (a gyro session's push may leave both out; one without the other is refused).  cols = 7:
    IMU samples (t, wx, wy, wz, ax, ay, az)"""
    if gyro is None:
        if frame_times is not None or gyro_samples is not None:
            raise ValueError(f"{name}: frame_times and gyro_samples need gyro input")
        return None, None, None
    if (frame_times is None) != (gyro_samples is None):
        raise ValueError(f"{name}: frame_times and gyro_samples go together")
    if frame_times is None:
        return None, None, None
    ft = np.ascontiguousarray(frame_times, dtype=np.float64).reshape(-1, 2)
    if ft.shape[0] != n_frames:
        raise ValueError(f"{name}: {n_frames} frames but {ft.shape[0]} frame times")
    if len(gyro_samples) != n_seqs:
        raise ValueError(f"{name}: {n_seqs} sequences but {len(gyro_samples)} sample arrays")
    smp = [np.asarray(x, dtype=np.float64).reshape(-1, cols) for x in gyro_samples]
    off = np.zeros(n_seqs + 1, dtype=np.int64)
    off[1:] = np.cumsum([x.shape[0] for x in smp])
    return ft, np.ascontiguousarray(np.concatenate(smp) if smp else np.zeros((0, cols))), off


def _pack_v_init(name, v_init, n_seqs):
    """v_init as a contiguous (n_seqs, 3) float64 array, or None (every sequence starts at rest)"""
    if v_init is None:
        return None
    v = np.ascontiguousarray(v_init, dtype=np.float64).reshape(-1, 3)
    if v.shape[0] != n_seqs:
        raise ValueError(f"{name}: {n_seqs} sequences but {v.shape[0]} initial velocities")
    return v


def _split_deskewed(out, npts):
    """(total, 3) deskewed points cut into one array per frame"""
    at = np.concatenate([[0], np.cumsum(npts)])
    return [out[a:b].copy() for a, b in zip(at[:-1], at[1:])]


_MOTIONS = {"increments": 0, "constant_velocity": 1}


def _motion(motion, name):
    if motion not in _MOTIONS:
        raise ValueError(f"{name}: motion must be one of {sorted(_MOTIONS)}, not {motion!r}")
    return _MOTIONS[motion]


# The arguments after the context of every odometry and voxel-downsample entry point, in C order with the names of
# include/dcreg_b200.h: the one place the binding and the tests know these signatures.
_RUN = "params n_seqs seq_offsets n_frames xyz frame_offsets stride cell_size"
_FILTERS = "source_voxel map_voxel source_max_points map_max_points"
_OUTPUTS = "T_prior T_out n_iterations converged status cov"
_PUSH = "seq_offsets n_frames xyz frame_offsets stride deltas"
_DOWNSAMPLE = "n_clouds xyz offsets stride voxel"
_ODOMETRY_ARGS = {name: " ".join(args).split() for name, args in {
    "dcreg_icp_run_odometry": (_RUN, "map_frames motion T_init deltas", _OUTPUTS, "log log_cap"),
    "dcreg_icp_run_odometry_voxel": (_RUN, "map_frames motion source_voxel map_voxel T_init deltas frame_points",
                                     _OUTPUTS, "log log_cap"),
    "dcreg_icp_run_odometry_voxel_n": (_RUN, "map_frames motion", _FILTERS, "T_init deltas frame_points", _OUTPUTS,
                                       "log log_cap"),
    "dcreg_icp_run_odometry_deskew": (_RUN, "map_frames motion", _FILTERS, "T_init deltas timestamps frame_points",
                                      _OUTPUTS, "deskewed_xyz log log_cap"),
    "dcreg_icp_run_odometry_map": (_RUN, "motion", _FILTERS, "max_distance T_init deltas timestamps frame_points",
                                   _OUTPUTS, "deskewed_xyz log log_cap"),
    "dcreg_icp_run_odometry_adaptive": (_RUN, "map_frames motion", _FILTERS,
                                        "max_distance adaptive T_init deltas timestamps frame_points", _OUTPUTS,
                                        "deskewed_xyz search_radius log log_cap"),
    "dcreg_icp_run_odometry_gyro": (_RUN, "map_frames motion", _FILTERS,
                                    "max_distance adaptive gyro T_init deltas timestamps frame_times samples",
                                    "sample_offsets frame_points", _OUTPUTS, "deskewed_xyz search_radius log log_cap"),
    "dcreg_icp_run_odometry_imu": (_RUN, "map_frames motion", _FILTERS,
                                   "max_distance adaptive imu T_init v_init deltas timestamps frame_times samples",
                                   "sample_offsets frame_points", _OUTPUTS, "deskewed_xyz search_radius velocity log",
                                   "log_cap"),
    "dcreg_odometry_open": ("params n_seqs cell_size map_frames motion", _FILTERS, "T_init"),
    "dcreg_odometry_open_map": ("params n_seqs cell_size motion", _FILTERS, "max_distance T_init"),
    "dcreg_odometry_open_adaptive": ("params n_seqs cell_size map_frames motion", _FILTERS,
                                     "max_distance adaptive T_init"),
    "dcreg_odometry_push": (_PUSH, "frame_points", _OUTPUTS, "log log_cap"),
    "dcreg_odometry_push_deskew": (_PUSH, "timestamps frame_points", _OUTPUTS, "deskewed_xyz log log_cap"),
    "dcreg_odometry_push_adaptive": (_PUSH, "timestamps frame_points", _OUTPUTS,
                                     "deskewed_xyz search_radius log log_cap"),
    "dcreg_odometry_open_gyro": ("params n_seqs cell_size map_frames motion", _FILTERS,
                                 "max_distance adaptive gyro T_init"),
    "dcreg_odometry_push_gyro": (_PUSH, "timestamps frame_times samples sample_offsets frame_points", _OUTPUTS,
                                 "deskewed_xyz search_radius log log_cap"),
    "dcreg_odometry_open_imu": ("params n_seqs cell_size map_frames motion", _FILTERS,
                                "max_distance adaptive imu T_init v_init"),
    "dcreg_odometry_push_imu": (_PUSH, "timestamps frame_times samples sample_offsets frame_points", _OUTPUTS,
                                "deskewed_xyz search_radius velocity log log_cap"),
    "dcreg_voxel_downsample": (_DOWNSAMPLE, "out_xyz out_offsets out_index"),
    "dcreg_voxel_downsample_n": (_DOWNSAMPLE, "max_points out_xyz out_offsets out_index"),
    "dcreg_voxel_downsample_spaced": (_DOWNSAMPLE, "max_points min_spacing out_xyz out_offsets out_index"),
}.items()}
_ODOMETRY_NAMES = {a for args in _ODOMETRY_ARGS.values() for a in args}


def _odometry_call(lib, h, entry, **values):
    """lib.<entry>(h, ...) with values laid out in the entry's order (_ODOMETRY_ARGS).  A pointer argument not given is
    NULL, a scalar not given is a ctypes error, and a value the entry does not take is left out: one set of values serves
    every entry point a call may pick."""
    unknown = values.keys() - _ODOMETRY_NAMES
    if unknown:
        raise TypeError(f"{entry}: no argument named {sorted(unknown)}")
    return getattr(lib, entry)(h, *(values.get(k) for k in _ODOMETRY_ARGS[entry]))


def _odometry_entry(op, radius=False, voxel_map=False, deskew=False, capped=False, filtered=False, gyro=False,
                    imu=False):
    """The entry point of op ("icp_run_odometry", "odometry_open" or "odometry_push") for a call with these settings: the
    narrowest that takes them all.  Each entry point names itself in dcreg_last_error."""
    if imu:
        return f"dcreg_{op}_imu"
    if gyro:
        return f"dcreg_{op}_gyro"
    if radius:
        return f"dcreg_{op}_adaptive"
    if voxel_map:
        return f"dcreg_{op}_map"
    if deskew:
        return f"dcreg_{op}_deskew"
    if capped:
        return f"dcreg_{op}_voxel_n"
    if filtered:
        return f"dcreg_{op}_voxel"
    return f"dcreg_{op}"


def pose_Rt(T):
    T = np.asarray(T, dtype=np.float64)
    return np.ascontiguousarray(np.concatenate([T[:3, :3].reshape(-1), T[:3, 3]]))


def compose_prior(T, D):
    """The next frame's prior T D of dcreg_icp_run_sequences, bit for bit as the device composes it: R' = R R_D and
    t' = R t_D + t, every entry ((a0 b0 + a1 b1) + a2 b2) [+ t] in FP64, one rounding per operation (elementwise NumPy
    ops, no matmul, no FMA), no re-orthonormalisation.  T, D: (..., 4, 4); returns (..., 4, 4) with the row [0, 0, 0, 1]."""
    T = np.asarray(T, dtype=np.float64)
    D = np.asarray(D, dtype=np.float64)
    shape = np.broadcast_shapes(T.shape, D.shape)
    out = np.zeros(shape)
    for c in range(4):
        col = (T[..., :3, 0] * D[..., 0:1, c] + T[..., :3, 1] * D[..., 1:2, c]) + T[..., :3, 2] * D[..., 2:3, c]
        if c == 3:
            col = col + T[..., :3, 3]
        out[..., :3, c] = col
    out[..., 3, 3] = 1.0
    return out


def map_points(T, P):
    """The local-map points of dcreg_icp_run_odometry, bit for bit as the device transforms them: frame points P (N, >=3)
    float32 under the pose T (4, 4), each coordinate ((r0 x + r1 y) + r2 z) + t in FP64 with one rounding per operation
    (elementwise NumPy ops, no matmul, no FMA), then one float32 rounding.  Returns (N, 3) float32."""
    T = np.asarray(T, dtype=np.float64)
    P = np.asarray(P, dtype=np.float32)[:, :3].astype(np.float64)
    out = np.empty((P.shape[0], 3), dtype=np.float32)
    for r in range(3):
        out[:, r] = (((T[r, 0] * P[:, 0] + T[r, 1] * P[:, 1]) + T[r, 2] * P[:, 2]) + T[r, 3]).astype(np.float32)
    return out


def constant_velocity_increment(T_prev, T):
    """The constant-velocity increment of dcreg_icp_run_odometry, inv(T_prev) T, bit for bit as the device forms it:
    R_D = R_prev^T R, t_D = R_prev^T (t - t_prev), the differences rounded first, every entry ((a0 b0 + a1 b1) + a2 b2)
    in FP64 with one rounding per operation.  T_prev, T: (4, 4); returns (4, 4) with the row [0, 0, 0, 1]."""
    A = np.asarray(T_prev, dtype=np.float64)
    B = np.asarray(T, dtype=np.float64)
    dt = B[:3, 3] - A[:3, 3]
    out = np.zeros((4, 4))
    for r in range(3):
        for c in range(3):
            out[r, c] = (A[0, r] * B[0, c] + A[1, r] * B[1, c]) + A[2, r] * B[2, c]
        out[r, 3] = (A[0, r] * dt[0] + A[1, r] * dt[1]) + A[2, r] * dt[2]
    out[3, 3] = 1.0
    return out


# The adaptive threshold of dcreg_icp_run_odometry_adaptive (dcreg_b200/csrc/adaptive_threshold.cuh): the same formulas
# and operation order in Python floats (FP64, one rounding per operation).  A state is (sse, n), (0.0, 0) at the anchor.
def adaptive_threshold_radius(state, initial_threshold, ceiling):
    """The search radius a sequence in `state` registers its next frame with, min(3 sigma, ceiling), bit for bit"""
    sse, n = state
    sigma = float(initial_threshold) if n == 0 else math.sqrt(float(sse) / float(n))
    r = 3.0 * sigma
    return r if r < float(ceiling) else float(ceiling)


def _rotation_angle(R):
    """The rotation angle of R (9 row-major floats) by se3_log's route: Shepperd's quaternion, 2 atan2(|v|, w)"""
    if not all(math.isfinite(x) for x in R):
        return math.nan
    tr = (R[0] + R[4]) + R[8]
    v = [0.0, 0.0, 0.0]
    if tr > 0.0:
        r = math.sqrt(tr + 1.0)
        w = 0.5 * r
        r = 0.5 / r
        v = [(R[7] - R[5]) * r, (R[2] - R[6]) * r, (R[3] - R[1]) * r]
    else:
        i = 0
        if R[4] > R[0]:
            i = 1
        if R[8] > R[4 * i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        r = math.sqrt(((R[4 * i] - R[4 * j]) - R[4 * k]) + 1.0)
        v[i] = 0.5 * r
        r = 0.5 / r
        w = (R[3 * k + j] - R[3 * j + k]) * r
        v[j] = (R[3 * j + i] + R[3 * i + j]) * r
        v[k] = (R[3 * k + i] + R[3 * i + k]) * r
    w = abs(w)
    n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
    n = math.sqrt(n2)
    if n2 < SE3_LOG_SMALL * SE3_LOG_SMALL:
        return (2.0 / w - (2.0 / 3.0) * n2 / ((w * w) * w)) * n
    return 2.0 * math.atan2(n, w)


def adaptive_threshold_error(T_prior, T_out, max_range):
    """e of one frame: with D = constant_velocity_increment(T_prior, T_out) (how far registration corrected the
    prediction), 2 max_range sin(theta / 2) + |t_D|.  NaN when a pose is not finite."""
    with np.errstate(invalid="ignore", over="ignore"):
        D = constant_velocity_increment(T_prior, T_out)
    theta = _rotation_angle([float(x) for x in D[:3, :3].reshape(-1)])
    t = [float(x) for x in D[:3, 3]]
    t2 = (t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]
    if not (math.isfinite(theta) and math.isfinite(t2)):
        return math.nan
    return (2.0 * float(max_range)) * math.sin(0.5 * theta) + math.sqrt(t2)


def adaptive_threshold_update(state, T_prior, T_out, min_motion, max_range):
    """The state after a frame that started from T_prior and returned T_out: e is a sample when finite and > min_motion"""
    sse, n = state
    e = adaptive_threshold_error(T_prior, T_out, max_range)
    if math.isfinite(e) and e > float(min_motion):
        return (float(sse) + e * e, int(n) + 1)
    return (float(sse), int(n))


# The motion compensation of dcreg_icp_run_odometry_deskew (dcreg_b200/csrc/se3.cuh): the same formulas, operation order
# and branch thresholds in FP64 NumPy.  A twist is xi = (rho, phi), Sophus's order.
SE3_LOG_SMALL = 1e-10       # |quaternion vector| below which 2 atan(n / w) / n takes its series
SE3_SMALL_ANGLE = 1e-3      # rotation angle below which A, B, C and the V^-1 factor take their series


def _cross(a, b):
    """a x b over the last axis, each entry a_i b_j - a_k b_l in FP64 (the device's order)"""
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def se3_log(D):
    """xi = Log(D) (6,) of a rigid motion D (4, 4), as se3.cuh forms it: the rotation's quaternion by Shepperd's rule
    (w >= 0), theta = 2 atan2(|v|, w) for every angle in [0, pi], rho = V^-1 t.  The exact identity gives exactly 0; a
    D with an entry that is not finite gives NaN."""
    D = np.asarray(D, dtype=np.float64)
    if not np.isfinite(D[:3]).all():
        return np.full(6, np.nan)
    R = [float(x) for x in D[:3, :3].reshape(-1)]
    t = np.array(D[:3, 3], dtype=np.float64)
    tr = (R[0] + R[4]) + R[8]
    v = [0.0, 0.0, 0.0]
    if tr > 0.0:
        r = math.sqrt(tr + 1.0)
        w = 0.5 * r
        r = 0.5 / r
        v = [(R[7] - R[5]) * r, (R[2] - R[6]) * r, (R[3] - R[1]) * r]
    else:
        i = 0
        if R[4] > R[0]:
            i = 1
        if R[8] > R[4 * i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        r = math.sqrt(((R[4 * i] - R[4 * j]) - R[4 * k]) + 1.0)
        v[i] = 0.5 * r
        r = 0.5 / r
        w = (R[3 * k + j] - R[3 * j + k]) * r
        v[j] = (R[3 * j + i] + R[3 * i + j]) * r
        v[k] = (R[3 * k + i] + R[3 * i + k]) * r
    if w < 0.0:
        w, v = -w, [-x for x in v]
    n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
    if n2 < SE3_LOG_SMALL * SE3_LOG_SMALL:
        f = 2.0 / w - (2.0 / 3.0) * n2 / ((w * w) * w)
    else:
        n = math.sqrt(n2)
        f = 2.0 * math.atan2(n, w) / n
    theta = f * math.sqrt(n2)
    phi = np.array([f * v[0], f * v[1], f * v[2]])
    if theta < SE3_SMALL_ANGLE:
        c = 1.0 / 12.0 + (theta * theta) / 720.0
    else:
        h = 0.5 * theta
        c = (1.0 - theta * math.cos(h) / (2.0 * math.sin(h))) / (theta * theta)
    a = _cross(phi, t)
    b = _cross(phi, a)
    return np.concatenate([(t - 0.5 * a) + c * b, phi])


def _exp_coeffs(t2):
    """A = sin(theta) / theta, B = (1 - cos(theta)) / theta^2, C = (theta - sin(theta)) / theta^3 for theta^2 = t2
    (array), with se3.cuh's series below SE3_SMALL_ANGLE"""
    theta = np.sqrt(t2)
    small = theta < SE3_SMALL_ANGLE
    with np.errstate(invalid="ignore", divide="ignore"):
        sn, cs = np.sin(theta), np.cos(theta)
        A = np.where(small, 1.0 - t2 / 6.0 * (1.0 - t2 / 20.0), sn / theta)
        B = np.where(small, 0.5 - t2 / 24.0 * (1.0 - t2 / 30.0), (1.0 - cs) / t2)
        C = np.where(small, 1.0 / 6.0 - t2 / 120.0 * (1.0 - t2 / 42.0), (theta - sn) / (t2 * theta))
    return A, B, C


def se3_exp(xi):
    """Exp(xi) (4, 4) of a twist xi (6,) = (rho, phi): Rodrigues for the rotation and t = V rho, with se3.cuh's
    coefficients"""
    xi = np.asarray(xi, dtype=np.float64)
    rho, phi = xi[:3], xi[3:]
    t2 = np.float64((phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2])
    A, B, C = (float(x) for x in _exp_coeffs(np.array(t2)))
    T = np.eye(4)
    E = np.eye(3)
    for c in range(3):                                      # column c = R e_c, formed as se3.cuh applies R to a point
        a = _cross(phi, E[c])
        T[:3, c] = (E[c] + A * a) + B * _cross(phi, a)
    c1 = _cross(phi, rho)
    T[:3, 3] = (rho + B * c1) + C * _cross(phi, c1)
    return T


def se3_exp_apply(xi, s, p):
    """Exp(s_i xi) p_i for every row (s (N,), p (N, 3) FP64), as se3.cuh applies it: R p + V rho' in FP64, no rounding
    to float32.  Returns (N, 3) float64."""
    s = np.asarray(s, dtype=np.float64)[:, None]
    rho, phi = s * xi[:3], s * xi[3:]
    t2 = (phi[:, 0] * phi[:, 0] + phi[:, 1] * phi[:, 1]) + phi[:, 2] * phi[:, 2]
    A, B, C = (x[:, None] for x in _exp_coeffs(t2))
    a = _cross(phi, p)
    c = _cross(phi, rho)
    return ((p + A * a) + B * _cross(phi, a)) + ((rho + B * c) + C * _cross(phi, c))


def deskew_points(P, timestamps, D):
    """Points of one frame deskewed to mid-sweep as dcreg_icp_run_odometry_deskew does it: p' = fl32(Exp((tau - 0.5)
    Log(D)) p) in FP64 with one float32 rounding, D (4, 4) the frame's increment, timestamps (N,) float32 in [0, 1].  A
    row is copied bit for bit (no arithmetic) when tau = 0.5, when Log(D) is zero or not finite, when the row has a
    non-finite coordinate, or when the result would have one.  P: (N, >=3).  Returns (N, 3) float32."""
    P = np.asarray(P, dtype=np.float32)
    if P.ndim != 2 or P.shape[1] < 3:
        raise ValueError("points must be (N, >=3)")
    xyz = np.array(P[:, :3])
    tau = np.asarray(timestamps, dtype=np.float32).reshape(-1)
    if tau.shape[0] != xyz.shape[0]:
        raise ValueError(f"deskew_points: {xyz.shape[0]} points but {tau.shape[0]} timestamps")
    xi = se3_log(D)
    if not np.isfinite(xi).all() or (xi == 0.0).all():
        return xyz
    s = tau.astype(np.float64) - 0.5
    move = (s != 0.0) & np.isfinite(xyz).all(axis=1)
    with np.errstate(over="ignore", invalid="ignore"):
        q = se3_exp_apply(xi, s[move], xyz[move].astype(np.float64)).astype(np.float32)
    ok = np.isfinite(q).all(axis=1)
    rows = np.nonzero(move)[0][ok]
    xyz[rows] = q[ok]
    return xyz


# The gyroscope rotation of dcreg_icp_run_odometry_gyro (dcreg_b200/csrc/se3.cuh): the same formulas and operation order
# in Python floats and elementwise NumPy (FP64, one rounding per operation, no FMA; sin and cos from libm).  samples:
# (n, 4) rows (t, wx, wy, wz) in the IMU frame, t strictly ascending.
GYRO_ORTHO_TOL = 1e-6       # the largest |R^T R - I| entry R_sensor_imu may have


def _so3_exp(phi):
    """Exp(phi) as 9 row-major floats: R_rr = 1 + B (phi_r^2 - t2), R_rc = A K_rc + B phi_r phi_c (se3::so3_exp)"""
    t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2]
    theta = math.sqrt(t2)
    if theta < SE3_SMALL_ANGLE:
        A = 1.0 - (t2 / 6.0) * (1.0 - t2 / 20.0)
        B = 0.5 - (t2 / 24.0) * (1.0 - t2 / 30.0)
    else:
        A = math.sin(theta) / theta
        B = (1.0 - math.cos(theta)) / t2
    K = [0.0, -phi[2], phi[1], phi[2], 0.0, -phi[0], -phi[1], phi[0], 0.0]
    return [1.0 + B * (phi[r] * phi[r] - t2) if r == c else A * K[3 * r + c] + B * (phi[r] * phi[c])
            for r in range(3) for c in range(3)]


def _mat3_mul(M, E):
    """M E as 9 row-major floats, every entry ((m0 e0 + m1 e1) + m2 e2)"""
    return [(M[3 * r] * E[c] + M[3 * r + 1] * E[3 + c]) + M[3 * r + 2] * E[6 + c] for r in range(3) for c in range(3)]


def _gyro_rate(R, bias, row):
    """R (omega - bias) of one sample row, each entry ((r0 d0 + r1 d1) + r2 d2)"""
    d = [float(row[1]) - bias[0], float(row[2]) - bias[1], float(row[3]) - bias[2]]
    return [(R[3 * r] * d[0] + R[3 * r + 1] * d[1]) + R[3 * r + 2] * d[2] for r in range(3)]


def _gyro_piece(M, w, d):
    """M Exp(w d)"""
    return _mat3_mul(M, _so3_exp([w[0] * d, w[1] * d, w[2] * d]))


def _gyro_setup(samples, R_sensor_imu, bias):
    S = np.asarray(samples, dtype=np.float64).reshape(-1, 4)
    R = [float(x) for x in np.asarray(R_sensor_imu, dtype=np.float64).reshape(9)]
    b = [float(x) for x in np.asarray(bias, dtype=np.float64).reshape(3)]
    return S, [float(t) for t in S[:, 0]], R, b


def gyro_rotation(samples, a, b, R_sensor_imu=np.eye(3), bias=(0.0, 0.0, 0.0)):
    """G(a -> b) (3, 3) as the device forms a prior's rotation: for a <= b the walk from a to b in time order, M = I then M
    = M Exp(w_j d_j) over the sample intervals [t_j, t_{j+1}) clipped to [a, b] (d_j > 0), w_j = R_sensor_imu (omega_j -
    bias) (zero-order hold).  It reads only the samples that bracket [a, b]: one at or before a and one at or after b
    must exist (ValueError otherwise).  a > b: G(b -> a)^T."""
    a, b = float(a), float(b)
    if a > b:
        return gyro_rotation(samples, b, a, R_sensor_imu, bias).T
    S, t, R, bs = _gyro_setup(samples, R_sensor_imu, bias)
    j = bisect.bisect_right(t, a) - 1
    if j < 0 or not t or t[-1] < b:
        raise ValueError(f"gyro_rotation: the samples do not bracket [{a!r}, {b!r}]")
    M = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    cur = a
    while cur < b:
        nxt = min(t[j + 1], b)
        M = _gyro_piece(M, _gyro_rate(R, bs, S[j]), nxt - cur)
        cur = nxt
        j += 1
    return np.array(M).reshape(3, 3)


def gyro_knots(samples, start, span, R_sensor_imu=np.eye(3), bias=(0.0, 0.0, 0.0)):
    """The knot table of the sweep [start, start + span] (se3::gyro_knots): knots at its mid-sweep time tm = start + 0.5
    span and at every sample time strictly inside the sweep other than tm, ascending, each a row of 16: the time, Q =
    G(tm -> time) as the walk from tm forms it (backwards, with negative durations, for knots before tm), the rate after
    the knot (of the last sample at or before it) and the rate before it (of the last sample strictly before it).  Needs a
    sample at or before start and one at or after the end.  Returns (K, 16) float64."""
    start, span = float(start), float(span)
    tm, end = start + 0.5 * span, start + span
    S, t, R, bs = _gyro_setup(samples, R_sensor_imu, bias)
    lo = bisect.bisect_right(t, start) - 1
    if lo < 0 or not t or t[-1] < end:
        raise ValueError(f"gyro_knots: the samples do not bracket the sweep [{start!r}, {end!r}]")
    jb, ja = bisect.bisect_left(t, tm) - 1, bisect.bisect_right(t, tm) - 1
    I = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    mid = [tm] + I + _gyro_rate(R, bs, S[ja]) + _gyro_rate(R, bs, S[jb])
    before, Q, cur, w = [], I, tm, mid[13:16]
    while jb > lo:                                      # the samples in (start, tm), newest first
        Q = _gyro_piece(Q, w, t[jb] - cur)
        cur = t[jb]
        k = [cur] + Q + _gyro_rate(R, bs, S[jb]) + _gyro_rate(R, bs, S[jb - 1])
        before.append(k)
        w = k[13:16]
        jb -= 1
    after, Q, cur, w = [], I, tm, mid[10:13]
    while ja + 1 < len(t) and t[ja + 1] < end:          # the samples in (tm, end)
        Q = _gyro_piece(Q, w, t[ja + 1] - cur)
        cur = t[ja + 1]
        ja += 1
        k = [cur] + Q + _gyro_rate(R, bs, S[ja]) + _gyro_rate(R, bs, S[ja - 1])
        after.append(k)
        w = k[10:13]
    return np.array(before[::-1] + [mid] + after)


def gyro_increment(samples, tm_prev, tm, T_prev2=None, T_prev=None, R_sensor_imu=np.eye(3), bias=(0.0, 0.0, 0.0)):
    """The increment D a non-anchor frame's prior is composed with (dcreg_icp_run_odometry_gyro): rotation G(tm_prev ->
    tm), translation that of constant_velocity_increment(T_prev2, T_prev) (zero right after the anchor: T_prev2 None)"""
    D = np.eye(4) if T_prev2 is None else constant_velocity_increment(T_prev2, T_prev)
    D[:3, :3] = gyro_rotation(samples, tm_prev, tm, R_sensor_imu, bias)
    return D


def deskew_points_gyro(P, timestamps, frame_time, tm_prev, samples, t_D=(0.0, 0.0, 0.0), R_sensor_imu=np.eye(3),
                       bias=(0.0, 0.0, 0.0)):
    """Points of one frame deskewed to mid-sweep as dcreg_icp_run_odometry_gyro does it (se3::deskew_point_gyro).
    frame_time = (start, span); point i's time is t = start + tau_i span, tm = start + 0.5 span.  G = G(tm -> t) from
    the sweep's knot table (gyro_knots): for t >= tm the last knot k at or before t, G = Q_k Exp(w_after (t - t_k)); for
    t < tm the first knot at or after t, G = Q_k Exp(w_before (t - t_k)).  p' = fl32(G p + s t_D), s = (t - tm) / (tm -
    tm_prev), every entry (((g0 x + g1 y) + g2 z) + s t_D).  A row is copied bit for bit when t = tm, when it has a
    non-finite coordinate, or when the result would have one or equal it.  P: (N, >=3).  Returns (N, 3) float32."""
    P = np.asarray(P, dtype=np.float32)
    if P.ndim != 2 or P.shape[1] < 3:
        raise ValueError("points must be (N, >=3)")
    xyz = np.array(P[:, :3])
    tau = np.asarray(timestamps, dtype=np.float32).reshape(-1)
    if tau.shape[0] != xyz.shape[0]:
        raise ValueError(f"deskew_points_gyro: {xyz.shape[0]} points but {tau.shape[0]} timestamps")
    start, span = float(frame_time[0]), float(frame_time[1])
    tm = start + 0.5 * span
    K = gyro_knots(samples, start, span, R_sensor_imu, bias)
    t = start + tau.astype(np.float64) * span
    rows = np.nonzero((t != tm) & np.isfinite(xyz).all(axis=1))[0]
    t = t[rows]
    fwd = t >= tm
    k = np.where(fwd, np.searchsorted(K[:, 0], t, side="right") - 1, np.searchsorted(K[:, 0], t, side="left"))
    w = np.where(fwd[:, None], K[k, 10:13], K[k, 13:16])
    phi = w * (t - K[k, 0])[:, None]
    t2 = (phi[:, 0] * phi[:, 0] + phi[:, 1] * phi[:, 1]) + phi[:, 2] * phi[:, 2]
    theta = np.sqrt(t2)
    small = theta < SE3_SMALL_ANGLE
    sn = np.array([math.sin(x) for x in theta]) if len(theta) else theta
    cs = np.array([math.cos(x) for x in theta]) if len(theta) else theta
    with np.errstate(invalid="ignore", divide="ignore"):
        A = np.where(small, 1.0 - (t2 / 6.0) * (1.0 - t2 / 20.0), sn / theta)
        B = np.where(small, 0.5 - (t2 / 24.0) * (1.0 - t2 / 30.0), (1.0 - cs) / t2)
    Kx = [np.zeros_like(t2), -phi[:, 2], phi[:, 1], phi[:, 2], np.zeros_like(t2), -phi[:, 0], -phi[:, 1], phi[:, 0],
          np.zeros_like(t2)]
    E = [1.0 + B * (phi[:, r] * phi[:, r] - t2) if r == c else A * Kx[3 * r + c] + B * (phi[:, r] * phi[:, c])
         for r in range(3) for c in range(3)]
    Q = K[k, 1:10]
    G = [(Q[:, 3 * r] * E[c] + Q[:, 3 * r + 1] * E[3 + c]) + Q[:, 3 * r + 2] * E[6 + c] for r in range(3) for c in range(3)]
    s = (t - tm) / (tm - float(tm_prev))
    tD = [float(x) for x in np.asarray(t_D, dtype=np.float64).reshape(3)]
    p = xyz[rows].astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        q = np.stack([(((G[3 * r] * p[:, 0] + G[3 * r + 1] * p[:, 1]) + G[3 * r + 2] * p[:, 2]) + s * tD[r])
                      for r in range(3)], axis=1).astype(np.float32)
    ok = np.isfinite(q).all(axis=1) & ~(q == xyz[rows]).all(axis=1)
    xyz[rows[ok]] = q[ok]
    return xyz


# The accelerometer prior of dcreg_icp_run_odometry_imu (se3::gyro_rotation with acc_bias, se3::imu_translation,
# se3::imu_velocity): the same formulas and operation order in Python floats (FP64, one rounding per operation, no FMA).
# samples: (n, 7) rows (t, wx, wy, wz, ax, ay, az) in the IMU frame, t strictly ascending.
def imu_preintegrate(samples, a, b, R_sensor_imu=np.eye(3), gyro_bias=(0.0, 0.0, 0.0), accel_bias=(0.0, 0.0, 0.0)):
    """(G, alpha, beta, gamma) over [a, b], a <= b: G = gyro_rotation(samples, a, b) bit for bit, and over every piece
    [u, u + d] of that walk, with M the walk's rotation at u and f = R_sensor_imu (acc_j - accel_bias) held over the
    piece, m = M f d (each entry ((m0 f0 + m1 f1) + m2 f2) d), alpha += m, beta += m ((b - u) - 0.5 d), gamma += m ((u -
    a) + 0.5 d).  It reads only the samples that bracket [a, b] (ValueError when they do not).  Returns (3, 3) and three
    (3,) arrays."""
    a, b = float(a), float(b)
    S = np.asarray(samples, dtype=np.float64).reshape(-1, 7)
    t = [float(x) for x in S[:, 0]]
    R = [float(x) for x in np.asarray(R_sensor_imu, dtype=np.float64).reshape(9)]
    bg = [float(x) for x in np.asarray(gyro_bias, dtype=np.float64).reshape(3)]
    ba = [float(x) for x in np.asarray(accel_bias, dtype=np.float64).reshape(3)]
    j = bisect.bisect_right(t, a) - 1
    if not a <= b or j < 0 or not t or t[-1] < b:
        raise ValueError(f"imu_preintegrate: the samples do not bracket [{a!r}, {b!r}]")
    M = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    al, be, ga = [0.0] * 3, [0.0] * 3, [0.0] * 3
    cur = a
    while cur < b:
        nxt = min(t[j + 1], b)
        d = nxt - cur
        row = S[j]
        f = _gyro_rate(R, ba, [0.0, float(row[4]), float(row[5]), float(row[6])])
        h = 0.5 * d
        wb, wg = (b - cur) - h, (cur - a) + h
        for r in range(3):
            m = ((M[3 * r] * f[0] + M[3 * r + 1] * f[1]) + M[3 * r + 2] * f[2]) * d
            al[r] = al[r] + m
            be[r] = be[r] + m * wb
            ga[r] = ga[r] + m * wg
        M = _gyro_piece(M, _gyro_rate(R, bg, row), d)
        cur = nxt
        j += 1
    return np.array(M).reshape(3, 3), np.array(al), np.array(be), np.array(ga)


def imu_translation(T_prev, v_prev, gravity, beta, dt):
    """t_D = dt R^T v + (0.5 dt^2) R^T g + beta, R = T_prev's rotation, every R^T x entry ((R_0r x0 + R_1r x1) + R_2r x2)
    (se3::imu_translation).  Returns (3,)."""
    R = [float(x) for x in np.asarray(T_prev, dtype=np.float64)[:3, :3].reshape(9)]
    v = [float(x) for x in np.asarray(v_prev, dtype=np.float64).reshape(3)]
    g = [float(x) for x in np.asarray(gravity, dtype=np.float64).reshape(3)]
    be = [float(x) for x in np.asarray(beta, dtype=np.float64).reshape(3)]
    dt = float(dt)
    c2 = 0.5 * (dt * dt)
    out = []
    for r in range(3):
        rv = (R[r] * v[0] + R[3 + r] * v[1]) + R[6 + r] * v[2]
        rg = (R[r] * g[0] + R[3 + r] * g[1]) + R[6 + r] * g[2]
        out.append((dt * rv + c2 * rg) + be[r])
    return np.array(out)


def imu_increment(samples, tm_prev, tm, T_prev, v_prev, gravity, R_sensor_imu=np.eye(3), gyro_bias=(0.0, 0.0, 0.0),
                  accel_bias=(0.0, 0.0, 0.0)):
    """The increment D a non-anchor frame's prior is composed with (dcreg_icp_run_odometry_imu): rotation G(tm_prev ->
    tm), translation imu_translation(T_prev, v_prev, gravity, beta, tm - tm_prev).  T_prior = compose_prior(T_prev, D).
    Returns (4, 4)."""
    G, _, beta, _ = imu_preintegrate(samples, tm_prev, tm, R_sensor_imu, gyro_bias, accel_bias)
    D = np.eye(4)
    D[:3, :3] = G
    D[:3, 3] = imu_translation(T_prev, v_prev, gravity, beta, float(tm) - float(tm_prev))
    return D


def imu_velocity(samples, tm_prev, tm, T_prev, T, gravity, R_sensor_imu=np.eye(3), gyro_bias=(0.0, 0.0, 0.0),
                 accel_bias=(0.0, 0.0, 0.0)):
    """A frame's velocity once it has stopped (dcreg_icp_run_odometry_imu): v = (t - t_prev) / dt + (R_prev gamma) / dt +
    (0.5 dt) g, dt = tm - tm_prev, every R_prev gamma entry ((r0 g0 + r1 g1) + r2 g2) (se3::imu_velocity).  T_prev, T:
    the two frames' poses.  Returns (3,)."""
    _, _, _, gamma = imu_preintegrate(samples, tm_prev, tm, R_sensor_imu, gyro_bias, accel_bias)
    return imu_velocity_from(T_prev, T, gravity, gamma, float(tm) - float(tm_prev))


def imu_velocity_from(T_prev, T, gravity, gamma, dt):
    """imu_velocity from a given gamma and dt"""
    A = np.asarray(T_prev, dtype=np.float64)
    B = np.asarray(T, dtype=np.float64)
    Rp = [float(x) for x in A[:3, :3].reshape(9)]
    g = [float(x) for x in np.asarray(gravity, dtype=np.float64).reshape(3)]
    gm = [float(x) for x in np.asarray(gamma, dtype=np.float64).reshape(3)]
    dt = float(dt)
    h = 0.5 * dt
    out = []
    for r in range(3):
        rg = (Rp[3 * r] * gm[0] + Rp[3 * r + 1] * gm[1]) + Rp[3 * r + 2] * gm[2]
        out.append(((float(B[r, 3]) - float(A[r, 3])) / dt + rg / dt) + h * g[r])
    return np.array(out)


VOXEL_LIMIT = 1 << 20    # voxel coordinates must lie in [-2^20, 2^20): 21 bits per axis in one 63-bit key


def _max_points(v, name="max_points"):
    """A voxel filter's cap as a C int: an integer >= 1 (bools and floats are refused)"""
    if isinstance(v, (bool, np.bool_)):
        raise ValueError(f"{name} must be an integer >= 1, not {v!r}")
    try:
        n = operator.index(v)
    except TypeError:
        raise ValueError(f"{name} must be an integer >= 1, not {v!r}") from None
    if not 1 <= n < 2 ** 31:
        raise ValueError(f"{name} must be an integer in [1, 2^31), not {n}")
    return n


def voxel_downsample(P, voxel, max_points=1, min_spacing=0.0):
    """The voxel filter of dcreg_voxel_downsample_n (min_spacing = 0) and dcreg_voxel_downsample_spaced, bit for bit:
    the voxel of a point is np.floor(p.astype(float64) * (1.0 / voxel)) per axis, rows with a non-finite coordinate have
    none and are dropped, and each voxel keeps its max_points points of smallest index (1: its first point,
    dcreg_voxel_downsample).  min_spacing > 0: going through a voxel's rows in ascending index, a row is kept iff fewer
    than max_points rows of its voxel are kept before it and each kept row q before it has ((px - qx)^2 + (py - qy)^2) +
    (pz - qz)^2 >= min_spacing * min_spacing in FP64 (KISS-ICP's AddPoints).  P: (N, >=3).  Returns (points (K, 3)
    float32, the kept rows' coordinates unchanged; index (K,) int64, their rows in P, ascending).  Raises ValueError for
    a voxel that is not finite and > 0, a max_points that is not an integer >= 1, a min_spacing that is not finite and
    >= 0, or a voxel coordinate outside [-2^20, 2^20)."""
    P = np.asarray(P, dtype=np.float32)
    if P.ndim != 2 or P.shape[1] < 3:
        raise ValueError("points must be (N, >=3)")
    max_points = _max_points(max_points)
    voxel, min_spacing = float(voxel), _min_spacing(min_spacing)
    if not (voxel > 0.0 and np.isfinite(voxel)):
        raise ValueError(f"voxel_downsample: voxel must be finite and > 0, not {voxel}")
    xyz = P[:, :3]
    rows = np.nonzero(np.isfinite(xyz).all(axis=1))[0]
    with np.errstate(invalid="ignore", over="ignore"):
        keys = np.floor(xyz[rows].astype(np.float64) * (1.0 / voxel))
    if not ((keys >= -VOXEL_LIMIT) & (keys < VOXEL_LIMIT)).all():
        raise ValueError("voxel_downsample: a voxel coordinate lies outside [-2^20, 2^20) (voxel too small for the "
                         "cloud's coordinates)")
    k = keys.astype(np.int64) + VOXEL_LIMIT
    ids = (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]
    # a stable sort by voxel keeps each voxel's rows ascending: a row's rank in its voxel is its distance to the voxel's
    # first sorted position
    order = np.argsort(ids, kind="stable")
    s = ids[order]
    at = np.arange(len(s))
    starts = np.ones(len(s), dtype=bool)
    starts[1:] = s[1:] != s[:-1]
    rank = at - np.maximum.accumulate(np.where(starts, at, 0))
    if min_spacing > 0.0 and max_points > 1:
        sel = order[_spaced_ranks(xyz[rows[order]], np.nonzero(starts)[0], max_points, min_spacing)]
    else:
        sel = order[rank < max_points]
    keep = rows[np.sort(sel)].astype(np.int64)
    return np.ascontiguousarray(xyz[keep]), keep


def _min_spacing(s):
    s = float(s)
    if not (s >= 0.0 and np.isfinite(s)):
        raise ValueError(f"min_spacing must be finite and >= 0 (0: no spacing), not {s}")
    return s


def _spaced_ranks(X, starts, max_points, min_spacing):
    """The spacing rule over voxels sorted into runs: X (N, 3) float32 rows, each voxel one run beginning at `starts`
    with its rows in ascending index.  Round r settles the rank-r row of every run still open, against that run's kept
    rows.  Returns the sorted positions kept, ascending."""
    n = len(X)
    length = np.append(starts[1:], n) - starts
    room = np.minimum(length, max_points)
    base = np.cumsum(room) - room                           # run g's kept rows: kept[base[g] : base[g] + count[g]]
    kept = np.empty((int(room.sum()), 3))                   # in FP64 (exact)
    count = np.zeros(len(starts), dtype=np.int64)
    flag = np.zeros(n, dtype=bool)
    s2 = min_spacing * min_spacing
    open_ = np.arange(len(starts))
    r = 0
    while len(open_):
        at = starts[open_] + r
        c = X[at].astype(np.float64)
        held = count[open_]
        ok = np.ones(len(open_), dtype=bool)
        row = np.repeat(np.arange(len(open_)), held)        # every (candidate, kept row of its run) pair at once
        d = c[row] - kept[np.repeat(base[open_], held) + np.arange(len(row)) - np.repeat(np.cumsum(held) - held, held)]
        ok[row[~((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] >= s2)]] = False
        g = open_[ok]
        flag[at[ok]] = True
        kept[base[g] + count[g]] = c[ok]
        count[g] += 1
        r += 1
        open_ = open_[(length[open_] > r) & (count[open_] < max_points)]
    return np.nonzero(flag)[0]


def _voxel_ids(xyz, voxel, name):
    """Packed voxel keys of the rows of xyz (K, 3) float32, all finite, as voxel_downsample forms them"""
    with np.errstate(invalid="ignore", over="ignore"):
        keys = np.floor(xyz.astype(np.float64) * (1.0 / voxel))
    if not ((keys >= -VOXEL_LIMIT) & (keys < VOXEL_LIMIT)).all():
        raise ValueError(f"{name}: a voxel coordinate lies outside [-2^20, 2^20) (voxel too small for the cloud's "
                         "coordinates)")
    k = keys.astype(np.int64) + VOXEL_LIMIT
    return (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]


def voxel_map_prune(X, voxel, max_distance, t):
    """The prune of the voxel map (dcreg_icp_run_odometry_map), bit for bit: every point of every voxel whose first point
    q (its row of smallest index in X) has ((qx - tx)^2 + (qy - ty)^2) + (qz - tz)^2 >= max_distance^2 is dropped, in
    FP64 from the float32 coordinates with one rounding per operation, max_distance^2 = max_distance * max_distance
    (KISS-ICP's RemovePointsFarFromLocation).  Voxels as in voxel_downsample; rows with a non-finite coordinate have no
    voxel and are dropped.  X: (N, >=3); t: the translation (3,).  Returns (points (K, 3) float32, the survivors' rows
    unchanged and in order; index (K,) int64, their rows in X)."""
    X = np.asarray(X, dtype=np.float32)
    if X.ndim != 2 or X.shape[1] < 3:
        raise ValueError("points must be (N, >=3)")
    voxel, max_distance = float(voxel), float(max_distance)
    if not (voxel > 0.0 and np.isfinite(voxel)):
        raise ValueError(f"voxel_map_prune: voxel must be finite and > 0, not {voxel}")
    if not max_distance > 0.0:
        raise ValueError(f"voxel_map_prune: max_distance must be > 0 (+inf: no pruning), not {max_distance}")
    xyz = X[:, :3]
    rows = np.nonzero(np.isfinite(xyz).all(axis=1))[0]
    ids = _voxel_ids(xyz[rows], voxel, "voxel_map_prune")
    order = np.argsort(ids, kind="stable")
    s = ids[order]
    starts = np.ones(len(s), dtype=bool)
    starts[1:] = s[1:] != s[:-1]
    at = np.arange(len(s))
    first = np.empty(len(s), dtype=np.int64)
    first[order] = order[np.maximum.accumulate(np.where(starts, at, 0))]     # each row's voxel's first row (of rows)
    q = xyz[rows[first]].astype(np.float64)
    d = q - np.asarray(t, dtype=np.float64).reshape(3)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = rows[~(d2 >= max_distance * max_distance)].astype(np.int64)
    return np.ascontiguousarray(xyz[keep]), keep


def voxel_map_update(M, P, T, voxel, max_points, max_distance, min_spacing=0.0):
    """One update of the voxel map of dcreg_icp_run_odometry_map, bit for bit: prune(cap(M ++ map_points(T, P)), t_T)
    with cap = voxel_downsample(., voxel, max_points, min_spacing) (M first: older points win, KISS-ICP's AddPoints;
    min_spacing: dcreg_set_map_spacing) and prune = voxel_map_prune at T's translation.  M: the map (K, 3) float32 (may
    be empty); P: the frame's points (N, >=3) in its sensor frame; T: its pose (4, 4).  Returns the new map (K', 3)
    float32."""
    M = np.asarray(M, dtype=np.float32).reshape(-1, 3)
    X = np.concatenate([M, map_points(T, P)])
    capped, _ = voxel_downsample(X, voxel, max_points, min_spacing)
    return voxel_map_prune(capped, voxel, max_distance, np.asarray(T, dtype=np.float64)[:3, 3])[0]


class IcpResult:
    def __init__(self, status, converged, iterations, T, logs, cov=None):
        self.status, self.converged, self.iterations, self.T, self.logs = status, converged, iterations, T, logs
        self.cov = cov
        self.metrics = None
        self.T_prior = None             # icp_run_sequences: the initial pose the frame started from
        self.n_points = None            # icp_run_odometry: the frame's points after the source filter
        self.deskewed = None            # icp_run_odometry (want_deskewed): those points after deskewing
        self.search_radius = None       # icp_run_odometry (adaptive / want_radius): the radius the frame registered with


def _trial_results(st, conv, n_it, T_out, logs, cap, cov=None):
    """One IcpResult per trial from a batched call's per-trial outputs.  logs: cap records per trial, or None.  A trial
    holds min(iterations, cap) records, one more when it aborted with NONFINITE_UPDATE before the cap (that abort
    writes the record of the failed iteration)."""
    out = []
    for b in range(len(st)):
        recs = []
        if logs is not None:
            nrec = min(n_it[b], cap)
            if st[b] == NONFINITE_UPDATE and n_it[b] < cap:
                nrec = n_it[b] + 1
            recs = [logs[b * cap + i] for i in range(nrec)]
        out.append(IcpResult(int(st[b]), bool(conv[b]), int(n_it[b]), T_out[b], recs, None if cov is None else cov[b]))
    return out


class Context:
    """One engine context per GPU (owns the stream, device buffers and the optional NCCL comm)."""

    _map_input_voxel = 0.0      # dcreg_set_map_input_voxel as set_map_input_voxel last set it

    def __init__(self, device: int = 0):
        self.lib = load_library()
        self._h = C.c_void_p()
        rc = self.lib.dcreg_create(device, C.byref(self._h))
        if rc != OK:
            msg = self.lib.dcreg_last_error(self._h).decode() if self._h else "no CUDA device"
            if self._h:
                self.lib.dcreg_destroy(self._h)
            self._h = None
            raise DcregError(rc, msg)
        self.n_source = 0
        self._lane_params = False

    # -- lifetime --
    def close(self):
        if getattr(self, "_h", None):
            self.lib.dcreg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc, allow=()):
        if rc != OK and rc not in allow:
            raise DcregError(rc, self.lib.dcreg_last_error(self._h).decode())
        return rc

    @property
    def stream(self) -> int:
        return int(self.lib.dcreg_stream(self._h) or 0)

    @property
    def launch_count(self) -> int:
        return int(self.lib.dcreg_launch_count(self._h))

    @property
    def loop_variant_launches(self) -> np.ndarray:
        """Loop-kernel launches since the context was created, one count per loop_plan.hpp variant (18, int64): which
        instantiation of the iteration kernel each call ran (include/dcreg_b200.h, dcreg_loop_variant_launches)."""
        out = np.zeros(LOOP_VARIANTS, np.int64)
        self._check(self.lib.dcreg_loop_variant_launches(self._h, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    # -- clouds --
    def set_source(self, xyz):
        a = _as_points(xyz)
        self._check(self.lib.dcreg_set_source(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0], a.shape[1]))
        self.n_source = a.shape[0]

    def set_target(self, xyz, cell_size: float):
        """A dense grid, or past 2^27 cells of the bounding box a sparse row index on which the batched calls and
        find_planes run as on a dense grid (include/dcreg_b200.h, dcreg_set_target)."""
        a = _as_points(xyz)
        self._check(self.lib.dcreg_set_target(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0], a.shape[1],
                                              float(cell_size)))

    def set_target_sparse(self, xyz, cell_size: float):
        """Identical to set_target (dcreg_set_target_sparse, kept for compatibility: include/dcreg_b200.h)."""
        a = _as_points(xyz)
        self._check(self.lib.dcreg_set_target_sparse(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0],
                                                     a.shape[1], float(cell_size)))

    def set_sparse_maps(self, enable: bool):
        """Sparse row indexes, instead of a refusal, for odometry's local maps and icp_run_pairs' targets too large for
        dense grids (include/dcreg_b200.h, dcreg_set_sparse_maps).  A session keeps the value it had when it opened."""
        self._check(self.lib.dcreg_set_sparse_maps(self._h, 1 if enable else 0))

    def set_map_spacing(self, min_spacing: float):
        """Minimum point spacing of odometry's map filter (include/dcreg_b200.h, dcreg_set_map_spacing): every local
        map's voxels keep points at least min_spacing apart, as api.voxel_downsample(..., min_spacing) keeps them (0, the
        default: the cap rule; KISS-ICP uses map_voxel / sqrt(map_max_points)).  A session keeps the value it had when it
        opened."""
        self._check(self.lib.dcreg_set_map_spacing(self._h, float(min_spacing)))

    def set_map_input_voxel(self, voxel: float):
        """The map-input filter of scan-to-map odometry (include/dcreg_b200.h, dcreg_set_map_input_voxel; KISS-ICP's
        Voxelize): with voxel > 0 the frames enter the local maps as voxel_downsample(frame, voxel) and register with
        voxel_downsample(voxel_downsample(frame, voxel), source_voxel, source_max_points), its NumPy twin (0, the
        default: the maps take the source).  Applies to icp_run_odometry, icp_run_odometry_map and the sessions (which
        keep the value they had when they opened), whatever their own voxel sizes."""
        self._check(self.lib.dcreg_set_map_input_voxel(self._h, float(voxel)))
        self._map_input_voxel = float(voxel)

    def set_prior_map(self, enable: int):
        """Localisation in a prior map (include/dcreg_b200.h, dcreg_set_prior_map): with 1, icp_run_odometry (window
        forms, map_frames >= 1) and the window sessions register every frame against the context's target instead of a
        local map, each sequence's first frame from its T_init (0, the default: local maps).  Anything but 0 or 1
        raises.  A session keeps the value it had when it opened, and local_map raises on it."""
        self._check(self.lib.dcreg_set_prior_map(self._h, int(enable)))

    def set_lane_params(self, enable: bool):
        """Per-lane solver settings (include/dcreg_b200.h, dcreg_set_lane_params): the batched calls' params point to one
        IcpParams per lane.  The Python calls set it themselves from their params argument (one IcpParams or a sequence
        of them), so this is for callers of the C functions.  A session keeps the value it had when it opened."""
        self._check(self.lib.dcreg_set_lane_params(self._h, 1 if enable else 0))
        self._lane_params = bool(enable)

    def _lanes(self, name, params, n):
        """params as a call with n lanes takes it: (entry 0, the library argument, whether it holds one entry per lane).
        params: one IcpParams for every lane, or a sequence of n, one per lane (a wrong length raises ValueError)."""
        if isinstance(params, IcpParams):
            return params, C.byref(params), False
        entries = list(params)
        if len(entries) != n:
            raise ValueError(f"{name}: {n} lanes but {len(entries)} parameter sets")
        arr = (IcpParams * n)(*entries)
        return arr[0], arr, True

    @contextlib.contextmanager
    def _lane_setting(self, per_lane: bool):
        """dcreg_set_lane_params as the params argument of the call inside needs it, restored afterwards"""
        prev = self._lane_params
        if per_lane != prev:
            self.set_lane_params(per_lane)
        try:
            yield
        finally:
            if per_lane != prev:
                self.set_lane_params(prev)

    # -- seams --
    def find_planes(self, T, search_radius: float, want_planes: bool = True):
        T = np.ascontiguousarray(T, dtype=np.float64)
        planes = np.empty((self.n_source, 4), dtype=np.float64) if want_planes else None
        npt = C.c_int64(0)
        self._check(self.lib.dcreg_find_planes(self._h, _dptr(T), float(search_radius),
                                               _dptr(planes) if want_planes else None, C.byref(npt)))
        return planes, int(npt.value)

    def reduce_normal_equations(self, src4, plane4, T, use_weight_derivative: bool):
        """Host arrays in, (out27, stats) out.  plane4 dtype float32 -> 32 B/slot, float64 -> 48 B/slot."""
        src4 = np.ascontiguousarray(src4, dtype=np.float32)
        assert src4.ndim == 2 and src4.shape[1] == 4
        plane4 = np.ascontiguousarray(plane4)
        is64 = plane4.dtype == np.float64
        if not is64:
            plane4 = plane4.astype(np.float32, copy=False)
        out = np.empty(27); stats = np.empty(3)
        prt = pose_Rt(T)
        self._check(self.lib.dcreg_reduce_normal_equations_host(
            self._h, src4.ctypes.data_as(C.POINTER(C.c_float)), plane4.ctypes.data_as(C.c_void_p), int(is64),
            src4.shape[0], _dptr(prt), int(bool(use_weight_derivative)), _dptr(out), _dptr(stats)))
        self.n_source = src4.shape[0]
        return out, stats

    def reduce_device(self, plane_is_f64: bool, T, use_weight_derivative: bool):
        """K1 over the ctx-resident source + planes (after find_planes / freeze_planes_f32)."""
        out = np.empty(27); stats = np.empty(3)
        prt = pose_Rt(T)
        fn = self.lib.dcreg_reduce_normal_equations_f64plane if plane_is_f64 else self.lib.dcreg_reduce_normal_equations
        planes = self.lib.dcreg_device_planes_f64(self._h) if plane_is_f64 else self.lib.dcreg_device_planes_f32(self._h)
        self._check(fn(self._h, self.lib.dcreg_device_source(self._h), planes, self.n_source, _dptr(prt),
                       int(bool(use_weight_derivative)), _dptr(out), _dptr(stats)))
        return out, stats

    def freeze_planes_f32(self):
        self._check(self.lib.dcreg_freeze_planes_f32(self._h))

    def time_reduce(self, plane_is_f64: bool, T, use_weight_derivative: bool, reps: int, flush_l2: bool) -> float:
        ms = C.c_float(0)
        prt = pose_Rt(T)
        self._check(self.lib.dcreg_time_reduce(self._h, int(plane_is_f64), _dptr(prt), int(bool(use_weight_derivative)),
                                               reps, int(flush_l2), C.byref(ms)))
        return float(ms.value)

    def time_iteration(self, params: IcpParams, T, what: int, reps: int) -> float:
        ms = C.c_float(0)
        T = np.ascontiguousarray(T, dtype=np.float64)
        self._check(self.lib.dcreg_time_iteration(self._h, C.byref(params), _dptr(T), int(what), int(reps), C.byref(ms)))
        return float(ms.value)

    def iteration_timeline(self, params: IcpParams, T, iters: int):
        """Phase time stamps (ns) of the last of `iters` real iterations from pose T: (blocks (n, 16), solve (16,))."""
        T = np.ascontiguousarray(T, dtype=np.float64)
        cap = 4096
        out = np.zeros((cap, 16), dtype=np.uint64)
        nb = C.c_int(0)
        self._check(self.lib.dcreg_iteration_timeline(self._h, C.byref(params), _dptr(T), int(iters),
                                                      out.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(nb)))
        return out[:nb.value].astype(np.int64), out[nb.value].astype(np.int64)

    def iteration_counters(self, enable: bool = True):
        out = (C.c_uint64 * 2)()
        self._check(self.lib.dcreg_iteration_counters(self._h, int(enable), out))
        return int(out[0]), int(out[1])

    def analyze_and_solve(self, H27, params: IcpParams):
        """DCReg::analyzeDegeneracy + solveDegenerateSystem on the device.  Returns (Analysis, dx, status)."""
        H27 = np.ascontiguousarray(H27, dtype=np.float64)
        a = Analysis(); dx = np.empty(6)
        rc = self._check(self.lib.dcreg_analyze_and_solve(self._h, _dptr(H27), C.byref(params), C.byref(a), _dptr(dx)),
                         allow=(NONFINITE_UPDATE,))
        return a, dx, rc

    def solve_pcg(self, A, b, P, max_iterations: int, tolerance: float):
        A = np.ascontiguousarray(A, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
        P = np.ascontiguousarray(P, dtype=np.float64)
        x = np.empty(6); it = C.c_int(0)
        self._check(self.lib.dcreg_solve_pcg(self._h, _dptr(A), _dptr(b), _dptr(P), max_iterations, tolerance,
                                             _dptr(x), C.byref(it)))
        return x, int(it.value)

    # -- outer loop --
    def icp_run(self, params: IcpParams, T_init, want_log: bool = True) -> IcpResult:
        """TestRunner::Point2PlaneICP_SO3_OpenMP (icp_test_runner.cpp:1611-2060), device correspondences."""
        T_init = np.ascontiguousarray(T_init, dtype=np.float64)
        T_out = np.empty((4, 4))
        cap = int(params.max_iterations) if want_log else 0
        logs = (IterLog * max(cap, 1))()
        n_it = C.c_int(0); conv = C.c_int(0)
        rc = self._check(self.lib.dcreg_icp_run(self._h, C.byref(params), _dptr(T_init), _dptr(T_out),
                                                logs if want_log else None, cap, C.byref(n_it), C.byref(conv)),
                         allow=(NOT_ENOUGH_POINTS, NONFINITE_UPDATE))
        nrec = min(n_it.value, cap)
        return IcpResult(rc, bool(conv.value), n_it.value, T_out, [logs[i] for i in range(nrec)])

    Point2PlaneICP_SO3 = icp_run

    def icp_enqueue(self, params: IcpParams, T_init):
        """Put a whole run on the context's stream without any host synchronisation (see icp_fetch)."""
        T_init = np.ascontiguousarray(T_init, dtype=np.float64)
        self._check(self.lib.dcreg_icp_enqueue(self._h, C.byref(params), _dptr(T_init)))

    def icp_fetch(self) -> IcpResult:
        """Wait for the stream; pose / iteration count / flags of the last enqueued run."""
        T_out = np.empty((4, 4)); n_it = C.c_int(0); conv = C.c_int(0)
        rc = self._check(self.lib.dcreg_icp_fetch(self._h, _dptr(T_out), C.byref(n_it), C.byref(conv)),
                         allow=(NOT_ENOUGH_POINTS, NONFINITE_UPDATE))
        return IcpResult(rc, bool(conv.value), n_it.value, T_out, [])

    def icp_run_batch(self, params, T_init, want_log: bool = False):
        """`num_runs` registrations side by side (icp_test_runner.cpp:331-345): T_init (B, 4, 4).  params: one IcpParams,
        or B of them, one per trial (per-lane settings, dcreg_set_lane_params).
        Returns a list of IcpResult, one per trial (logs only when want_log)."""
        T_init = np.ascontiguousarray(T_init, dtype=np.float64).reshape(-1, 4, 4)
        B = T_init.shape[0]
        p0, parg, per_lane = self._lanes("icp_run_batch", params, B)
        T_out = np.empty((B, 4, 4))
        n_it = (C.c_int * B)(); conv = (C.c_int * B)(); st = (C.c_int * B)()
        cap = int(p0.max_iterations) if want_log else 0
        logs = (IterLog * max(cap * B, 1))() if want_log else None
        with self._lane_setting(per_lane):
            self._check(self.lib.dcreg_icp_run_batch(self._h, parg, B, _dptr(T_init), _dptr(T_out), n_it, conv, st, logs,
                                                     cap))
        return _trial_results(st, conv, n_it, T_out, logs, cap)

    def _run_batched(self, name, call, params, n, n_poses, noun, T_init, want_log, want_cov, deltas=None,
                     want_prior=False):
        """The steps the batched calls share: check T_init (n_poses of them, one per `noun`) and deltas, allocate the
        outputs of n trials, run call(o) (the library function with o's outputs) and build one IcpResult per trial.  An
        empty batch goes to the library as it is and gets BAD_ARG, like every other malformed batch."""
        o = types.SimpleNamespace(n=0, T_init=None, deltas=None, T_prior=None, T_out=None, n_it=None, conv=None, st=None,
                                  cov=None, logs=None, cap=0)
        if n == 0 or n_poses == 0:
            self._check(call(o))
        o.T_init = np.ascontiguousarray(T_init, dtype=np.float64).reshape(-1, 4, 4)
        if o.T_init.shape[0] != n_poses:
            raise ValueError(f"{name}: {n_poses} {noun} but {o.T_init.shape[0]} initial poses")
        if deltas is not None:
            o.deltas = np.ascontiguousarray(deltas, dtype=np.float64).reshape(-1, 4, 4)
            if o.deltas.shape[0] != n:
                raise ValueError(f"{name}: {n} frames but {o.deltas.shape[0]} increments")
        o.n = n
        o.T_prior = np.empty((n, 4, 4)) if want_prior else None
        o.T_out = np.empty((n, 4, 4))
        o.n_it = (C.c_int * n)(); o.conv = (C.c_int * n)(); o.st = (C.c_int * n)()
        o.cov = np.empty((n, 6, 6)) if want_cov else None
        o.cap = int(params.max_iterations) if want_log else 0
        o.logs = (IterLog * max(o.cap * n, 1))() if want_log else None
        self._check(call(o))
        out = _trial_results(o.st, o.conv, o.n_it, o.T_out, o.logs, o.cap, o.cov)
        if want_prior:
            for r, Tp in zip(out, o.T_prior):
                r.T_prior = Tp
        return out

    def icp_run_scans(self, params, scans, T_init, want_log: bool = False, want_cov: bool = False):
        """Different scans (a list of (N_b, >=3) point arrays) against the context's target, side by side, each from its
        own initial pose (T_init (B, 4, 4)).  The context's own source is left as it was.  Returns a list of IcpResult,
        one per scan (logs only when want_log, .cov the post-loop 6x6 covariance when want_cov)."""
        xyz, off = _pack(scans)
        B = len(scans)
        p0, parg, per_lane = self._lanes("icp_run_scans", params, B)

        def call(o):
            return self.lib.dcreg_icp_run_scans(self._h, parg, o.n, _fptr(xyz), _iptr(off), 3, _optr(o.T_init),
                                                _optr(o.T_out), o.n_it, o.conv, o.st, _optr(o.cov), o.logs, o.cap)
        with self._lane_setting(per_lane):
            return self._run_batched("icp_run_scans", call, p0, B, B, "scans", T_init, want_log, want_cov)

    def icp_run_sequences(self, params, sequences, T_init, deltas=None, want_log: bool = False,
                          want_cov: bool = False):
        """Sequences of frames against the context's target (`sequences`: a list of lists of (N, >=3) point arrays).
        Inside a sequence the frames run one after another on the device, frame k+1 starting from
        compose_prior(frame k's result, deltas[k]); the sequences run side by side.  T_init (S, 4, 4): the prior of each
        sequence's first frame.  deltas: (n_frames, 4, 4) increments over all frames in order (a sequence's last entry is
        unused), or None for identity.  Returns a list of IcpResult, one per frame in order, with .T_prior the pose the
        frame started from (logs only when want_log, .cov when want_cov).  The context's own source is left as it was."""
        seq_off, xyz, off = _pack_sequences(sequences)
        S, n = len(sequences), int(seq_off[-1])
        p0, parg, per_lane = self._lanes("icp_run_sequences", params, S)

        def call(o):
            return self.lib.dcreg_icp_run_sequences(
                self._h, parg, S, seq_off.ctypes.data_as(C.POINTER(C.c_int)), o.n, _fptr(xyz), _iptr(off), 3,
                _optr(o.T_init), _optr(o.deltas), _optr(o.T_prior), _optr(o.T_out), o.n_it, o.conv, o.st, _optr(o.cov),
                o.logs, o.cap)
        with self._lane_setting(per_lane):
            return self._run_batched("icp_run_sequences", call, p0, n, S, "sequences", T_init, want_log, want_cov,
                                     deltas, want_prior=True)

    def voxel_downsample(self, clouds, voxel: float, max_points: int = 1, min_spacing: float = 0.0):
        """dcreg_voxel_downsample_n of every cloud (a list of (N_b, >=3) arrays) in one call on the device, each voxel
        keeping up to max_points points (min_spacing > 0: dcreg_voxel_downsample_spaced, at least min_spacing apart): a
        list of (points (K_b, 3) float32, index (K_b,) int64), as api.voxel_downsample gives for each cloud alone."""
        max_points = _max_points(max_points)
        xyz, off = _pack(clouds)
        n = len(clouds)
        total = int(off[-1]) if n else 0
        pts = np.empty((max(total, 1), 3), dtype=np.float32)
        idx = np.empty(max(total, 1), dtype=np.int64)
        kept = np.zeros(n + 1, dtype=np.int64)
        entry = "dcreg_voxel_downsample_n" if min_spacing == 0.0 else "dcreg_voxel_downsample_spaced"
        self._check(_odometry_call(self.lib, self._h, entry, n_clouds=n, xyz=_fptr(xyz), offsets=_iptr(off), stride=3,
                                   voxel=float(voxel), max_points=max_points, min_spacing=float(min_spacing),
                                   out_xyz=_fptr(pts), out_offsets=_iptr(kept), out_index=_iptr(idx)))
        return [(pts[a:b].copy(), idx[a:b].copy()) for a, b in zip(kept[:-1], kept[1:])]

    def icp_run_odometry(self, params, sequences, T_init, deltas=None, motion: str = "increments",
                         map_frames: int = 10, cell_size=None, want_log: bool = False, want_cov: bool = False,
                         source_voxel: float = 0.0, map_voxel: float = 0.0, source_max_points: int = 1,
                         map_max_points: int = 1, timestamps=None, want_deskewed: bool = False, adaptive=None,
                         want_radius: bool = False, gyro=None, frame_times=None, gyro_samples=None, imu=None,
                         imu_samples=None, v_init=None, want_velocity: bool = False):
        """Scan-to-map odometry (`sequences`: a list of lists of (N, >=3) point arrays): frame k of a sequence registers
        against the local map of the frames [k - map_frames, k) before it, each placed at its own registered pose
        (map_points), starting from compose_prior(frame k-1's result, D).  motion "increments": D = deltas[k-1]
        (deltas: (n_frames, 4, 4) over all frames in order, or None for identity); "constant_velocity": D =
        constant_velocity_increment(T_out[k-2], T_out[k-1]) (identity after the anchor; deltas must be None).  The first
        frame of each sequence is its anchor: not registered, T = T_prior = T_init[s].  cell_size: the maps' grid cell
        (default search_radius).  source_voxel / map_voxel (0: no filter): voxel_downsample every frame in its sensor
        frame, and every local map in world coordinates (dcreg_icp_run_odometry_voxel); source_max_points /
        map_max_points: the points each voxel of those filters keeps (dcreg_icp_run_odometry_voxel_n).  Returns a list of
        IcpResult, one per frame in order, with .T_prior and .n_points, the frame's points after the source filter (logs
        only when want_log, .cov when want_cov).  Needs no target; the context's source and target are left as they
        were.  timestamps (nested like `sequences`: one float32 array per frame, each point's fraction of its sweep in
        [0, 1]): deskew every registered frame with the increment its prior used (dcreg_icp_run_odometry_deskew);
        want_deskewed: .deskewed holds each frame's kept points after deskewing ((n_points, 3) float32).
        adaptive (an AdaptiveThreshold): every frame's search radius follows its sequence's motion-model error under
        the ceiling params.search_radius (dcreg_icp_run_odometry_adaptive; the twin is adaptive_threshold_*), and
        .search_radius holds the radius each frame registered with (0 for anchors); want_radius: .search_radius also
        without the threshold (that entry point with adaptive = NULL).
        gyro (a Gyro), frame_times ((n_frames, 2) (start, span) in seconds over all frames in order) and gyro_samples (one
        (n_s, 4) array (t, wx, wy, wz) per sequence): every non-anchor frame's prior rotation, and with timestamps its
        deskew rotation, come from the integrated rates (dcreg_icp_run_odometry_gyro; the twin is gyro_rotation,
        gyro_increment and deskew_points_gyro); motion must be "constant_velocity".  .search_radius as with adaptive.
        imu (an Imu), frame_times and imu_samples (one (n_s, 7) array (t, wx, wy, wz, ax, ay, az) per sequence) instead
        of gyro: the gyro's rotation, and every non-anchor frame's prior translation from the previous frame's velocity
        and the preintegrated specific force (dcreg_icp_run_odometry_imu; the twin is imu_preintegrate, imu_increment
        and imu_velocity).  v_init ((n_seqs, 3), None: zero): every sequence's velocity at its first frame; want_velocity:
        .velocity holds every frame's world-frame velocity at its mid-sweep time."""
        return self._odometry("icp_run_odometry", params, sequences, T_init, deltas, motion, map_frames, None, cell_size,
                              want_log, want_cov, source_voxel, map_voxel, source_max_points, map_max_points, timestamps,
                              want_deskewed, adaptive, want_radius, gyro, frame_times, gyro_samples, imu, imu_samples,
                              v_init, want_velocity)

    def icp_run_odometry_map(self, params, sequences, T_init, deltas=None, motion: str = "increments", *,
                             map_voxel: float, max_distance: float, cell_size=None, want_log: bool = False,
                             want_cov: bool = False, source_voxel: float = 0.0, source_max_points: int = 1,
                             map_max_points: int = 1, timestamps=None, want_deskewed: bool = False, adaptive=None,
                             want_radius: bool = False, gyro=None, frame_times=None, gyro_samples=None, imu=None,
                             imu_samples=None, v_init=None, want_velocity: bool = False):
        """icp_run_odometry with a persistent voxel map per sequence instead of the window (dcreg_icp_run_odometry_map,
        KISS-ICP's VoxelHashMap): frame k registers against M_k, where M_1 = voxel_map_update(empty, F_s(anchor),
        T_init[s]) and M_{k+1} = voxel_map_update(M_k, F_s(frame k), T_out[k], map_voxel, map_max_points,
        max_distance).  map_voxel must be > 0; max_distance > 0 (inf: nothing is pruned, and the outputs are those of
        icp_run_odometry with map_frames >= the longest sequence).  The arguments are icp_run_odometry's in the same
        positions, without map_frames; map_voxel and max_distance are keyword-only."""
        return self._odometry("icp_run_odometry_map", params, sequences, T_init, deltas, motion, 0,
                              float(max_distance), cell_size, want_log, want_cov, source_voxel, map_voxel,
                              source_max_points, map_max_points, timestamps, want_deskewed, adaptive, want_radius, gyro,
                              frame_times, gyro_samples, imu, imu_samples, v_init, want_velocity)

    def _odometry(self, name, params, sequences, T_init, deltas, motion, map_frames, max_distance, cell_size, want_log,
                  want_cov, source_voxel, map_voxel, source_max_points, map_max_points, timestamps, want_deskewed,
                  adaptive, want_radius, gyro=None, frame_times=None, gyro_samples=None, imu=None, imu_samples=None,
                  v_init=None, want_velocity=False):
        """icp_run_odometry (max_distance None: the window of map_frames frames) and icp_run_odometry_map (map_frames
        0: the voxel map pruned at max_distance)"""
        motion = _motion(motion, name)
        source_max_points = _max_points(source_max_points, "source_max_points")
        map_max_points = _max_points(map_max_points, "map_max_points")
        seq_off, xyz, off = _pack_sequences(sequences)
        S, n = len(sequences), int(seq_off[-1])
        params, parg, per_lane = self._lanes(name, params, S)
        cell = float(params.search_radius if cell_size is None else cell_size)
        if imu is not None and (gyro is not None or gyro_samples is not None):
            raise ValueError(f"{name}: imu and gyro input are exclusive (imu carries the gyro)")
        if imu is None and (imu_samples is not None or v_init is not None or want_velocity):
            raise ValueError(f"{name}: imu_samples, v_init and want_velocity need imu input")
        with_radius = adaptive is not None or want_radius or gyro is not None or imu is not None
        entry = _odometry_entry("icp_run_odometry", radius=with_radius, voxel_map=max_distance is not None,
                                deskew=timestamps is not None or want_deskewed,
                                capped=source_max_points != 1 or map_max_points != 1,
                                filtered=source_voxel != 0.0 or map_voxel != 0.0 or self._map_input_voxel > 0.0,
                                gyro=gyro is not None, imu=imu is not None)
        if imu is not None:
            ft, smp, smp_off = _pack_gyro(name, imu, frame_times, imu_samples, n, S, cols=7)
        else:
            ft, smp, smp_off = _pack_gyro(name, gyro, frame_times, gyro_samples, n, S)
        v0 = _pack_v_init(name, v_init, S)
        vel = np.zeros((max(n, 1), 3)) if want_velocity else None
        ts = _pack_timestamps([t for s in timestamps for t in s] if timestamps is not None else None,
                              off if off is not None else np.zeros(1, np.int64), name)
        npts = np.diff(off) if off is not None else np.zeros(0, dtype=np.int64)
        if entry != "dcreg_icp_run_odometry":       # the others return each frame's points after the source filter
            npts = np.zeros(max(n, 1), dtype=np.int64)
        desk = np.empty((max(int(off[-1]) if off is not None else 0, 1), 3), np.float32) if want_deskewed else None
        radius = np.zeros(max(n, 1)) if with_radius else None

        def call(o):
            return _odometry_call(
                self.lib, self._h, entry, params=parg, n_seqs=S, seq_offsets=seq_off.ctypes.data_as(C.POINTER(C.c_int)),
                n_frames=o.n, xyz=_fptr(xyz), frame_offsets=_iptr(off), stride=3, cell_size=cell,
                map_frames=int(map_frames), motion=motion, source_voxel=float(source_voxel), map_voxel=float(map_voxel),
                source_max_points=source_max_points, map_max_points=map_max_points,
                max_distance=0.0 if max_distance is None else float(max_distance),
                adaptive=None if adaptive is None else C.byref(adaptive), T_init=_optr(o.T_init), deltas=_optr(o.deltas),
                timestamps=_fptr(ts), frame_points=_iptr(npts), T_prior=_optr(o.T_prior), T_out=_optr(o.T_out),
                n_iterations=o.n_it, converged=o.conv, status=o.st, cov=_optr(o.cov), deskewed_xyz=_fptr(desk),
                search_radius=_optr(radius), log=o.logs, log_cap=o.cap,
                gyro=None if gyro is None else C.byref(gyro), frame_times=_optr(ft), samples=_optr(smp),
                sample_offsets=_iptr(smp_off), imu=None if imu is None else C.byref(imu), v_init=_optr(v0),
                velocity=_optr(vel))
        with self._lane_setting(per_lane):
            out = self._run_batched(name, call, params, n, S, "sequences", T_init, want_log, want_cov, deltas,
                                    want_prior=True)
        if want_velocity:
            for r, v in zip(out, vel):
                r.velocity = v.copy()
        for r, c in zip(out, npts):
            r.n_points = int(c)
        if with_radius:
            for r, x in zip(out, radius):
                r.search_radius = float(x)
        if want_deskewed:
            for r, d in zip(out, _split_deskewed(desk, npts[:n])):
                r.deskewed = d
        return out

    def odometry_map_session(self, params, n_seqs: int, T_init, motion: str = "increments", *,
                             map_voxel: float, max_distance: float, cell_size=None, source_voxel: float = 0.0,
                             source_max_points: int = 1, map_max_points: int = 1, adaptive=None, gyro=None, imu=None,
                             v_init=None):
        """Open the context's odometry session with icp_run_odometry_map's voxel map (dcreg_odometry_open_map): the
        OdometrySession of odometry_session, whose pushes give byte for byte what one icp_run_odometry_map call over the
        recording gives, and whose local_map(s) returns sequence s's current map.  The arguments are odometry_session's
        in the same positions, without map_frames; map_voxel and max_distance are keyword-only."""
        return self._open_session("odometry_map_session", params, n_seqs, T_init, motion, 0, float(max_distance),
                                  cell_size, source_voxel, map_voxel, source_max_points, map_max_points, adaptive, gyro,
                                  imu, v_init)

    def odometry_session(self, params, n_seqs: int, T_init, motion: str = "increments", map_frames: int = 10,
                         cell_size=None, source_voxel: float = 0.0, map_voxel: float = 0.0, source_max_points: int = 1,
                         map_max_points: int = 1, adaptive=None, gyro=None, imu=None, v_init=None):
        """Open the context's odometry session (dcreg_odometry_open): icp_run_odometry's settings for n_seqs sequences
        whose frames come in pushes (OdometrySession.push).  T_init (n_seqs, 4, 4): the pose of each sequence's first
        frame.  Pushing a recording in any chunks gives byte for byte what one icp_run_odometry call over it gives.
        One session per context; use it as a context manager, or close() it.  gyro (a Gyro): dcreg_odometry_open_gyro,
        whose pushes take frame_times and gyro_samples and return .search_radius.  imu (an Imu) and v_init ((n_seqs, 3),
        None: zero): dcreg_odometry_open_imu, whose pushes take frame_times and imu_samples and return .search_radius
        and, with want_velocity, .velocity."""
        return self._open_session("odometry_session", params, n_seqs, T_init, motion, map_frames, None, cell_size,
                                  source_voxel, map_voxel, source_max_points, map_max_points, adaptive, gyro, imu,
                                  v_init)

    def _open_session(self, name, params, n_seqs, T_init, motion, map_frames, max_distance, cell_size, source_voxel,
                      map_voxel, source_max_points, map_max_points, adaptive, gyro=None, imu=None, v_init=None):
        """odometry_session (max_distance None) and odometry_map_session (map_frames 0), as in _odometry"""
        motion = _motion(motion, name)
        source_max_points = _max_points(source_max_points, "source_max_points")
        map_max_points = _max_points(map_max_points, "map_max_points")
        T0 = np.ascontiguousarray(T_init, dtype=np.float64).reshape(-1, 4, 4)
        if T0.shape[0] != n_seqs:
            raise ValueError(f"{name}: {n_seqs} sequences but {T0.shape[0]} initial poses")
        params, parg, per_lane = self._lanes(name, params, int(n_seqs))
        cell = float(params.search_radius if cell_size is None else cell_size)
        # dcreg_odometry_open_adaptive's pushes return .search_radius
        if imu is not None and gyro is not None:
            raise ValueError(f"{name}: imu and gyro input are exclusive (imu carries the gyro)")
        if imu is None and v_init is not None:
            raise ValueError(f"{name}: v_init needs imu input")
        entry = _odometry_entry("odometry_open", radius=adaptive is not None, voxel_map=max_distance is not None,
                                gyro=gyro is not None, imu=imu is not None)
        v0 = _pack_v_init(name, v_init, int(n_seqs))
        with self._lane_setting(per_lane):
            self._check(_odometry_call(
                self.lib, self._h, entry, params=parg, n_seqs=int(n_seqs), cell_size=cell, map_frames=int(map_frames),
                motion=motion, source_voxel=float(source_voxel), map_voxel=float(map_voxel),
                source_max_points=source_max_points, map_max_points=map_max_points,
                max_distance=0.0 if max_distance is None else float(max_distance),
                adaptive=None if adaptive is None else C.byref(adaptive), gyro=None if gyro is None else C.byref(gyro),
                imu=None if imu is None else C.byref(imu), T_init=_dptr(T0), v_init=_optr(v0)))
        return OdometrySession(self, params, int(n_seqs), adaptive=adaptive is not None, gyro=gyro is not None,
                               imu=imu is not None)

    def icp_run_pairs(self, params, sources, targets, T_init, cell_size=None, want_log: bool = False,
                      want_cov: bool = False, metrics_threshold=None):
        """Pairs of clouds, each source (a list of (N_b, >=3) arrays) against its own target (a list of (M_b, >=3) arrays),
        side by side, each from its own initial pose (T_init (B, 4, 4)).  cell_size: the targets' grid cell (default
        params.search_radius).  Needs no set_target / set_source and leaves the context's clouds as they were.  Returns a
        list of IcpResult, one per pair (logs only when want_log, .cov the post-loop 6x6 covariance when want_cov,
        .metrics the point_to_point_metrics dict at the pair's final pose when metrics_threshold is given)."""
        xyz_s, off_s = _pack(sources)
        xyz_t, off_t = _pack(targets)
        B = len(sources)
        if len(targets) != B:
            raise ValueError(f"icp_run_pairs: {B} sources but {len(targets)} targets")
        params, parg, per_lane = self._lanes("icp_run_pairs", params, B)
        cell = float(params.search_radius if cell_size is None else cell_size)
        met = np.empty((B, 4)) if metrics_threshold is not None else None

        def call(o):
            return self.lib.dcreg_icp_run_pairs(
                self._h, parg, o.n, _fptr(xyz_s), _iptr(off_s), _fptr(xyz_t), _iptr(off_t), 3, cell,
                _optr(o.T_init), _optr(o.T_out), o.n_it, o.conv, o.st, _optr(o.cov),
                float(metrics_threshold) if met is not None and o.n else 0.0, _optr(met) if o.n else None, o.logs, o.cap)
        with self._lane_setting(per_lane):
            out = self._run_batched("icp_run_pairs", call, params, B, B, "pairs", T_init, want_log, want_cov)
        if met is not None:
            for r, m in zip(out, met):
                r.metrics = {"rmse": m[0], "fitness": m[1], "chamfer": m[2], "n_valid": int(m[3])}
        return out

    def icp_run_host_planes(self, params: IcpParams, T_init, plane_fn, want_log: bool = True) -> IcpResult:
        """Same loop with caller-supplied correspondences: plane_fn(T 4x4) -> (planes (N,4) f64, n_corr_pt)."""
        T_init = np.ascontiguousarray(T_init, dtype=np.float64)
        T_out = np.empty((4, 4))
        cap = int(params.max_iterations) if want_log else 0
        logs = (IterLog * max(cap, 1))()
        n = self.n_source
        err = []

        def _cb(user, Tp, planes_p, npt_p):
            try:
                T = np.ctypeslib.as_array(Tp, shape=(16,)).reshape(4, 4).copy()
                planes, npt = plane_fn(T)
                dst = np.ctypeslib.as_array(planes_p, shape=(n * 4,))
                dst[:] = np.ascontiguousarray(planes, dtype=np.float64).reshape(-1)
                npt_p[0] = int(npt)
                return 0
            except Exception as e:  # pragma: no cover
                err.append(e)
                return 1

        cb = PLANE_CALLBACK(_cb)
        n_it = C.c_int(0); conv = C.c_int(0)
        rc = self.lib.dcreg_icp_run_host_planes(self._h, C.byref(params), _dptr(T_init), cb, None, _dptr(T_out),
                                                logs if want_log else None, cap, C.byref(n_it), C.byref(conv))
        if err:
            raise err[0]
        self._check(rc, allow=(NOT_ENOUGH_POINTS, NONFINITE_UPDATE))
        nrec = min(n_it.value, cap)
        return IcpResult(rc, bool(conv.value), n_it.value, T_out, [logs[i] for i in range(nrec)])

    def last_covariance(self):
        cov = np.empty((6, 6))
        self._check(self.lib.dcreg_last_covariance(self._h, _dptr(cov)))
        return cov

    def point_to_point_metrics(self, T, error_threshold: float):
        """calculatePointToPointError on the device: returns dict(rmse, fitness, chamfer, n_valid)."""
        T = np.ascontiguousarray(T, dtype=np.float64)
        out = np.empty(4)
        self._check(self.lib.dcreg_point_to_point_metrics(self._h, _dptr(T), float(error_threshold), _dptr(out)))
        return {"rmse": out[0], "fitness": out[1], "chamfer": out[2], "n_valid": int(out[3])}

    # -- multi-GPU --
    def comm_unique_id(self) -> bytes:
        buf = (C.c_uint8 * 128)()
        self._check(self.lib.dcreg_comm_unique_id(self._h, buf))
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self.lib.dcreg_comm_init(self._h, buf, rank, nranks))

    @property
    def comm_mode(self) -> int:
        """0 no communicator, 1 ncclAllReduce fallback, 2 in-kernel peer-memory all-reduce."""
        return int(self.lib.dcreg_comm_mode(self._h))

    def comm_destroy(self):
        self._check(self.lib.dcreg_comm_destroy(self._h))

    def set_global_source_count(self, n_total: int):
        self._check(self.lib.dcreg_set_global_source_count(self._h, int(n_total)))


class OdometrySession:
    """The context's odometry session (Context.odometry_session): frames pushed as they arrive, each sequence's local-map
    window and motion-model state kept on the device from one push to the next."""

    def __init__(self, ctx: Context, params: IcpParams, n_seqs: int, adaptive: bool = False, gyro: bool = False,
                 imu: bool = False):
        self.ctx, self.params, self.n_seqs = ctx, params, n_seqs
        self.adaptive = adaptive        # opened with an AdaptiveThreshold: every push returns .search_radius
        self.gyro = gyro                # opened with a Gyro: pushes take frame_times and gyro_samples
        self.imu = imu                  # opened with an Imu: pushes take frame_times and imu_samples
        self.open = True

    def push(self, frames_per_seq, deltas=None, want_log: bool = False, want_cov: bool = False, timestamps=None,
             want_deskewed: bool = False, frame_times=None, gyro_samples=None, imu_samples=None,
             want_velocity: bool = False):
        """The next frames of every sequence (dcreg_odometry_push): frames_per_seq, a list of n_seqs lists, possibly
        empty, of (N, >=3) point arrays.  deltas: (frames, 4, 4) increments over the pushed frames in order (entry k maps
        frame k's result to the next frame's prior in its sequence, which may come in a later push), or None for
        identity.  Returns one list of IcpResult per sequence, as icp_run_odometry gives them (.T_prior, .n_points; logs
        only when want_log, .cov when want_cov).  timestamps / want_deskewed: as in icp_run_odometry, nested like
        frames_per_seq (dcreg_odometry_push_deskew).  frame_times ((frames, 2) over the pushed frames in order) and
        gyro_samples (one (n_s, 4) array per sequence, holding the samples that bracket every pushed frame's interval
        from the previous mid-sweep to its sweep's end): a gyro session's input (dcreg_odometry_push_gyro).
        frame_times and imu_samples (one (n_s, 7) array per sequence, the same bracketing): an IMU session's input
        (dcreg_odometry_push_imu); want_velocity: .velocity as in icp_run_odometry.  A push that fails raises DcregError
        and leaves the session as it was."""
        ctx = self.ctx
        if len(frames_per_seq) != self.n_seqs:
            raise ValueError(f"odometry push: {self.n_seqs} sequences but {len(frames_per_seq)} frame lists")
        seq_off, xyz, off = _pack_sequences(frames_per_seq)
        n = int(seq_off[-1])
        D = None
        if deltas is not None:
            D = np.ascontiguousarray(deltas, dtype=np.float64).reshape(-1, 4, 4)
            if D.shape[0] != n:
                raise ValueError(f"odometry push: {n} frames but {D.shape[0]} increments")
        m = max(n, 1)
        T_prior = np.empty((m, 4, 4)); T_out = np.empty((m, 4, 4))
        npts = np.zeros(m, dtype=np.int64)
        n_it = (C.c_int * m)(); conv = (C.c_int * m)(); st = (C.c_int * m)()
        cov = np.empty((m, 6, 6)) if want_cov else None
        cap = int(self.params.max_iterations) if want_log else 0
        logs = (IterLog * max(cap * n, 1))() if want_log else None
        radius = np.zeros(m) if self.adaptive or self.gyro or self.imu else None
        if not self.imu and (imu_samples is not None or want_velocity):
            raise ValueError("odometry push: imu_samples and want_velocity need a session opened with imu input")
        if self.imu:
            if gyro_samples is not None:
                raise ValueError("odometry push: an imu session takes imu_samples, not gyro_samples")
            ft, smp, smp_off = _pack_gyro("odometry push", True, frame_times, imu_samples, n, self.n_seqs, cols=7)
        else:
            ft, smp, smp_off = _pack_gyro("odometry push", self.gyro or None, frame_times, gyro_samples, n, self.n_seqs)
        vel = np.zeros((m, 3)) if want_velocity else None
        ts = _pack_timestamps([t for s in timestamps for t in s] if timestamps is not None else None,
                              off if off is not None else np.zeros(1, np.int64), "odometry push")
        desk = np.empty((max(int(off[-1]) if off is not None else 0, 1), 3), np.float32) if want_deskewed else None
        entry = _odometry_entry("odometry_push", radius=self.adaptive, deskew=timestamps is not None or want_deskewed,
                                gyro=self.gyro, imu=self.imu)
        ctx._check(_odometry_call(
            ctx.lib, ctx._h, entry, seq_offsets=seq_off.ctypes.data_as(C.POINTER(C.c_int)), n_frames=n, xyz=_fptr(xyz),
            frame_offsets=_iptr(off), stride=3, deltas=_optr(D), timestamps=_fptr(ts), frame_points=_iptr(npts),
            T_prior=_dptr(T_prior), T_out=_dptr(T_out), n_iterations=n_it, converged=conv, status=st, cov=_optr(cov),
            deskewed_xyz=_fptr(desk), search_radius=_optr(radius), log=logs, log_cap=cap, frame_times=_optr(ft),
            samples=_optr(smp), sample_offsets=_iptr(smp_off), velocity=_optr(vel)))
        res = _trial_results(st[:n], conv[:n], n_it[:n], T_out, logs, cap, cov)
        if want_velocity:
            for r, v in zip(res, vel):
                r.velocity = v.copy()
        for r, Tp, c in zip(res, T_prior, npts):
            r.T_prior, r.n_points = Tp, int(c)
        if radius is not None:
            for r, x in zip(res, radius):
                r.search_radius = float(x)
        if want_deskewed:
            for r, d in zip(res, _split_deskewed(desk, npts[:n])):
                r.deskewed = d
        return [res[a:b] for a, b in zip(seq_off[:-1], seq_off[1:])]

    def local_map(self, s: int):
        """Sequence s's current voxel map (a session of Context.odometry_map_session, dcreg_odometry_local_map): M after
        its last committed frame, (K, 3) float32 in map order (empty before its first frame)."""
        ctx, lib = self.ctx, self.ctx.lib
        n = C.c_int64(0)
        rc = lib.dcreg_odometry_local_map(ctx._h, int(s), None, 0, C.byref(n))
        if n.value == 0:
            ctx._check(rc)
            return np.zeros((0, 3), np.float32)
        out = np.empty((n.value, 3), np.float32)
        ctx._check(lib.dcreg_odometry_local_map(ctx._h, int(s), _fptr(out), n.value, C.byref(n)))
        return out

    def close(self):
        if self.open and self.ctx._h:
            self.ctx._check(self.ctx.lib.dcreg_odometry_close(self.ctx._h))
        self.open = False

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

"""dcreg_b200 - H100 (sm_90a) point-to-plane ICP + Schur-decoupled degeneracy engine (hot path of JokerJohn/DCReg).

The product is the sm_90a CUDA library ``libdcreg_b200.so`` behind the C ABI in ``include/dcreg_b200.h``;
this package is its thin ctypes host binding.  There is no CPU fallback.
"""
from .api import (Context, DcregError, IcpParams, Analysis, IterLog, default_params, load_library, DET, HAND, STATUS,
                  LIB_PATH, EXPORTS, pose_Rt, compose_prior, map_points,
                  constant_velocity_increment)

__all__ = ["Context", "DcregError", "IcpParams", "Analysis", "IterLog", "default_params", "load_library", "DET",
           "HAND", "STATUS", "LIB_PATH", "EXPORTS", "pose_Rt", "compose_prior", "map_points",
           "constant_velocity_increment"]

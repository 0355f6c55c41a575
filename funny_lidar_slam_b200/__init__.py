"""funny_lidar_slam_b200 — H100-native (sm_90a) scan-matching hot path behind the reference's
RegistrationInterface (include/registration/registration_interface.h:11-20 upstream).

The product is the C-ABI shared library built from csrc/ (include/fls_b200.h); this package holds the
host-side mirror of the reference interface used by tests and bench.py.  There is no CPU fallback: every
compute call raises if libfls_b200.so is missing or no sm_90 device is present.
"""
from ._abi import (FLS_ICP_P2P, FLS_LOAM_FULL, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, FlsConfig, FlsMatchStats,  # noqa: F401
                   default_config)

__version__ = "0.1.0"

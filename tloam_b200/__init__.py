"""tloam_b200 -- H100-native (sm_90a) TLS scan-to-map registration behind T-LOAM's RegistrationInterface.

The product is the C-ABI CUDA library `libtloam_b200.so` (sources in tloam_b200/csrc, boundary in
include/tloam_b200.h).  This package is only the Python host-side mirror of the reference interface plus the
synthetic-scene generator used by tests and bench.py.  Importing it never touches oracle/.
"""
from .occupancy import save_occupancy_map  # noqa: F401
from .registration import (BatchRegistration, DistanceField, Frame, Frontier, GlobalRegistrationResult,  # noqa: F401
                           LocalRegistration, LoopResult, LoopVerifyResult,
                           OccupancyGrid, PlanField, PlanPath, PoseGraphResult, PoseGraphRobustResult, RegistrationError,
                           TerrainMap, default_config, packed_scan, packed_time)

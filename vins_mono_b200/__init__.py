"""vins_mono_b200 — H100-native (sm_90a) hot paths of VINS-Mono behind a C ABI (include/vinsb200/*.h).

The product is lib/libvinsb200.so (hand-written CUDA for sm_90a + host glue); this package is a thin
ctypes mirror of the reference's host classes for tests and benchmarks.  There is no CPU fallback:
loading fails loudly when the library is missing, creating a tracker fails when no CUDA device exists.
"""
from ._abi import VinsError  # noqa: F401
from .tracker import FeatureTracker, TrackerBatch, TrackerConfig, load_library, LIB_PATH  # noqa: F401
from .estimator import Estimator, EstimatorBatch, EstimatorConfig, debug_projection_factor, debug_imu_factor  # noqa: F401
from .replay import ReplaySession  # noqa: F401
from .pose_graph import PoseGraph, PoseGraphBatch, PoseGraphError, debug_four_dof_error  # noqa: F401

"""The C ABI of lib/libvinsb200.so (include/vinsb200/*.h) as ctypes sees it: the signature of every declared function, the
mirrors of the header structs, and the handle bases the classes of this package are built on.  tests/test_ctypes_abi.py
checks the table and the structs against the headers."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libvinsb200.so")


class TrackerConfig(C.Structure):  # vt_config
    _fields_ = [("rows", C.c_int), ("cols", C.c_int), ("max_cnt", C.c_int), ("min_dist", C.c_int), ("freq", C.c_int),
                ("equalize", C.c_int), ("fisheye", C.c_int), ("focal_length", C.c_int), ("f_threshold", C.c_double),
                ("camera_model", C.c_int), ("intrinsics", C.c_double * 8), ("fisheye_mask", C.c_void_p),
                ("device", C.c_int), ("xi", C.c_double)]


class EstimatorConfig(C.Structure):  # ve_config
    _fields_ = [("window_size", C.c_int), ("max_features", C.c_int), ("num_iterations", C.c_int),
                ("estimate_extrinsic", C.c_int), ("estimate_td", C.c_int), ("focal_length", C.c_double),
                ("keyframe_parallax", C.c_double), ("acc_n", C.c_double), ("gyr_n", C.c_double), ("acc_w", C.c_double),
                ("gyr_w", C.c_double), ("g_norm", C.c_double), ("init_depth", C.c_double), ("td", C.c_double),
                ("tr", C.c_double), ("row", C.c_double), ("tic", C.c_double * 3), ("ric", C.c_double * 9),
                ("device", C.c_int)]


class PoseGraphConfig(C.Structure):  # vp_config
    _fields_ = [("max_keyframes", C.c_int), ("fast_relocalization", C.c_int), ("device", C.c_int), ("max_anchors", C.c_int)]


class LoopConfig(C.Structure):  # vp_loop_config
    _fields_ = [("rows", C.c_int), ("cols", C.c_int), ("intrinsics", C.c_double * 8), ("ric9", C.c_double * 9), ("tic3", C.c_double * 3),
                ("brief_pattern", C.c_void_p), ("max_window", C.c_int), ("max_corners", C.c_int)]


class LoopResult(C.Structure):  # vp_loop_result
    _fields_ = [("accepted", C.c_int), ("n_matches", C.c_int), ("n_inliers", C.c_int), ("n_points", C.c_int),
                ("loop_info", C.c_double * 8), ("old_R9", C.c_double * 9), ("old_T3", C.c_double * 3)]


class AttachJob(C.Structure):  # vp_attach_job
    _fields_ = [("member", C.c_int), ("index", C.c_int), ("vio_P3", C.c_void_p), ("vio_Qwxyz", C.c_void_p), ("img", C.c_void_p),
                ("row_stride", C.c_size_t), ("img_on_device", C.c_int), ("n", C.c_int), ("point_3d", C.c_void_p),
                ("point_uv", C.c_void_p), ("point_norm", C.c_void_p), ("point_id", C.c_void_p)]


class ReplaySequence(C.Structure):  # vr_sequence
    _fields_ = [("images", C.c_void_p), ("row_stride", C.c_size_t), ("frame_stride", C.c_size_t), ("n_images", C.c_int),
                ("images_on_device", C.c_int), ("stamps", C.c_void_p), ("n_imu", C.c_int), ("imu_t", C.c_void_p),
                ("acc", C.c_void_p), ("gyr", C.c_void_p)]


# Arrays and handles go in as c_void_p; a scalar written through a pointer is passed by byref as POINTER(<its type>).
V, I, D, Z, S = C.c_void_p, C.c_int, C.c_double, C.c_size_t, C.c_char_p
IP, FP, DP, LLP = (C.POINTER(t) for t in (C.c_int, C.c_float, C.c_double, C.c_longlong))
VP = C.POINTER(V)

# name: (restype, argtypes) for every function the headers declare
SIGNATURES = {
    # tracker.h
    "vt_create": (I, [C.POINTER(TrackerConfig), VP]),
    "vt_destroy": (None, [V]),
    "vt_last_error": (S, [V]),
    "vt_read_image": (I, [V, V, Z, D, I]),
    "vt_read_image_device": (I, [V, V, Z, D, I]),
    "vt_count": (I, [V]),
    "vt_get": (I, [V] * 6),
    "vt_node_image": (I, [V, V, Z, D, IP]),
    "vt_node_image_device": (I, [V, V, Z, D, IP]),
    "vt_node_pack": (I, [V, I] + [V] * 6),
    "vt_batch_create": (I, [C.POINTER(TrackerConfig), I, VP]),
    "vt_batch_destroy": (None, [V]),
    "vt_batch_size": (I, [V]),
    "vt_batch_member": (V, [V, I]),
    "vt_batch_last_error": (S, [V]),
    "vt_batch_read_image": (I, [V, V, V, Z, V, V, I]),
    "vt_batch_node_image": (I, [V, V, V, Z, V, I, V, V]),
    "vt_batch_last_timing": (I, [V, FP, IP]),
    "vt_batch_set_profile": (I, [V, I]),
    "vt_batch_kernel_times": (I, [V, V, V]),
    "vt_last_timing": (I, [V, FP, IP]),
    "vt_set_profile": (I, [V, I]),
    "vt_kernel_times": (I, [V, V, V]),
    "vt_last_traffic": (I, [V, DP, DP]),
    "vt_debug_equalized": (I, [V, I, V, IP, IP]),
    "vt_debug_gftt": (I, [V, V, Z, V, I, V, IP, V]),
    "vt_debug_lk": (I, [V, V, V, Z, V, I, V, V]),
    "vt_debug_fundamental_ransac": (I, [V, V, I, D, D, V]),
    "vt_debug_fundamental_ransac_model": (I, [V, V, I, D, D, V, V]),
    "vt_debug_lift_projective": (I, [V, V, I, V]),
    "vt_debug_lift_projective_model": (I, [I, V, D, V, I, V]),
    "vt_debug_disc_half_widths": (I, [I, V]),
    # estimator.h
    "ve_create": (I, [C.POINTER(EstimatorConfig), VP]),
    "ve_destroy": (None, [V]),
    "ve_last_error": (S, [V]),
    "ve_clear_state": (I, [V]),
    "ve_set_seed": (I, [V, I, V, V, V]),
    "ve_process_imu": (I, [V, D, V, V]),
    "ve_process_image": (I, [V, I, V, V, D]),
    "ve_get_states": (I, [V, V, DP]),
    "ve_info": (I, [V, V, V]),
    "ve_get_prior": (I, [V, I, V, V, IP, V]),
    "ve_last_timing": (I, [V, V, IP]),
    "ve_process_imu_batch": (I, [V, I, V, V, V]),
    "ve_set_profile": (I, [V, I]),
    "ve_kernel_times": (I, [V, V, V]),
    "ve_last_traffic": (I, [V, DP, DP]),
    "ve_window_size": (I, [V]),
    "ve_get_latest_imu": (I, [V, V, V, V]),
    "ve_get_extrinsic": (I, [V, V, V]),
    "ve_batch_create": (I, [C.POINTER(EstimatorConfig), I, VP]),
    "ve_batch_destroy": (None, [V]),
    "ve_batch_size": (I, [V]),
    "ve_batch_groups": (I, [V]),
    "ve_batch_member": (V, [V, I]),
    "ve_batch_last_error": (S, [V]),
    "ve_batch_process_image": (I, [V] * 7),
    "ve_batch_last_timing": (I, [V, V, IP]),
    "ve_batch_set_profile": (I, [V, I]),
    "ve_batch_kernel_times": (I, [V, V, V]),
    "ve_batch_sync": (I, [V]),
    "ve_debug_projection_factor": (I, [V, V, I, D, D, D, I, V]),
    "ve_debug_imu_factor": (I, [V, D, V, V, I] + [V] * 6),
    "ve_debug_ex_rotation": (I, [I, V, V, V, I] + [V] * 5),
    "ve_debug_relative_rt": (I, [V, I, V, V, IP]),
    "ve_debug_solve_pnp": (I, [V, V, I, V, V]),
    "ve_debug_sfm_construct": (I, [I, I, V, V, I] + [V] * 4 + [D, V, V, IP, V, V, IP, DP]),
    "ve_debug_initial_structure": (I, [I, V, I] + [V] * 7 + [I] + [V] * 6 + [D, D] + [V] * 6 + [DP]),
    "ve_get_features": (I, [V, I, I] + [V] * 6),
    "ve_get_headers": (I, [V, V]),
    "ve_set_relo_frame": (I, [V, D, I, I, V, V, V]),
    "ve_get_relocalization": (I, [V, V]),
    "ve_init_info": (I, [V, V]),
    "ve_solver_debug": (I, [V, V]),
    # pose_graph.h
    "vp_create": (I, [C.POINTER(PoseGraphConfig), VP]),
    "vp_destroy": (None, [V]),
    "vp_last_error": (S, [V]),
    "vp_new_sequence": (I, [V]),
    "vp_add_keyframe": (I, [V, D, V, V, I, V, IP, V, V]),
    "vp_update_loop": (I, [V, I, V]),
    "vp_optimize": (I, [V]),
    "vp_sync": (I, [V]),
    "vp_correct_pose": (I, [V] * 5),
    "vp_get_drift": (I, [V] * 4),
    "vp_get_keyframe": (I, [V, I, V, IP, V]),
    "vp_get_path": (I, [V, I] + [V] * 4),
    "vp_info": (I, [V, V, V]),
    "vp_last_timing": (I, [V, FP, IP]),
    "vp_save": (I, [V, S]),
    "vp_load": (I, [V, S]),
    "vp_batch_create": (I, [C.POINTER(PoseGraphConfig), I, VP]),
    "vp_batch_destroy": (None, [V]),
    "vp_batch_size": (I, [V]),
    "vp_batch_member": (V, [V, I]),
    "vp_batch_last_error": (S, [V]),
    "vp_batch_optimize": (I, [V, V, V]),
    "vp_batch_sync": (I, [V]),
    "vp_batch_last_timing": (I, [V, V, IP]),
    "vp_debug_four_dof_error": (I, [V, V, I, I, V]),
    # loop_verify.h
    "vp_loop_enable": (I, [V, C.POINTER(LoopConfig)]),
    "vp_batch_loop_enable": (I, [V, C.POINTER(LoopConfig)]),
    "vp_attach_keyframe": (I, [V, I, V, V, V, Z, I, V, V, V, V, IP]),
    "vp_find_connection": (I, [V, I, I, C.POINTER(LoopResult), I, V]),
    "vp_batch_find_connection": (I, [V, V, V, V, I, V, V]),
    "vp_loop_last_timing": (I, [V, V]),
    "vp_batch_loop_last_timing": (I, [V, V]),
    "vp_debug_brief_blur": (I, [V, I, I, V]),
    "vp_debug_fast": (I, [V, I, I, I, V]),
    "vp_debug_brief": (I, [V, I, I, V, I, V, V]),
    "vp_debug_match": (I, [I, V, I, V, V]),
    "vp_debug_pnp": (I, [I, V, V, V, IP, V]),
    # loop_attach.h
    "vp_batch_attach_keyframes": (I, [V, I, V, V, V]),
    # loop_camera.h
    "vp_loop_enable_camera": (I, [V, C.POINTER(LoopConfig), I, D]),
    "vp_batch_loop_enable_camera": (I, [V, C.POINTER(LoopConfig), I, D]),
    "vp_debug_lift": (I, [I, V, D, I, V, V]),
    # replay.h
    "vr_open": (I, [I, V, V, V, VP]),
    "vr_open_batch": (I, [V, V, V, VP]),
    "vr_close": (None, [V]),
    "vr_last_error": (S, [V]),
    "vr_advance": (I, [V, I]),
    "vr_stats": (I, [V, I, IP, LLP, DP, DP]),
    "vr_trajectory": (I, [V, I, I, V, V]),
    "vr_debug_imu_batches": (I, [I, V, V, V, I, V, I, V, V, V, V]),
    "vr_prop_create": (V, []),
    "vr_prop_destroy": (None, [V]),
    "vr_prop_predict": (I, [V, D, V, V, V]),
    "vr_prop_update": (I, [V, D] + [V] * 8 + [I] + [V] * 3),
    "vr_prop_update_from_estimator": (I, [V, V, D, I, V, V, V]),
    "vr_format_result_row": (I, [D, V, V, V, S, I]),
    "vr_decode_pointcloud": (I, [I] + [V] * 9),
    "vr_decode_relo_message": (I, [I] + [V] * 5 + [IP]),
    "vr_queue_relo": (I, [V, I, D, D, I, I, V, V, V]),
}

_lib = None


def load_library():
    """Loads libvinsb200.so once and applies SIGNATURES.  Raises if it has not been built (python vins_mono_b200/build.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python vins_mono_b200/build.py` (no CPU fallback exists)")
        lib = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = lib
    return _lib


def ptr(a):
    """The data pointer of a numpy array as a c_void_p argument; None stays NULL."""
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def f64(a):
    return np.ascontiguousarray(a, np.float64)


class VinsError(RuntimeError):
    """A call into the library failed; status is its negative return value (-1 invalid, -2 no device, -3 CUDA,
    -4 capacity)."""

    def __init__(self, status, msg):
        super().__init__(f"vinsb200 error {status}: {msg}")
        self.status = status


def check(rc, name):
    """The status of a handle-free call: raises VinsError when it is negative, returns it otherwise."""
    if rc < 0:
        raise VinsError(rc, f"{name} failed with status {rc}")
    return rc


class _Closed:
    """The library as a closed handle sees it: every call raises before it can pass a NULL or freed handle."""

    def __getattr__(self, name):
        raise VinsError(-1, f"{name} on a closed handle")


_CLOSED = _Closed()


class Handle:
    """A library handle, owned or borrowed.  An owned one is destroyed by close() or by garbage collection; a borrowed one
    is a batch member and holds its batch, so the batch outlives it.  After close() every call raises VinsError.
    Subclasses name their family's destroy and last-error functions."""
    _destroy = _last_error = ""
    h = _owner = None

    def _open(self, create, *args):
        """Calls create(*args, &handle) and owns the handle it returns."""
        self.lib = load_library()
        h = C.c_void_p()
        rc = getattr(self.lib, create)(*args, C.byref(h))
        if rc != 0:
            raise VinsError(rc, f"{create} failed with status {rc} (-1 = invalid configuration, -2 = no CUDA device; this "
                                "library has no CPU path)")
        self.h = h

    @classmethod
    def _borrow(cls, batch, handle):
        self = cls.__new__(cls)
        self.lib, self.h, self._owner = batch.lib, C.c_void_p(handle), batch
        return self

    def _check(self, rc):
        if rc < 0:
            raise VinsError(rc, getattr(self.lib, self._last_error)(self.h).decode())
        return rc

    def close(self):
        if self.h is not None and self._owner is None:
            getattr(self.lib, self._destroy)(self.h)
        self.h, self._owner, self.lib = None, None, _CLOSED

    def __del__(self):
        self.close()


class Batch(Handle):
    """An owned handle whose members (borrowed handles) are listed in self.members; close() detaches them first.  The
    members and the batch reference each other, so a batch dropped without close() goes with the next garbage collection."""
    members = ()

    def close(self):
        for m in self.members:
            m.close()
        super().close()

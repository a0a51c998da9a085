"""ctypes loader for librobotoc_b200.so (built in-tree by __graft_entry__.build()).

Fails loudly when the library is missing: there is no CPU / PyTorch fallback for the hot path.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ROBOTOC_B200_LIB", os.path.join(_HERE, "librobotoc_b200.so"))  # env override: A/B builds


class rbt_dims(ctypes.Structure):
    _fields_ = [("nv", ctypes.c_int), ("nu", ctypes.c_int), ("ns_max", ctypes.c_int), ("n_passive", ctypes.c_int)]


class rbt_stage_ctrl(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("sto", ctypes.c_int), ("sto_next", ctypes.c_int), ("ns", ctypes.c_int),
                ("nf", ctypes.c_int), ("ngrids_in_phase", ctypes.c_int), ("contact_mask", ctypes.c_int),
                ("ineq_gate", ctypes.c_int), ("dt", ctypes.c_double)]


_lib = None

# every symbol include/robotoc_b200.h declares
EXPORTS = [
    "rbt_layout_get", "rbt_ulayout_get", "rbt_device_info", "rbt_version",
    "rbt_create", "rbt_destroy", "rbt_set_schedule", "rbt_dev_ptr", "rbt_buf_doubles", "rbt_bind_buffer", "rbt_upload",
    "rbt_download", "rbt_upload_bytes", "rbt_download_info", "rbt_check_info", "rbt_set_fxx_structure", "rbt_set_time_segments", "rbt_riccati_backward", "rbt_riccati_forward",
    "rbt_riccati_solve_host", "rbt_stage_layout_get", "rbt_stage_setup", "rbt_condense",
    "rbt_expand_and_step_sizes", "rbt_update", "rbt_trial_doubles", "rbt_line_search_trials", "rbt_line_search_trial_dev", "rbt_line_search_filter", "rbt_line_search_clear_history", "rbt_eval_kkt", "rbt_set_slack_and_dual_positive", "rbt_initial_state_direction", "rbt_set_joint_limits", "rbt_linearize_joint_limits", "rbt_set_robot_model", "rbt_linearize_inverse_dynamics", "rbt_set_contact_gains", "rbt_linearize_contact_kinematics", "rbt_linearize_state_equation", "rbt_iteration_host", "rbt_iteration_host_bytes", "rbt_iteration_host_wire", "rbt_iteration_host_resident", "rbt_set_wire_cost_structure", "rbt_wire_doubles", "rbt_wire_layout_get", "rbt_pack_wire", "rbt_set_condense_event", "rbt_step_doubles", "rbt_pack_step", "rbt_allgather_step", "rbt_sync", "rbt_last_error", "rbt_launch_count",
    "rbt_unconstr_create", "rbt_unconstr_destroy", "rbt_unconstr_dev_ptr", "rbt_unconstr_buf_doubles",
    "rbt_unconstr_upload", "rbt_unconstr_download", "rbt_unconstr_download_info", "rbt_unconstr_backward",
    "rbt_unconstr_forward", "rbt_unconstr_solve_host", "rbt_unconstr_sync", "rbt_unconstr_last_error",
    "rbt_unconstr_launch_count", "rbt_unconstr_stage_layout_get", "rbt_unconstr_stage_setup", "rbt_unconstr_condense",
    "rbt_unconstr_expand_and_step_sizes", "rbt_unconstr_update", "rbt_unconstr_iteration_host",
]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -c 'import __graft_entry__ as g; "
            "g.build()'` at the repo root. robotoc_b200 has no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH)
    c_int, c_dbl, c_vp, c_ll = ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_longlong
    pd = ctypes.POINTER(ctypes.c_double)
    L.rbt_layout_get.argtypes = [ctypes.POINTER(rbt_dims), ctypes.c_char_p]
    L.rbt_layout_get.restype = c_int
    L.rbt_ulayout_get.argtypes = [c_int, ctypes.c_char_p]
    L.rbt_ulayout_get.restype = c_int
    L.rbt_device_info.argtypes = [c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.c_char_p, c_int]
    L.rbt_device_info.restype = c_int
    L.rbt_version.restype = ctypes.c_char_p
    L.rbt_create.argtypes = [ctypes.POINTER(rbt_dims), c_int, c_int, c_int, ctypes.POINTER(c_vp)]
    L.rbt_destroy.argtypes = [c_vp]
    L.rbt_set_schedule.argtypes = [c_vp, ctypes.POINTER(rbt_stage_ctrl), c_int, c_dbl]
    L.rbt_dev_ptr.argtypes = [c_vp, c_int]
    L.rbt_dev_ptr.restype = c_vp
    L.rbt_buf_doubles.argtypes = [c_vp, c_int]
    L.rbt_buf_doubles.restype = c_ll
    L.rbt_bind_buffer.argtypes = [c_vp, c_int, c_vp]
    L.rbt_upload.argtypes = [c_vp, c_int, c_vp, c_vp]
    L.rbt_download.argtypes = [c_vp, c_int, c_vp, c_vp]
    L.rbt_download_info.argtypes = [c_vp, c_vp, c_vp]
    L.rbt_set_fxx_structure.argtypes = [c_vp, c_int]
    L.rbt_set_time_segments.argtypes = [c_vp, c_int]
    L.rbt_eval_kkt.argtypes = [c_vp, c_vp]
    L.rbt_line_search_trials.argtypes = [c_vp, c_int, c_dbl, c_vp, c_vp, c_vp, c_vp]
    L.rbt_line_search_trial_dev.argtypes = [c_vp]
    L.rbt_line_search_trial_dev.restype = c_vp
    L.rbt_line_search_filter.argtypes = [c_vp, c_int, c_dbl, c_dbl, c_dbl, c_dbl, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.rbt_line_search_clear_history.argtypes = [c_vp, c_vp]
    L.rbt_step_doubles.argtypes = [c_vp]
    L.rbt_pack_step.argtypes = [c_vp, c_vp, c_vp]
    L.rbt_allgather_step.argtypes = [c_vp, c_vp, c_vp, c_vp]
    L.rbt_set_slack_and_dual_positive.argtypes = [c_vp, c_vp]
    L.rbt_initial_state_direction.argtypes = [c_vp, c_vp, c_vp]
    L.rbt_check_info.argtypes = [c_vp, ctypes.POINTER(c_int), c_vp]
    L.rbt_upload_bytes.argtypes = [c_vp, c_int]
    L.rbt_upload_bytes.restype = c_ll
    L.rbt_riccati_backward.argtypes = [c_vp, c_int, c_vp]
    L.rbt_riccati_forward.argtypes = [c_vp, c_vp]
    L.rbt_riccati_solve_host.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.rbt_stage_layout_get.argtypes = [c_vp, ctypes.c_char_p]
    L.rbt_stage_setup.argtypes = [c_vp, c_vp, c_vp]
    L.rbt_condense.argtypes = [c_vp, c_vp]
    L.rbt_set_condense_event.argtypes = [c_vp, c_vp]
    L.rbt_expand_and_step_sizes.argtypes = [c_vp, c_vp]
    L.rbt_update.argtypes = [c_vp, c_vp]
    L.rbt_iteration_host.argtypes = [c_vp] * 9
    L.rbt_iteration_host_bytes.argtypes = [c_vp, c_int, ctypes.POINTER(c_ll), ctypes.POINTER(c_ll)]
    L.rbt_iteration_host_wire.argtypes = [c_vp] * 10
    L.rbt_iteration_host_resident.argtypes = [c_vp] * 9
    L.rbt_set_joint_limits.argtypes = [c_vp, c_vp]
    L.rbt_linearize_joint_limits.argtypes = [c_vp, c_vp]
    L.rbt_set_robot_model.argtypes = [c_vp, c_vp]
    L.rbt_linearize_inverse_dynamics.argtypes = [c_vp, c_vp]
    L.rbt_set_contact_gains.argtypes = [c_vp, c_vp]
    L.rbt_linearize_contact_kinematics.argtypes = [c_vp, c_vp]
    L.rbt_linearize_state_equation.argtypes = [c_vp, c_vp]
    L.rbt_set_wire_cost_structure.argtypes = [c_vp, c_int]
    L.rbt_wire_doubles.argtypes = [c_vp, c_vp, c_int, c_int]
    L.rbt_wire_layout_get.argtypes = [c_vp, c_vp, c_int, c_int, c_int, c_vp]
    L.rbt_pack_wire.argtypes = [c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_ll]
    L.rbt_sync.argtypes = [c_vp, c_vp]
    L.rbt_last_error.argtypes = [c_vp]
    L.rbt_last_error.restype = ctypes.c_char_p
    L.rbt_launch_count.argtypes = [c_vp]
    L.rbt_launch_count.restype = c_ll
    L.rbt_unconstr_create.argtypes = [c_int, c_int, c_dbl, c_int, c_int, ctypes.POINTER(c_vp)]
    L.rbt_unconstr_destroy.argtypes = [c_vp]
    L.rbt_unconstr_dev_ptr.argtypes = [c_vp, c_int]
    L.rbt_unconstr_dev_ptr.restype = c_vp
    L.rbt_unconstr_buf_doubles.argtypes = [c_vp, c_int]
    L.rbt_unconstr_buf_doubles.restype = c_ll
    L.rbt_unconstr_upload.argtypes = [c_vp, c_int, c_vp, c_vp]
    L.rbt_unconstr_download.argtypes = [c_vp, c_int, c_vp, c_vp]
    L.rbt_unconstr_download_info.argtypes = [c_vp, c_vp, c_vp]
    L.rbt_unconstr_backward.argtypes = [c_vp, c_int, c_vp]
    L.rbt_unconstr_forward.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_solve_host.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.rbt_unconstr_sync.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_last_error.argtypes = [c_vp]
    L.rbt_unconstr_last_error.restype = ctypes.c_char_p
    L.rbt_unconstr_launch_count.argtypes = [c_vp]
    L.rbt_unconstr_launch_count.restype = c_ll
    L.rbt_unconstr_stage_layout_get.argtypes = [c_int, c_int, ctypes.c_char_p]
    L.rbt_unconstr_stage_setup.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_condense.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_expand_and_step_sizes.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_update.argtypes = [c_vp, c_vp]
    L.rbt_unconstr_iteration_host.argtypes = [c_vp] * 9
    _ = pd
    _lib = L
    return L

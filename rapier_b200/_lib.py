"""Loader of the CUDA library (rapier_b200/csrc/librapier_b200.so) and its ctypes prototypes.

The product path has NO fallback: if the shared library is missing, or no CUDA device is usable,
loading / world creation raises.  (tests/emul builds a host emulation of the kernel logic for CI
boxes without a GPU; it is loaded only by tests/emul_lib.py, never from here.)
"""
import ctypes as C
import os

from . import _abi as A

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "librapier_b200.so")
if os.environ.get("RAPIER_B200_DEBUG_LIB") == "1":   # profiling experiments only (-DRB_DEBUG build of the same sources)
    LIB_PATH = os.path.join(HERE, "csrc", "librapier_b200_dbg.so")
elif os.environ.get("RAPIER_B200_DEBUG_LIB"):        # ... or another CUDA build of the same sources, by file name (A/B timing of kernels)
    LIB_PATH = os.path.join(HERE, "csrc", os.path.basename(os.environ["RAPIER_B200_DEBUG_LIB"]))

EXPORTS = [
    "rb_abi_version", "rb_last_error", "rb_integration_parameters_default", "rb_world_create",
    "rb_world_destroy", "rb_world_set_params", "rb_world_set_scene", "rb_world_set_body_states",
    "rb_world_step", "rb_world_synchronize", "rb_world_get_body_states", "rb_world_num_bodies",
    "rb_world_get_counters", "rb_world_enable_profiling", "rb_world_get_contact_pairs",
    "rb_world_debug_read", "rb_world_label_components", "rb_world_set_owned_bodies",
    "rb_world_state_buffer", "rb_world_import_states", "rb_world_import_states_from", "rb_world_state_buffers", "rb_world_stream", "rb_world_set_stream",
    "rb_world_step_host", "rb_debug_kat", "rb_world_get_quarantine", "rb_world_get_sleeping", "rb_world_wake_up", "rb_world_set_halo_bodies", "rb_world_import_halo", "rb_world_reserve", "rb_world_insert", "rb_world_remove_bodies", "rb_world_reserve_joints", "rb_world_insert_joints", "rb_world_remove_joints", "rb_world_update_joints",
    "rb_world_set_body_forces", "rb_world_set_next_kinematic_positions", "rb_world_drain_collision_events", "rb_world_drain_contact_force_events",
    "rb_world_add_hull", "rb_convex_hull",
]


def declare(L):
    """Attach argtypes/restypes of include/rapier_b200.h to a loaded library."""
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.rb_abi_version.restype = C.c_int
    L.rb_last_error.restype = C.c_char_p
    L.rb_integration_parameters_default.argtypes = [C.POINTER(A.RbIntegrationParameters)]
    L.rb_world_create.restype = vp
    L.rb_world_create.argtypes = [C.POINTER(A.RbIntegrationParameters), C.c_int]
    L.rb_world_destroy.argtypes = [vp]
    L.rb_world_set_params.argtypes = [vp, C.POINTER(A.RbIntegrationParameters)]
    L.rb_world_set_scene.argtypes = [vp, i32, vp, i32, vp, i32, vp]
    L.rb_world_set_body_states.argtypes = [vp, i32, vp, vp, vp]
    L.rb_world_step.argtypes = [vp, C.POINTER(C.c_float), i32, i32]
    L.rb_world_synchronize.argtypes = [vp]
    L.rb_world_get_body_states.argtypes = [vp, vp, vp]
    L.rb_world_num_bodies.argtypes = [vp]
    L.rb_world_get_counters.argtypes = [vp, C.POINTER(A.RbCounters)]
    L.rb_world_enable_profiling.argtypes = [vp, i32]
    L.rb_world_get_contact_pairs.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    L.rb_world_debug_read.restype = i64
    L.rb_world_debug_read.argtypes = [vp, C.c_char_p, vp, i64]
    L.rb_world_label_components.argtypes = [vp, vp]
    L.rb_world_set_owned_bodies.argtypes = [vp, vp]
    L.rb_world_state_buffer.argtypes = [vp, C.POINTER(vp), C.POINTER(i64)]
    L.rb_world_import_states.argtypes = [vp, vp, vp, i32]
    L.rb_world_import_states_from.argtypes = [vp, vp, vp, i32]
    L.rb_world_state_buffers.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_int64)]
    L.rb_world_stream.restype = vp
    L.rb_world_stream.argtypes = [vp]
    L.rb_world_set_stream.argtypes = [vp, vp]
    L.rb_world_step_host.argtypes = [vp, C.POINTER(C.c_float), vp, vp]
    L.rb_world_get_quarantine.argtypes = [vp, vp, i32]
    L.rb_world_get_sleeping.argtypes = [vp, vp]
    L.rb_world_wake_up.argtypes = [vp, i32, vp]
    L.rb_world_set_halo_bodies.argtypes = [vp, vp]
    L.rb_world_import_halo.argtypes = [vp]
    L.rb_world_reserve.argtypes = [vp, i32, i32]
    L.rb_world_insert.argtypes = [vp, i32, vp, i32, vp, C.POINTER(i32), C.POINTER(i32)]
    L.rb_world_remove_bodies.argtypes = [vp, i32, vp]
    L.rb_world_reserve_joints.argtypes = [vp, i32, i32]
    L.rb_world_insert_joints.argtypes = [vp, i32, vp, vp]
    L.rb_world_remove_joints.argtypes = [vp, i32, vp]
    L.rb_world_update_joints.argtypes = [vp, i32, vp, vp, i32]
    L.rb_world_set_body_forces.argtypes = [vp, i32, vp, vp, vp]
    L.rb_world_set_next_kinematic_positions.argtypes = [vp, i32, vp, vp]
    L.rb_world_drain_collision_events.argtypes = [vp, i32, vp]
    L.rb_world_drain_contact_force_events.argtypes = [vp, i32, vp]
    L.rb_debug_kat.argtypes = [C.c_char_p, vp, i32, vp, i32]
    L.rb_world_add_hull.restype = i32
    L.rb_world_add_hull.argtypes = [vp, i32, vp, i32, vp, vp]
    L.rb_convex_hull.restype = i32
    L.rb_convex_hull.argtypes = [i32, vp, C.POINTER(i32), vp, C.POINTER(i32), vp, vp]
    return L


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  rapier_b200 has no CPU fallback.")
        _lib = declare(C.CDLL(LIB_PATH))
    return _lib

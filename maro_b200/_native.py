"""Loader for the CUDA library (``libmaro_b200.so``, built in-tree by ``__graft_entry__.build()``).

There is deliberately no CPU fallback: if the extension is missing or no GPU is present, the product fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MARO_B200_LIB") or os.path.join(_HERE, "libmaro_b200.so")  # (override: A/B builds of tools/build_variant.py)
_lib = None

#: every symbol ``include/maro_b200.h`` declares
EXPORTS = (
    "maro_last_error", "maro_abi_version", "maro_cim_create", "maro_cim_destroy", "maro_cim_set_stream",
    "maro_cim_step", "maro_cim_step_device", "maro_cim_reset", "maro_cim_set_topology", "maro_cim_query",
    "maro_cim_query_device", "maro_cim_attr_id", "maro_cim_attr_slots", "maro_cim_read_frame",
    "maro_cim_frame_words", "maro_cim_ticks", "maro_cim_counters", "maro_cim_snapshot_frames",
    "maro_cim_random_policy_device", "maro_cim_pinned_buffers", "maro_cim_step_pinned", "maro_cim_rollout_device", "maro_cim_pinned_granularity", "maro_cim_submit_pinned", "maro_cim_wait_pinned",
    "maro_cim_rl_state_dim", "maro_cim_rl_state_device", "maro_cim_rl_state_f32_device", "maro_cim_rl_reward_device", "maro_cim_rl_reward_batch_device", "maro_cim_rl_action_device", "maro_cim_rl_action_ex_device",
    "maro_bike_pinned_buffers", "maro_bike_step_pinned",
    "maro_bike_create", "maro_bike_destroy", "maro_bike_set_stream", "maro_bike_decision_words", "maro_bike_step",
    "maro_bike_step_device", "maro_bike_reset", "maro_bike_query", "maro_bike_attr_id", "maro_bike_attr_slots",
    "maro_bike_read_frame", "maro_bike_frame_words", "maro_bike_ticks", "maro_bike_counters", "maro_bike_snapshot_frames",
    "maro_bike_greedy_policy_device", "maro_bike_set_transfer_seeds", "maro_bike_rollout_device",
    "maro_cim_set_query_layout", "maro_bike_set_query_layout", "maro_vm_set_query_layout",
    "maro_cim_save", "maro_cim_load", "maro_bike_save", "maro_bike_load", "maro_vm_save", "maro_vm_load",
    "maro_vm_create", "maro_vm_destroy", "maro_vm_set_stream", "maro_vm_decision_words", "maro_vm_step",
    "maro_vm_step_device", "maro_vm_pinned_buffers", "maro_vm_step_pinned", "maro_vm_reset", "maro_vm_query",
    "maro_vm_attr_id", "maro_vm_attr_slots", "maro_vm_read_frame", "maro_vm_frame_words", "maro_vm_ticks",
    "maro_vm_counters", "maro_vm_snapshot_frames", "maro_vm_best_fit_policy_device", "maro_vm_rollout_device",
)


class NativeLibraryError(RuntimeError):
    pass


def lib():
    """Return the loaded library (ctypes.CDLL) with argtypes declared; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  maro_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, u32 = C.c_void_p, C.c_int32, C.c_uint32
    L.maro_last_error.restype = C.c_char_p
    L.maro_abi_version.restype = C.c_int
    L.maro_cim_create.argtypes = [vp, i32, vp, C.POINTER(vp)]
    L.maro_cim_destroy.argtypes = [vp]
    L.maro_cim_set_stream.argtypes = [vp, vp, i32]
    L.maro_cim_step.argtypes = [vp, vp, vp, vp, vp, vp]
    L.maro_cim_step_device.argtypes = [vp, vp, vp, vp, vp, vp]
    L.maro_cim_reset.argtypes = [vp, vp]
    L.maro_cim_set_topology.argtypes = [vp, i32, vp]
    L.maro_cim_query.argtypes = [vp, vp, i32, i32, vp, i32, vp, i32, vp, i32, vp, vp]
    L.maro_cim_query_device.argtypes = [vp, vp, i32, i32, vp, i32, vp, i32, vp, i32, vp, vp]
    L.maro_cim_attr_id.argtypes = [vp, i32, C.c_char_p]
    L.maro_cim_attr_id.restype = i32
    L.maro_cim_attr_slots.argtypes = [vp, i32, i32]
    L.maro_cim_attr_slots.restype = i32
    L.maro_cim_read_frame.argtypes = [vp, i32, vp, i32]
    L.maro_cim_frame_words.argtypes = [vp]
    L.maro_cim_frame_words.restype = i32
    L.maro_cim_ticks.argtypes = [vp, vp]
    L.maro_cim_counters.argtypes = [vp, vp]
    L.maro_cim_snapshot_frames.argtypes = [vp, i32, vp, i32, vp]
    L.maro_cim_random_policy_device.argtypes = [vp, vp, vp, u32, u32]
    L.maro_cim_pinned_granularity.argtypes = [vp]
    L.maro_cim_pinned_granularity.restype = i32
    L.maro_cim_submit_pinned.argtypes = [vp, i32, i32, i32, i32, i32]
    L.maro_cim_wait_pinned.argtypes = [vp, i32, i32]
    L.maro_cim_rollout_device.argtypes = [vp, i32, u32, u32, i32, vp, vp, vp]
    L.maro_cim_rl_state_dim.argtypes = [vp, i32, i32, i32]
    L.maro_cim_rl_state_dim.restype = i32
    L.maro_cim_rl_state_device.argtypes = [vp, vp, i32, vp, i32, vp, i32, vp]
    L.maro_cim_rl_state_f32_device.argtypes = [vp, vp, i32, vp, i32, vp, i32, vp]
    L.maro_cim_rl_reward_device.argtypes = [vp, vp, vp, vp, i32, C.c_double, C.c_double, vp]
    L.maro_cim_rl_reward_batch_device.argtypes = [vp, vp, vp, i32, vp, i32, C.c_double, C.c_double, vp]
    L.maro_cim_rl_action_device.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp]
    L.maro_cim_rl_action_ex_device.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, vp]
    pvp = C.POINTER(vp)
    for name in ("maro_cim_pinned_buffers", "maro_bike_pinned_buffers", "maro_vm_pinned_buffers"):
        getattr(L, name).argtypes = [vp, pvp, pvp, pvp, pvp, pvp]
    for name in ("maro_cim_step_pinned", "maro_bike_step_pinned", "maro_vm_step_pinned"):
        getattr(L, name).argtypes = [vp, i32, i32, i32]
    L.maro_bike_create.argtypes = [vp, vp, C.POINTER(vp)]
    L.maro_bike_destroy.argtypes = [vp]
    L.maro_bike_set_stream.argtypes = [vp, vp, i32]
    L.maro_bike_decision_words.argtypes = [vp]
    L.maro_bike_decision_words.restype = i32
    L.maro_bike_step.argtypes = [vp, vp, vp, vp, vp, vp]
    L.maro_bike_step_device.argtypes = [vp, vp, vp, vp, vp, vp]
    L.maro_bike_reset.argtypes = [vp, vp]
    L.maro_bike_query.argtypes = [vp, vp, i32, i32, vp, i32, vp, i32, vp, i32, vp, vp]
    L.maro_bike_attr_id.argtypes = [vp, i32, C.c_char_p]
    L.maro_bike_attr_id.restype = i32
    L.maro_bike_attr_slots.argtypes = [vp, i32, i32]
    L.maro_bike_attr_slots.restype = i32
    L.maro_bike_read_frame.argtypes = [vp, i32, vp, i32]
    L.maro_bike_frame_words.argtypes = [vp]
    L.maro_bike_frame_words.restype = i32
    L.maro_bike_ticks.argtypes = [vp, vp]
    L.maro_bike_counters.argtypes = [vp, vp]
    L.maro_bike_snapshot_frames.argtypes = [vp, i32, vp, i32, vp]
    L.maro_bike_greedy_policy_device.argtypes = [vp, vp, vp]
    L.maro_bike_set_transfer_seeds.argtypes = [vp, vp]
    L.maro_bike_rollout_device.argtypes = [vp, i32, vp, vp]
    for name in ("maro_cim_set_query_layout", "maro_bike_set_query_layout", "maro_vm_set_query_layout"):
        getattr(L, name).argtypes = [vp, i32]
    for pre in ("maro_cim", "maro_bike", "maro_vm"):
        getattr(L, pre + "_save").argtypes = [vp, C.c_char_p, i32]
        getattr(L, pre + "_load").argtypes = [vp, C.c_char_p]
    for pre in ("maro_vm",):  # same shapes as the citi_bike entry points
        getattr(L, pre + "_create").argtypes = [vp, vp, C.POINTER(vp)]
        getattr(L, pre + "_destroy").argtypes = [vp]
        getattr(L, pre + "_set_stream").argtypes = [vp, vp, i32]
        getattr(L, pre + "_decision_words").argtypes = [vp]
        getattr(L, pre + "_decision_words").restype = i32
        getattr(L, pre + "_step").argtypes = [vp, vp, vp, vp, vp, vp]
        getattr(L, pre + "_step_device").argtypes = [vp, vp, vp, vp, vp, vp]
        getattr(L, pre + "_reset").argtypes = [vp, vp]
        getattr(L, pre + "_query").argtypes = [vp, vp, i32, i32, vp, i32, vp, i32, vp, i32, vp, vp]
        getattr(L, pre + "_attr_id").argtypes = [vp, i32, C.c_char_p]
        getattr(L, pre + "_attr_id").restype = i32
        getattr(L, pre + "_attr_slots").argtypes = [vp, i32, i32]
        getattr(L, pre + "_attr_slots").restype = i32
        getattr(L, pre + "_read_frame").argtypes = [vp, i32, vp, i32]
        getattr(L, pre + "_frame_words").argtypes = [vp]
        getattr(L, pre + "_frame_words").restype = i32
        getattr(L, pre + "_ticks").argtypes = [vp, vp]
        getattr(L, pre + "_counters").argtypes = [vp, vp]
        getattr(L, pre + "_snapshot_frames").argtypes = [vp, i32, vp, i32, vp]
    L.maro_vm_best_fit_policy_device.argtypes = [vp, vp, vp]
    L.maro_vm_rollout_device.argtypes = [vp, i32, vp, vp]
    if L.maro_abi_version() != _abi.ABI_VERSION:
        raise NativeLibraryError("libmaro_b200.so ABI version mismatch; rebuild")
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise RuntimeError(lib().maro_last_error().decode())

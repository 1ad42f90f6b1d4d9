"""CPU: the small-topology instantiation of the CIM step (replica_step<G, false, kSmall = true>, the resident kernel's form with
the control state held between ctl_load and ctl_store) under the host emulator, against the golden reference traces and the
oracle; and the due rings (per-vessel, per-stop accumulators of the discharges) against the calendar queue they replace."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emul
from helpers import CASES, assert_snapshots_equal, case_topology, drive, load_golden
from maro_b200 import _abi
from oracle.cim_oracle import CimOracle

SRC = os.path.join(os.path.dirname(emul.SRC), "emul_small.cpp")
LIB = os.path.join(os.path.dirname(emul.LIB), "libmaro_emul_small.so")
_lib = None


def emul_lib():
    """the emulator (tests/_emul_src/emul.cpp) plus the small-topology step (emul_small.cpp), built like emul.lib()"""
    global _lib
    if _lib is None:
        deps = [SRC, emul.SRC, os.path.join(os.path.dirname(SRC), "warp_emul.hpp"), os.path.join(emul.CORE, "cim_core.cuh"),
                os.path.join(emul.CORE, "cim_host.hpp")]
        if not os.path.isfile(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-ffp-contract=off", "-DMARO_HOST_EMULATION",
                                   "-I", os.path.dirname(SRC), "-I", os.path.join(os.path.dirname(emul.HERE), "include"),
                                   "-shared", "-fPIC", SRC, "-o", LIB])
        L = C.CDLL(LIB)
        L.emul_create.restype = C.c_void_p
        L.emul_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.emul_destroy.argtypes = [C.c_void_p]
        L.emul_small_step.argtypes = [C.c_void_p] * 5
        L.emul_small_ok.argtypes = [C.c_void_p]
        L.emul_due_ring_slots.argtypes = [C.c_void_p]
        L.emul_step.argtypes = [C.c_void_p] * 5
        L.emul_frame_words.argtypes = [C.c_void_p]
        L.emul_max_actions.argtypes = [C.c_void_p]
        L.emul_read_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.emul_read_snapshot.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.emul_tick.argtypes = [C.c_void_p, C.c_int]
        L.emul_counters.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib = L
    return _lib


class _Env:
    """one replica under the emulator; `small` steps through replica_step<G, false, kSmall = true>"""

    def __init__(self, spec, topo, lanes=0, small=True):
        self._topo, self._keep = _abi.topology_struct(topo)
        cfg = _abi.MaroCimConfig()
        cfg.n_replicas = 1
        cfg.start_tick = spec.get("start_tick", 0)
        cfg.snapshot_resolution = spec.get("snapshot_resolution", 1)
        cfg.max_snapshots = int(spec.get("max_snapshots") or 0)
        cfg.max_actions = 2
        self._h = emul_lib().emul_create(C.byref(self._topo), 1, C.byref(cfg), lanes)
        assert self._h
        self.small = small
        self.A = emul_lib().emul_max_actions(self._h)
        self.frame_words = emul_lib().emul_frame_words(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            emul_lib().emul_destroy(self._h)
            self._h = None

    def step1(self, actions=None):
        dec = np.zeros((1, 8), np.int32)
        met = np.zeros((1, 3), np.int64)
        a = n = None
        if actions is not None:
            src = np.asarray(actions, np.int32).reshape(1, -1, 4)
            a = np.zeros((1, self.A, 4), np.int32)
            a[:, :src.shape[1]] = src
            n = np.full(1, src.shape[1], np.int32)
        args = (self._h, None if a is None else a.ctypes.data, None if n is None else n.ctypes.data, dec.ctypes.data,
                met.ctypes.data)
        if self.small:
            assert emul_lib().emul_small_step(*args) == 1
        else:
            emul_lib().emul_step(*args)
        return int(dec[0, 6]), dec[0], met[0]

    def frame(self):
        out = np.zeros(self.frame_words, np.int32)
        emul_lib().emul_read_frame(self._h, 0, out.ctypes.data)
        return out

    def snapshot(self, frame_index, rep=0):
        out = np.zeros(self.frame_words, np.int32)
        return out if emul_lib().emul_read_snapshot(self._h, rep, frame_index, out.ctypes.data) else None

    def tick(self):
        return emul_lib().emul_tick(self._h, 0)

    def counters(self):
        out = np.zeros(4, np.int64)
        emul_lib().emul_counters(self._h, 0, out.ctypes.data)
        return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_small_kernel_matches_reference_trace(name):
    spec = CASES[name]
    topo = case_topology(spec)
    e = _Env(spec, topo)
    if not emul_lib().emul_small_ok(e._h):
        pytest.skip("shape outside the small-topology instantiation (noise, volume, resolution or size)")
    gold = load_golden(name)
    rows, final, dec, st = drive(lambda a: e.step1(a), spec)
    assert rows.shape == gold["steps"].shape
    if not np.array_equal(rows, gold["steps"]):
        bad = np.argwhere(rows != gold["steps"])[0]
        raise AssertionError(f"step {bad[0]} col {bad[1]}: got {rows[bad[0]]} want {gold['steps'][bad[0]]}")
    assert final.tolist() == gold["final_metrics"].tolist()
    assert e.tick() == int(gold["final_tick"])
    assert st == 1
    assert e.step1(None)[0] == 2
    if "frames" in gold:
        assert_snapshots_equal(e.snapshot, gold, topo)
    o = CimOracle(topo, spec.get("start_tick", 0), spec.get("snapshot_resolution", 1), spec.get("max_snapshots"))
    drive(lambda a: o.step(a), spec)
    assert e.counters().tolist() == o.counters().tolist()
    assert np.array_equal(e.frame(), o.frame())


def test_small_instantiation_covers_the_noise_free_toy_cases():
    """the cases above are not all skipped: the noise-free toy topologies take the small instantiation and the due rings"""
    for name in ("toy4p_l00_300_rand_r0", "toy4p_l00_1120_null"):
        spec = CASES[name]
        e = _Env(spec, case_topology(spec))
        assert emul_lib().emul_small_ok(e._h) == 1, name
        assert emul_lib().emul_due_ring_slots(e._h) == 4, name  # toy.4p: route length 3 -> 4 slots per vessel


def _with_repeated_stop_tick(topo):
    """the same episode, except that vessel 0 reaches its last stop at the tick of the one before (both after the episode)"""
    hi = int(topo.stop_offset[1])
    arr = topo.stop_arrival.copy()
    assert arr[hi - 2] >= topo.max_tick
    arr[hi - 1] = arr[hi - 2]
    topo.stop_arrival = arr
    return topo


@pytest.mark.parametrize("lanes", [0, 1])
def test_repeated_stop_tick_falls_back_to_the_queue(lanes):
    """a vessel whose stop ticks do not strictly increase: no due rings (nor the small instantiation); the calendar queue
    runs the episode, which is the golden one (the repeated tick lies after it)"""
    name = "toy4p_l00_300_rand_r0"
    spec, gold = CASES[name], load_golden(name)
    topo = _with_repeated_stop_tick(case_topology(spec))
    e = _Env(spec, topo, lanes, small=False)
    assert emul_lib().emul_due_ring_slots(e._h) == 0
    assert emul_lib().emul_small_ok(e._h) == 0
    rows, final, _, st = drive(lambda a: e.step1(a), spec)
    assert np.array_equal(rows, gold["steps"]) and final.tolist() == gold["final_metrics"].tolist() and st == 1
    o = CimOracle(case_topology(spec))
    drive(lambda a: o.step(a), spec)
    assert e.counters().tolist() == o.counters().tolist()
    assert np.array_equal(e.frame(), o.frame())

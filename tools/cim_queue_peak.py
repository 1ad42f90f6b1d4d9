"""High-water mark of the CIM calendar queue (dynamic events outstanding at once) against the configured capacity `QN`.

The device code is compiled for the host with -DMARO_TRACK_QPEAK (tests/_emul_src/emul.cpp, thread-per-lane emulator) and an
episode is played per seed with a random agent.  Build container only; used to size `queue_capacity` head-room claims in DESIGN.md.
Noise-free handles with delay lines and due rings (toy.*_l0.0: every vessel's stop ticks increase strictly) do not use the
queue at all (`QN = 0`): their peak is 0 and `queue_capacity` does not apply to them.

    python tools/cim_queue_peak.py global_trade.22p_l0.8 500 4096 4097 4098
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import emul  # noqa: E402

from maro_b200.scenarios.cim.topology import build_topology  # noqa: E402

topology, durations = sys.argv[1], int(sys.argv[2])
seeds = [int(x) for x in sys.argv[3:]] or [None]
out = "/tmp/libmaro_emul_qpeak.so"
subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-ffp-contract=off", "-DMARO_HOST_EMULATION", "-DMARO_TRACK_QPEAK",
                       "-I", os.path.dirname(emul.SRC), "-I", os.path.join(ROOT, "include"), "-shared", "-fPIC", emul.SRC, "-o", out])
emul.LIB = out
for seed in seeds:
    topo = build_topology(topology, durations) if seed is None else build_topology(topology, durations, seed=seed)
    for agent in ("noop", "random"):
        e = emul.EmulEnv(topo, lanes=32)
        peak = C.c_int.in_dll(emul.lib(), "maro_emul_qpeak")
        peak.value = 0
        rng = np.random.default_rng(7)
        st, dec, _ = e.step1(None)
        n = 0
        while st == 0:
            a = None
            if agent == "random":  # dec: tick, port, vessel, load scope, discharge scope, early discharge, status
                load, dis = int(dec[3]), int(dec[4])
                if rng.random() < 0.5 and load > 0:
                    a = [[dec[2], dec[1], int(rng.integers(0, load + 1)), 0]]
                elif dis > 0:
                    a = [[dec[2], dec[1], int(rng.integers(0, dis + 1)), 1]]
            st, dec, _ = e.step1(a)
            n += 1
        print(f"{topology} seed {seed} agent {agent}: {n} decisions, status {st}, queue peak {peak.value}")

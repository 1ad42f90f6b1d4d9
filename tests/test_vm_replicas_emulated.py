"""CPU: the replica-class harness of tests/test_gpu_vm_replicas.py (tests/vm_helpers.py, ``VmClasses``) on the
emulator-backed batch, host stepping and end state: the agent, the active and reset schedules, the BAD_ACTION class and
the oracle replay run on any machine, with the device logic under the host emulator instead of the kernels."""
import numpy as np
import pytest

from emul_batch import EmulVmBatch
from vm_helpers import VM_CASES, VmClasses, vm_topology

P, B = 3, 6
BAD = (2, 3)


@pytest.mark.parametrize("name", ["synth_120_oversub_mixed", "synth_160_tight_budget"])
def test_vm_replica_classes_emulated(name):
    spec = VM_CASES[name]
    topo = vm_topology(spec)
    res, ms = spec.get("snapshot_resolution", 1), spec.get("max_snapshots")
    env = EmulVmBatch(topo, B, res, ms)
    h = VmClasses(env, topo, P, res, ms, bad=BAD)
    h.first_step()
    h.host_steps(4, 1)
    h.reset(h.c % 4 == 1)
    h.host_steps(6, 5)
    assert h.bad_seen and h.last[BAD[0], 6] in (-1, 2)  # BAD_ACTION, then FINISHED if stepped again
    assert (h.last[np.arange(P) != BAD[0], 6] != -1).all()
    h.reset((h.last[:, 6] != 0) | (h.c % 4 == 2))
    h.host_steps(30, 11)
    h.check_end(with_counters=False)  # (the emulated reset starts a fresh emulator: its counters do not persist)

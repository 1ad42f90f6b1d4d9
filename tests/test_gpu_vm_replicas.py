"""GPU (-m gpu): vm_scheduling with replicas that really diverge, at every launch shape `maro_vm_create` picks.

Replica r belongs to class r % 37 (tests/vm_helpers.py, ``VmClasses``): its agent, active mask and reset schedule depend
on the class only, so each step is checked batch-wide (every replica against its class representative, bit for bit) and
per class (each representative against its own VmOracle).  Anything that leaks between warps of a CTA (the per-warp float64
scratch, the rollout kernel's per-warp decision / metrics / action slots), between CTAs or between grid-stride passes, or
that indexes the float64 lift of a batched query by the wrong replica, shows up as a class whose members disagree.

Each case runs host ``step()`` with actions, empty action lists, inactive replicas and masked resets (one class answers
a decision with the wrong VM and must end in BAD_ACTION alone), then ``step_device`` on device tensors, then fused
``rollout_device`` launches of uneven length until every class is done, and finally compares frames, counters, the
snapshot ring and one batched query with the oracles.  The launch shape of each case is read from the profiler trace of\nthe same configuration."""
import json
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import yaml

from vm_helpers import VM_CASES, VmClasses, gen, vm_topology

pytestmark = pytest.mark.gpu

P = 37
BAD = (6, 1)  # class 6 answers its second decision with a VM id no VM has (and is not among the first reset's classes)


def _n_sm():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _topology(name):
    from maro_b200.scenarios.vm_scheduling.data import build_vm_topology

    if name == "hier_1130":
        from test_vm_oracle_golden import CONFIG_1130

        conf = yaml.safe_load(CONFIG_1130)
        conf["VM_TABLE"] = VM_CASES["toy_5_first"]["conf"]["VM_TABLE"]
        conf["CPU_READINGS"] = VM_CASES["toy_5_first"]["conf"]["CPU_READINGS"]
        return build_vm_topology(conf, 0, 5), 1, None
    if name == "synth_640":  # 640 PMs: the 4-warp rollout kernel needs the opt-in shared-memory carve-out
        conf = gen.config("vm_synth", [(32, 128, 185, 120), (16, 112, 100, 60)], 32, 10, BUFFER_TIME_BUDGET=3)
        return build_vm_topology(conf, 0, 60), 2, 8
    spec = VM_CASES[name]
    return vm_topology(spec), spec.get("snapshot_resolution", 1), spec.get("max_snapshots")


def _trace(fn, tmp_path):
    """run fn under torch.profiler: [(kernel name, grid x, block x)]"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as fp:
        events = json.load(fp)["traceEvents"]
    return [(e["name"], e["args"]["grid"][0], e["args"]["block"][0]) for e in events if e.get("cat") == "kernel"]


def _one_launch(kernels, kernel):
    got = [(int(m.group(1)), g, b) for name, g, b in kernels for m in [re.search(kernel + r"<(\d+)>", name)] if m]
    assert len(got) == 1, (kernel, kernels)
    return got[0]


def _probe(name, B, out_dir):
    """print the (warps, grid, block) of one vm_step_kernel and one vm_rollout_kernel launch of a fresh handle"""
    import torch

    from maro_b200.batch import VmBatch

    topo, res, ms = _topology(name)
    env = VmBatch(topo, B, res, ms)
    env.set_stream(torch.cuda.current_stream().cuda_stream)
    dec = torch.zeros((B, env.dec_words), dtype=torch.int32, device="cuda")
    met = torch.zeros((B, 16), dtype=torch.int64, device="cuda")
    step = _trace(lambda: env.step_device(dec.data_ptr(), met.data_ptr()), pathlib.Path(out_dir))
    roll = _trace(lambda: env.rollout_device(dec.data_ptr(), met.data_ptr(), 1), pathlib.Path(out_dir))
    print(json.dumps([_one_launch(step, "vm_step_kernel"), _one_launch(roll, "vm_rollout_kernel")]))
    env.close()


def _launch_shapes(name, B, tmp_path):
    """the probe, in a process of its own: the trace then does not depend on what earlier tests in this process did with
    the profiler"""
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = {[here, os.path.dirname(here)]!r}; import test_gpu_vm_replicas as t; "
            f"t._probe({name!r}, {B}, {str(tmp_path)!r})")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return [tuple(x) for x in json.loads(r.stdout.strip().splitlines()[-1])]


# (topology, B or "two_pass" = 48 nSM + 37, warps per CTA the batch must get)
CASES = [("synth_120_oversub_mixed", 37, 1), ("synth_120_oversub_mixed", 300, 2), ("synth_120_oversub_mixed", "two_pass", 4),
         ("synth_160_tight_budget", 37, 1), ("synth_160_tight_budget", 300, 2), ("synth_160_tight_budget", "two_pass", 4),
         ("hier_1130", 300, 2), ("synth_640", 600, 4)]


@pytest.mark.parametrize("name,B,warps", CASES, ids=[f"{n}-B{b}" for n, b, _ in CASES])
def test_vm_diverging_replicas_match_their_oracles(name, B, warps, tmp_path):
    import torch

    from maro_b200.batch import VmBatch

    n_sm = _n_sm()
    B = 48 * n_sm + P if B == "two_pass" else B
    topo, res, ms = _topology(name)
    env = VmBatch(topo, B, res, ms)
    h = VmClasses(env, topo, P, res, ms, bad=BAD)
    grid_want = min(-(-B // warps), 48 // warps * n_sm)
    if B > 48 * n_sm:
        assert grid_want < -(-B // warps)  # a second grid-stride pass
    assert _launch_shapes(name, B, tmp_path) == [(warps, grid_want, warps * 32)] * 2

    # phase 1: host step() with actions, n_actions, active; masked resets mid-episode
    quarter = h.c % 4 == 1
    h.first_step()
    h.host_steps(4, 1)
    h.reset(quarter)
    h.host_steps(6, 5)
    assert h.bad_seen and h.last[BAD[0], 6] in (-1, 2)  # BAD_ACTION, then FINISHED if stepped again
    assert (h.last[np.arange(P) != BAD[0], 6] != -1).all()
    # a later reset that also hits classes already DONE / FINISHED (the BAD_ACTION class among them)
    finished = h.last[:, 6] != 0
    again = finished | (h.c % 4 == 2)
    h.reset(again)
    h.host_steps(6, 11)

    # phase 2: step_device with device-resident actions, n_actions and active
    env.set_stream(torch.cuda.current_stream().cuda_stream)
    dec_t = torch.from_numpy(env.decisions.copy()).cuda()
    met_t = torch.from_numpy(env.metrics.copy()).cuda()
    for i in range(17, 25):
        acts, nact, active, per_class = h.inputs(i, active_every=1000 if i == 24 else 5)  # the last step: every class
        inputs = [torch.from_numpy(x).cuda() for x in (acts, nact, active)]  # (held until the step has run)
        env.step_device(dec_t.data_ptr(), met_t.data_ptr(), *(t.data_ptr() for t in inputs))
        h.check(dec_t.cpu().numpy(), met_t.cpu().numpy(), per_class[2], h.oracle_step(per_class), f"device step {i}")
    assert (dec_t.cpu().numpy()[:, 6] != 3).all()

    # phase 3: fused rollouts in uneven launches until every class is done, then one more launch.  Classes whose episode
    # has ended start a new one first (the rollout kernel starts a freshly reset replica whatever its last row says).
    h.reset(h.last[:, 6] != 0)
    everyone = np.ones(P, bool)
    chunks = [1, 3, 50] + [4000] * 4
    for n in chunks:
        env.rollout_device(dec_t.data_ptr(), met_t.data_ptr(), n)
        outs = h.rollout_model(n)
        h.check(dec_t.cpu().numpy(), met_t.cpu().numpy(), everyone, outs, f"rollout of {n}")
        if (h.last[:, 6] != 0).all():
            break
    assert (h.last[:, 6] != 0).all()
    env.rollout_device(dec_t.data_ptr(), met_t.data_ptr(), 5)
    outs = h.rollout_model(5)
    d, m = dec_t.cpu().numpy(), met_t.cpu().numpy()
    assert (d[:, 6] == 2).all() and (np.delete(d, 6, axis=1) == 0).all() and (m == 0).all()
    h.check(d, m, everyone, outs, "launch after the end")

    # phase 4: end state against the oracles
    h.check_end()
    env.close()

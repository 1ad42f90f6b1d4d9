"""GPU (-m gpu): a masked reset leaves the caller's pinned staging buffers alone.

A caller may fill the pinned action / n_actions / active rows for the next ``step_pinned``, reset some finished replicas,
then step.  The reset must neither write those rows nor change what the step computes: every scenario is checked
against a twin handle that gets the same inputs through ``step()``.  Each test runs with zero-copy steps (the default at
this size) and with bulk copies (``MARO_B200_ZEROCOPY=0``, read when the handle is created)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B = 64


def _pair(monkeypatch, zero_copy, make):
    if zero_copy:
        monkeypatch.delenv("MARO_B200_ZEROCOPY", raising=False)
    else:
        monkeypatch.setenv("MARO_B200_ZEROCOPY", "0")
    try:
        return make(), make()
    finally:
        monkeypatch.delenv("MARO_B200_ZEROCOPY", raising=False)


def _inputs(agent, dec, step, rng, A):
    """per-replica actions from each replica's own decision row, some empty action lists, some inactive replicas"""
    acts = np.zeros((B, A, 4), np.int32)
    for i in range(B):
        acts[i, 0] = agent(dec[i], i, step)
    nact = np.ones(B, np.int32)
    nact[rng.choice(np.arange(4, B), 6, replace=False)] = 0
    nact[1] = 0
    active = np.ones(B, np.uint8)
    active[rng.choice(np.arange(4, B), 9, replace=False)] = 0
    active[2] = 0
    return acts, nact, active


def _reset_then_step(x, y, agent, step, rng, use_view):
    """fill x's pinned inputs, reset x and y under the same mask, check the inputs survived, step both and compare"""
    p_act, p_nact, p_active, p_dec, p_met = x.pinned()
    acts, nact, active = _inputs(agent, p_dec.copy(), step, rng, x.max_actions)
    p_act[...] = acts
    p_nact[...] = nact
    p_active[...] = active
    keep = [p_act.tobytes(), p_nact.tobytes(), p_active.tobytes()]
    if use_view:
        p_active[:4] = 0  # (the replicas whose action rows a reset could clobber stay out of the mask)
        active[:4] = 0
        keep[2] = p_active.tobytes()
        x.reset(p_active)
        y.reset(active.copy())
    else:
        mask = np.zeros(B, np.uint8)
        mask[4:] = rng.random(B - 4) < 0.3
        mask[[7, B - 1]] = 1
        x.reset(mask)
        y.reset(mask)
    assert p_act.tobytes() == keep[0], "reset(mask) wrote into the pinned action rows"
    assert p_nact.tobytes() == keep[1], "reset(mask) wrote into the pinned n_actions"
    assert p_active.tobytes() == keep[2], "reset(mask) wrote into the pinned active mask"
    x.step_pinned(True, True, True)
    dy, my = y.step(acts, nact, active)
    live = active.astype(bool)
    assert np.array_equal(p_dec[:, 6], dy[:, 6])
    assert (p_dec[~live, 6] == 3).all()
    assert np.array_equal(p_dec[live], dy[live]) and np.array_equal(p_met[live], my[live])
    return p_dec.copy()


def _drive(x, y, agent, rounds):
    rng = np.random.default_rng(7)
    dx, _ = x.step(None)
    dx = dx.copy()
    dy, _ = y.step(None)
    assert np.array_equal(dx, dy)
    step = 1
    for _ in range(3):
        acts = np.stack([agent(dx[i], i, step) for i in range(B)]).reshape(B, 1, 4)
        dx = x.step(acts)[0].copy()
        assert np.array_equal(dx, y.step(acts)[0])
        step += 1
    for before in rounds:
        if before:
            before()
        for use_view in (False, True):
            _reset_then_step(x, y, agent, step, rng, use_view)
            step += 1


@pytest.mark.parametrize("zero_copy", [True, False], ids=["zerocopy", "bulk"])
def test_cim_masked_reset_keeps_pinned_inputs(monkeypatch, zero_copy):
    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology
    from oracle.cim_oracle import policy_random

    topo = build_topology("toy.4p_ssdd_l0.0", 200)
    x, y = _pair(monkeypatch, zero_copy, lambda: CimBatch(topo, B, device=0))

    def agent(dec, i, step):
        return policy_random(dec, 3, i, step)

    def end_sessions():  # reading device state ends the live session: the next reset takes the direct path
        assert np.array_equal(x.read_frame(5), y.read_frame(5))

    # first with the session live (the reset rides on each replica's next command row), then the direct path
    _drive(x, y, agent, [None, end_sessions])
    x.close()
    y.close()


@pytest.mark.parametrize("zero_copy", [True, False], ids=["zerocopy", "bulk"])
def test_bike_masked_reset_keeps_pinned_inputs(monkeypatch, zero_copy):
    from bike_helpers import BIKE_CASES, bike_config, greedy_py
    from maro_b200.batch import BikeBatch
    from maro_b200.scenarios.citi_bike.data import build_bike_topology

    spec = BIKE_CASES["toy_1440_greedy_res10"]
    topo = build_bike_topology(bike_config(spec["data"]), 0, spec["durations"], transfer_seed=77)
    seeds = np.arange(500, 500 + B, dtype=np.uint32)

    def make():
        env = BikeBatch(topo, B, spec["snapshot_resolution"], spec.get("max_snapshots"))
        env.set_transfer_seeds(seeds)
        env.reset()
        return env

    x, y = _pair(monkeypatch, zero_copy, make)
    _drive(x, y, lambda dec, i, step: np.asarray(greedy_py(dec), np.int32), [None])
    x.close()
    y.close()


@pytest.mark.parametrize("zero_copy", [True, False], ids=["zerocopy", "bulk"])
def test_vm_masked_reset_keeps_pinned_inputs(monkeypatch, zero_copy):
    from maro_b200.batch import VmBatch
    from vm_helpers import VM_CASES, vm_topology

    spec = VM_CASES["synth_120_oversub_mixed"]
    topo = vm_topology(spec)
    x, y = _pair(monkeypatch, zero_copy, lambda: VmBatch(topo, B, 1, None))

    def agent(dec, i, step):
        if dec[6] != 0:
            return np.asarray([-1, -1, 0, 0], np.int32)
        return np.asarray([dec[1], 0, dec[12 + (i + step) % dec[10]], 0], np.int32)

    _drive(x, y, agent, [None])
    x.close()
    y.close()


def test_work_counters_start_at_zero_in_reused_device_memory():
    """No reset writes the cumulative work counters, so a new handle must start them at zero even when its state blocks
    land in device memory a closed handle of this process used (the allocator hands the same blocks back)."""
    from bike_helpers import BIKE_CASES, bike_config
    from maro_b200.batch import BikeBatch, CimBatch, VmBatch
    from maro_b200.scenarios.citi_bike.data import build_bike_topology
    from maro_b200.scenarios.cim.topology import build_topology
    from vm_helpers import VM_CASES, vm_topology

    spec = BIKE_CASES["toy_1440_greedy_res10"]
    makers = [lambda: CimBatch(build_topology("toy.4p_ssdd_l0.0", 100), B, device=0),
              lambda: BikeBatch(build_bike_topology(bike_config(spec["data"]), 0, spec["durations"]), B,
                                spec["snapshot_resolution"], spec.get("max_snapshots")),
              lambda: VmBatch(vm_topology(VM_CASES["synth_120_oversub_mixed"]), B, 1, None)]
    for make in makers:
        for _ in range(2):
            env = make()
            assert (env.counters() == 0).all()
            for _ in range(5):
                env.step(None)
            assert (env.counters()[:, 0] == 5).all()
            env.close()

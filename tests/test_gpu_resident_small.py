"""GPU (-m gpu): the small-topology instantiation of the resident kernel (cim_resident_kernel<G, false, 1, true>, chosen at
create for noise-free small topologies; MARO_B200_RES_SMALL=0/1 forces it off / on where allowed) against the general
noise-free one, bit for bit: decision and metrics rows, the snapshot ring read back through snapshot_list queries, and the
state written back to device memory at the end of every launch."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SMALL_TOPOLOGIES = ["toy.4p_ssdd_l0.0", "toy.5p_ssddd_l0.0", "toy.6p_sssbdd_l0.0"]


def _make(topology, ticks, B, small, monkeypatch):
    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology

    monkeypatch.setenv("MARO_B200_RES_SMALL", "1" if small else "0")
    env = CimBatch(build_topology(topology, ticks), B, device=0)
    monkeypatch.delenv("MARO_B200_RES_SMALL")
    return env


def _resident_kernels(env, B):
    """names of the resident-kernel instantiations one short rollout launches"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    dec = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    met = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    env.set_stream(torch.cuda.current_stream().cuda_stream)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        env.rollout_device(dec.data_ptr(), met.data_ptr(), 2, 1, 0, 0)
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "cim_resident_kernel" in e.name}


def _run(env, B, chunk, launches, ticks):
    """`launches` fused rollouts of `chunk` env-steps (Env.reset once every replica is done); per launch the decision and
    metrics rows, the written-back state (frames, ticks, counters) and every snapshot row through snapshot_list queries"""
    import torch

    env.set_stream(torch.cuda.current_stream().cuda_stream)
    dec = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    met = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    n_ports, n_vessels = env.node_counts()["ports"], env.node_counts()["vessels"]
    pattrs = ["empty", "full", "on_shipper", "on_consignee", "booking", "shortage", "fulfillment", "acc_booking",
              "acc_shortage", "acc_fulfillment", "transfer_cost", "capacity"]
    vattrs = ["empty", "full", "remaining_space", "early_discharge", "last_loc_idx", "next_loc_idx", "past_stop_list",
              "future_stop_list", "future_stop_tick_list"]
    out, resets = [], 0
    for _ in range(launches):
        if bool((dec[:, 6] != 0).all().item()):
            env.reset()
            resets += 1
        env.rollout_device(dec.data_ptr(), met.data_ptr(), chunk, 1, 7, 3)
        torch.cuda.synchronize()
        frames = np.arange(ticks, dtype=np.int32)
        out.append({
            "dec": dec.cpu().numpy().copy(), "met": met.cpu().numpy().copy(),
            "frame": np.stack([env.read_frame(i) for i in range(B)]), "ticks": env.ticks().copy(), "counters": env.counters().copy(),
            "ports": env.query("ports", frames, np.arange(n_ports), pattrs),
            "vessels": env.query("vessels", frames, np.arange(n_vessels), vattrs),
        })
    return out, resets


@pytest.mark.parametrize("chunk,launches", [(1, 90), (7, 14), (64, 3)])
@pytest.mark.parametrize("topology", SMALL_TOPOLOGIES)
def test_small_instantiation_matches_general(topology, chunk, launches, monkeypatch):
    ticks, B = 40, 96
    small = _make(topology, ticks, B, True, monkeypatch)
    general = _make(topology, ticks, B, False, monkeypatch)
    assert any("true>" in n for n in _resident_kernels(small, B)), "the small-topology kernel was not selected"
    assert not any("true>" in n for n in _resident_kernels(general, B))
    small.reset()
    general.reset()
    got, r1 = _run(small, B, chunk, launches, ticks)
    want, r2 = _run(general, B, chunk, launches, ticks)
    assert r1 == r2 and r1 >= 1, "the rollouts must cross an episode end"
    for k, (a, b) in enumerate(zip(got, want)):
        for key in b:
            assert np.array_equal(a[key], b[key], equal_nan=a[key].dtype.kind == "f"), (topology, chunk, k, key)
    small.close()
    general.close()


@pytest.mark.parametrize("topology", ["toy.4p_ssdd_l0.8", "global_trade.22p_l0.0", "global_trade.22p_l0.8"])
def test_small_instantiation_not_selected(topology, monkeypatch):
    """order / buffer noise (the general kernel) or more ports than a lane group's width: never the small kernel, even when
    forced"""
    B = 32
    env = _make(topology, 40, B, True, monkeypatch)
    names = _resident_kernels(env, B)
    assert names and not any("true>" in n for n in names), names
    env.close()


@pytest.mark.parametrize("small", [True, False])
def test_session_resets_keep_counters(small, monkeypatch):
    """host session (the resident kernel stays up between Env.step calls, Env.reset of finished replicas rides on their
    next command row) against the per-step kernel: decision and metrics rows every step, and the cumulative work counters,
    which an in-place reset must carry over"""
    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology
    from oracle.cim_oracle import policy_random

    topo, B = build_topology("toy.4p_ssdd_l0.0", 30), 64
    monkeypatch.setenv("MARO_B200_RES_SMALL", "1" if small else "0")
    session = CimBatch(topo, B, device=0)
    monkeypatch.setenv("MARO_B200_SESSION", "0")
    per_step = CimBatch(topo, B, device=0)
    monkeypatch.delenv("MARO_B200_SESSION")
    monkeypatch.delenv("MARO_B200_RES_SMALL")
    acts = np.zeros((B, session.max_actions, 4), np.int32)
    resets = 0
    for k in range(120):
        got = [x.copy() for x in session.step(acts)]
        want = [x.copy() for x in per_step.step(acts)]
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), k
        for i in range(B):
            acts[i, 0] = policy_random(got[0][i], 0, i, k)
        done = (got[0][:, 6] != 0).astype(np.uint8)
        if done.any():
            session.reset(done)
            per_step.reset(done)
            resets += 1
    assert resets >= 2
    assert np.array_equal(session.counters(), per_step.counters())
    assert np.array_equal(session.ticks(), per_step.ticks())
    session.close()
    per_step.close()

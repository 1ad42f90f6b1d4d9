"""GPU (-m gpu): fused rollouts write a decision's snapshot row only when the launch ends on that decision, and noise-free
small topologies keep their discharges on per-vessel due rings.  Checked against a handle that launches the per-step kernel
once per env-step (snapshots written eagerly), advanced by the same steps with the same agent: after EVERY rollout launch the
snapshot ring (every row through snapshot_list queries, and which frame each row holds), the decision and metrics rows, the
written-back frames, the ticks and the work counters are identical -- including launches that end in the middle of a tick
with more decisions due in it, and sliced rollouts."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOPOLOGIES = ["toy.4p_ssdd_l0.0", "toy.5p_ssddd_l0.0", "toy.6p_sssbdd_l0.0"]
SEED, BASE = 7, 3
PATTRS = ["empty", "full", "on_shipper", "on_consignee", "booking", "shortage", "fulfillment", "acc_booking", "acc_shortage",
          "acc_fulfillment", "transfer_cost", "capacity"]
VATTRS = ["empty", "full", "remaining_space", "early_discharge", "last_loc_idx", "next_loc_idx", "past_stop_list",
          "future_stop_list", "future_stop_tick_list"]


def _state(env, B, ticks, dec, met):
    n_ports, n_vessels = env.node_counts()["ports"], env.node_counts()["vessels"]
    frames = np.arange(ticks, dtype=np.int32)
    return {
        "dec": dec.copy(), "met": met.copy(),
        "frame": np.stack([env.read_frame(i) for i in range(B)]), "ticks": env.ticks().copy(), "counters": env.counters().copy(),
        "rows": [sorted(env.snapshot_frames(i).tolist()) for i in range(B)],
        "ports": env.query("ports", frames, np.arange(n_ports), PATTRS),
        "vessels": env.query("vessels", frames, np.arange(n_vessels), VATTRS),
    }


def _assert_same(got, want, what):
    for key in want:
        if key == "rows":
            assert got[key] == want[key], (what, key)
        else:
            assert np.array_equal(got[key], want[key], equal_nan=want[key].dtype.kind == "f"), (what, key)


class _PerStep:
    """the reference side: one per-step kernel launch per env-step, the rollout's device agent evaluated on the host"""

    def __init__(self, topo, B):
        from maro_b200.batch import CimBatch

        self.env = CimBatch(topo, B, device=0)
        self.B = B
        self.dec = np.zeros((B, 8), np.int32)
        self.met = np.zeros((B, 3), np.int64)

    def reset(self):
        self.env.reset()

    def launch(self, n_steps):
        """what one fused rollout of n_steps does: every replica steps until its episode reports done (that row stays)"""
        from oracle.cim_oracle import policy_random

        live = np.ones(self.B, bool)
        acts = np.zeros((self.B, self.env.max_actions, 4), np.int32)
        for _ in range(n_steps):
            if not live.any():
                break
            for i in np.flatnonzero(live):
                acts[i, 0] = policy_random(self.dec[i], SEED, i + BASE, int(self.dec[i, 7]))
            d, m = self.env.step(acts, active=live.astype(np.uint8))
            self.dec[live] = d[live]
            self.met[live] = m[live]
            live &= ~np.isin(self.dec[:, 6], (1, 2))


def _pair(topology, ticks, B, monkeypatch, slice_steps=None):
    import torch

    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology

    topo = build_topology(topology, ticks)
    if slice_steps:
        monkeypatch.setenv("MARO_B200_RES_SLICE_STEPS", str(slice_steps))
    roll = CimBatch(topo, B, device=0)
    monkeypatch.delenv("MARO_B200_RES_SLICE_STEPS", raising=False)
    monkeypatch.setenv("MARO_B200_SESSION", "0")
    ref = _PerStep(topo, B)
    monkeypatch.delenv("MARO_B200_SESSION")
    roll.set_stream(torch.cuda.current_stream().cuda_stream)
    return roll, ref


def _compare(roll, ref, B, ticks, chunk, launches):
    """returns (episode resets, launches that ended on a decision with another decision of the same tick still due)"""
    import torch

    dec = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    met = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    resets, mid_tick = 0, 0
    prev = None
    for k in range(launches):
        if bool((dec[:, 6] != 0).all().item()):
            roll.reset()
            ref.reset()
            resets += 1
            prev = None
        roll.rollout_device(dec.data_ptr(), met.data_ptr(), chunk, 1, SEED, BASE)
        torch.cuda.synchronize()
        ref.launch(chunk)
        d, m = dec.cpu().numpy(), met.cpu().numpy()
        _assert_same(_state(roll, B, ticks, d, m), _state(ref.env, B, ticks, ref.dec, ref.met), (chunk, k))
        if chunk == 1 and prev is not None:  # this launch returned another decision of the tick the previous one ended on
            mid_tick += int(np.sum((d[:, 6] == 0) & (prev[:, 6] == 0) & (d[:, 0] == prev[:, 0])))
        prev = d.copy()
    return resets, mid_tick


@pytest.mark.parametrize("chunk,launches", [(1, 70), (2, 40), (7, 14), (64, 3)])
@pytest.mark.parametrize("topology", TOPOLOGIES)
def test_rollout_snapshots_match_per_step(topology, chunk, launches, monkeypatch):
    ticks, B = 40, 64
    roll, ref = _pair(topology, ticks, B, monkeypatch)
    resets, mid_tick = _compare(roll, ref, B, ticks, chunk, launches)
    assert resets >= 1, "the rollouts must cross an episode end"
    if chunk == 1:
        assert mid_tick > 0, "no launch ended with another decision of its tick still due"
    roll.close()
    ref.env.close()


@pytest.mark.parametrize("chunk,launches", [(7, 14), (64, 3)])
def test_sliced_rollout_snapshots_match_per_step(chunk, launches, monkeypatch):
    ticks, B = 40, 64
    roll, ref = _pair("toy.4p_ssdd_l0.0", ticks, B, monkeypatch, slice_steps=3)
    resets, _ = _compare(roll, ref, B, ticks, chunk, launches)
    assert resets >= 1
    roll.close()
    ref.env.close()


def test_checkpoint_mid_episode_continues_bit_for_bit(tmp_path):
    """a checkpoint saved mid-episode (due rings and their cursors in the replica blocks) continues exactly as the
    handle it was taken from"""
    import torch

    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology

    ticks, B = 60, 64
    topo = build_topology("toy.4p_ssdd_l0.0", ticks)
    a, b = CimBatch(topo, B, device=0), CimBatch(topo, B, device=0)
    stream = torch.cuda.current_stream().cuda_stream
    a.set_stream(stream)
    b.set_stream(stream)
    da = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    ma = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    a.rollout_device(da.data_ptr(), ma.data_ptr(), 23, 1, SEED, BASE)
    torch.cuda.synchronize()
    path = str(tmp_path / "mid.ckpt")
    a.save(path)
    b.load(path)
    db, mb = da.clone(), ma.clone()
    assert bool((da[:, 6] == 0).all().item()), "the checkpoint must be taken mid-episode"
    for _ in range(3):
        a.rollout_device(da.data_ptr(), ma.data_ptr(), 17, 1, SEED, BASE)
        b.rollout_device(db.data_ptr(), mb.data_ptr(), 17, 1, SEED, BASE)
        torch.cuda.synchronize()
        _assert_same(_state(b, B, ticks, db.cpu().numpy(), mb.cpu().numpy()),
                     _state(a, B, ticks, da.cpu().numpy(), ma.cpu().numpy()), "after load")
    a.close()
    b.close()


def _with_repeated_stop_tick(topo):
    """the same episode, except that vessel 0 reaches its last stop at the tick of the one before (both after the episode)"""
    hi = int(topo.stop_offset[1])
    arr = topo.stop_arrival.copy()
    assert arr[hi - 2] >= topo.max_tick
    arr[hi - 1] = arr[hi - 2]
    topo.stop_arrival = arr
    return topo


def test_repeated_stop_tick(monkeypatch):
    """a replacement instance whose stop ticks do not strictly increase is refused by a handle that keeps due rings; a
    handle created with it runs the calendar queue and gives the same episode"""
    import torch

    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology

    ticks, B = 40, 32
    env = CimBatch(build_topology("toy.4p_ssdd_l0.0", ticks), B, device=0)
    with pytest.raises(Exception, match="strictly increase"):
        env.set_topology(0, _with_repeated_stop_tick(build_topology("toy.4p_ssdd_l0.0", ticks)))
    queue = CimBatch(_with_repeated_stop_tick(build_topology("toy.4p_ssdd_l0.0", ticks)), B, device=0)
    stream = torch.cuda.current_stream().cuda_stream
    env.set_stream(stream)
    queue.set_stream(stream)
    d1 = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    m1 = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    d2, m2 = d1.clone(), m1.clone()
    for _ in range(4):
        env.rollout_device(d1.data_ptr(), m1.data_ptr(), 16, 1, SEED, BASE)
        queue.rollout_device(d2.data_ptr(), m2.data_ptr(), 16, 1, SEED, BASE)
        torch.cuda.synchronize()
        _assert_same(_state(queue, B, ticks, d2.cpu().numpy(), m2.cpu().numpy()),
                     _state(env, B, ticks, d1.cpu().numpy(), m1.cpu().numpy()), "queue vs due rings")
    env.close()
    queue.close()

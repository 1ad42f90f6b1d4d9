"""GPU (-m gpu): the launch shapes maro_cim_create / maro_bike_create pick from the batch size and the SM count, and the ones
the MARO_B200_* tuning overrides force, each pinned twice: bit for bit against the CPU oracle on sampled replicas (every lane
group of one full warp, a group in a middle CTA, the last live groups), and for the whole batch against a handle that runs the
per-step kernel with one replica per warp (MARO_B200_SPREAD=1, the path the golden traces pin).

Packed shapes put 32 / G replicas into one warp (G lanes each): ballots, match_any results and shuffles are shifted / narrowed
to the group, and the resident kernel lays out mbarriers, decision slots and state blocks per group.  A leak between groups
only shows when neighbours disagree, so the replicas here run different topology seeds (replica_topology = r % 3), per-replica
hashed agents, subset stepping and masked resets mid-episode, on batches whose last warp and last CTA are partly empty.

Every case reads, from the torch.profiler trace, which instantiation ran (template arguments in the kernel name) and with which
grid and block, so an override that is silently ignored fails the case."""
import json
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SPREAD_REF = {"MARO_B200_SPREAD": 1, "MARO_B200_SESSION": 0}
TUNING = ["MARO_B200_SPREAD", "MARO_B200_RES_SPREAD", "MARO_B200_RES_DENSE", "MARO_B200_RES_SMALL", "MARO_B200_LANES",
          "MARO_B200_ZEROCOPY", "MARO_B200_RES_WARPS", "MARO_B200_ROLL_WARPS", "MARO_B200_RES_SLICE_STEPS", "MARO_B200_SESSION"]
PORT_ATTRS = ["empty", "full", "on_shipper", "on_consignee", "booking", "shortage", "fulfillment", "acc_booking",
              "acc_shortage", "acc_fulfillment", "transfer_cost", "capacity"]
VESSEL_ATTRS = ["empty", "full", "remaining_space", "early_discharge", "last_loc_idx", "next_loc_idx", "future_stop_list"]


def _n_sm():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _batch_mod32(lo, hi):
    """a batch size in [lo, hi] that is 5 mod 32: the last warp and the last CTA are partly empty"""
    b = (lo + hi) // 2
    b += (5 - b) % 32
    if b > hi:
        b -= 32
    assert lo <= b <= hi and b % 32 == 5, (lo, hi, b)
    return b


def _cim_topologies(name, ticks, multi):
    """one topology, or three instances of it with different seeds (replica r runs instance r % 3)"""
    from maro_b200.scenarios.cim.topology import build_topology

    if not multi:
        return [build_topology(name, ticks)]
    return [build_topology(name, ticks, seed=s) for s in (101, 202, 303)]


def _clean_env(monkeypatch):
    for k in TUNING:
        monkeypatch.delenv(k, raising=False)


def _make(cls, monkeypatch, overrides, *args, **kw):
    """a handle created under `overrides` (read only at create), which are unset again afterwards"""
    _clean_env(monkeypatch)
    for k, v in overrides.items():
        monkeypatch.setenv(k, str(v))
    try:
        return cls(*args, **kw)
    finally:
        _clean_env(monkeypatch)


def _cim(monkeypatch, overrides, topos, B, **kw):
    from maro_b200.batch import CimBatch

    rt = (np.arange(B) % len(topos)).astype(np.int32) if len(topos) > 1 else None
    return _make(CimBatch, monkeypatch, overrides, topos, B, replica_topology=rt, device=0, **kw)


def _trace(fn, tmp_path):
    """run fn under torch.profiler: [(kernel name, grid, block)], [memcpy names], fn's result"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as fp:
        events = json.load(fp)["traceEvents"]
    kernels = [(e["name"], e.get("args", {}).get("grid"), e.get("args", {}).get("block")) for e in events if e.get("cat") == "kernel"]
    copies = [e["name"] for e in events if e.get("cat") == "gpu_memcpy"]
    for name, grid, block in kernels:
        assert grid is not None and block is not None, f"the profiler trace carries no launch dimensions for {name}"
    return kernels, copies, out


def _launches(kernels, kernel):
    """(template arguments, grid x, block x) of every launch of `kernel` in a trace"""
    out = []
    for name, grid, block in kernels:
        m = re.search(kernel + r"<([^<>]*)>", name)
        if m:
            targs = tuple(True if a == "true" else False if a == "false" else int(a) for a in (x.strip() for x in m.group(1).split(",")))
            out.append((targs, int(grid[0]), int(block[0])))
    return out


def _one_launch(kernels, kernel):
    got = _launches(kernels, kernel)
    assert len(got) == 1, (kernel, [k[0] for k in kernels])
    return got[0]


def _sample(B, groups_per_warp, replicas_per_cta):
    """every group of the first (full) warp, a group of a middle CTA, the last live groups"""
    mid = (B // replicas_per_cta // 2) * replicas_per_cta + groups_per_warp + 1
    return sorted({*range(groups_per_warp), min(mid, B - 1), B - 2, B - 1})


def _assert_rows(got, want, what, gpw):
    if not np.array_equal(got, want):
        bad = np.argwhere((got != want).reshape(len(got), -1).any(1))[:, 0]
        r = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} replicas differ, first {r} (group {r % gpw} of its warp): "
                             f"got {got[r].tolist()} want {want[r].tolist()}")


def _assert_state(x, ref, gpw, frames, P, V):
    """ticks, counters, every replica's written-back frame, the ring rows through one batched query"""
    _assert_rows(x.ticks().reshape(-1, 1), ref.ticks().reshape(-1, 1), "ticks", gpw)
    _assert_rows(x.counters(), ref.counters(), "counters", gpw)
    B = x.n_replicas
    _assert_rows(np.stack([x.read_frame(i) for i in range(B)]), np.stack([ref.read_frame(i) for i in range(B)]), "frames", gpw)
    fr = np.asarray(frames, np.int32)
    for node, n, attrs in (("ports", P, PORT_ATTRS), ("vessels", V, VESSEL_ATTRS)):
        a, b = x.query(node, fr, np.arange(n), attrs), ref.query(node, fr, np.arange(n), attrs)
        _assert_rows(np.nan_to_num(a, nan=-1.5), np.nan_to_num(b, nan=-1.5), f"{node} ring rows", gpw)


def _query_frames(ticks, B):
    n = max(4, min(ticks, 200000 // B))
    return np.unique(np.linspace(0, ticks - 1, n).astype(np.int32))


def _replay_steps(o, tape):
    """the oracle against one replica's per-step tape [(reset, active, actions or None, decision row, metrics row)]"""
    for k, (reset, active, act, dec, met) in enumerate(tape):
        if reset:
            o.reset()
        if not active:
            continue
        st, d, m = o.step(act)
        assert d[:7].tolist() == dec[:7].tolist(), (k, d, dec)
        if st != 2:
            assert m.tolist() == met.tolist(), (k, m, met)


def _replay_rollouts(o, launches, r, seed, base):
    """the oracle against one replica's fused rollouts [(reset before, trace rows [n][8], decision row, metrics row at the end)],
    the hashed agent replayed from the traced rows"""
    from oracle.cim_oracle import policy_random

    prev, over = None, False
    for L, (reset, rows, end_dec, end_met) in enumerate(launches):
        if reset:
            o.reset()
            prev, over = None, False
        last = None
        for j, row in enumerate(rows):
            if over:  # the launch repeats the DONE row; a later one answers FINISHED
                assert row[6] in (1, 2), (L, j, row)
                continue
            act = None if prev is None else np.asarray([policy_random(prev, seed, r + base, int(prev[7]))], np.int32)
            st, d, m = o.step(act)
            assert d[:7].tolist() == row[:7].tolist(), (L, j, d, row)
            prev, last, over = row, (st, d, m), st != 0
        if last is not None and last[0] in (0, 1):
            assert end_dec[:7].tolist() == last[1][:7].tolist() and end_met.tolist() == last[2].tolist(), (L, end_dec, last)


def _oracle_final(o, x, r):
    """the oracle's frame, work counters and last snapshot rows against replica r's"""
    assert np.array_equal(x.read_frame(r), o.frame()), r
    assert x.counters()[r].tolist() == o.counters().tolist(), r
    for f in x.snapshot_frames(r)[-3:]:
        assert np.array_equal(x.snapshot_row(int(f), r), o.snapshot(int(f))), (r, int(f))


# ---- CIM per-step kernel ---------------------------------------------------------------------------------------------


def _step_loop(x, ref, B, path, sample, tmp_path, seed=5, resets=(9, 23), max_actions=1, lists=False, trace_at=1):
    """Drive the tested handle and the reference with the same actions (the hashed agent, evaluated by the reference handle on
    the tested handle's rows), random subset stepping and masked resets; every step's decision and metrics rows of the whole
    batch must agree.  Returns the profiler trace of step `trace_at` and the per-step tapes of the sampled replicas."""
    import torch

    s = torch.cuda.current_stream().cuda_stream
    dev = path == "device"
    ref.set_stream(s)
    if dev:  # (a host-step handle keeps its own non-blocking stream: a live session must not hold up torch's stream)
        x.set_stream(s)
    bufs = [(torch.zeros((B, 8), dtype=torch.int32, device="cuda"), torch.zeros((B, 3), dtype=torch.int64, device="cuda"))
            for _ in range(2)]
    d_act = torch.zeros((B, max_actions, 4), dtype=torch.int32, device="cuda")
    d_rows = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(seed)
    tapes = {r: [] for r in sample}
    cur = np.zeros((B, 8), np.int32)
    traced = None
    for k in range(100000):
        reset = np.zeros(B, np.uint8)
        if k in resets:  # neighbours end up in different episodes, at different ticks
            reset = (rng.random(B) < 0.3).astype(np.uint8)
            x.reset(reset)
            ref.reset(reset)
        active = None if k % 3 == 0 else (rng.random(B) < 0.75).astype(np.uint8)
        acts = nact = None
        if k > 0:
            d_rows.copy_(torch.from_numpy(cur))
            ref.random_policy_device(d_rows.data_ptr(), d_act.data_ptr(), seed, 0)
            acts = d_act.cpu().numpy()
            if lists:  # action lists: the LOAD part, then a DISCHARGE of 0; some replicas without any action
                acts[:, 1] = acts[:, 0]
                acts[:, 1, 2] = 0
                acts[:, 1, 3] = 1
                nact = np.where(np.arange(B) % 7 == k % 7, 0, 1 + (k % 2)).astype(np.int32)
                d_act.copy_(torch.from_numpy(acts))
        d_active = torch.from_numpy(active).cuda() if dev and active is not None else None
        d_n = torch.from_numpy(nact).cuda() if dev and nact is not None else None
        outs = []
        for e, (dd, dm) in zip((x, ref), bufs):
            def go(e=e, dd=dd, dm=dm):
                if dev:
                    e.step_device(dd.data_ptr(), dm.data_ptr(), d_act.data_ptr() if acts is not None else 0,
                                  d_n.data_ptr() if d_n is not None else 0, d_active.data_ptr() if d_active is not None else 0)
                    return None
                d, m = e.step(acts, nact, active)
                return d.copy(), m.copy()
            if k == trace_at and e is x:
                kernels, copies, out = _trace(go, tmp_path)
                traced = (kernels, copies)
            else:
                out = go()
            if dev:
                torch.cuda.synchronize()
                out = (dd.cpu().numpy().copy(), dm.cpu().numpy().copy())
            outs.append(out)
        (d0, m0), (d1, m1) = outs
        _assert_rows(d0, d1, f"decision rows after step {k}", 32)
        _assert_rows(m0, m1, f"metrics rows after step {k}", 32)
        cur = d0
        on = np.ones(B, bool) if active is None else active.astype(bool)
        for r in sample:
            a = None
            if acts is not None:
                a = acts[r, :(1 if nact is None else nact[r])].copy()
            tapes[r].append((bool(reset[r]), bool(on[r]), a, d0[r].copy(), m0[r].copy()))
        if k > max(resets) and active is None and (d0[:, 6] != 0).all():
            break
    return traced, tapes


def _packed_step_batch(target_w, nsm, gpw):
    """B for which the create-time rule picks `target_w` warps per CTA: it halves W while ceil(B / (W * gpw)) < nSM, so W = w
    for w * gpw * (nSM - 1) < B <= 2 * w * gpw * (nSM - 1) below the widest CTA shared memory allows"""
    if target_w == 1:
        return _batch_mod32(1, 2 * gpw * (nsm - 1))
    lo = target_w * gpw * (nsm - 1) + 1
    return _batch_mod32(lo, lo + 64) if target_w == 8 else _batch_mod32(lo, 2 * target_w * gpw * (nsm - 1))


@pytest.mark.parametrize("target_w,path", [(1, "host"), (2, "device"), (4, "host_dma"), (8, "device")])
@pytest.mark.parametrize("topology,multi", [("toy.4p_ssdd_l0.0", False), ("toy.4p_ssdd_l0.8", True)])
def test_step_packed_g8(topology, multi, target_w, path, monkeypatch, tmp_path):
    """the packed per-step kernel (MARO_B200_SPREAD=0: four replicas per warp) at each CTA size the create-time rule picks for
    these blocks; host step() through zero-copy and through bulk DMA copies (MARO_B200_ZEROCOPY=0), and step_device"""
    from oracle.cim_oracle import CimOracle

    nsm, gpw, ticks = _n_sm(), 4, 60
    B = _packed_step_batch(target_w, nsm, gpw)
    topos = _cim_topologies(topology, ticks, multi)
    over = {"MARO_B200_SPREAD": 0, "MARO_B200_SESSION": 0}
    if path == "host_dma":
        over["MARO_B200_ZEROCOPY"] = 0
    x = _cim(monkeypatch, over, topos, B)
    ref = _cim(monkeypatch, SPREAD_REF, topos, B)
    sample = _sample(B, gpw, gpw * min(target_w, 4))
    (kernels, copies), tapes = _step_loop(x, ref, B, path, sample, tmp_path)
    (W, G, general, spread), _, block = _one_launch(kernels, "cim_step_kernel")
    assert (G, general, spread, block) == (8, multi, False, W * 32), (G, general, spread, block)
    if target_w < 8:
        assert W == target_w, (B, W)
    else:  # the widest CTA shared memory allows for these blocks (at least 4 warps), not narrowed for this batch
        assert W in (4, 8) and -(-B // (W * gpw)) >= nsm, (B, W)
    assert not _launches(kernels, "cim_resident_kernel")
    if path == "host_dma":
        assert any("HtoD" in c for c in copies) and any("DtoH" in c for c in copies), copies
    else:
        assert not copies, copies
    for r in sample:
        o = CimOracle(topos[r % len(topos)])
        _replay_steps(o, tapes[r])
        _oracle_final(o, x, r)
    _assert_state(x, ref, gpw, _query_frames(ticks, B), 4, topos[0].n_vessels)
    x.close()
    ref.close()


@pytest.mark.parametrize("lanes", [16, 32])
@pytest.mark.parametrize("topology,multi", [("toy.4p_ssdd_l0.0", False), ("toy.4p_ssdd_l0.8", True)])
def test_step_wide_groups(topology, multi, lanes, monkeypatch, tmp_path):
    """the per-step kernel with 16 and 32 lanes per replica (MARO_B200_LANES; two replicas per warp, and one), not spread"""
    from oracle.cim_oracle import CimOracle

    ticks, B = 60, 293
    gpw = 32 // lanes
    topos = _cim_topologies(topology, ticks, multi)
    x = _cim(monkeypatch, {"MARO_B200_LANES": lanes, "MARO_B200_SPREAD": 0, "MARO_B200_SESSION": 0}, topos, B)
    ref = _cim(monkeypatch, SPREAD_REF, topos, B)
    sample = _sample(B, gpw, gpw)
    (kernels, copies), tapes = _step_loop(x, ref, B, "device", sample, tmp_path)
    (W, G, general, spread), _, block = _one_launch(kernels, "cim_step_kernel")
    assert (G, general, spread, block) == (lanes, multi, False, W * 32)
    for r in sample:
        o = CimOracle(topos[r % len(topos)])
        _replay_steps(o, tapes[r])
        _oracle_final(o, x, r)
    _assert_state(x, ref, gpw, _query_frames(ticks, B), 4, topos[0].n_vessels)
    x.close()
    ref.close()


# ---- CIM resident kernel: fused rollouts -------------------------------------------------------------------------------


def _rollout_vs_steps(x, ref, B, chunks, reset_before, sample, tmp_path, seed=7, base=3):
    """Fused rollouts of the tested handle against one (agent, step) launch pair per env-step on the reference: each launch's
    trace rows up to the replica's DONE / FINISHED row, and the decision / metrics rows it ends with.  Returns the trace of
    the first launch and the per-launch records of the sampled replicas."""
    import torch

    s = torch.cuda.current_stream().cuda_stream
    x.set_stream(s)
    ref.set_stream(s)
    dx = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    mx = torch.zeros((B, 3), dtype=torch.int64, device="cuda")
    dr, mr = torch.zeros_like(dx), torch.zeros_like(mx)
    act = torch.zeros((B, 1, 4), dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(seed)
    records = {r: [] for r in sample}
    traced = None
    L = 0
    while L < len(chunks) or not bool((dx[:, 6] != 0).all()):  # (then more launches of the last size until every episode ended)
        n = chunks[min(L, len(chunks) - 1)]
        assert L < len(chunks) + 50
        reset = np.zeros(B, np.uint8)
        if L in reset_before:
            reset = (rng.random(B) < 0.35).astype(np.uint8)
            x.reset(reset)
            ref.reset(reset)
        trace = torch.full((n, B, 8), -7, dtype=torch.int32, device="cuda")
        launch = lambda: x.rollout_device(dx.data_ptr(), mx.data_ptr(), n, 1, seed, base, trace.data_ptr())  # noqa: E731
        if L == 0:
            traced = _trace(launch, tmp_path)[:2]
        else:
            launch()
        rows, mets = [], []
        for _ in range(n):
            ref.random_policy_device(dr.data_ptr(), act.data_ptr(), seed, base)
            ref.step_device(dr.data_ptr(), mr.data_ptr(), act.data_ptr())
            rows.append(dr.clone())
            mets.append(mr.clone())
        want, wmet = torch.stack(rows), torch.stack(mets)
        stopped = want[:, :, 6] != 0
        first = torch.where(stopped.any(0), stopped.int().argmax(0), torch.full_like(stopped[0], n - 1, dtype=torch.int64))
        upto = torch.arange(n, device="cuda")[:, None] <= first[None, :]
        bad = ((trace != want).any(-1) & upto).any(0)
        if bool(bad.any()):
            r = int(bad.nonzero()[0])
            j = int(((trace[:, r] != want[:, r]).any(-1) & upto[:, r]).nonzero()[0])
            raise AssertionError(f"launch {L} ({n} steps), replica {r}, step {j}: got {trace[j, r].tolist()} want {want[j, r].tolist()}")
        after = trace[:, :, 6][~upto]
        assert bool(((after == 1) | (after == 2)).all()), L
        idx = first.view(1, B, 1)
        end_d = want.gather(0, idx.expand(1, B, 8))[0]
        end_m = wmet.gather(0, idx.expand(1, B, 3))[0]
        live = end_d[:, 6] != 2  # (a replica that started the launch finished answers FINISHED; its metrics words are not compared)
        assert bool((dx[:, 6] == end_d[:, 6]).all()), L
        assert bool((dx[live] == end_d[live]).all()) and bool((mx[live] == end_m[live]).all()), L
        t, d, m = trace.cpu().numpy(), dx.cpu().numpy(), mx.cpu().numpy()
        for r in sample:
            records[r].append((bool(reset[r]), t[:, r].copy(), d[r].copy(), m[r].copy()))
        L += 1
    return traced, records


def _res_expect(kernels, B, G, spread, W=None):
    """the one resident launch of a trace: its template arguments, after checking the grid and block against the replica layout
    (one replica per warp when spread, 32 / G per warp when packed)"""
    targs, grid, block = _one_launch(kernels, "cim_resident_kernel")
    w = block // 32
    if W is not None:
        assert w == W, (w, W)
    gpw = 1 if spread else 32 // G
    assert targs[0] == G and grid == -(-B // (w * gpw)), (targs, grid, block, B)
    return targs


ROLLOUT_CASES = [
    # id, topology, multi-seed, overrides, (G, kGeneral, kMinBlocks, kSmall), warps per CTA
    ("packed-general", "toy.4p_ssdd_l0.8", True, {"MARO_B200_RES_SPREAD": 0}, (8, True, 1, False), 8),
    ("packed-small-4p", "toy.4p_ssdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1}, (8, False, 1, True), 8),
    ("packed-small-5p", "toy.5p_ssddd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1}, (8, False, 1, True), 8),
    ("packed-small-6p", "toy.6p_sssbdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1}, (8, False, 1, True), 8),
    ("register-capped", "toy.4p_ssdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_DENSE": 1}, (8, False, 3, False), 8),
    ("g16-small-4p", "toy.4p_ssdd_l0.0", False, {"MARO_B200_LANES": 16, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1},
     (16, False, 1, True), 8),
    ("g16-4p", "toy.4p_ssdd_l0.0", False, {"MARO_B200_LANES": 16, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0},
     (16, False, 1, False), 8),
    ("g16-small-6p", "toy.6p_sssbdd_l0.0", False, {"MARO_B200_LANES": 16, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1},
     (16, False, 1, True), 8),
    ("g16-6p", "toy.6p_sssbdd_l0.0", False, {"MARO_B200_LANES": 16, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0},
     (16, False, 1, False), 8),
    ("g32-small-sliced-4p", "toy.4p_ssdd_l0.0", False,
     {"MARO_B200_LANES": 32, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 1, "MARO_B200_RES_SLICE_STEPS": 3}, (32, False, 1, True), 8),
    ("g32-sliced-6p", "toy.6p_sssbdd_l0.0", False,
     {"MARO_B200_LANES": 32, "MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0, "MARO_B200_RES_SLICE_STEPS": 3}, (32, False, 1, False), 8),
    ("res-warps-1", "toy.4p_ssdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0, "MARO_B200_RES_WARPS": 1},
     (8, False, 1, False), 1),
    ("res-warps-2", "toy.4p_ssdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0, "MARO_B200_RES_WARPS": 2},
     (8, False, 1, False), 2),
    ("roll-warps-1", "toy.4p_ssdd_l0.0", False, {"MARO_B200_RES_SPREAD": 0, "MARO_B200_RES_SMALL": 0, "MARO_B200_ROLL_WARPS": 1},
     (8, False, 1, False), 1),
]


@pytest.mark.parametrize("case", ROLLOUT_CASES, ids=[c[0] for c in ROLLOUT_CASES])
def test_rollout_shapes(case, monkeypatch, tmp_path):
    """fused rollouts (uneven chunks: single steps, launches that end mid-tick and ones that cross an episode end, masked resets
    between launches) on each resident instantiation and CTA size"""
    from oracle.cim_oracle import CimOracle

    _, topology, multi, over, expect, W = case
    ticks, B = 60, 357
    G = expect[0]
    gpw = 32 // G
    topos = _cim_topologies(topology, ticks, multi)
    x = _cim(monkeypatch, over, topos, B)
    ref = _cim(monkeypatch, SPREAD_REF, topos, B)
    sample = _sample(B, gpw, gpw * W)
    (kernels, _), records = _rollout_vs_steps(x, ref, B, [1, 2, 7, 1, 13, 40, 3, 1000], {3, 5}, sample, tmp_path)
    assert _res_expect(kernels, B, G, False, W) == expect
    for r in sample:
        o = CimOracle(topos[r % len(topos)])
        _replay_rollouts(o, records[r], r, 7, 3)
        _oracle_final(o, x, r)
    _assert_state(x, ref, gpw, _query_frames(ticks, B), topos[0].n_ports, topos[0].n_vessels)
    x.close()
    ref.close()


# ---- CIM resident kernel: host session ---------------------------------------------------------------------------------


@pytest.mark.parametrize("topology,multi", [("toy.4p_ssdd_l0.0", False), ("toy.4p_ssdd_l0.8", True)])
def test_session_packed(topology, multi, monkeypatch, tmp_path):
    """maro_cim_step through the packed resident session (MARO_B200_RES_SPREAD=0) against the spread per-step handle: action
    lists, None actions, subset stepping, masked resets that ride on the next command row, inspection mid-session"""
    from oracle.cim_oracle import CimOracle

    ticks, B = 60, 101
    topos = _cim_topologies(topology, ticks, multi)
    x = _cim(monkeypatch, {"MARO_B200_RES_SPREAD": 0}, topos, B, max_actions=2)
    ref = _cim(monkeypatch, SPREAD_REF, topos, B, max_actions=2)
    assert x.pinned_granularity() == 32 and ref.pinned_granularity() == 0  # (a session of 8-warp CTAs, 4 replicas per warp)
    sample = _sample(B, 4, 32)
    _, tapes = _step_loop(x, ref, B, "host", sample, tmp_path, max_actions=2, lists=True, trace_at=None)
    # (a device synchronise would wait for the live session kernel: reading the ticks ends the session first, and inside the
    # trace, after the step that relaunches it)
    x.ticks()
    k2, _, _ = _trace(lambda: (x.step(None), x.ticks()), tmp_path)
    targs = _res_expect(k2, B, 8, False, 8)
    assert targs[:3] == (8, multi, 1) and not _launches(k2, "cim_step_kernel"), targs
    ref.step(None)
    for r in sample:
        o = CimOracle(topos[r % len(topos)])
        _replay_steps(o, tapes[r])
        o.step(None)
        _oracle_final(o, x, r)
    _assert_state(x, ref, 4, _query_frames(ticks, B), topos[0].n_ports, topos[0].n_vessels)
    x.close()
    ref.close()


# ---- CIM at the sizes the benchmark runs, no overrides -------------------------------------------------------------------


@pytest.mark.parametrize("B", [8192, 65536])
def test_natural_cim_shapes(B, monkeypatch, tmp_path, capsys):
    """toy.4p_ssdd_l0.0 at 8 192 and 65 536 replicas with the shapes create picks on this device: packed resident lane groups
    (spread only while B <= 32 * nSM), the register-capped instantiation once the packed grid is more than 5 * nSM CTAs deep;
    at 65 536 the host step() is the packed per-step kernel behind bulk copies"""
    import torch

    from oracle.cim_oracle import CimOracle

    nsm, ticks, ms = _n_sm(), 150, 16
    topos = _cim_topologies("toy.4p_ssdd_l0.0", ticks, False)
    x = _cim(monkeypatch, {}, topos, B, max_snapshots=ms)
    ref = _cim(monkeypatch, SPREAD_REF, topos, B, max_snapshots=ms)
    spread = B <= 32 * nsm
    dense = not spread and -(-B // 32) > 5 * nsm
    assert not spread
    sample = _sample(B, 4, 32)
    (kernels, _), records = _rollout_vs_steps(x, ref, B, [1, 7, 30, 64], {3}, sample, tmp_path)
    targs = _res_expect(kernels, B, 8, spread, 8)
    if dense:
        assert targs == (8, False, 3, False), targs
    else:
        assert targs[:3] == (8, False, 1), targs
    with capsys.disabled():
        print(f"\n[B={B}, {nsm} SMs] resident rollout: cim_resident_kernel<{', '.join(str(a).lower() for a in targs)}>")
    for r in sample:
        o = CimOracle(topos[0], max_snapshots=ms)
        _replay_rollouts(o, records[r], r, 7, 3)
        _oracle_final(o, x, r)
    frames = np.arange(ticks - ms, ticks, 5, dtype=np.int32)
    _assert_state(x, ref, 4, frames, 4, topos[0].n_vessels)
    if B > 16384:  # a short stretch of host step(): no session (the grid is not resident at once), bulk copies
        x.reset()
        ref.reset()
        d_rows = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
        d_act = torch.zeros((B, 1, 4), dtype=torch.int32, device="cuda")
        cur = None
        for k in range(12):
            acts = None
            if k:
                d_rows.copy_(torch.from_numpy(cur))
                ref.random_policy_device(d_rows.data_ptr(), d_act.data_ptr(), 9, 0)
                acts = d_act.cpu().numpy()
            active = None if k % 2 == 0 else (np.arange(B) % 3 != k % 3).astype(np.uint8)
            if k == 1:
                k1, copies, (d0, m0) = _trace(lambda: tuple(a.copy() for a in x.step(acts, None, active)), tmp_path)
                (W, G, general, sp), _, block = _one_launch(k1, "cim_step_kernel")
                assert (G, general, sp, block) == (8, False, False, W * 32) and -(-B // (W * 4)) >= nsm
                assert not _launches(k1, "cim_resident_kernel")
                assert any("HtoD" in c for c in copies) and any("DtoH" in c for c in copies), copies
            else:
                d0, m0 = (a.copy() for a in x.step(acts, None, active))
            d1, m1 = ref.step(acts, None, active)
            _assert_rows(d0, d1, f"host step {k}", 4)
            _assert_rows(m0, m1, f"host step {k} metrics", 4)
            cur = d0
        _assert_rows(x.counters(), ref.counters(), "counters", 4)
    x.close()
    ref.close()


# ---- citi_bike ---------------------------------------------------------------------------------------------------------


def _bike_setup(B, durations, monkeypatch, overrides):
    from bike_helpers import BIKE_CASES, bike_config
    from maro_b200.batch import BikeBatch
    from maro_b200.scenarios.citi_bike.data import build_bike_topology

    conf = bike_config(BIKE_CASES["toy_1440_greedy_res10"]["data"])
    topo = build_bike_topology(conf, 0, durations, transfer_seed=77)
    seeds = (1000 + 7 * np.arange(B)).astype(np.uint32)
    envs = []
    for over in (overrides, {"MARO_B200_SPREAD": 1}):
        e = _make(BikeBatch, monkeypatch, over, topo, B, 10)
        e.set_transfer_seeds(seeds)
        e.reset()
        envs.append(e)
    make_topo = lambda r: build_bike_topology(conf, 0, durations, transfer_seed=int(seeds[r]))  # noqa: E731
    return envs, topo, make_topo


def _bike_kernel(kernels):
    got = {l[0] for l in _launches(kernels, "bike_step_kernel")}
    assert len(got) == 1, got
    return got.pop()


def _bike_rollouts(x, ref, B, chunks, tmp_path):
    """fused rollouts (greedy agent on the device) of both handles, compared after every launch"""
    import torch

    bufs = [(torch.zeros((B, x.dec_words), dtype=torch.int32, device="cuda"), torch.zeros((B, 3), dtype=torch.int64, device="cuda"))
            for _ in range(2)]
    for e in (x, ref):
        e.set_stream(torch.cuda.current_stream().cuda_stream)
    traced = None
    for L, n in enumerate(chunks):
        for e, (d, m) in zip((x, ref), bufs):
            if L == 0 and e is x:
                traced = _trace(lambda: e.rollout_device(d.data_ptr(), m.data_ptr(), n), tmp_path)[0]
            else:
                e.rollout_device(d.data_ptr(), m.data_ptr(), n)
        torch.cuda.synchronize()
        (d0, m0), (d1, m1) = bufs
        _assert_rows(d0.cpu().numpy(), d1.cpu().numpy(), f"rollout {L} decision rows", 32)
        _assert_rows(m0.cpu().numpy(), m1.cpu().numpy(), f"rollout {L} metrics rows", 32)
        _assert_rows(x.ticks().reshape(-1, 1), ref.ticks().reshape(-1, 1), f"rollout {L} ticks", 32)
        if bool((d0[:, 6] != 0).all()):  # (every replica holds its DONE row and final metrics; a further launch answers FINISHED)
            break
    assert bool((bufs[0][0][:, 6] == 1).all())
    return traced, bufs[0][1].cpu().numpy()


def _bike_state(x, ref, samples, gpw):
    _assert_rows(x.counters(), ref.counters(), "counters", gpw)
    B = x.n_replicas
    _assert_rows(np.stack([x.read_frame(i) for i in range(B)]), np.stack([ref.read_frame(i) for i in range(B)]), "frames", gpw)
    S = x.topology.n_stations
    frames = np.unique(np.linspace(0, x.ring_rows() - 1, max(4, min(x.ring_rows(), 100000 // B))).astype(np.int32))
    attrs = ["bikes", "shortage", "trip_requirement", "fulfillment", "extra_cost", "transfer_cost", "failed_return"]
    _assert_rows(x.query("stations", frames, np.arange(S), attrs), ref.query("stations", frames, np.arange(S), attrs), "ring rows", gpw)


def test_bike_packed(monkeypatch, tmp_path):
    """citi_bike's packed per-step kernel (MARO_B200_SPREAD=0) with per-replica transfer seeds and subset stepping, and its
    fused rollouts, against the spread kernel and per-seed oracles"""
    import torch

    from oracle.bike_oracle import BikeOracle

    B, durations = 229, 400
    (x, ref), topo, make_topo = _bike_setup(B, durations, monkeypatch, {"MARO_B200_SPREAD": 0})
    S = topo.n_stations
    G = 8 if S <= 8 else (16 if S <= 16 else 32)
    gpw = 32 // G
    assert gpw > 1, "the toy trace needs a sub-warp lane group for a packed shape"
    sample = _sample(B, gpw, gpw * 2)
    s = torch.cuda.current_stream().cuda_stream
    x.set_stream(s)
    ref.set_stream(s)
    bufs = [(torch.zeros((B, x.dec_words), dtype=torch.int32, device="cuda"), torch.zeros((B, 3), dtype=torch.int64, device="cuda"))
            for _ in range(2)]
    act = torch.zeros((B, 1, 4), dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(2)
    tapes = {r: [] for r in sample}
    names = {}
    for k in range(100000):
        active = None if k % 3 == 0 else (rng.random(B) < 0.7).astype(np.uint8)
        d_active = torch.from_numpy(active).cuda() if active is not None else None
        if k:
            x.greedy_policy_device(bufs[0][0].data_ptr(), act.data_ptr())
        for e, (d, m) in zip((x, ref), bufs):
            go = lambda e=e, d=d, m=m: e.step_device(d.data_ptr(), m.data_ptr(), act.data_ptr() if k else 0, 0,  # noqa: E731
                                                     d_active.data_ptr() if d_active is not None else 0)
            if k == 0:
                names[e is x] = _bike_kernel(_trace(go, tmp_path)[0])
            else:
                go()
        torch.cuda.synchronize()
        (d0, m0), (d1, m1) = ((d.cpu().numpy(), m.cpu().numpy()) for d, m in bufs)
        _assert_rows(d0, d1, f"decision rows after step {k}", gpw)
        _assert_rows(m0, m1, f"metrics rows after step {k}", gpw)
        a = act.cpu().numpy()
        on = np.ones(B, bool) if active is None else active.astype(bool)
        for r in sample:
            tapes[r].append((False, bool(on[r]), a[r].copy() if k else None, d0[r].copy(), m0[r].copy()))
        if active is None and (d0[:, 6] != 0).all():
            break
    assert names[True][1:] == (G, False) and names[False] == (4, G, True), names
    for r in sample:
        o = BikeOracle(make_topo(r), 10)
        for k, (_, on, a, dec, met) in enumerate(tapes[r]):
            if on:
                st, d, m = o.step(a)
                assert d.tolist() == dec.tolist() and (st == 2 or m.tolist() == met.tolist()), (r, k)
        assert np.array_equal(x.read_frame(r), o.frame()) and x.counters()[r].tolist() == o.counters().tolist(), r
    _bike_state(x, ref, sample, gpw)
    # fused rollouts of a second episode
    x.reset()
    ref.reset()
    before = x.counters()
    kernels, met = _bike_rollouts(x, ref, B, [1, 5, 37, 1000, 3000], tmp_path)
    assert _bike_kernel(kernels)[1:] == (G, False)
    for r in sample:
        o = BikeOracle(make_topo(r), 10)
        _, om = o.run_episode(1)
        assert om.tolist() == met[r].tolist() and np.array_equal(x.read_frame(r), o.frame()), r
        assert (x.counters()[r] - before[r]).tolist() == o.counters().tolist(), r
    _bike_state(x, ref, sample, gpw)
    x.close()
    ref.close()


def test_natural_bike_shape(monkeypatch, tmp_path, capsys):
    """citi_bike just past the spread threshold (B = 128 * nSM + 7, no overrides): packed; fused rollouts against the forced
    spread handle and per-seed oracles"""
    from oracle.bike_oracle import BikeOracle

    nsm = _n_sm()
    B = 128 * nsm + 7
    (x, ref), topo, make_topo = _bike_setup(B, 300, monkeypatch, {})
    S = topo.n_stations
    G = 8 if S <= 8 else (16 if S <= 16 else 32)
    gpw = 32 // G
    kernels, met = _bike_rollouts(x, ref, B, [1, 64, 5000], tmp_path)
    W, g, spread = _bike_kernel(kernels)
    assert (g, spread) == (G, False), (W, g, spread)
    with capsys.disabled():
        print(f"\n[B={B}, {nsm} SMs] citi_bike: bike_step_kernel<{W}, {g}, false>")
    sample = _sample(B, gpw, gpw * W)
    for r in sample:
        o = BikeOracle(make_topo(r), 10)
        _, om = o.run_episode(1)
        assert om.tolist() == met[r].tolist() and np.array_equal(x.read_frame(r), o.frame()), r
        assert x.counters()[r].tolist() == o.counters().tolist(), r
    _bike_state(x, ref, sample, gpw)
    x.close()
    ref.close()

"""Shared helpers for the vm_scheduling tests."""
import importlib.util
import os

import numpy as np

from maro_b200 import _abi
from maro_b200.scenarios.vm_scheduling.data import build_vm_topology

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

_spec = importlib.util.spec_from_file_location("gen_vm_golden", os.path.join(GOLDEN, "gen_vm_golden.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
VM_CASES = gen.CASES


def vm_topology(spec):
    st = spec.get("start_tick", 0)
    return build_vm_topology(dict(spec["conf"]), st, st + spec["durations"])


def load_vm_golden(name):
    return np.load(os.path.join(GOLDEN, f"vm_{name}.npz"))


def metrics_vector(met_row):
    """int64[16] metrics row -> the 14 numbers of the golden files (floats decoded)."""
    d = _abi.vm_metrics_dict(met_row)
    return np.asarray([d[k] for k in gen.METRICS] + [d["latency_due_to_agent"], d["latency_due_to_resource"],
                                                      d["total_oversubscriptions"], d["total_overload_pms"],
                                                      d["total_overload_vms"]], np.float64)


def drive_vm(step_fn, gold, n_pm):
    """Replays the recorded action tape.  step_fn(actions or None) -> (status, dec row, metrics row)."""
    rows, valid, mets = [], [], []
    st, dec, met = step_fn(None)
    k = 0
    while st == 0:
        rows.append([dec[0], dec[1], dec[2], dec[3], dec[4], dec[5], dec[8], dec[9], dec[10]])
        v = np.full(n_pm, -1, np.int32)
        v[:dec[10]] = dec[12:12 + dec[10]]
        valid.append(v)
        mets.append(metrics_vector(met))
        a = gold["actions"][k]
        k += 1
        st, dec, met = step_fn(None if a[1] < 0 else a.reshape(1, 4))
    return (np.asarray(rows, np.int64).reshape(-1, 9), np.asarray(valid, np.int32).reshape(-1, n_pm),
            np.asarray(mets, np.float64).reshape(-1, 14), metrics_vector(met), st, dec)


def assert_metrics_close(got, want, what=""):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    if (err > 1e-9).any():
        bad = np.argwhere(err > 1e-9)[0]
        raise AssertionError(f"{what} metrics differ at {bad.tolist()}: got {got[tuple(bad)]!r} want {want[tuple(bad)]!r}")


def vm_named_frames(words_by_frame, topo):
    lay, fw = _abi.vm_frame_layout(topo)
    w = np.asarray(words_by_frame, np.int32)
    out = {}
    for node, attrs in lay.items():
        for a, (off, n, _) in attrs.items():
            x = w[:, off:off + n]
            out[f"{node}/{a}"] = x.view(np.float32) if a in _abi.VM_FLOAT_ATTRS else x
    return out


def assert_vm_snapshots_equal(get_snapshot, gold, topo):
    frames = gold["frames"].tolist()
    rows = []
    for f in frames:
        s = get_snapshot(int(f))
        assert s is not None, f"frame {f} missing"
        rows.append(s)
    named = vm_named_frames(rows, topo)
    for key, val in named.items():
        g = gold[key]
        if val.dtype == np.float32:
            ok = np.allclose(val, g, rtol=1e-6, atol=1e-7)
        else:
            ok = np.array_equal(val, g)
        if not ok:
            bad = np.argwhere(val != g)[0]
            raise AssertionError(f"{key} differs first at {bad.tolist()} (frame {frames[bad[0]]}): got {val[tuple(bad)]} want {g[tuple(bad)]}")


# ---- replica classes: diverging replicas that can still be checked batch-wide ----------------------------------------
# Replica r belongs to class r % P.  The agent, the active mask and the reset schedule are functions of (class, step)
# only, so every member of a class must produce its representative's rows bit for bit (the representative of class c is
# replica c), and each representative must follow its own oracle.  With P coprime to the warp and CTA sizes, the members
# of a class sit in different warps, CTAs and grid-stride passes, and neighbours in a warp belong to different classes.

EXACT_WORDS = [0, 2, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15]  # every metrics word except total_incomes (1), total_profit (3)
FLOAT_WORDS = [1, 3]
BAD_VM_ID = -7  # no VM has this id: an action naming it names the wrong VM
MARO_VM_DEC_VM_ID, MARO_VM_DEC_STATUS, MARO_VM_DEC_N_VALID, MARO_VM_DEC_EXT, MARO_VM_DEC_HEAD = 1, 6, 10, 11, 12  # decision row words (maro_b200.h)


def class_hash(c, k):
    """32-bit mix of (class, ordinal), vectorised"""
    u = np.uint64
    h = (np.asarray(c, u) * u(0x9E3779B1) + np.asarray(k, u) * u(0x85EBCA77) + u(0x165667B1)) & u(0xFFFFFFFF)
    h ^= h >> u(15)
    h = (h * u(0x2C1B3C6D)) & u(0xFFFFFFFF)
    h ^= h >> u(12)
    return h


def class_agent(dec, c, k, n_pm, bad=None):
    """actions [P][4] and n_actions [P] of the representatives' decision rows `dec`, class ids `c`, decision ordinals `k`:
    a hashed valid PM, best fit from the remaining-cores extension, a postponement by 1 or 2 steps, or an empty action
    list; `bad` = (class, ordinal) answers that one decision with a VM id no VM has"""
    P = len(c)
    h = class_hash(c, k)
    kind = (h % np.uint64(8)).astype(np.int64)
    n = dec[:, MARO_VM_DEC_N_VALID].astype(np.int64)
    live = dec[:, MARO_VM_DEC_STATUS] == 0
    rows = np.arange(P)
    pick = dec[rows, MARO_VM_DEC_HEAD + ((h >> np.uint64(8)) % np.maximum(n, 1).astype(np.uint64)).astype(np.int64)]
    rem = dec[:, MARO_VM_DEC_HEAD + n_pm:MARO_VM_DEC_HEAD + 2 * n_pm].astype(np.int64)
    rem = np.where(np.arange(n_pm)[None, :] < n[:, None], rem, np.iinfo(np.int64).max)
    best = dec[rows, MARO_VM_DEC_HEAD + np.argmin(rem, axis=1)]
    act = np.zeros((P, 4), np.int32)
    act[:, 0] = dec[:, MARO_VM_DEC_VM_ID]
    act[:, 2] = np.where((kind == 3) | (kind == 4), best, pick)
    post = kind == 5
    act[post, 1] = 1
    act[post, 2] = 1 + ((h[post] >> np.uint64(4)) % np.uint64(2)).astype(np.int32)
    nact = np.where(kind == 6, 0, 1).astype(np.int32)
    if bad is not None:
        hit = (c == bad[0]) & (k == bad[1]) & live
        act[hit] = [BAD_VM_ID, 0, 0, 0]
        nact[hit] = 1
    act[~live] = [-1, -1, 0, 0]
    nact[~live] = 0
    return act, nact


class VmClasses:
    """Lockstep driver of a vm_scheduling batch (the CUDA handle or the emulator-backed one) against one VmOracle per class."""

    def __init__(self, env, topo, P, res=1, max_snapshots=None, bad=None):
        from oracle.vm_oracle import VmOracle

        self.env, self.topo, self.P, self.B, self.N = env, topo, P, env.n_replicas, topo.n_pm
        self.res, self.max_snapshots = res, max_snapshots
        self.cls = np.arange(self.B) % P
        self.c = np.arange(P)
        self.oracles = [VmOracle(topo, res, max_snapshots) for _ in range(P)]
        self.k = np.zeros(P, np.int64)  # decisions each class has answered
        self.last = np.zeros((P, env.dec_words), np.int32)  # last non-INACTIVE representative rows
        self.last_met = np.zeros((P, 16), np.int64)
        self.bad = bad
        self.bad_seen = False
        self.uncounted = np.zeros((P, 4), np.int64)  # oracle counters of steps the device does not count (BAD_ACTION)
        lay, _ = _abi.vm_frame_layout(topo)
        self.pm_off = {a: v[0] for a, v in lay["pms"].items()}

    # -- one step -------------------------------------------------------------------------------------------------------
    def inputs(self, step, active_every=5):
        """(actions [B][A][4], n_actions [B], active [B] u8, per-class (act, nact, active))"""
        act, nact = class_agent(self.last, self.c, self.k, self.N, self.bad)
        on = (class_hash(self.c, step + 100000) % np.uint64(active_every)) != 0
        acts = np.zeros((self.B, self.env.max_actions, 4), np.int32)
        acts[:, 0] = act[self.cls]
        return acts, nact[self.cls], on[self.cls].astype(np.uint8), (act, nact, on)

    def oracle_step(self, per_class):
        act, nact, on = per_class
        outs = {}
        for c in np.flatnonzero(on):
            o = self.oracles[c]
            was_decision = self.last[c, MARO_VM_DEC_STATUS] == 0
            hit_bad = self.bad is not None and c == self.bad[0] and was_decision and nact[c] and act[c, 0] == BAD_VM_ID
            before = o.counters()
            outs[c] = o.step(act[c] if nact[c] else None)
            if hit_bad:
                assert outs[c][0] == -1, outs[c][0]
                self.uncounted[c] += o.counters() - before
                self.bad_seen = True
            if was_decision:
                self.k[c] += 1
        return outs

    def check(self, dec, met, on, outs, what=""):
        """batch-wide: every active replica equals its representative; inactive replicas answer INACTIVE; every active
        representative equals its oracle"""
        live = on[self.cls]
        reps = self.cls[live]
        if not np.array_equal(dec[live], dec[reps]) or not np.array_equal(met[live], met[reps]):
            bad = np.flatnonzero(live)[np.flatnonzero((dec[live] != dec[reps]).any(1) | (met[live] != met[reps]).any(1))[0]]
            raise AssertionError(f"{what}: replica {bad} (class {self.cls[bad]}) differs from its representative")
        assert (dec[~live, MARO_VM_DEC_STATUS] == 3).all(), what
        for c, (st, od, om) in outs.items():
            self.compare(c, dec[c], met[c], st, od, om, f"{what} class {c}")
            self.last[c], self.last_met[c] = dec[c], met[c]

    def compare(self, c, d, m, st, od, om, what):
        """header, valid PM ids and remaining-cores extension of a decision row (word 11, the extension's offset, is not
        part of the oracle's rows); whole rows otherwise; metrics exact but for the two float64 sums"""
        assert d[MARO_VM_DEC_STATUS] == st, (what, d[MARO_VM_DEC_STATUS], st)
        if st == 0:
            n = int(od[MARO_VM_DEC_N_VALID])
            assert d[:11].tolist() == od[:11].tolist(), (what, d[:11], od[:11])
            ids = od[MARO_VM_DEC_HEAD:MARO_VM_DEC_HEAD + n]
            assert d[MARO_VM_DEC_HEAD:MARO_VM_DEC_HEAD + n].tolist() == ids.tolist(), what
            ext = int(d[MARO_VM_DEC_EXT])
            assert ext == MARO_VM_DEC_HEAD + self.N, what
            f = self.oracles[c].frame()
            want = f[self.pm_off["cpu_cores_capacity"] + ids] - f[self.pm_off["cpu_cores_allocated"] + ids]
            assert d[ext:ext + n].tolist() == want.tolist(), (what, d[ext:ext + n], want)
        else:
            assert d[:len(od)].tolist() == od.tolist(), (what, d[:12], od[:12])
        if st == -1:
            return  # (the device also reports the metrics at a BAD_ACTION row; the oracle leaves them zero)
        assert np.array_equal(m[EXACT_WORDS], om[EXACT_WORDS]), (what, m, om)
        fm, fo = m[FLOAT_WORDS].view(np.float64), om[FLOAT_WORDS].view(np.float64)
        assert (np.abs(fm - fo) <= 1e-9 * np.maximum(1.0, np.abs(fo))).all(), (what, fm, fo)

    # -- resets, host stepping, fused rollouts ----------------------------------------------------------------------------
    def reset(self, classes):
        """masked reset of every member of `classes` (bool [P]) on the batch and on their oracles; the counters stay"""
        self.env.reset(classes[self.cls].astype(np.uint8))
        for c in np.flatnonzero(classes):
            self.oracles[c].reset()
        self.last[classes] = 0  # (a fresh episode ignores actions: the agent sends none)
        self.last[classes, MARO_VM_DEC_STATUS] = 2

    def first_step(self):
        dec, met = self.env.step(None)
        outs = {c: o.step(None) for c, o in enumerate(self.oracles)}
        self.check(dec, met, np.ones(self.P, bool), outs, "first step")

    def host_steps(self, steps, first_step_index, reset_at=None):
        """`steps` host step() calls with actions / n_actions / active; reset_at: {step index: classes to reset first}"""
        for i in range(first_step_index, first_step_index + steps):
            if reset_at and i in reset_at:
                self.reset(reset_at[i])
            acts, nact, active, per_class = self.inputs(i)
            dec, met = self.env.step(acts, nact, active)
            self.check(dec, met, per_class[2], self.oracle_step(per_class), f"host step {i}")

    def rollout_model(self, n_steps):
        """what one fused launch of `n_steps` does to every class: best fit while the row is a decision, stop at the first
        row that is not"""
        outs = {}
        for c, o in enumerate(self.oracles):
            row = self.last[c]
            for _ in range(n_steps):
                st, od, om = o.step(o.best_fit(row).reshape(1, 4) if row[MARO_VM_DEC_STATUS] == 0 else None)
                outs[c] = (st, od, om)
                row = od
                if st != 0:
                    break
        return outs

    # -- end state ----------------------------------------------------------------------------------------------------------
    def held_frames(self, c):
        o = self.oracles[c]
        total = -(-(self.topo.max_tick - self.topo.start_tick) // self.res)
        return [f for f in range(total) if o.snapshot(f) is not None]

    def check_end(self, with_counters=True):
        env = self.env
        members = self.c + self.P * ((self.B - 1 - self.c) // self.P)  # the last member of every class
        for c in range(self.P):
            assert np.array_equal(env.read_frame(int(members[c])), self.oracles[c].frame()), f"frame of class {c}"
            held = self.held_frames(c)
            assert env.snapshot_frames(c).tolist() == held, (c, env.snapshot_frames(c), held)
            assert env.snapshot_frames(int(members[c])).tolist() == held, c
        if with_counters:
            want = np.stack([o.counters() for o in self.oracles]) - self.uncounted
            got = env.counters()
            assert np.array_equal(got, want[self.cls]), (np.argwhere(got != want[self.cls])[:4], got[:4], want[:4])
        # one batched query over every representative x every frame any of them holds x all PMs x all 14 attributes
        frames = sorted(set(f for c in range(self.P) for f in self.held_frames(c)))
        attrs = list(_abi.VM_NODE_ATTRS["pms"])
        q = env.query("pms", frames, np.arange(self.N), attrs, self.c).reshape(self.P, len(frames), self.N, len(attrs))
        want = np.zeros(q.shape, np.float64)
        for c in range(self.P):
            for fi, f in enumerate(frames):
                row = self.oracles[c].snapshot(f)
                if row is None:
                    continue
                for ai, a in enumerate(attrs):
                    w = row[self.pm_off[a]:self.pm_off[a] + self.N]
                    want[c, fi, :, ai] = w.view(np.float32) if a in _abi.VM_FLOAT_ATTRS else w
        isf = np.asarray([a in _abi.VM_FLOAT_ATTRS for a in attrs])
        assert np.array_equal(q[..., ~isf], want[..., ~isf]), np.argwhere(q[..., ~isf] != want[..., ~isf])[:4]
        assert np.allclose(q[..., isf], want[..., isf], rtol=1e-6, atol=1e-7)
        for c in range(self.P):  # the float64 lift indexes the replicas of a batched query like a query of one replica
            one = env.query("pms", frames, np.arange(self.N), attrs, [c]).reshape(q.shape[1:])
            assert np.array_equal(one, q[c]), f"batched query row of class {c} differs from its own query"

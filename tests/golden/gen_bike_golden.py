"""Generate golden citi_bike traces from the UNMODIFIED reference (oracle/_ref).

    bash oracle/build_ref.sh && python tests/golden/gen_bike_golden.py

Datasets: the frozen toy.3s_4t slice in tests/golden/bike_toy (generated once by the reference's own toy pipeline — its
trip generator is unseeded, hence frozen) and the reference's own test fixtures tests/data/citi_bike/case_{1,2}
(converted to .bin with the reference's BinaryConverter into tests/golden/bike_case_{1,2}).  The agent reads
``decision_event.action_scope`` at every decision (lazy in the reference) and plays either the null policy or the greedy
top-1 policy of examples/citi_bike/greedy/launcher.py; ``np.random.seed`` pins the transfer-time stream.
Output: tests/golden/bike_<case>.npz.
"""
import multiprocessing as mp
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = "/root/reference"

TOY_DECISION = """decision:
  extra_cost_mode: source
  resolution: 20
  effective_time_mean: 20
  effective_time_std: 5
  supply_water_mark_ratio: 0.8
  demand_water_mark_ratio: 0.2
  action_scope:
    low: 0
    high: 1
    filters:
      - type: "distance"
        num: 80
      - type: "requirements"
        num: 40
      - type: "trip_window"
        windows: 10
        num: 20
time_zone: "America/New_York"
"""

CASES = {
    "toy_1440_null_res10": dict(data="bike_toy", durations=1440, policy=0, snapshot_resolution=10, np_seed=11),
    "toy_1440_greedy_res10": dict(data="bike_toy", durations=1440, policy=1, snapshot_resolution=10, np_seed=128),
    "toy_600_greedy_res1": dict(data="bike_toy", durations=600, policy=1, snapshot_resolution=1, np_seed=5),
    "toy_2000_greedy_res7_ring12": dict(data="bike_toy", durations=2000, policy=1, snapshot_resolution=7, max_snapshots=12,
                                        np_seed=77),
    # start_tick > 0: mid-day entry into the trace (trip picker skips ahead, day features of the entry day)
    "toy_start700_500_greedy_res5": dict(data="bike_toy", start_tick=700, durations=500, policy=1, snapshot_resolution=5, np_seed=9),
    # found by tools/fuzz_cim_bike_parity.py: this seed draws a transfer time of -2 -> the DeliverBike event is filed under a
    # tick that has already run and never executes (3 bikes vanish), event_buffer.py:166-175
    "toy_start300_773_negative_transfer": dict(data="bike_toy", start_tick=300, durations=773, policy=1, snapshot_resolution=20,
                                               np_seed=41130),
    # 26 synthetic stations (tests/golden/bike_synth_gen.py): every action-scope filter DROPS neighbours (distance 14 ->
    # requirements 9 -> trip_window 5 x 4; decision_strategy.py:15-163).  Snapshot resolution 7 does not divide the decision
    # resolution 20, so the trip-window filter's per-frame cache holds mid-frame values (its staleness is part of the trace)
    "synth26_1440_greedy_res7": dict(data="bike_synth26", durations=1440, policy=1, snapshot_resolution=7, np_seed=3),
    "synth26_900_null_res10_ring3": dict(data="bike_synth26", durations=900, policy=0, snapshot_resolution=10, max_snapshots=3,
                                         np_seed=8),
    "synth26_start400_600_greedy_res1": dict(data="bike_synth26", start_tick=400, durations=600, policy=1, snapshot_resolution=1,
                                             np_seed=21),
    # found by tools/fuzz_cim_bike_parity.py (bike_filter_spec(15)): at tick 144 the action of the tick's LAST decision event draws a
    # transfer time of 0; the reference's event list keeps its tail on the removed decision event (event_linked_list.py:86-92
    # does not update `_tail`), the DeliverBike appended to the running tick is lost and two bikes vanish
    "synth26_lost_same_tick_delivery": dict(
        data="bike_synth26", durations=300, policy=1, snapshot_resolution=7, np_seed=95996,
        decision_text=('decision:\n  extra_cost_mode: target\n  resolution: 5\n  effective_time_mean: 7\n  effective_time_std: 4\n'
                       '  supply_water_mark_ratio: 0.73\n  demand_water_mark_ratio: 0.18\n  action_scope:\n    low: 0.27\n    high: 0.73\n'
                       '    filters:\n      - type: "requirements"\n        num: 3\ntime_zone: "America/New_York"\n')),
    "case1_30_null": dict(data="bike_case_1", durations=30, policy=0, snapshot_resolution=1, np_seed=1),
    "case2_30_greedy": dict(data="bike_case_2", durations=30, policy=1, snapshot_resolution=1, np_seed=2),
}

STATION_ATTRS = ("bikes", "capacity", "extra_cost", "failed_return", "fulfillment", "holiday", "id", "min_bikes",
                 "shortage", "temperature", "transfer_cost", "trip_requirement", "weather", "weekday")


def data_config_dir(name, decision_text=None):
    """tests/golden/<name>/ holds trips.bin, weather bin, station + distance csv and (for the reference's cases) the
    decision config; returns a temp folder with a config.yml of absolute paths."""
    src = os.path.join(HERE, name)
    d = tempfile.mkdtemp()
    if name == "bike_toy":
        body = TOY_DECISION
        files = dict(trip_data="trips.bin", weather_data="KNYC_daily.bin", stations_init_data="station_meta.csv",
                     distance_adj_data="distance_adj.csv")
    else:
        body = decision_text or open(os.path.join(src, "decision.yml")).read()
        files = dict(trip_data="trips.bin", weather_data="weathers.bin", stations_init_data="stations.csv",
                     distance_adj_data="distance_adj.csv")
    with open(os.path.join(d, "config.yml"), "w") as fp:
        fp.write(body)
        for k, v in files.items():
            fp.write(f'{k}: "{os.path.join(src, v)}"\n')
    return d


def greedy(dec_event):
    """examples/citi_bike/greedy/launcher.py:35-65 with top_k = 1."""
    import heapq

    top = []
    for cand, v in dec_event.action_scope.items():
        if cand == dec_event.station_idx:
            continue
        heapq.heappush(top, (v, cand))
        if len(top) > 1:
            heapq.heappop(top)
    v, cand = top[0]
    return v, cand


def prepare_reference_cases():
    """Convert the reference's csv fixtures to .bin once (BinaryConverter), keep them under tests/golden."""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref", "_stubs"))
    os.environ["SKIP_DEPLOYMENT"] = "TRUE"
    import yaml
    from maro.data_lib import BinaryConverter

    base = os.path.join(REF, "tests/data/citi_bike")
    for case in ("case_1", "case_2"):
        dst = os.path.join(HERE, "bike_" + case)
        if os.path.isfile(os.path.join(dst, "trips.bin")):
            continue
        os.makedirs(dst, exist_ok=True)
        conv = BinaryConverter(os.path.join(dst, "trips.bin"), os.path.join(base, "trips.meta.yml"))
        conv.add_csv(os.path.join(base, case, "trips.csv"))
        conv.flush()
        conv = BinaryConverter(os.path.join(dst, "weathers.bin"), os.path.join(base, "weather.meta.yml"))
        conv.add_csv(os.path.join(base, "weather.csv"))
        conv.flush()
        for f in ("stations.csv", "distance_adj.csv"):
            shutil.copy(os.path.join(base, case, f), os.path.join(dst, f))
        with open(os.path.join(base, case, "config.yml")) as fp:
            conf = yaml.safe_load(fp)
        with open(os.path.join(dst, "decision.yml"), "w") as fp:
            yaml.safe_dump({"decision": conf["decision"], "time_zone": conf["time_zone"]}, fp, sort_keys=False)
    # the reference's data_lib test metas (tests/data/data_lib/case_{1,2}/meta.yml, kept as tests/golden/data_lib/trips_tz*.meta.yml)
    # on their trips.csv (= tests/golden/data_lib/trips_case_1.csv): byte-identity cases of tests/test_data_lib.py
    dl = os.path.join(HERE, "data_lib")
    for meta, out in (("trips_tz_events.meta.yml", "trips_case_1_tz_events.bin"), ("trips_tz.meta.yml", "trips_case_1_tz.bin")):
        if not os.path.isfile(os.path.join(dl, out)):
            conv = BinaryConverter(os.path.join(dl, out), os.path.join(dl, meta))
            conv.add_csv(os.path.join(dl, "trips_case_1.csv"))
            conv.flush()
            del conv


def run_case(name, spec, out_dir=None):
    os.environ["SKIP_DEPLOYMENT"] = "TRUE"
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref", "_stubs"))
    from maro.simulator import Env
    from maro.simulator.scenarios.citi_bike.common import Action, DecisionType

    np.random.seed(spec["np_seed"])
    env = Env("citi_bike", data_config_dir(spec["data"], spec.get("decision_text")), start_tick=spec.get("start_tick", 0), durations=spec["durations"],
              snapshot_resolution=spec["snapshot_resolution"], max_snapshots=spec.get("max_snapshots"))
    S = len(env.snapshot_list["stations"])
    rows, scopes = [], []
    metrics, dec, done = env.step(None)
    while not done:
        scope = dec.action_scope  # read at every decision
        rows.append([dec.tick, dec.station_idx, dec.frame_index, 0 if dec.type == DecisionType.Supply else 1, len(scope),
                     int(metrics["trip_requirements"]), int(metrics["bike_shortage"]), int(metrics["operation_number"])])
        sv = np.full(S, -1, np.int64)
        for k, v in scope.items():
            sv[k] = int(v)
        scopes.append(sv)
        if spec["policy"] == 1:
            v, cand = greedy(dec)
            action = Action(dec.station_idx, cand, int(v)) if dec.type == DecisionType.Supply else Action(cand, dec.station_idx, int(v))
        else:
            action = None
        metrics, dec, done = env.step(action)
    sl = env.snapshot_list
    frames = sorted(sl.get_frame_index_list())
    out = {"steps": np.asarray(rows, np.int64).reshape(-1, 8), "scopes": np.asarray(scopes, np.int64).reshape(-1, S),
           "final_metrics": np.asarray([int(metrics["trip_requirements"]), int(metrics["bike_shortage"]),
                                        int(metrics["operation_number"])], np.int64),
           "final_tick": np.asarray(env.tick), "frames": np.asarray(frames, np.int32)}
    for a in STATION_ATTRS:
        out["stations/" + a] = sl["stations"][frames::a].reshape(len(frames), S).astype(np.int32)
    out["matrices/trips_adj"] = sl["matrices"][frames::"trips_adj"].reshape(len(frames), S * S).astype(np.int32)
    np.savez_compressed(os.path.join(out_dir or HERE, f"bike_{name}.npz"), **out)
    print(name, "steps", len(rows), "final", out["final_metrics"].tolist(), "tick", env.tick, flush=True)


if __name__ == "__main__":
    prepare_reference_cases()
    names = sys.argv[1:] or list(CASES)
    ctx = mp.get_context("spawn")
    for n in names:
        p = ctx.Process(target=run_case, args=(n, CASES[n]))
        p.start()
        p.join()
        if p.exitcode != 0:
            raise SystemExit(f"case {n} failed")

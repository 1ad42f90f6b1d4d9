#!/bin/bash
# Round-end measurement session on one H100: default bench line, the north-star matrix, the secondary workloads.
tag=${1:-r2}
mkdir -p gpurun_out
cp maro_b200/libmaro_b200.so gpurun_out/${tag}_lib.so
timeout 900 python bench.py > gpurun_out/${tag}_bench_default.json 2> gpurun_out/${tag}_bench_default.err; echo "default rc=$?"
timeout 600 python bench.py --impl reference --steps 200 --warmup 5 > gpurun_out/${tag}_bench_reference.json 2> gpurun_out/${tag}_bench_reference.err; echo "reference rc=$?"
timeout 1500 python bench.py --matrix --steps 1280 --warmup 20 --cpu-seconds 3 > gpurun_out/${tag}_bench_matrix.json 2> gpurun_out/${tag}_bench_matrix.err; echo "matrix rc=$?"
timeout 600 python bench.py --scenario citi_bike --replicas 4096 --steps 2000 --cpu-seconds 3 > gpurun_out/${tag}_bench_bike_4096.json 2> gpurun_out/${tag}_bench_bike_4096.err; echo "bike rc=$?"
timeout 600 python bench.py --scenario vm_scheduling --replicas 2048 --steps 400 --warmup 5 --cpu-seconds 3 > gpurun_out/${tag}_bench_vm_2048.json 2> gpurun_out/${tag}_bench_vm_2048.err; echo "vm rc=$?"
timeout 600 python bench.py --topology global_trade.22p_l0.8 --ticks 500 --seeds 8 --steps 640 --cpu-seconds 3 > gpurun_out/${tag}_bench_22p_l08_1024env_8seeds.json 2> gpurun_out/${tag}_bench_22p.err; echo "22p rc=$?"
python - <<PY
import json, glob
for f in sorted(glob.glob("gpurun_out/${tag}_bench_*.json")):
    try:
        d = json.load(open(f))
    except Exception as ex:
        print(f, "unreadable", ex); continue
    if "matrix" in d:
        for e in d["matrix"]:
            print("  matrix", e.get("scenario"), e.get("replicas_per_gpu"), "value %.3g" % (e.get("value") or 0), "e2e %.3g" % ((e.get("e2e") or {}).get("value") or 0),
                  "frac %.3f" % ((e.get("roofline") or {}).get("frac") or 0), e.get("error", ""))
    else:
        print(f, "value %.4g" % d.get("value", 0), "e2e %.4g" % ((d.get("e2e") or {}).get("value") or 0), "frac %.3f" % ((d.get("roofline") or {}).get("frac") or 0))
PY

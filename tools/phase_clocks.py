"""Cycles per replica env-step of each phase of the CIM step, measured inside the resident rollout kernel.

    python tools/phase_clocks.py [--topology toy.4p_ssdd_l0.0] [--replicas 1024] [--ticks 1000] [--launches 200] [--chunk 64]

Builds the -DMARO_PHASE_CLOCKS variant of the library with tools/build_variant.py (unless --lib names a built one), runs
fused rollouts with the hashed device agent (the shape bench.py times) and prints, per phase, the clock64() cycles the leader
lane of a replica spent there, divided by the env-steps run.  The marks themselves cost a few cycles each, so the total
is a little above the product build's chain; use the table for where the time goes, bench.py for how much there is."""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["agent", "action apply", "vessel scan", "bucket", "delay line", "orders", "arrivals", "decision snapshot",
          "post-step (acc + snapshot + wait + resets)", "metrics / store"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--topology", default="toy.4p_ssdd_l0.0")
    ap.add_argument("--replicas", type=int, default=1024)
    ap.add_argument("--ticks", type=int, default=1000)
    ap.add_argument("--chunk", type=int, default=64)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--lib", default="", help="an already built -DMARO_PHASE_CLOCKS library")
    args = ap.parse_args()
    lib = args.lib
    if not lib:
        out = subprocess.check_output([sys.executable, os.path.join(ROOT, "tools", "build_variant.py"), "phase",
                                       "-DMARO_PHASE_CLOCKS"], text=True)
        lib = out.strip().splitlines()[-1]
    os.environ["MARO_B200_LIB"] = os.path.abspath(lib)
    sys.path.insert(0, ROOT)
    import torch

    from maro_b200 import _native
    from maro_b200.batch import CimBatch
    from maro_b200.scenarios.cim.topology import build_topology

    L = _native.lib()
    L.maro_cim_phase_clocks.argtypes = [C.c_void_p, C.c_int32]
    slots = (C.c_uint64 * (len(PHASES) + 2))()

    def read(clear):
        _native.check(L.maro_cim_phase_clocks(C.addressof(slots), int(clear)))
        return list(slots)

    B = args.replicas
    env = CimBatch(build_topology(args.topology, args.ticks), B, device=0)
    dec = torch.zeros((B, 8), dtype=torch.int32, device="cuda")
    met = torch.zeros((B, 3), dtype=torch.int64, device="cuda")

    def run(n):
        for _ in range(n):
            if bool((dec[:, 6] != 0).all().item()):
                env.reset()
            env.rollout_device(dec.data_ptr(), met.data_ptr(), args.chunk, 1, 0, 0)

    run(args.warmup)
    read(True)
    run(args.launches)
    acc = read(True)
    env.close()
    steps, ticks = acc[len(PHASES)], acc[len(PHASES) + 1]
    total = sum(acc[:len(PHASES)])
    name = torch.cuda.get_device_name(0)
    print(f"{args.topology}, {B} envs, {args.launches} launches x {args.chunk} env-steps on {name}: "
          f"{steps} replica env-steps, {ticks / max(steps, 1):.2f} ticks per env-step")
    print(f"| phase | cycles / env-step | share |")
    print(f"|---|---:|---:|")
    for p, c in zip(PHASES, acc):
        print(f"| {p} | {c / steps:.0f} | {100.0 * c / total:.1f} % |")
    print(f"| **total** | **{total / steps:.0f}** | |")


if __name__ == "__main__":
    main()

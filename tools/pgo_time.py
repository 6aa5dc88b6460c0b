"""Time optimize::graph_optimizer on the GPU (b200_graph_optimize) against the CPU oracle's single-thread time, on the loop-closure
graphs of workloads/synth.make_pose_graph.  g2o itself is not part of this project and is not timed here.

    python tools/pgo_time.py [--sizes 500 2000 4000] [--runs 2] [--no-oracle]

Per size and run: device time split into linearisation, envelope assembly + factorisation and substitution + trial step; host wall time
of the call; LM iterations and trials; kernel launches; envelope size and the flops of one envelope factorisation."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[500, 2000, 4000])
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    from stella_vslam_b200 import optimize
    from workloads import synth
    try:
        gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        gpu = "unknown"
    print(json.dumps(dict(gpu=gpu)))
    opt = optimize.graph_optimizer()
    opt.optimize(synth.make_pose_graph(100, seed=0))          # warm-up: context, module load, arena
    for n in a.sizes:
        g = synth.make_pose_graph(n, seed=n)
        for run in range(a.runs):
            r = opt.optimize(g)
            row = dict(n_keyframes=n, run=run, edges=len(g["e_v1"]), iterations=r["iterations"], trials=r["trials"], launches=r["launches"],
                       envelope_doubles=r["envelope_doubles"], factor_gflop=r["factor_flops"] / 1e9,
                       lin_ms=round(r["lin_ms"], 3), factor_ms=round(r["factor_ms"], 3), solve_ms=round(r["solve_ms"], 3),
                       device_ms=round(r["lin_ms"] + r["factor_ms"] + r["solve_ms"], 3), wall_ms=round(r["total_ms"], 3),
                       factor_gflops_per_s=round(r["factor_flops"] * r["trials"] / max(r["factor_ms"], 1e-6) / 1e6, 1))
            if run == 0 and not a.no_oracle:
                import pgo_oracle as O
                t = time.perf_counter()
                ref = O.graph_optimize(g)
                row["oracle_ms"] = round(1e3 * (time.perf_counter() - t), 1)
                row["oracle_iterations"] = ref["iterations"]
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()

"""Joint-torque cost (b200sqp_set_joint_torque_cost) on the H100: what the term costs a solve.  One JSON line.

bench.py's whole-body configuration -- N = 100 intervals (3.5 s at dt = 0.035 s), batch 256 of stance / walk / slow_walk instances at random
phases, sqpIteration 1, cold start (b200sqp_reset before every solve) -- solved as bench.py solves it: one handle per node count, every group on
its own CUDA stream from its own host thread.  Two such sets of handles, term off and term on (weights 1e-3 on every joint), are timed
alternately in one process after a warm-up.  Per setting: median and spread of the wall time of one solve of the whole batch (all groups,
ended by a device synchronise), the stage times (b200sqp_get_stage_times: LQ approximation, QP, line search, K1b) summed over the groups, and
the launches summed over the groups.  The card's name and power limit are printed beside the numbers.
"""
import argparse
import json
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from bench import build_batch  # noqa: E402
from wb_humanoid_mpc_b200 import abi, model_loader  # noqa: E402
from wb_humanoid_mpc_b200.solver import B200SqpSolver, stack_instances  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--horizon", type=float, default=3.5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--weight", type=float, default=1e-3)
    args = ap.parse_args()
    import torch

    model = model_loader.load_packaged_model()
    insts = build_batch(model, args.batch, 0, args.horizon, ["stance", "walk", "slow_walk"], random_phase=True)
    by_n = {}
    for i in insts:
        by_n.setdefault(len(i["t_nodes"]), []).append(i)
    st = abi.default_settings(model, sqp_iteration=1)
    settings = {}
    for name, w in (("off", None), ("on", np.full(model["nj"], args.weight))):
        groups = []
        for n, gi in sorted(by_n.items()):
            s = B200SqpSolver(model, st)
            s.set_joint_torque_cost(w)
            s.upload(stack_instances(gi))
            groups.append((s, torch.cuda.Stream()))
        settings[name] = groups
    pool = ThreadPoolExecutor(max_workers=len(by_n))

    def solve_all(groups):
        def work(g):
            g[0].reset()
            g[0].solve(g[1].cuda_stream)
        t = time.perf_counter()
        list(pool.map(work, groups))
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t)

    times = {k: [] for k in settings}
    stages = {k: [] for k in settings}
    for r in range(args.warmup + args.reps):
        for name, groups in settings.items():   # alternating, so that drifts of the shared machine hit both settings alike
            ms = solve_all(groups)
            if r >= args.warmup:
                times[name].append(ms)
                stages[name].append(np.sum([list(g[0].benchmarks()) for g in groups], axis=0))
    out = dict(card=card(), batch=len(insts), groups=[(n, len(gi)) for n, gi in sorted(by_n.items())], weight=args.weight,
               stage_keys=["lq", "qp", "linesearch", "lq_k1b"])
    for name, groups in settings.items():
        t = np.array(times[name])
        out[name] = dict(ms_median=round(float(np.median(t)), 3), ms_spread=round(float(t.max() - t.min()), 3),
                         stage_ms_median_summed_over_groups=[round(float(v), 4) for v in np.median(np.array(stages[name], dtype=float), axis=0)],
                         launches=int(sum(g[0].launch_count() for g in groups)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()

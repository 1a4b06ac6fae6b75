"""Device-resident receding horizon (SURVEY.md section 8(f)-2): `--cycles` MPC cycles of a batch of whole-body instances, every cycle
b200sqp_build_instances shifting the previous solution and rebuilding the references ON THE DEVICE, then b200sqp_solve running one SQP iteration (the
shipped real-time iteration).  No state or input trajectory crosses PCIe inside the loop; per cycle the host sends 44 bytes per instance (gait id,
gait start, command).  Prints one JSON line.

--sim tracking (default): perfect tracking -- the measured state of the next cycle is the previous plan interpolated at the new time
(build_instances(warm = 1, x0 = NULL)); cycles are --mpc-dt apart.
--sim rollout: the reference's dummy simulation -- after every solve b200sqp_rollout_policy simulates one MRT step (--mrt-dt, default 1/80 s as in
WBMpcDummySimNode.cpp) under the new policy with the ODE45 roll-out, and build_instances(warm = 2) takes the simulated state as the next measured
state; cycles are --mrt-dt apart.  --push S adds a seeded N(0, S) perturbation to the base velocity of the first measured state.  Reports the
roll-out's host-timed milliseconds per cycle (enqueue to collected results)."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from wb_humanoid_mpc_b200 import abi, model_loader  # noqa: E402
from wb_humanoid_mpc_b200.solver import B200SqpSolver  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--cycles", type=int, default=120)
ap.add_argument("--horizon", type=float, default=3.5)
ap.add_argument("--mpc-dt", type=float, default=1.0 / 60.0, help="time between MPC cycles (mpcDesiredFrequency 60 Hz, task.info:115)")
ap.add_argument("--gait", default="walk")
ap.add_argument("--sim", choices=["tracking", "rollout"], default="tracking")
ap.add_argument("--mrt-dt", type=float, default=1.0 / 80.0, help="--sim rollout: simulated time per cycle (the MRT step of WBMpcDummySimNode.cpp)")
ap.add_argument("--push", type=float, default=0.0, help="--sim rollout: std of a seeded perturbation of the first state's base velocity [m/s, rad/s]")
ap.add_argument("--feedback", type=int, default=1, help="--sim rollout: simulate the linear feedback policy (use_feedback_policy)")
args = ap.parse_args()

import torch  # noqa: E402

model = model_loader.load_packaged_model()
rollout = args.sim == "rollout"
st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=int(rollout and args.feedback))
insts = bench.build_batch(model, args.batch, 0, args.horizon, [args.gait])
x0 = np.array([i["x0"] for i in insts])
cmd = np.array([i["cmd"] for i in insts])
start = np.zeros(args.batch)
gaits = [args.gait] * args.batch
solver = B200SqpSolver(model, st)
n0 = solver.build_instances(0.0, args.horizon, x0, gaits, start, cmd)
solver.solve()
first = solver.iterations_log()[:, 0]
node_counts, ls_ms, ro_ms, ro_bad = {n0}, [], [], 0
step = args.mrt_dt if rollout else args.mpc_dt
if rollout:
    xs = x0.copy()
    xs[:, 29:35] += np.random.default_rng(0).normal(0.0, args.push, (args.batch, 6)) if args.push > 0 else 0.0
    r = solver.rollout_policy(0.0, step, x_start=xs)   # cycle 0's roll-out (also the warm-up of the kernel)
    ro_bad += int(r["status"].any())
torch.cuda.synchronize()
t_begin = time.perf_counter()
for c in range(1, args.cycles + 1):
    n = solver.build_instances(c * step, args.horizon, None, gaits, start, cmd, warm="rollout" if rollout else True)
    node_counts.add(n)
    solver.solve()
    ls_ms.append(solver.benchmarks()[2])
    if rollout:
        t0 = time.perf_counter()
        r = solver.rollout_policy(c * step, step)
        ro_ms.append(1e3 * (time.perf_counter() - t0))
        ro_bad += int(r["status"].any())
torch.cuda.synchronize()
dt = time.perf_counter() - t_begin
last = solver.iterations_log()[:, 0]
sol = solver.primal_solution()
g0 = np.sqrt(first[:, 2] + first[:, 3])
g1 = np.sqrt(last[:, 2] + last[:, 3])
out = {"metric": "SQP solves/sec (G1 whole-body, N=100, batched), receding horizon on the device", "value": args.batch * args.cycles / dt, "unit": "solves/s",
       "cycles": args.cycles, "batch": args.batch, "ms_per_cycle": 1e3 * dt / args.cycles, "node_counts_seen": sorted(int(v) for v in node_counts),
       "h2d_bytes_per_cycle": int(args.batch * (4 + 8 + 32)), "d2h_bytes_per_cycle": 12,
       "constraint_violation_first_cycle_median": float(np.median(g0)), "constraint_violation_last_cycle_median": float(np.median(g1)),
       "full_steps_last_cycle": int((last[:, 8] == 1.0).sum()), "linesearch_ms_first_last": [float(ls_ms[0]), float(ls_ms[-1])],
       "status_ok": bool(not sol["status"].any() and ro_bad == 0)}
if rollout:
    out.update(sim="rollout", mrt_dt=step, push=args.push, feedback=bool(args.feedback), rollout_ms_per_cycle_median=float(np.median(ro_ms)),
               rollout_ms_per_cycle_mean=float(np.mean(ro_ms)), rollout_steps_last_cycle_median=[float(v) for v in np.median(r["n_steps"], axis=0)],
               d2h_bytes_per_cycle=12 + int(args.batch * (58 * 8 + 35 * 8 + 5 * 4)))
print(json.dumps(out))

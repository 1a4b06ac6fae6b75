"""Device-resident receding horizon (SURVEY.md section 8(f)-2): `--cycles` MPC cycles of a batch of whole-body instances, every cycle
b200sqp_build_instances shifting the previous solution and rebuilding the references ON THE DEVICE, then b200sqp_solve running one SQP iteration (the
shipped real-time iteration).  No state or input trajectory crosses PCIe inside the loop; per cycle the host sends 44 bytes per instance (gait id,
gait start, command).  Prints one JSON line.

--sim tracking (default): perfect tracking -- the measured state of the next cycle is the previous plan interpolated at the new time
(build_instances(warm = 1, x0 = NULL)); cycles are --mpc-dt apart.
--sim rollout: the reference's dummy simulation -- after every solve b200sqp_rollout_policy simulates one MRT step (--mrt-dt, default 1/80 s as in
WBMpcDummySimNode.cpp) under the new policy with the ODE45 roll-out, and build_instances(warm = 2) takes the simulated state as the next measured
state; cycles are --mrt-dt apart.  --push S adds a seeded N(0, S) perturbation to the base velocity of the first measured state.  Reports the
roll-out's host-timed milliseconds per cycle (enqueue to collected results).
--model centroidal: the same loop on the centroidal MPC, with the defaults of its task.info (horizon 1.2 s, 80 Hz); also reports the builder's
milliseconds per cycle and share of the cycle, and the last cycle's stage times (LQ approximation, QP, line search).  With --sim rollout the
roll-out is b200sqp_cen_rollout_policy with the centroidal task.info settings, --mrt-dt defaults to 1/100 s (one MRT step of
CentroidalMpcDummySimNode per MPC cycle), --push perturbs the normalized momentum x[0:6], and the policy is feed-forward unless --feedback is
given (useFeedbackPolicy false in that task.info)."""
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
ap.add_argument("--model", choices=["wb", "centroidal"], default="wb", help="the whole-body MPC, or the centroidal MPC (b200sqp_cen_create)")
ap.add_argument("--horizon", type=float, default=None, help="default: timeHorizon of the model's task.info (3.5 s whole-body, 1.2 s centroidal)")
ap.add_argument("--mpc-dt", type=float, default=None,
                help="time between MPC cycles; default: mpcDesiredFrequency of the model's task.info (60 Hz whole-body, 80 Hz centroidal)")
ap.add_argument("--gait", default="walk")
ap.add_argument("--sim", choices=["tracking", "rollout"], default="tracking")
ap.add_argument("--mrt-dt", type=float, default=None,
                help="--sim rollout: simulated time per cycle; default: the MRT step of the model's dummy simulation (1/80 s whole-body, 1/100 s centroidal)")
ap.add_argument("--push", type=float, default=0.0,
                help="--sim rollout: std of a seeded perturbation of the first state's base velocity [m/s, rad/s] (centroidal: normalized momentum)")
ap.add_argument("--feedback", type=int, nargs="?", const=1, default=None,
                help="--sim rollout: simulate the linear feedback policy (use_feedback_policy); default 1 whole-body, 0 centroidal")
ap.add_argument("--gait-sequence", default=None,
                help="gait commands as gait@time,... (e.g. stance@0,walk@0.5,run@3,walk@5,stance@7): stateful gait schedule on the device, every "
                     "instance commanded the gait of the current time; replaces --gait")
args = ap.parse_args()
cen = args.model == "centroidal"
if cen and args.gait_sequence:
    ap.error("--model centroidal: the stateful gait schedule serves whole-body handles only; use --gait")
if args.horizon is None:
    args.horizon = 1.2 if cen else 3.5
if args.mpc_dt is None:
    args.mpc_dt = 1.0 / 80.0 if cen else 1.0 / 60.0
if args.mrt_dt is None:
    args.mrt_dt = 1.0 / 100.0 if cen else 1.0 / 80.0
if args.feedback is None:
    args.feedback = 0 if cen else 1
sequence = None
if args.gait_sequence:
    sequence = [(g, float(t)) for g, t in (item.split("@") for item in args.gait_sequence.split(","))]
    args.gait = sequence[0][0]


def commanded(t):
    return [g for g, ts in sequence if ts <= t + 1e-9][-1] if sequence else args.gait

import torch  # noqa: E402

def centroidal_batch(model, batch):
    """perturbed centroidal states (zero momentum, as tools/bench_centroidal.py) and velocity commands of bench.build_batch's distribution"""
    rng = np.random.default_rng(bench.SEED)
    x0s, cmds = [], []
    for _ in range(batch):
        x = np.array(model["x_init"], float)
        x[6:8] += rng.uniform(-0.02, 0.02, 2)
        x[9:12] += rng.uniform(-0.05, 0.05, 3)
        x[12:] += rng.uniform(-0.1, 0.1, model["nj"])
        x0s.append(x)
        cmds.append([rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)])
    return np.array(x0s), np.array(cmds)


model = model_loader.load_packaged_model("g1_centroidal" if cen else "g1_wb")
rollout = args.sim == "rollout"
st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=int(rollout and args.feedback))
if cen:
    x0, cmd = centroidal_batch(model, args.batch)
else:
    insts = bench.build_batch(model, args.batch, 0, args.horizon, [args.gait])
    x0 = np.array([i["x0"] for i in insts])
    cmd = np.array([i["cmd"] for i in insts])
start = np.zeros(args.batch)
gaits = [args.gait] * args.batch
solver = B200SqpSolver(model, st)
if sequence:
    solver.set_gait_schedule(True)
n0 = solver.build_instances(0.0, args.horizon, x0, gaits, start, cmd)
solver.solve()
first = solver.iterations_log()[:, 0]
node_counts, ls_ms, ro_ms, ro_bad = {n0}, [], [], 0
step = args.mrt_dt if rollout else args.mpc_dt
if rollout:
    xs = x0.copy()
    pushed = slice(0, 6) if cen else slice(29, 35)   # normalized momentum / base velocity
    xs[:, pushed] += np.random.default_rng(0).normal(0.0, args.push, (args.batch, 6)) if args.push > 0 else 0.0
    rollout_policy = solver.cen_rollout_policy if cen else solver.rollout_policy
    r = rollout_policy(0.0, step, x_start=xs)   # cycle 0's roll-out (also the warm-up of the kernel)
    ro_bad += int(r["status"].any())
torch.cuda.synchronize()
t_begin = time.perf_counter()
build_s = 0.0
for c in range(1, args.cycles + 1):
    gaits = [commanded(c * step)] * args.batch
    tb = time.perf_counter()
    n = solver.build_instances(c * step, args.horizon, None, gaits, start, cmd, warm="rollout" if rollout else True)
    build_s += time.perf_counter() - tb   # (b200sqp_build_instances returns after its last kernel)
    node_counts.add(n)
    solver.solve()
    ls_ms.append(solver.benchmarks()[2])
    if rollout:
        t0 = time.perf_counter()
        r = rollout_policy(c * step, step)
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
               d2h_bytes_per_cycle=12 + int(args.batch * (model["nx"] * 8 + 35 * 8 + 5 * 4)))
if cen:
    bm = solver.benchmarks()
    out.update(metric=f"SQP solves/sec (G1 centroidal, N={round(args.horizon / model['sqp']['dt'])}, batched), receding horizon on the device", model="centroidal",
               horizon=args.horizon, mpc_dt=step, builder_ms_per_cycle=1e3 * build_s / args.cycles, builder_share_of_cycle=build_s / dt,
               stage_ms_last_cycle={"lq": float(bm[0]), "qp": float(bm[1]), "linesearch": float(bm[2])})
if sequence:
    out.update(gait_sequence=args.gait_sequence, simulated_seconds=args.cycles * step, builder_ms_per_cycle=1e3 * build_s / args.cycles,
               builder_share_of_cycle=build_s / dt)
print(json.dumps(out))

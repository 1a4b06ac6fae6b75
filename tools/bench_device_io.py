"""Device-pointer I/O of the closed loop against the host-pointer path, for a batched simulator whose robot states live in CUDA tensors.  For the
whole-body and the centroidal MPC, at each `--batches` size, on a plain handle (every instance walking) and on a mixed fleet (stance / walk /
slow_walk at random phases: several node-count groups), after a cold build and one solve:
  tick   joint_actions on states that are already in a CUDA tensor.  Host path: the states go to the host (tensor.cpu()), b200sqp_joint_actions
         runs and waits, and q_des / qd_des / tau go back to the device (what a GPU simulator has to do with it).  Device path:
         joint_actions_device into preallocated tensors.  Reported per tick: the host-blocking time (until the call returns) and the end-to-end
         time (host clock around the call and a torch.cuda.synchronize), median over `--ticks`.
  cycle  one MPC cycle, a warm build + one SQP iteration, with x0 from the CUDA tensor (build_instances_dev) against x0 copied to the host
         first; host clock around build + solve + wait, median over `--cycles`.
Reads the card's name, power limit and max SM clock in the same process.  Prints one JSON line."""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import mrt_ref  # noqa: E402
from wb_humanoid_mpc_b200 import abi, model_loader  # noqa: E402
from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batches", type=int, nargs="+", default=[256, 1024])
ap.add_argument("--ticks", type=int, default=200)
ap.add_argument("--cycles", type=int, default=10)
ap.add_argument("--warmup", type=int, default=10)
args = ap.parse_args()

import torch  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("bench_device_io: no CUDA device; the device-pointer paths have no CPU path")
DEV = torch.device("cuda", 0)
HORIZON = {"wb": 1.1, "centroidal": 1.2}   # the horizons of the closed-loop tests
MIXED = ["stance", "walk", "slow_walk"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return out.stdout.strip()


def inputs(model, batch, rng, cen):
    x0s, cmds = [], []
    for _ in range(batch):
        x = np.array(model["x_init"], float)
        if cen:
            x[:6] += rng.uniform(-0.1, 0.1, 6)
            x[12:] += rng.uniform(-0.1, 0.1, model["nj"])
        else:
            x[2] = model["reference"]["defaultBaseHeight"]
            x[6:29] += rng.uniform(-0.1, 0.1, 23)
        x0s.append(x)
        cmds.append([rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)])
    return np.array(x0s), np.array(cmds)


def median_ms(fn, n):
    blocking, e2e = [], []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        blocking.append((t1 - t0) * 1e3)
        e2e.append((t2 - t0) * 1e3)
    return statistics.median(blocking), statistics.median(e2e)


def run(fam, batch, mixed):
    cen = fam == "centroidal"
    model = model_loader.load_packaged_model("g1_centroidal" if cen else "g1_wb")
    rng = np.random.default_rng(7)
    x0, cmd = inputs(model, batch, rng, cen)
    solver = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1))
    if mixed:
        gaits = [MIXED[b % 3] for b in range(batch)]
        starts = np.array([0.5 if g == "stance" else -rng.uniform(0.0, model["gaits"][g]["switchingTimes"][-1]) for g in gaits])
        h = B200SqpFleet(solver)
    else:
        gaits, starts, h = ["walk"] * batch, np.zeros(batch), solver
    h.build_instances(0.0, HORIZON[fam], x0, gaits, starts, cmd)
    h.solve()
    nj = model["nj"]
    rs = torch.tensor(mrt_ref.random_robot_states(rng, batch, nj, base=x0[:, 6:] if cen else x0), device=DEV)
    t = 0.005
    out = h.joint_actions_device(t, rs)
    joints = torch.empty((3, batch, nj), dtype=torch.float64, device=DEV)

    def host_tick():
        a = h.joint_actions(t, rs.cpu().numpy())
        joints.copy_(torch.from_numpy(np.stack([a["q_des"], a["qd_des"], a["tau"]])), non_blocking=False)

    def dev_tick():
        h.joint_actions_device(t, rs, out=out)

    res = {}
    for name, fn in (("host", host_tick), ("device", dev_tick)):
        median_ms(fn, args.warmup)
        b, e = median_ms(fn, args.ticks)
        res[f"tick_{name}_blocking_ms"], res[f"tick_{name}_e2e_ms"] = b, e
    assert torch.isfinite(out["tau"]).all() and not out["status"].any()
    x0d = torch.tensor(x0, device=DEV)
    cyc = {"host": lambda t0: h.build_instances(t0, HORIZON[fam], x0d.cpu().numpy(), gaits, starts, cmd, warm=True),
           "device": lambda t0: h.build_instances(t0, HORIZON[fam], x0d, gaits, starts, cmd, warm=True)}
    t0 = 0.0
    for name, build in cyc.items():
        ms = []
        for k in range(args.warmup + args.cycles):
            t0 += 0.01
            s = time.perf_counter()
            build(t0)
            h.solve()
            ms.append((time.perf_counter() - s) * 1e3)
        res[f"cycle_{name}_ms"] = statistics.median(ms[args.warmup:])
    if mixed:
        res["n_groups"] = h.n_groups
        h.close()
    solver.close()
    return res


out = dict(ticks=args.ticks, cycles=args.cycles, card=card(), results={})
for batch in args.batches:
    for fam in ("wb", "centroidal"):
        for kind in ("plain", "mixed"):
            out["results"][f"{fam}/{kind}/B{batch}"] = run(fam, batch, kind == "mixed")
out["card_after"] = card()
print(json.dumps(out))

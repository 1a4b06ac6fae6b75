"""MRT-side queries (b200sqp_mrt_query / _dev) at production batch size: for the whole-body MPC (B = 256 over a 3.5 s horizon, N = 100 +
event nodes) and a centroidal batch, a cold build + one solve with settings.create_value_function = use_feedback_policy = 1, then, timed with
CUDA events around `--calls` calls each:
  query_host    mrt_query(t, x) with both outputs on host arrays (x uploaded, the kernel, dfdxx / dfdx / K copied back, collected);
  query_device  mrt_query_device(t, x) into CUDA tensors (the kernel alone, stream-ordered);
  download_path the way without the query: value_function() (b200sqp_download_value_function, every node's P and p) and
                primal_solution(K), then the host interpolation of one time for every instance (mrt_query_ref.py).
Every path's result is checked against the host restatement first.  The card name and power limit are read in the same process.  Prints
one JSON line."""
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
import bench  # noqa: E402
import mrt_query_ref  # noqa: E402
from wb_humanoid_mpc_b200 import abi, model_loader  # noqa: E402
from wb_humanoid_mpc_b200.solver import B200SqpSolver  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--calls", type=int, default=200)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--download-calls", type=int, default=3)
args = ap.parse_args()

import torch  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("bench_mrt_queries: no CUDA device; the query kernel has no CPU path")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return out.stdout.strip()


def centroidal_batch(model, batch, rng):
    x0s, cmds = [], []
    for _ in range(batch):
        x = np.array(model["x_init"], float)
        x[6:8] += rng.uniform(-0.02, 0.02, 2)
        x[9:12] += rng.uniform(-0.05, 0.05, 3)
        x[12:] += rng.uniform(-0.1, 0.1, model["nj"])
        x0s.append(x)
        cmds.append([rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)])
    return np.array(x0s), np.array(cmds)


def timed(fn, n):
    """CUDA events around each call (the host path waits inside the call, so its events bracket the whole round trip)"""
    ms = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return dict(median_ms=statistics.median(ms), mean_ms=statistics.fmean(ms), min_ms=min(ms), calls=n)


def restate_all(t, inp, P, p, K, x):
    return [mrt_query_ref.query(t, inp["t_nodes"][b], inp["node_event"][b], P=P[b], p=p[b], K=K[b], x=x[b]) for b in range(len(x))]


def run(name):
    cen = name == "centroidal"
    model = model_loader.load_packaged_model("g1_centroidal" if cen else "g1_wb")
    horizon = 1.2 if cen else 3.5
    rng = np.random.default_rng(bench.SEED)
    if cen:
        x0, cmd = centroidal_batch(model, args.batch, rng)
    else:
        insts = bench.build_batch(model, args.batch, 0, horizon, ["walk"])
        x0, cmd = np.array([i["x0"] for i in insts]), np.array([i["cmd"] for i in insts])
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1, create_value_function=1))
    s.build_instances(0.0, horizon, x0, ["walk"] * args.batch, np.zeros(args.batch), cmd)
    s.solve()
    B, nx, nu = args.batch, model["nx"], model["nu"]
    x = x0 + rng.normal(0.0, 0.01, x0.shape)
    xd = torch.tensor(x, dtype=torch.float64, device="cuda")
    t = 0.2113
    # correctness first: both paths against the restatement over the downloads
    inp, sol = s.download_instances(), s.primal_solution()
    P, p = s.value_function()
    ref = restate_all(t, inp, P, p, sol["K"], x)
    host, dev = s.mrt_query(t, x), s.mrt_query_device(t, xd)
    torch.cuda.synchronize()
    worst = 0.0
    for k in ("dfdxx", "dfdx", "K"):
        r = np.array([q[k] for q in ref])
        for got in (host[k], dev[k].cpu().numpy()):
            worst = max(worst, float(np.max(np.abs(got - r)) / np.max(np.abs(r))))
    for _ in range(args.warmup):
        s.mrt_query(t, x)
        s.mrt_query_device(t, xd)
    torch.cuda.synchronize()

    def download_path():
        Pd, pd = s.value_function()
        Kd = s.primal_solution()["K"]
        restate_all(t, inp, Pd, pd, Kd, x)

    res = dict(n_nodes=int(s.n_nodes), max_rel_err=worst, query_host=timed(lambda: s.mrt_query(t, x), args.calls),
               query_device=timed(lambda: s.mrt_query_device(t, xd), args.calls), download_path=timed(download_path, args.download_calls))
    n = int(s.n_nodes)
    res["bytes_query_read"] = B * (2 * nx * nx + 2 * nx + 2 * nu * nx + nx) * 8   # what the kernel must read (two nodes, two stages, x)
    res["bytes_query_out"] = B * (nx * nx + nx + nu * nx) * 8
    res["bytes_download"] = B * (n * (nx * nx + nx) + (n - 1) * nu * nx) * 8 + B * (n * nx + (n - 1) * nu) * 8
    s.close()
    return res


res = dict(batch=args.batch, card=card())
for fam in ("wb", "centroidal"):
    res[fam] = run(fam)
res["card_after"] = card()
print(json.dumps(res))

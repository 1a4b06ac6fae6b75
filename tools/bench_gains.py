"""Per-instance gains (b200sqp_set_gains) on the H100: what they cost and what they are for.  One JSON line.

  solve   whole-body (N = 100, batch 256, sqpIteration 1, cold start: b200sqp_reset before every solve) and centroidal (horizon 1.2 s,
          batch 256) solve time under three settings, timed alternately in one process: gains never set; every instance set to the model's
          values; distinct seeded gains per instance.  Median and spread (max - min) of the host-clock solve (reset + solve + wait) and the
          median of each stage time (b200sqp_get_stage_times).  The distinct setting is the one whose models no longer share L1 between the
          CTAs of different instances.
  apply   b200sqp_set_gains (host records, synchronous) and b200sqp_set_gains_dev (device records, CUDA events on the stream) for 256 and
          1024 instances.
  --sweep one closed loop (device roll-out, a seeded --push of the base velocity, automatic resets) over 256 candidate gain sets sampled
          log-uniformly around the task.info values: each candidate's survival (mean episode length) and velocity tracking error, ranked.
The card's name and power limit are printed beside the numbers."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from test_emu_gains import model_gains  # noqa: E402
from wb_humanoid_mpc_b200 import abi, model_loader  # noqa: E402
from wb_humanoid_mpc_b200.solver import B200SqpSolver  # noqa: E402

SCALED = ("Q_diag", "R_diag", "Qf_diag", "foot_cost_w", "torso_w", "jlim_mu", "coll_mu", "fric_mu", "momxy_mu")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def sample_gains(model, rng, n, spread):
    """n gain sets: every weight group and penalty mu of the model scaled by one log-uniform factor in [1/spread, spread] per set"""
    base = model_gains(model)
    out = {k: np.stack([np.asarray(base[k])] * n) for k in abi.GAIN_FIELDS}
    for k in SCALED:
        f = np.exp(rng.uniform(-np.log(spread), np.log(spread), n))
        out[k] = out[k] * f.reshape((n,) + (1,) * (out[k].ndim - 1))
    return out


def handle(fam, batch, horizon, iters=1, rng=None):
    import test_gpu_builder
    import test_gpu_cen_builder

    model = model_loader.load_packaged_model("g1_wb" if fam == "wb" else "g1_centroidal")
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=iters))
    x0, cmd = (test_gpu_builder if fam == "wb" else test_gpu_cen_builder).make_inputs(model, rng or np.random.default_rng(0), batch)
    s.build_instances(0.0, horizon, x0, ["walk"] * batch, np.zeros(batch), cmd)
    return model, s, x0, cmd


def part_solve(fam, batch, horizon, reps, warmup):
    settings = {}
    for name in ("never", "defaults", "distinct"):
        model, s, _, _ = handle(fam, batch, horizon)
        if name == "defaults":
            s.set_gains(np.arange(batch), s.default_gains())
        elif name == "distinct":
            s.set_gains(np.arange(batch), sample_gains(model, np.random.default_rng(1), batch, 2.0))
        settings[name] = s
    times = {k: [] for k in settings}
    stages = {k: [] for k in settings}
    for r in range(warmup + reps):
        for name, s in settings.items():   # alternating, so that drifts of the shared machine hit every setting alike
            t = time.perf_counter()
            s.reset()
            s.solve()
            dt = time.perf_counter() - t
            if r >= warmup:
                times[name].append(1e3 * dt)
                stages[name].append(s.benchmarks())
    out = {}
    for name in settings:
        t = np.array(times[name])
        st = np.median(np.array([[b[k] for k in sorted(b)] if isinstance(b, dict) else list(b) for b in stages[name]], dtype=float), axis=0)
        out[name] = dict(ms_median=float(np.median(t)), ms_spread=float(t.max() - t.min()), stage_ms_median=[round(float(v), 4) for v in st])
    return out


def part_apply(reps):
    import torch

    out = {}
    for batch in (256, 1024):
        model, s, _, _ = handle("wb", batch, 1.1)
        g = sample_gains(model, np.random.default_rng(2), batch, 2.0)
        idx = np.arange(batch)
        host = []
        for _ in range(reps):
            t = time.perf_counter()
            s.set_gains(idx, g)
            host.append(1e3 * (time.perf_counter() - t))
        rows = torch.from_numpy(abi.pack_gains(g)).cuda()
        dev = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            s.set_gains_device(idx, rows)
            b.record()
            torch.cuda.synchronize()
            dev.append(a.elapsed_time(b))
        out[str(batch)] = dict(host_ms_median=float(np.median(host)), dev_ms_median=float(np.median(dev)))
    return out


def part_sweep(args):
    """one closed loop of 256 candidates: every instance walks under the same command from the same pushed state"""
    B, dt = 256, 1.0 / 80.0
    model, s, x0, cmd = handle("wb", 1, args.horizon)
    x0 = np.repeat(x0, B, axis=0)
    x0[:, 29:35] += np.random.default_rng(args.seed).normal(0.0, args.push, (1, 6))   # one push, the same for every candidate
    cmd = np.repeat(np.array([[0.5, 0.0, model["reference"]["defaultBaseHeight"], 0.0]]), B, axis=0)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1))
    s.set_gait_schedule(True)
    s.set_auto_reset(on_solve_failure=True, on_rollout_failure=True, max_height_deviation=0.25, max_pitch_deviation=0.5, max_roll_deviation=0.5)
    gaits = ["walk"] * B
    s.build_instances(0.0, args.horizon, x0, gaits, np.zeros(B), cmd)
    s.set_reset_states(x0, gaits)
    cand = sample_gains(model, np.random.default_rng(args.seed), B, args.spread)
    s.set_gains(np.arange(B), cand)
    err, resets = np.zeros(B), np.zeros(B, dtype=int)
    t = 0.0
    for c in range(args.cycles):
        s.solve()
        ro = s.rollout_policy(t, dt)
        t += dt
        err += np.abs(ro["x"][:, 29] - cmd[:, 0])   # base x velocity against the command
        s.build_instances(t, args.horizon, None, gaits, np.zeros(B), cmd, warm="rollout")
        resets += s.episodes()["reset"]
    survival = t / (resets + 1)
    order = np.lexsort((err, -survival))
    ranked = [dict(candidate=int(i), survival_s=round(float(survival[i]), 4), resets=int(resets[i]), tracking_err=round(float(err[i] / args.cycles), 5),
                   scale={k: round(float(np.ravel(cand[k][i])[0] / max(np.ravel(model_gains(model)[k])[0], 1e-300)), 4) for k in SCALED})
              for i in order]
    return dict(cycles=args.cycles, push=args.push, spread=args.spread, seed=args.seed, ranked=ranked)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sweep", action="store_true", help="only the candidate sweep")
    ap.add_argument("--cycles", type=int, default=160)
    ap.add_argument("--push", type=float, default=0.3)
    ap.add_argument("--spread", type=float, default=3.0, help="the candidates scale each term by a log-uniform factor in [1/spread, spread]")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--horizon", type=float, default=1.1)
    args = ap.parse_args()
    out = dict(card=card())
    if args.sweep:
        out["sweep"] = part_sweep(args)
    else:
        out["wb_solve"] = part_solve("wb", 256, 3.5, args.reps, args.warmup)
        out["cen_solve"] = part_solve("cen", 256, 1.2, args.reps, args.warmup)
        out["apply"] = part_apply(args.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

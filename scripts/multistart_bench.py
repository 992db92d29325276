#!/usr/bin/env python3
"""Time multi-start solving to a tolerance two ways, and measure what the seeds recover:

  UR5 at B = 8192 targets, S in {1, 8, 32}: the task set of examples/arm_ur5_reach_batched.py with
      the targets of examples/arm_ur5_reach_multistart_batched.py (FK of configurations uniform
      within the limits, one shared home pose as seed 0), tol = 1e-5, max_steps = 200;
  G1 + CoM at B = 2048 targets, S = 4: the workload of scripts/converge_bench.py (tol = the median
      error after a 40-step rollout), seeds 1..3 = the start with its joints moved by N(0, 0.1).

  (a) one BatchedIK.converge_multistart launch;
  (b) BatchedIK.converge on the tiled [B*S, nq] seeds (targets repeated S times), then the winner
      per target with torch ops (smallest error, NaN as +inf, lowest index on ties).

Both run on the same seeds, are captured in CUDA graphs and timed over --regions regions (median
and spread), each region behind an L2 flush and a short device-side spin, as bench.py does.
Reported per case: the converged fraction of (a) and of (b), the distribution of the rounds (a)
ran and of the steps (b) ran, and the card name and power limit from a read-only nvidia-smi query
in the same run.  Prints one JSON line per case.

    python scripts/multistart_bench.py [--regions 11]
"""

import argparse
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from scripts.converge_bench import card, g1  # noqa: E402


def ur5(B, S):
    spec = importlib.util.spec_from_file_location(
        "reach_ms", os.path.join(ROOT, "examples", "arm_ur5_reach_multistart_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    ik, task, q0, targets = ex.setup(B)
    qs = ik.sample_seeds(q0, S, generator=torch.Generator(device="cuda").manual_seed(1))
    return ik, [task], qs, targets, ex.TOL


def g1_seeds(B, S):
    ik, tasks, q0, targets, tol = g1(B)
    qs = q0[:, None].repeat(1, S, 1)
    g = torch.Generator(device="cuda").manual_seed(1)
    qs[:, 1:, 7:] += 0.1 * torch.randn(qs[:, 1:, 7:].shape, device="cuda", generator=g)
    return ik, tasks, qs.contiguous(), targets, tol


def pick(res, B, S):
    """The winner of each target among the tiled converge results."""
    e = res.error.reshape(B, S)
    key = torch.where(torch.isnan(e), torch.full_like(e, float("inf")), e)
    seed = torch.argmin(key, dim=1)  # the first minimum: the lowest index on ties
    rows = torch.arange(B, device=e.device) * S + seed
    return res.q[rows], res.error[rows], seed, res.steps[rows], res.status[rows]


def dist(x):
    x = x.cpu().numpy()
    return {"mean": round(float(x.mean()), 2),
            "p50_p90_p99_max": [int(np.percentile(x, p)) for p in (50, 90, 99)] + [int(x.max())]}


def measure(name, setup, B, S, max_steps, regions):
    ik, tasks, qs, targets, tol = setup(B, S)
    dev = qs.device
    flat = qs.reshape(B * S, -1)
    t_flat = targets.repeat_interleave(S, dim=0).contiguous()
    res_a = ik.converge_multistart(qs, targets, tasks, tol, max_steps)
    res_b = ik.converge(flat, t_flat, tasks, tol, max_steps)
    win_b = pick(res_b, B, S)
    torch.cuda.synchronize()
    out_a = [torch.empty((B, ik.nq), device=dev), torch.empty(B, device=dev)] + [
        torch.empty(B, device=dev, dtype=torch.int32) for _ in range(3)]
    out_b = [torch.empty_like(flat), torch.empty(B * S, device=dev)] + [
        torch.empty(B * S, device=dev, dtype=torch.int32) for _ in range(2)]
    variants = {
        "a_multistart": lambda: ik.converge_multistart(qs, targets, tasks, tol, max_steps, *out_a),
        "b_tiled_converge_and_select": lambda: pick(ik.converge(flat, t_flat, tasks, tol, max_steps, *out_b), B, S),
    }
    graphs = {}
    for v, fn in variants.items():
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            fn()  # warm-up outside the capture
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        g.replay()
        torch.cuda.synchronize()
        graphs[v] = g
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    flush = torch.empty(2 * l2, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {v: [] for v in graphs}
    for _ in range(regions):
        for v, g in graphs.items():  # variants interleaved region by region
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda._sleep(300000)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) * 1e3)
    cname, power = card()
    out = {"workload": name, "card": cname, "power_limit": power, "targets": B, "seeds": S, "tol": tol,
           "max_steps": max_steps, "regions": regions,
           "timing": "median over regions, one CUDA-graph replay after an L2 flush"}
    for v, ts in times.items():
        out[v] = {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
    out["b_over_a"] = round(out["b_tiled_converge_and_select"]["us"] / out["a_multistart"]["us"], 3)
    conv_b = (win_b[1] <= tol)
    out["converged_fraction"] = {"a": round(res_a.converged.float().mean().item(), 5),
                                 "b": round(conv_b.float().mean().item(), 5),
                                 "seed0_alone": round(res_b.converged.reshape(B, S)[:, 0].float().mean().item(), 5)}
    out["a_rounds"] = dist(res_a.steps)
    out["b_steps_all_seeds"] = dist(res_b.steps)
    out["a_winner_seed_gt0"] = int((res_a.seed > 0).sum())
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    for S in (1, 8, 32):
        measure("ur5_workspace", ur5, 8192, S, 200, args.regions)
    measure("g1_com", g1_seeds, 2048, 4, 200, args.regions)


if __name__ == "__main__":
    main()

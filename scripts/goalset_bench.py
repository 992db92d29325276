#!/usr/bin/env python3
"""Time goal-set solving to a tolerance three ways, and measure what each solves:

  UR5 at B = 8192 instances, G = 8 goals, S = 4 seeds: examples/arm_ur5_grasp_goalset_batched.py
      (half of each instance's goals FK of configurations uniform within the limits, half out of
      reach; seed 0 the home pose, the others uniform within the limits), tol = 1e-5,
      max_steps = 200;
  G1 + CoM at B = 2048 instances, G = 2, S = 4 (G S = 8, the tree kernel's limit): the workload of
      scripts/multistart_bench.py (tol = the median error after a 40-step rollout, seeds 1..3 =
      the start with its joints moved by N(0, 0.1)), goal 0 the instance's targets row and goal 1
      the row of the previous instance.

  (a) one BatchedIK.converge_goalset launch;
  (b) BatchedIK.converge_multistart on the B G tiled targets rows, then the winner per instance
      with torch ops (smallest error, NaN as +inf, lowest goal on ties);
  (c) BatchedIK.converge on the B G S tiled rows, then the winner per instance with torch ops.

All run on the same seeds, are captured in CUDA graphs and timed over --regions regions (median
and spread), each region behind an L2 flush and a short device-side spin, as
scripts/multistart_bench.py does.  Reported per case: the solved fraction of each (a and b must
agree: a member follows the same trajectory in both until its group stops), the distribution of
the rounds (a) ran and of the rounds or steps (b) and (c) ran, and the card name and power limit
from a read-only nvidia-smi query in the same run.  Prints one JSON line per case.

    python scripts/goalset_bench.py [--regions 11]
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

from scripts.converge_bench import card  # noqa: E402
from scripts.multistart_bench import dist, g1_seeds  # noqa: E402


def ur5(B, G, S):
    spec = importlib.util.spec_from_file_location(
        "grasp_gs", os.path.join(ROOT, "examples", "arm_ur5_grasp_goalset_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    ik, task, q0, goals, _ = ex.setup(B)
    assert goals.shape[1] == G
    qs = ik.sample_seeds(q0, S, generator=torch.Generator(device="cuda").manual_seed(1))
    return ik, [task], qs, goals, ex.TOL


def g1(B, G, S):
    ik, tasks, qs, targets, tol = g1_seeds(B, S)
    goals = torch.stack([targets.roll(g, 0) for g in range(G)], dim=1).contiguous()
    return ik, tasks, qs, goals, tol


def pick(q, error, steps, B, K):
    """The winner of each instance among K tiled results per instance."""
    e = error.reshape(B, K)
    key = torch.where(torch.isnan(e), torch.full_like(e, float("inf")), e)
    k = torch.argmin(key, dim=1)  # the first minimum: the lowest index on ties
    rows = torch.arange(B, device=e.device) * K + k
    return q[rows], error[rows], k, steps[rows]


def measure(name, setup, B, G, S, max_steps, regions):
    ik, tasks, qs, goals, tol = setup(B, G, S)
    dev = qs.device
    nq = ik.nq
    qs_b = qs.repeat_interleave(G, dim=0).contiguous()  # [B G, S, nq]: each goal's seeds
    t_b = goals.reshape(B * G, -1).contiguous()
    qs_c = qs[:, None].expand(B, G, S, nq).reshape(B * G * S, nq).contiguous()  # member j = g S + s
    t_c = goals.repeat_interleave(S, dim=1).reshape(B * G * S, -1).contiguous()
    res_a = ik.converge_goalset(qs, goals, tasks, tol, max_steps)
    res_b = ik.converge_multistart(qs_b, t_b, tasks, tol, max_steps)
    res_c = ik.converge(qs_c, t_c, tasks, tol, max_steps)
    win_b = pick(res_b.q, res_b.error, res_b.steps, B, G)
    win_c = pick(res_c.q, res_c.error, res_c.steps, B, G * S)
    torch.cuda.synchronize()
    i32 = dict(device=dev, dtype=torch.int32)
    out_a = [torch.empty((B, nq), device=dev), torch.empty(B, device=dev)] + [torch.empty(B, **i32) for _ in range(4)]
    out_b = [torch.empty((B * G, nq), device=dev), torch.empty(B * G, device=dev)] + [
        torch.empty(B * G, **i32) for _ in range(3)]
    out_c = [torch.empty_like(qs_c), torch.empty(B * G * S, device=dev)] + [
        torch.empty(B * G * S, **i32) for _ in range(2)]

    def run_b():
        r = ik.converge_multistart(qs_b, t_b, tasks, tol, max_steps, *out_b)
        return pick(r.q, r.error, r.steps, B, G)

    def run_c():
        r = ik.converge(qs_c, t_c, tasks, tol, max_steps, *out_c)
        return pick(r.q, r.error, r.steps, B, G * S)

    variants = {
        "a_goalset": lambda: ik.converge_goalset(qs, goals, tasks, tol, max_steps, *out_a),
        "b_tiled_multistart_and_select": run_b,
        "c_tiled_converge_and_select": run_c,
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
    out = {"workload": name, "card": cname, "power_limit": power, "instances": B, "goals": G, "seeds": S,
           "tol": tol, "max_steps": max_steps, "regions": regions,
           "timing": "median over regions, one CUDA-graph replay after an L2 flush"}
    for v, ts in times.items():
        out[v] = {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
    a_us = out["a_goalset"]["us"]
    out["b_over_a"] = round(out["b_tiled_multistart_and_select"]["us"] / a_us, 3)
    out["c_over_a"] = round(out["c_tiled_converge_and_select"]["us"] / a_us, 3)
    out["solved_fraction"] = {"a": round(res_a.converged.float().mean().item(), 5),
                              "b": round((win_b[1] <= tol).float().mean().item(), 5),
                              "c": round((win_c[1] <= tol).float().mean().item(), 5)}
    out["solved_a_equals_b"] = bool(torch.equal(res_a.converged, win_b[1] <= tol))
    out["a_rounds"] = dist(res_a.steps)
    out["b_rounds_all_goals"] = dist(res_b.steps)
    out["c_steps_all_members"] = dist(res_c.steps)
    out["a_goal_histogram"] = torch.bincount(res_a.goal.long(), minlength=G).cpu().tolist()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    measure("ur5_grasp_goals", ur5, 8192, 8, 4, 200, args.regions)
    measure("g1_com", g1, 2048, 2, 4, 200, args.regions)


if __name__ == "__main__":
    main()

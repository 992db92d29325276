#!/usr/bin/env python3
"""Time separate position and orientation tolerances (``orientation_tol`` of
``BatchedIK.converge``) against the default stopping test, alternated region by region in one run:

  UR5 at B = 65536: examples/arm_ur5_reach_batched.py with tol = 1e-9, so that both tests run
      the instances to max_steps = 100 (but for the few whose step fails, reported in "steps");
      the difference is the per-step cost of the test;
  G1: examples/humanoid_g1_reach_batched.py at B = 4096 (every frame task and the CoM in the
      stopping set, tol = 2 mm, orientation_tol = 0.02 rad, max_steps = 200); the default test
      cannot stop this set, so it runs every instance to max_steps.

Each variant is captured in a CUDA graph and timed over --regions regions (median and spread),
each region behind an L2 flush and a short device-side spin.  Reported: time per call and per
step, the steps taken, the solved fraction, and the card name and power limit from a read-only
nvidia-smi query in the same run.  Prints one JSON line per workload.

    python scripts/pose_tol_bench.py [--regions 11]
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
from scripts.multistart_bench import dist  # noqa: E402


def example(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "examples", name + ".py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    return ex


def timed(variants, regions):
    """Median and spread (us) of one graph replay per variant, interleaved region by region."""
    graphs = {}
    for v, fn in variants.items():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        g.replay()
        torch.cuda.synchronize()
        graphs[v] = g
    flush = torch.empty(2 * torch.cuda.get_device_properties(0).L2_cache_size, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {v: [] for v in graphs}
    for _ in range(regions):
        for v, g in graphs.items():
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda._sleep(300000)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) * 1e3)
    return {v: {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
            for v, ts in times.items()}


def outs(ik, B):
    return dict(q_out=torch.empty((B, ik.nq), device="cuda"), error=torch.empty(B, device="cuda"),
                steps=torch.empty(B, device="cuda", dtype=torch.int32),
                status=torch.empty(B, device="cuda", dtype=torch.int32))


def ur5(regions, B=65536, max_steps=100, tol=1e-9):
    ik, task, q0, targets = example("arm_ur5_reach_batched").setup(B)
    o_old, o_new = outs(ik, B), outs(ik, B)
    t = timed({"default_test": lambda: ik.converge(q0, targets, [task], tol, max_steps, **o_old),
               "pose_tol": lambda: ik.converge(q0, targets, [task], tol, max_steps, orientation_tol=tol, **o_new)},
              regions)
    torch.cuda.synchronize()
    out = {"workload": "ur5_to_max_steps", "instances": B, "tol": tol, "orientation_tol": tol,
           "max_steps": max_steps, "steps": {"default_test": dist(o_old["steps"]), "pose_tol": dist(o_new["steps"])}}
    for v, r in t.items():
        out[v] = dict(r, us_per_step=round(r["us"] / max_steps, 3))
    out["pose_tol_over_default"] = round(t["pose_tol"]["us"] / t["default_test"]["us"], 4)
    return out


def g1(regions, B=4096, max_steps=200):
    ex = example("humanoid_g1_reach_batched")
    ik, stop, q0, targets = ex.setup(B)
    o_old, o_new = outs(ik, B), outs(ik, B)
    t = timed({"default_test": lambda: ik.converge(q0, targets, stop, ex.TOL, max_steps, **o_old),
               "pose_tol": lambda: ik.converge(q0, targets, stop, ex.TOL, max_steps,
                                               orientation_tol=ex.ORIENTATION_TOL, **o_new)}, regions)
    torch.cuda.synchronize()
    out = {"workload": "g1_reach_example", "instances": B, "tol": ex.TOL, "orientation_tol": ex.ORIENTATION_TOL,
           "max_steps": max_steps, **t,
           "default_over_pose_tol": round(t["default_test"]["us"] / t["pose_tol"]["us"], 3),
           "solved_fraction": {"default_test": round((o_old["error"] <= ex.TOL).float().mean().item(), 5),
                               "pose_tol": round((o_new["error"] <= ex.TOL).float().mean().item(), 5)},
           "steps": {"default_test": dist(o_old["steps"]), "pose_tol": dist(o_new["steps"])}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    name, power = card()
    for fn in (ur5, g1):
        out = fn(args.regions)
        out.update(card=name, power_limit=power, regions=args.regions,
                   timing="median over regions, one CUDA-graph replay after an L2 flush, variants alternated")
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

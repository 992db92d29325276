#!/usr/bin/env python3
"""Time the backward of a converged solve against the solve itself, on the two workloads of
scripts/converge_bench.py:

  UR5 at B = 65536: the task set of examples/arm_ur5_reach_batched.py, tol = 1e-5, max_steps = 200;
  G1 + CoM at B = 16384: the humanoid task set of the tests, max_steps = 200, tol as in
      converge_bench.py.

  (a) one BatchedIK.converge launch;
  (b) one BatchedIK.converge_vjp launch at (a)'s solutions with a random grad_q: the backward
      pass that loss.backward() runs through converge's q.

Both are captured in CUDA graphs and timed over --regions regions (median reported), each region
behind an L2 flush and a short device-side spin, alternating (a) and (b).  The card name and power
limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line per workload.

    python scripts/converge_grad_bench.py [--regions 11]
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import converge_bench as cb  # noqa: E402


def measure(name, setup, B, max_steps, regions):
    ik, tasks, q0, targets, tol = setup(B)
    dev = q0.device
    res = ik.converge(q0, targets, tasks, tol, max_steps)
    q_star = res.q.clone()
    grad_q = torch.randn(q_star.shape, device=dev, generator=torch.Generator(dev).manual_seed(0))
    out_a = [torch.empty_like(q0), torch.empty(B, device=dev), torch.empty(B, device=dev, dtype=torch.int32),
             torch.empty(B, device=dev, dtype=torch.int32)]
    gt = torch.empty((B, ik.target_stride), device=dev)
    st = torch.empty(B, device=dev, dtype=torch.int32)
    variants = {
        "a_converge": lambda: ik.converge(q0, targets, tasks, tol, max_steps, *out_a),
        "b_converge_vjp": lambda: ik.converge_vjp(q_star, targets, grad_q, gt, st),
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
        for v, g in graphs.items():
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda._sleep(300000)  # the host queues the region meanwhile
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) * 1e3)
    cname, power = cb.card()
    out = {"workload": name, "card": cname, "power_limit": power, "batch": B, "tol": tol, "max_steps": max_steps,
           "regions": regions, "timing": "median over regions; one CUDA-graph replay after an L2 flush"}
    for v, ts in times.items():
        out[v] = {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
    out["b_over_a"] = round(out["b_converge_vjp"]["us"] / out["a_converge"]["us"], 4)
    out["converged_fraction"] = round(float(res.converged.float().mean()), 5)
    out["vjp_not_posdef"] = int((st == 4).sum())
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    measure("ur5", cb.ur5, 65536, 200, args.regions)
    measure("g1_com", cb.g1, 16384, 200, args.regions)


if __name__ == "__main__":
    main()

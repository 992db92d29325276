#!/usr/bin/env python3
"""Time solving to a tolerance three ways, on two workloads:

  UR5 at B = 65536: the task set of examples/arm_ur5_reach_batched.py (one FrameTask(tool0),
      dt = 1e-2, damping = 1e-8, targets FK(q0 + delta)), tol = 1e-5, max_steps = 200;
  G1 + CoM at B = 16384: the humanoid task set of the tests (five frame tasks, posture, CoM;
      the tree kernel), max_steps = 200.  The stopping test takes the CoM task and the frame tasks
      whose six costs are all non-zero (the two ankles): a component with zero cost is not driven
      to zero.  The posture task keeps them from reaching zero error, so tol is the median error
      after a 40-step rollout (about half the instances stop before step 40).

  (a) one BatchedIK.converge launch;
  (b) one BatchedIK.rollout of a fixed step count equal to the largest `steps` (a) returned;
  (c) the host-driven loop a user writes without converge: rollout in chunks of 10 steps, then
      pk_task_terms_batched per stopping task, a reduction and a host synchronisation, until every
      instance has converged or max_steps is reached (not graph-captured: it branches on the host).

(a) and (b) are captured in CUDA graphs and timed over --regions regions (median reported), each
region behind an L2 flush and a short device-side spin, as bench.py does; (c) is timed with a
host clock around the whole loop, after the same flush.  The distribution of `steps` is reported.
The card name and power limit come from a read-only nvidia-smi query in the same run.  Prints one
JSON line per workload.

    python scripts/converge_bench.py [--regions 11]
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as exc:  # pragma: no cover
        return torch.cuda.get_device_name(0), f"unknown ({exc})"


def ur5(B):
    import importlib.util

    spec = importlib.util.spec_from_file_location("reach", os.path.join(ROOT, "examples", "arm_ur5_reach_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    ik, task, q0, targets = ex.setup(B)
    return ik, [task], q0, targets, ex.TOL


def g1(B):
    from pink_b200 import BatchedIK, _cabi
    from tests import helpers

    sc = helpers.humanoid_scenario("g1_description", B, with_com=True)
    ik = BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, safety_break=sc.safety_break,
                   batch_size=B)
    _, targets, _ = sc.problem()
    tasks = [t for k, t in enumerate(ik.tasks) if int(ik.prob.tasks[k].type) == _cabi.PK_TASK_COM
             or (int(ik.prob.tasks[k].type) == _cabi.PK_TASK_FRAME and min(ik.prob.tasks[k].cost) > 0)]
    q0 = torch.as_tensor(sc.q32, device="cuda")
    targets = torch.as_tensor(targets, device="cuda").contiguous()
    q40, _, _ = ik.rollout(q0, targets, 40)
    tol = float("%.3g" % float(task_error(ik, tasks, q40, targets).median()))
    return ik, tasks, q0, targets, tol


def task_error(ik, tasks, q, targets):
    from pink_b200 import _cabi

    err = torch.zeros(q.shape[0], device="cuda")
    for t in tasks:
        k = next(k for k, t0 in enumerate(ik.tasks) if t0 is t)
        rows = 3 if int(ik.prob.tasks[k].type) == _cabi.PK_TASK_COM else 6
        e, _ = ik.engine.task_terms(ik.prob, k, rows, q, targets)
        err = torch.maximum(err, torch.linalg.vector_norm(e, dim=1))
    return err


def host_loop(ik, tasks, q0, targets, tol, max_steps, chunk=10):
    """rollout in chunks, then the task errors and a synchronisation; returns (q, steps run)."""
    q = q0.clone()
    done = 0
    while done < max_steps:
        n = min(chunk, max_steps - done)
        q, _, _ = ik.rollout(q, targets, n)
        done += n
        if bool((task_error(ik, tasks, q, targets) <= tol).all()):  # synchronises
            break
    return q, done


def measure(name, setup, B, max_steps, regions):
    ik, tasks, q0, targets, tol = setup(B)
    dev = q0.device
    res = ik.converge(q0, targets, tasks, tol, max_steps)
    torch.cuda.synchronize()
    steps = res.steps.cpu().numpy()
    k_max = int(steps.max())
    out_a = [torch.empty_like(q0), torch.empty(B, device=dev), torch.empty(B, device=dev, dtype=torch.int32),
             torch.empty(B, device=dev, dtype=torch.int32)]
    q_b = torch.empty_like(q0)
    v_b = torch.empty((B, ik.nv), device=dev)
    s_b = torch.empty(B, device=dev, dtype=torch.int32)
    variants = {
        "a_converge": lambda: ik.converge(q0, targets, tasks, tol, max_steps, *out_a),
        "b_rollout_fixed_steps": lambda: ik.rollout(q0, targets, max(k_max, 1), q_b, v_b, s_b),
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
    host_loop(ik, tasks, q0, targets, tol, max_steps)  # warm-up
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    flush = torch.empty(2 * l2, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {v: [] for v in list(graphs) + ["c_host_loop"]}
    c_steps = 0
    for _ in range(regions):
        for v, g in graphs.items():  # variants interleaved region by region
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda._sleep(300000)  # the host queues the region meanwhile
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) * 1e3)
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, c_steps = host_loop(ik, tasks, q0, targets, tol, max_steps)
        torch.cuda.synchronize()
        times["c_host_loop"].append((time.perf_counter() - t0) * 1e6)
    cname, power = card()
    out = {"workload": name, "card": cname, "power_limit": power, "batch": B, "tol": tol, "max_steps": max_steps,
           "regions": regions, "timing": "median over regions; (a), (b) one CUDA-graph replay after an L2 flush, "
                                         "(c) host clock around the loop after an L2 flush"}
    for v, ts in times.items():
        out[v] = {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
    out["b_rollout_fixed_steps"]["steps"] = max(k_max, 1)
    out["c_host_loop"]["steps"] = c_steps
    a = out["a_converge"]["us"]
    for v in ("b_rollout_fixed_steps", "c_host_loop"):
        out[v]["a_speedup"] = round(out[v]["us"] / a, 3)
    conv = res.converged.cpu().numpy()
    out["converged_fraction"] = round(float(conv.mean()), 5)
    out["steps"] = {"mean": round(float(steps.mean()), 2),
                    "p50_p90_p99_max": [int(np.percentile(steps, p)) for p in (50, 90, 99)] + [k_max],
                    "mean_over_warps_of_warp_max": round(float(steps[: B // 32 * 32].reshape(-1, 32).max(1).mean()), 2)}
    out["failed_instances"] = int(((res.status.cpu().numpy() & 3) != 0).sum())
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    measure("ur5", ur5, 65536, 200, args.regions)
    measure("g1_com", g1, 16384, 200, args.regions)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Time a K-step closed loop with per-step targets on the benchmark workload (UR5, FrameTask(tool0)
+ PostureTask, default limits, B = 65536 per call), four ways:

  (a) a CUDA graph of K x (BatchedIK.solve + engine.integrate) on the per-step target slices;
  (b) one BatchedIK.rollout_trajectory launch without records;
  (c) one rollout_trajectory launch with all three records (q, v and status of every step);
  (d) for context, the fixed-target BatchedIK.rollout of the same K steps on the first step's
      targets (one launch of the PDL instantiation of the chain kernel).

Each variant is captured in a CUDA graph and timed over --regions regions (median reported), each
region behind an L2 flush and a short device-side spin, as bench.py does.  The card name and power
limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line.

    python scripts/rollout_trajectory_bench.py [--batch 65536] [--steps 20] [--regions 11]
"""

import argparse
import json
import math
import os
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    B, K = args.batch, args.steps

    from pink_b200 import BatchedIK, FrameTask, PostureTask, workloads
    from pink_b200.engine import get_engine
    from pink_b200.limits import ConfigurationLimit, VelocityLimit
    from pink_b200.robots import load_robot_description

    device = torch.device("cuda", 0)
    model = load_robot_description("ur5_description").model
    eng = get_engine(model, device)
    table = eng.table
    rng = np.random.default_rng(workloads.SEED)
    q = workloads.sample_configurations(table, B, rng)
    qt = workloads.perturb_configurations(table, q, rng)
    q0 = torch.as_tensor(q, dtype=torch.float32, device=device)
    oMf, _ = eng.forward_kinematics(torch.as_tensor(qt, dtype=torch.float32, device=device))
    base = oMf[:, table.frame_names.index("tool0")].reshape(B, 12).contiguous()
    # per-step targets: the sinusoid of examples/arm_ur5.py (0.1 m, 2 rad/s, one phase per arm) on p_y
    phase = torch.as_tensor(rng.uniform(0.0, 2.0 * math.pi, size=B), dtype=torch.float32, device=device)
    t = workloads.UR5_DT * torch.arange(K, dtype=torch.float32, device=device)
    rows = base.unsqueeze(0).repeat(K, 1, 1)
    rows[:, :, 7] += 0.1 * torch.sin(2.0 * t[:, None] + phase[None, :])
    rows = rows.contiguous()

    frame_task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    frame_task.set_target(base)
    posture_task = PostureTask(cost=1e-3)
    posture_task.set_target(workloads.ur5_posture_reference(model))
    ik = BatchedIK(model, [frame_task, posture_task], workloads.UR5_DT, damping=workloads.UR5_DAMPING,
                   limits=[ConfigurationLimit(model), VelocityLimit(model)], safety_break=True, device=device,
                   batch_size=B)

    q_a = torch.empty_like(q0)
    v_a = torch.empty((B, 6), device=device)
    s_a = torch.empty((B,), dtype=torch.int32, device=device)

    def loop():
        src = q0
        for s in range(K):
            ik.solve(src, rows[s], v_a, s_a)
            eng.integrate(src, v_a, workloads.UR5_DT, out=q_a)
            src = q_a

    results = {}

    def fused(record):
        def run():
            results[record] = ik.rollout_trajectory(q0, rows, K, record=record)
        return run

    def fixed():
        results["fixed"] = ik.rollout(q0, rows[0], K)

    variants = {"a_graph_solve_integrate": loop, "b_trajectory": fused(False), "c_trajectory_records": fused(True),
                "d_rollout_fixed_targets": fixed}
    graphs = {}
    for name, fn in variants.items():
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):
            fn()  # warm-up outside the capture
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        g.replay()
        torch.cuda.synchronize()
        graphs[name] = g

    l2 = torch.cuda.get_device_properties(device).L2_cache_size
    flush = torch.empty(2 * l2, dtype=torch.uint8, device=device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {name: [] for name in graphs}
    for _ in range(args.regions):
        for name, g in graphs.items():  # variants interleaved region by region
            flush.zero_()
            torch.cuda.synchronize()
            torch.cuda._sleep(300000)  # the host queues the region meanwhile
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3)

    name, power = card()
    out = {"card": name, "power_limit": power, "batch": B, "steps": K, "regions": args.regions,
           "timing": "median over regions, each one CUDA-graph replay after an L2 flush"}
    for v, ts in times.items():
        med = float(np.median(ts))
        out[v] = {"us_per_call": round(med, 2), "us_per_step": round(med / K, 3),
                  "spread_us": [round(min(ts), 2), round(max(ts), 2)]}
    # bytes per instance-step: the 48 B targets row read; (c) also writes 24 B q + 24 B v + 4 B status
    for v, nbytes in (("b_trajectory", 48), ("c_trajectory_records", 100)):
        out[v]["GB_per_s_targets_and_records"] = round(nbytes * B * K / (out[v]["us_per_call"] * 1e-6) / 1e9, 1)
    a_ms = out["a_graph_solve_integrate"]["us_per_call"]
    for v in ("b_trajectory", "c_trajectory_records", "d_rollout_fixed_targets"):
        out[v]["speedup_vs_a"] = round(a_ms / out[v]["us_per_call"], 3)
    # the variants compute the same loop (no instance fails a step here)
    rb, rc = results[False], results[True]
    torch.cuda.synchronize()
    out["max_abs_q_b_minus_a"] = float((rb.q - q_a).abs().max())
    out["b_equals_c"] = bool(torch.equal(rb.q, rc.q) and torch.equal(rb.v, rc.v))
    out["failed_instances"] = int((rb.status & 7).ne(0).sum())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

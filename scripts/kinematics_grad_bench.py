#!/usr/bin/env python3
"""Time the differentiable forward kinematics (pink_b200.kinematics) on three workloads:

  UR5 at B = 65536 with [tool0];
  UR5 at B = 65536 with the six link frames and tool0;
  G1 at B = 16384 with both feet, both hands (wrist-yaw links), the pelvis and the CoM.

  (a) one pk_frame_placements_batched launch (the forward);
  (b) one pk_frame_placements_vjp_batched launch with random gradients of every output (the
      backward that loss.backward() runs);
  (c) one pk_forward_kinematics_batched launch: every frame of the model (and the CoM on G1);
  (d) the same outputs from forward kinematics written in plain torch ops in this script,
      forward and backward (torch.autograd), as a user would write it without the library.

Each is captured in a CUDA graph and timed over --regions regions (median reported), each region
behind an L2 flush and a short device-side spin, alternating the variants.  Bytes per instance are
those the launch must move (q, the requested frames, the gradients), and the bandwidth is those
bytes over the median time, against NVIDIA's 3.35 TB/s data-sheet figure for the H100 SXM.  The
card name and power limit come from a read-only nvidia-smi query in the same run.  Prints one JSON
line per workload.

    python scripts/kinematics_grad_bench.py [--regions 11]
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
from pink_b200 import kinematics, workloads  # noqa: E402
from pink_b200.engine import get_engine  # noqa: E402
from tests import helpers  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet

UR5_LINKS = ["shoulder_link", "upper_arm_link", "forearm_link", "wrist_1_link", "wrist_2_link", "wrist_3_link", "tool0"]
G1_FRAMES = ["left_ankle_roll_link", "right_ankle_roll_link", "left_wrist_yaw_link", "right_wrist_yaw_link", "pelvis"]


class TorchFK:
    """Forward kinematics of the requested frames and the CoM in plain torch ops, batched (the
    region (d) baseline; differentiable by torch.autograd)."""

    def __init__(self, table, frames, com, dev):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), dtype=torch.float32, device=dev)  # noqa: E731
        self.m = table
        self.frames = frames
        self.com = com
        self.jR, self.jp, self.axis = t(table.joint_R), t(table.joint_p), t(table.axis)
        self.fR, self.fp = t(table.frame_R), t(table.frame_p)
        self.mass_host = np.asarray(table.mass, dtype=np.float64)  # tested on the host: no sync in a capture
        self.mass, self.cl, self.M = t(self.mass_host), t(table.com), float(self.mass_host.sum())

    def __call__(self, q):
        m, B = self.m, q.shape[0]
        rq = 7 if m.free_flyer else 0
        if m.free_flyer:
            u = q[:, 3:7] / torch.linalg.vector_norm(q[:, 3:7], dim=1, keepdim=True)
            x, y, z, w = u.unbind(1)
            R0 = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                              2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                              2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(B, 3, 3)
            p0 = q[:, 0:3]
        else:
            R0 = torch.eye(3, device=q.device).expand(B, 3, 3)
            p0 = torch.zeros((B, 3), device=q.device)
        Rs, ps = [], []
        for j in range(m.njoints):
            par = int(m.parent[j])
            Rp, pp = (R0, p0) if par < 0 else (Rs[par], ps[par])
            a = self.axis[j]
            qj = q[:, rq + j]
            if int(m.jtype[j]) == 0:
                K = torch.stack([torch.zeros_like(a[0]), -a[2], a[1], a[2], torch.zeros_like(a[0]), -a[0],
                                 -a[1], a[0], torch.zeros_like(a[0])]).reshape(3, 3)
                s, c = torch.sin(qj)[:, None, None], torch.cos(qj)[:, None, None]
                Rm = torch.eye(3, device=q.device) + s * K + (1 - c) * (K @ K)
                Rl, pl = self.jR[j] @ Rm, self.jp[j].expand(B, 3)
            else:
                Rl, pl = self.jR[j].expand(B, 3, 3), self.jp[j] + qj[:, None] * (self.jR[j] @ a)
            Rs.append(Rp @ Rl)
            ps.append(pp + (Rp @ pl[..., None])[..., 0])
        out = []
        for f in self.frames:
            b = int(m.frame_body[f])
            Rb, pb = (R0, p0) if b == -1 else (Rs[b], ps[b]) if b >= 0 else (torch.eye(3, device=q.device).expand(
                B, 3, 3), torch.zeros((B, 3), device=q.device))
            out.append(torch.cat([Rb @ self.fR[f], (pb + (Rb @ self.fp[f][:, None])[..., 0])[..., None]], -1))
        oMf = torch.stack(out, 1)
        com = None
        if self.com:
            acc = 0.0
            for b in range(-1, m.njoints):
                if self.mass_host[b + 1] == 0.0:
                    continue
                Rb, pb = (R0, p0) if b < 0 else (Rs[b], ps[b])
                acc = acc + self.mass[b + 1] * (pb + (Rb @ self.cl[b + 1][:, None])[..., 0])
            com = acc / self.M
        return oMf, com


def measure(name, robot, B, frame_names, com, regions):
    _, model, table = helpers.load(robot)
    dev = torch.device("cuda", 0)
    frames = [table.frame_names.index(n) for n in frame_names]
    F = len(frames)
    q = torch.as_tensor(workloads.sample_configurations(table, B, np.random.default_rng(0)), dtype=torch.float32,
                        device=dev).contiguous()
    gen = torch.Generator(dev).manual_seed(1)
    W = torch.randn((B, F, 3, 4), device=dev, generator=gen)
    Wc = torch.randn((B, 3), device=dev, generator=gen) if com else None
    eng = get_engine(model, dev)
    tfk = TorchFK(table, frames, com, dev)
    qg = q.clone().requires_grad_(True)

    def torch_fwd_bwd():
        qg.grad = None
        oMf, c = tfk(qg)
        loss = (oMf * W).sum() + ((c * Wc).sum() if com else 0.0)
        loss.backward()

    # the torch baseline computes what the kernels compute
    with torch.no_grad():
        o_ref, c_ref = tfk(q)
    fp = kinematics.frame_placements(model, q, frames, com=com)
    fwd_err = float((fp.oMf - o_ref).abs().max())
    torch_fwd_bwd()
    g_lib = kinematics.frame_placements_vjp(model, q, frames, W, Wc)
    grad_err = float(((qg.grad - g_lib).abs().max(1).values / qg.grad.abs().max(1).values.clamp_min(1e-12)).max())
    variants = {
        "a_forward": lambda: kinematics.frame_placements(model, q, frames, com=com),
        "b_vjp": lambda: kinematics.frame_placements_vjp(model, q, frames, W, Wc),
        "c_fk_all_frames": lambda: eng.forward_kinematics(q, want_com=com),
        "d_torch_fwd_bwd": torch_fwd_bwd,
    }
    graphs = {}
    for v, fn in variants.items():
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
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
    nq = table.nq
    out_b = 4 * (12 * F + (3 if com else 0))
    bytes_per_instance = {
        "a_forward": 4 * nq + out_b,
        "b_vjp": 4 * nq + out_b + 4 * nq,
        "c_fk_all_frames": 4 * nq + 4 * (12 * table.nframes + (3 if com else 0)),
    }
    cname, power = cb.card()
    out = {"workload": name, "card": cname, "power_limit": power, "batch": B, "frames": frame_names, "com": com,
           "regions": regions, "timing": "median over regions; one CUDA-graph replay after an L2 flush",
           "torch_forward_max_abs_diff": fwd_err, "torch_grad_max_rel_diff": grad_err}
    for v, ts in times.items():
        r = {"us": round(float(np.median(ts)), 1), "spread_us": [round(min(ts), 1), round(max(ts), 1)]}
        if v in bytes_per_instance:
            bpi = bytes_per_instance[v]
            bw = bpi * B / (np.median(ts) * 1e-6)
            r.update({"bytes_per_instance": bpi, "GB_per_s": round(bw / 1e9, 1),
                      "of_3.35TB_per_s": round(bw / HBM_BYTES_PER_S, 4)})
        out[v] = r
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=11)
    args = ap.parse_args()
    measure("ur5_tool0", "ur5_description", 65536, ["tool0"], False, args.regions)
    measure("ur5_links", "ur5_description", 65536, UR5_LINKS, False, args.regions)
    measure("g1_feet_hands_pelvis_com", "g1_description", 16384, G1_FRAMES, True, args.regions)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""A batch of G1-class humanoids reaching with both wrists, solved to separate position and
orientation tolerances: 2 mm and 0.02 rad.

The task set is the G1 set of the benchmark's humanoid configuration (pelvis, both ankles, both
wrists, posture, CoM; no barrier).  Several of its frame tasks leave axes unweighed: the pelvis
has position cost 0 and both wrists have orientation cost 0.  The default stopping test of
``BatchedIK.converge`` measures each task's whole 6-vector, so it can never stop on this set:
the unweighed components are never driven to zero.  With ``orientation_tol`` the test counts
only the weighed components, translations in metres against ``tol`` and rotation angles in
radians against ``orientation_tol``, so every frame task and the CoM can be in the stopping set.

Each humanoid starts at a random configuration.  Its targets are taken at a configuration that
moves only its arm joints: the wrists get new position targets while the feet, the pelvis and the
CoM hold, and the posture task keeps pulling toward the start.  The example prints the solved
fraction and the percentiles of the steps taken.

    python examples/humanoid_g1_reach_batched.py --batch 4096 --max-steps 200
"""

import argparse

import numpy as np
import torch

import pink_b200 as pink
from pink_b200 import workloads
from pink_b200.model import JointModelFreeFlyer
from pink_b200.robots import load_robot_description
from pink_b200.solve_ik import describe_problem
from pink_b200.tasks import ComTask, FrameTask, PostureTask

DT = 1.0 / 200.0
TOL = 2e-3  # m, for the translations and the CoM
ORIENTATION_TOL = 2e-2  # rad
ARMS = ("shoulder", "elbow", "wrist")


def setup(batch: int = 4096, device: str = "cuda", seed: int = 0, sigma: float = 0.15):
    """``(ik, stop_tasks, q0 [batch, nq], targets [batch, target_stride])``: every frame task and
    the CoM in ``stop_tasks``; the targets at the start with the arm joints moved by N(0, sigma)."""
    robot = load_robot_description("g1_description", root_joint=JointModelFreeFlyer())
    model = robot.model
    table = model.table()
    rng = np.random.default_rng(seed)
    q = workloads.sample_configurations(table, batch, rng, near_limit_fraction=0.0)
    qt = q.copy()
    arms = [7 + i for i, n in enumerate(table.joint_names) if any(a in n for a in ARMS)]
    qt[:, arms] = workloads.perturb_configurations(table, q, rng, sigma=sigma)[:, arms]
    target = pink.Configuration(model, robot.data, torch.as_tensor(qt, dtype=torch.float32, device=device))
    frames = []
    for frame, pc, oc in workloads.G1_FRAME_TASKS:
        t = FrameTask(frame, position_cost=pc, orientation_cost=oc)
        t.set_target(target.get_transform_frame_to_world(frame))
        frames.append(t)
    posture = PostureTask(cost=workloads.G1_POSTURE_COST)
    posture.set_target(torch.as_tensor(q, dtype=torch.float32, device=device))
    com = ComTask(cost=workloads.G1_COM_COST)
    com.set_target(target.get_center_of_mass())
    tasks = frames + [posture, com]
    ik = pink.BatchedIK(model, tasks, DT, damping=workloads.G1_DAMPING, safety_break=False, batch_size=batch,
                        device=device)
    # the targets row in the layout of the problem (ik.target_layout)
    _, parts, _ = describe_problem(model, batch, tasks, DT, workloads.G1_DAMPING,
                                   [model.configuration_limit, model.velocity_limit], False)
    targets = torch.cat([p.to(device=device, dtype=torch.float32) for p in parts], dim=1).contiguous()
    q0 = torch.as_tensor(q, dtype=torch.float32, device=device).contiguous()
    return ik, frames + [com], q0, targets


def run(batch: int = 4096, max_steps: int = 200, device: str = "cuda", seed: int = 0, tol: float = TOL,
        orientation_tol: float = ORIENTATION_TOL, verbose: bool = False):
    """The :class:`pink_b200.batched.Convergence` of the batch."""
    ik, stop_tasks, q0, targets = setup(batch, device, seed)
    res = ik.converge(q0, targets, stop_tasks, tol, max_steps, orientation_tol=orientation_tol)
    if verbose:
        steps = res.steps[res.converged].float().cpu().numpy()
        pct = np.percentile(steps, [50, 90, 99]) if steps.size else [float("nan")] * 3
        print(f"{batch} G1 humanoids, every frame task and the CoM within {tol * 1e3:g} mm and "
              f"{orientation_tol:g} rad: solved {res.converged.float().mean().item():.4f}; steps of the solved "
              f"p50 {pct[0]:.0f}, p90 {pct[1]:.0f}, p99 {pct[2]:.0f} (max_steps {max_steps})")
    return res


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument("--batch", type=int, default=4096)
    parser.add_argument("--max-steps", type=int, default=200)
    args = parser.parse_args()
    run(args.batch, args.max_steps, verbose=True)

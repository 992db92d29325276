#!/usr/bin/env python3
"""The closed loop of the reference's ``examples/arm_ur5.py`` for a batch of arms.

Every instance tracks its own end-effector target (a sinusoid with an instance-specific
phase) with ``FrameTask(tool0) + PostureTask`` under the default limits; ``solve_ik`` and
``integrate_inplace`` are the reference's calls, with a leading batch dimension.  With
``--fused`` the whole trajectory of targets is built up front as one ``[steps, batch, 12]``
tensor and the loop runs in a single ``BatchedIK.rollout_trajectory`` launch.

    python examples/arm_ur5_batched.py --batch 65536 --steps 200 [--fused]
"""

import argparse
import math

import numpy as np
import torch

import pink_b200 as pink
from pink_b200 import solve_ik
from pink_b200.robots import load_robot_description
from pink_b200.tasks import FrameTask, PostureTask
from pink_b200.utils import custom_configuration_vector


def run(batch: int = 4096, steps: int = 100, device: str = "cuda", dt: float = 1.0 / 200.0, seed: int = 0,
        fused: bool = False):
    """Returns ``(final position error per instance [batch], final configurations)``.  ``fused``:
    one trajectory rollout instead of a ``solve_ik`` + ``integrate_inplace`` call per step."""
    robot = load_robot_description("ur5_description", root_joint=None)
    end_effector_task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    posture_task = PostureTask(cost=1e-3)
    tasks = [end_effector_task, posture_task]

    q_ref = custom_configuration_vector(robot, shoulder_lift_joint=1.0, shoulder_pan_joint=1.0, elbow_joint=1.0)
    rng = np.random.default_rng(seed)
    q0 = q_ref + 0.05 * rng.standard_normal((batch, robot.model.nq))
    configuration = pink.Configuration(robot.model, robot.data, torch.as_tensor(q0, dtype=torch.float32, device=device))
    posture_task.set_target(q_ref)  # one posture target shared by all instances
    targets = configuration.get_transform_frame_to_world("tool0")  # [batch, 3, 4] = [R | p]
    phase = torch.as_tensor(rng.uniform(0.0, 2.0 * math.pi, size=batch), dtype=torch.float32, device=targets.device)

    if fused:
        # tool0 target rows [R | p] row-major (p_y at 7, p_z at 11) for every step, then one launch
        end_effector_task.set_target(targets)  # fixes the layout: 12 floats per instance and step
        ik = pink.BatchedIK(robot.model, tasks, dt, batch_size=batch)
        times, t = [], 0.0
        for _ in range(steps):
            times.append(2.0 * t)
            t += dt
        rows = targets.reshape(1, batch, 12).repeat(steps, 1, 1)
        rows[:, :, 7] = 0.5 + 0.1 * torch.sin(torch.tensor(times, dtype=torch.float32, device=targets.device)[:, None]
                                              + phase)
        rows[:, :, 11] = 0.2
        res = ik.rollout_trajectory(configuration.q_device, rows, record=False)
        if bool((res.status & 7).any()):  # no solution, outside the limits or not positive definite
            raise pink.PinkError(f"{int(((res.status & 7) != 0).sum())} arms failed a step")
        configuration.update(res.q)
        targets = rows[-1].reshape(batch, 3, 4)
        reached = configuration.get_transform_frame_to_world("tool0")
        error = torch.linalg.norm(reached[:, :, 3] - targets[:, :, 3], dim=1)
        return error, configuration.q

    t = 0.0
    for _ in range(steps):
        targets[:, 1, 3] = 0.5 + 0.1 * torch.sin(2.0 * t + phase)
        targets[:, 2, 3] = 0.2
        end_effector_task.set_target(targets)
        velocity = solve_ik(configuration, tasks, dt, solver="quadprog")  # [batch, 6]
        configuration.integrate_inplace(velocity, dt)
        t += dt
    reached = configuration.get_transform_frame_to_world("tool0")
    error = torch.linalg.norm(reached[:, :, 3] - targets[:, :, 3], dim=1)
    return error, configuration.q


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--fused", action="store_true", help="one rollout_trajectory launch for the whole loop")
    args = ap.parse_args()
    err, _ = run(args.batch, args.steps, fused=args.fused)
    print(f"{args.batch} arms, {args.steps} steps: position error median {err.median().item():.4f} m, "
          f"max {err.max().item():.4f} m")

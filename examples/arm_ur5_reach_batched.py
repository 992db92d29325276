#!/usr/bin/env python3
"""The reaching loop of the reference's ``examples/inverse_kinematics_ur10.py`` for a batch of
UR5 arms: ``while norm(task.compute_error(configuration)) > stop_thres`` step the IK, per
instance, in one ``BatchedIK.converge`` launch.

Every instance starts at its own configuration ``q0`` and reaches for the end-effector pose of
``q0 + delta`` (reachable by construction) with a single ``FrameTask``.  The reference stops at
``stop_thres = 1e-8``; in fp32 a pose resolves to about 1e-7, so this example stops at 1e-5
(a tolerance below about 1e-6 may run to ``max_steps``).

    python examples/arm_ur5_reach_batched.py --batch 65536 --max-steps 200
"""

import argparse

import numpy as np
import torch

import pink_b200 as pink
from pink_b200.robots import load_robot_description
from pink_b200.tasks import FrameTask
from pink_b200.utils import custom_configuration_vector

DT = 1e-2
DAMPING = 1e-8
TOL = 1e-5


def setup(batch: int = 4096, device: str = "cuda", seed: int = 0, sigma: float = 0.2):
    """``(ik, task, q0 [batch, 6], targets [batch, 12])`` of the example's problem."""
    robot = load_robot_description("ur5_description", root_joint=None)
    task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    q_ref = custom_configuration_vector(robot, shoulder_lift_joint=-1.0, elbow_joint=1.5, wrist_1_joint=-1.0)
    rng = np.random.default_rng(seed)
    q0 = q_ref + 0.3 * rng.standard_normal((batch, robot.model.nq))
    q_goal = q0 + sigma * rng.standard_normal((batch, robot.model.nq))
    goal = pink.Configuration(robot.model, robot.data, torch.as_tensor(q_goal, dtype=torch.float32, device=device))
    task.set_target(goal.get_transform_frame_to_world("tool0"))  # [batch, 3, 4] = [R | p]
    ik = pink.BatchedIK(robot.model, [task], DT, damping=DAMPING, batch_size=batch)
    q0 = torch.as_tensor(q0, dtype=torch.float32, device=device).contiguous()
    targets = goal.get_transform_frame_to_world("tool0").reshape(batch, 12).contiguous()
    return ik, task, q0, targets


def run(batch: int = 4096, max_steps: int = 200, device: str = "cuda", seed: int = 0, tol: float = TOL,
        verbose: bool = False):
    """Returns the :class:`pink_b200.batched.Convergence` of the batch."""
    ik, task, q0, targets = setup(batch, device, seed)
    res = ik.converge(q0, targets, [task], tol, max_steps)
    if verbose:
        steps = res.steps.float().cpu().numpy()
        p50, p90, p99 = np.percentile(steps, [50, 90, 99])
        print(f"converged: {res.converged.float().mean().item():.4f} of {batch} arms (tol {tol:g})")
        print(f"steps: median {p50:.0f}, p90 {p90:.0f}, p99 {p99:.0f}, max {int(steps.max())}")
    return res


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument("--batch", type=int, default=4096)
    parser.add_argument("--max-steps", type=int, default=200)
    parser.add_argument("--tol", type=float, default=TOL)
    args = parser.parse_args()
    run(args.batch, args.max_steps, tol=args.tol, verbose=True)

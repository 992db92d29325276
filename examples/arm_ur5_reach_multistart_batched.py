#!/usr/bin/env python3
"""Reaching targets anywhere in a UR5's workspace from one home pose, with and without seeds.

Every target is the end-effector pose of a configuration drawn uniformly within the joint
limits (reachable by construction), and every arm starts at the same home pose.  A differential
IK step only follows the local gradient of the task error, so from that one start some targets
are not reached within ``max_steps``: the loop stalls against a joint limit or settles in a local
minimum.  ``BatchedIK.converge_multistart`` starts each target from S seeds at once (seed 0 the
home pose, the others uniform within the limits, :meth:`BatchedIK.sample_seeds`) and stops a
target as soon as one of its seeds reaches ``tol``.  The example prints the converged fraction
and the step percentiles for S = 1 and S = 8.

    python examples/arm_ur5_reach_multistart_batched.py --batch 8192 --max-steps 200
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


def setup(batch: int = 8192, device: str = "cuda", seed: int = 0):
    """``(ik, task, q_home [batch, 6], targets [batch, 12])``: targets = FK of configurations
    uniform within the limits, one shared home pose."""
    robot = load_robot_description("ur5_description", root_joint=None)
    model = robot.model
    task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    q_home = custom_configuration_vector(robot, shoulder_lift_joint=-1.0, elbow_joint=1.5, wrist_1_joint=-1.0)
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(model.lowerPositionLimit), np.asarray(model.upperPositionLimit)
    q_goal = rng.uniform(lo, hi, size=(batch, model.nq))
    goal = pink.Configuration(model, robot.data, torch.as_tensor(q_goal, dtype=torch.float32, device=device))
    task.set_target(goal.get_transform_frame_to_world("tool0"))
    ik = pink.BatchedIK(model, [task], DT, damping=DAMPING, batch_size=batch)
    q0 = torch.as_tensor(np.tile(q_home, (batch, 1)), dtype=torch.float32, device=device).contiguous()
    targets = goal.get_transform_frame_to_world("tool0").reshape(batch, 12).contiguous()
    return ik, task, q0, targets


def run(batch: int = 8192, num_seeds: int = 8, max_steps: int = 200, device: str = "cuda", seed: int = 0,
        tol: float = TOL, verbose: bool = False):
    """The :class:`pink_b200.batched.MultistartConvergence` of the batch with ``num_seeds`` seeds."""
    ik, task, q0, targets = setup(batch, device, seed)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    seeds = ik.sample_seeds(q0, num_seeds, generator=g)
    res = ik.converge_multistart(seeds, targets, [task], tol, max_steps)
    if verbose:
        steps = res.steps.float().cpu().numpy()
        p50, p90, p99 = np.percentile(steps, [50, 90, 99])
        print(f"S = {num_seeds:2d}: converged {res.converged.float().mean().item():.4f} of {batch} targets "
              f"(tol {tol:g}); steps median {p50:.0f}, p90 {p90:.0f}, p99 {p99:.0f}, max {int(steps.max())}")
    return res


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument("--batch", type=int, default=8192)
    parser.add_argument("--max-steps", type=int, default=200)
    parser.add_argument("--tol", type=float, default=TOL)
    args = parser.parse_args()
    for s in (1, 8):
        run(args.batch, s, args.max_steps, tol=args.tol, verbose=True)

#!/usr/bin/env python3
"""Reaching the best of several candidate tool poses per instance, as a grasp planner does.

Each instance has G = 8 candidate tool poses (grasps).  Four of them, at random positions in the
list, are end-effector poses of configurations drawn uniformly within the joint limits
(reachable by construction); the other four are the same kind of pose moved out to 2 m from the
base, beyond the arm's reach.  Every arm starts at the same home pose.
``BatchedIK.converge_goalset`` solves every instance toward all of its candidates from S = 4
seeds at once (seed 0 the home pose, the others uniform within the limits) and stops an
instance as soon as one (goal, seed) pair reaches ``tol``.  The winner is the pair with the
smallest error then, with ties going to the earlier goal, so the candidates may be listed in
order of preference.  The example prints the solved fraction and how often each candidate was
chosen.

    python examples/arm_ur5_grasp_goalset_batched.py --batch 8192 --max-steps 200
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
NUM_GOALS = 8
FAR = 2.0  # m from the base: out of the UR5's reach (about 0.85 m from the shoulder)


def setup(batch: int = 8192, device: str = "cuda", seed: int = 0):
    """``(ik, task, q_home [batch, 6], goals [batch, 8, 12], reachable [batch, 8])``."""
    robot = load_robot_description("ur5_description", root_joint=None)
    model = robot.model
    task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    q_home = custom_configuration_vector(robot, shoulder_lift_joint=-1.0, elbow_joint=1.5, wrist_1_joint=-1.0)
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(model.lowerPositionLimit), np.asarray(model.upperPositionLimit)
    q_goal = rng.uniform(lo, hi, size=(batch * NUM_GOALS, model.nq))
    conf = pink.Configuration(model, robot.data, torch.as_tensor(q_goal, dtype=torch.float32, device=device))
    poses = conf.get_transform_frame_to_world("tool0").reshape(batch, NUM_GOALS, 3, 4).clone()
    # half the candidates of each instance, at random places in its list, out of reach
    reachable = torch.as_tensor(np.argsort(rng.random((batch, NUM_GOALS)), axis=1) < NUM_GOALS // 2, device=device)
    p = poses[..., 3]
    far = p / torch.linalg.vector_norm(p, dim=-1, keepdim=True).clamp_min(1e-6) * FAR
    poses[..., 3] = torch.where(reachable[..., None], p, far)
    task.set_target(poses[:, 0])
    ik = pink.BatchedIK(model, [task], DT, damping=DAMPING, batch_size=batch)
    q0 = torch.as_tensor(np.tile(q_home, (batch, 1)), dtype=torch.float32, device=device).contiguous()
    goals = poses.reshape(batch, NUM_GOALS, 12).contiguous()
    return ik, task, q0, goals, reachable


def run(batch: int = 8192, num_seeds: int = 4, max_steps: int = 200, device: str = "cuda", seed: int = 0,
        tol: float = TOL, verbose: bool = False):
    """The :class:`pink_b200.batched.GoalsetConvergence` of the batch, and which goals were
    reachable."""
    ik, task, q0, goals, reachable = setup(batch, device, seed)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    seeds = ik.sample_seeds(q0, num_seeds, generator=g)
    res = ik.converge_goalset(seeds, goals, [task], tol, max_steps)
    if verbose:
        solved = res.converged
        hist = torch.bincount(res.goal[solved].long(), minlength=NUM_GOALS).cpu().tolist()
        steps = res.steps.float().cpu().numpy()
        p50, p90 = np.percentile(steps, [50, 90])
        print(f"G = {NUM_GOALS}, S = {num_seeds}: solved {solved.float().mean().item():.4f} of {batch} instances "
              f"(tol {tol:g}); rounds median {p50:.0f}, p90 {p90:.0f}, max {int(steps.max())}")
        print("chosen goal histogram (solved instances):", hist)
    return res, reachable


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument("--batch", type=int, default=8192)
    parser.add_argument("--seeds", type=int, default=4)
    parser.add_argument("--max-steps", type=int, default=200)
    parser.add_argument("--tol", type=float, default=TOL)
    args = parser.parse_args()
    run(args.batch, args.seeds, args.max_steps, tol=args.tol, verbose=True)

#!/usr/bin/env python3
"""Choosing the approach angle of a grasp by gradient descent through the IK solution.

Each instance grasps a vertical cylinder standing somewhere in front of a UR5.  The gripper
(``tool0``, approach along its z axis) reaches the cylinder horizontally from a yaw angle theta
about the cylinder's axis, so the target pose is a differentiable function of theta.  Every
iteration solves all instances with ``BatchedIK.converge``, evaluates the forearm frame of the
solutions with ``kinematics.frame_placements`` and takes an Adam step on theta that raises the
forearm (loss ``-z``): ``theta -> target -> converge -> frame_placements(q*) -> loss``, with the
gradient through ``converge`` (one implicit-gradient launch) and through the forward kinematics
(one reverse-sweep launch).  The example prints the converged fraction and the mean forearm
height before and after.

    python examples/arm_ur5_grasp_angle_grad_batched.py --batch 4096 --iters 5
"""

import argparse

import numpy as np
import torch

import pink_b200 as pink
from pink_b200 import kinematics
from pink_b200.robots import load_robot_description
from pink_b200.tasks import FrameTask
from pink_b200.utils import custom_configuration_vector

DT = 1e-2
DAMPING = 1e-8
TOL = 1e-5
STANDOFF = 0.12  # m from the cylinder's axis to tool0 along the approach


def grasp_targets(centres: torch.Tensor, theta: torch.Tensor) -> torch.Tensor:
    """``[B, 12]`` tool poses ``[R | p]`` that approach the cylinders at ``centres [B, 3]``
    horizontally from yaw ``theta [B]``: z (approach) = (cos, sin, 0), x = down, y = z x x."""
    c, s = torch.cos(theta), torch.sin(theta)
    z0, one = torch.zeros_like(c), torch.ones_like(c)
    R = torch.stack([torch.stack([z0, -s, c], -1), torch.stack([z0, c, s], -1), torch.stack([-one, z0, z0], -1)], -2)
    p = centres - STANDOFF * torch.stack([c, s, z0], -1)
    return torch.cat([R, p[..., None]], -1).reshape(-1, 12)


def setup(batch: int = 4096, device: str = "cuda", seed: int = 0):
    """``(model, ik, task, q0 [B, 6], centres [B, 3], theta0 [B])``: cylinders on an arc in front
    of the arm, each first approached straight out from the base."""
    robot = load_robot_description("ur5_description", root_joint=None)
    model = robot.model
    task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    rng = np.random.default_rng(seed)
    phi = rng.uniform(-0.8, 0.8, batch)
    r = rng.uniform(0.45, 0.6, batch)
    h = rng.uniform(0.1, 0.35, batch)
    centres = torch.as_tensor(np.stack([r * np.cos(phi), r * np.sin(phi), h], 1), dtype=torch.float32, device=device)
    theta0 = torch.as_tensor(phi + rng.uniform(-0.3, 0.3, batch), dtype=torch.float32, device=device)
    task.set_target(grasp_targets(centres, theta0).reshape(batch, 3, 4))
    ik = pink.BatchedIK(model, [task], DT, damping=DAMPING, batch_size=batch)
    q_home = custom_configuration_vector(robot, shoulder_lift_joint=-1.2, elbow_joint=1.5, wrist_1_joint=-1.9,
                                         wrist_2_joint=-1.57)
    q0 = torch.as_tensor(np.tile(q_home, (batch, 1)), dtype=torch.float32, device=device).contiguous()
    return model, ik, task, q0, centres, theta0


def run(batch: int = 4096, iters: int = 5, lr: float = 0.05, max_steps: int = 400, device: str = "cuda",
        seed: int = 0, verbose: bool = False):
    """``dict`` with the converged fraction and the mean forearm height (over the instances
    converged at both ends) before and after, and the loss of every iteration."""
    model, ik, task, q0, centres, theta0 = setup(batch, device, seed)
    theta = theta0.clone().requires_grad_(True)
    opt = torch.optim.Adam([theta], lr=lr)
    q_start = q0
    record = []
    for it in range(iters + 1):
        targets = grasp_targets(centres, theta).contiguous()
        res = ik.converge(q_start, targets, [task], TOL, max_steps)
        fp = kinematics.frame_placements(model, res.q, ["forearm_link"])
        z = fp.oMf[:, 0, 2, 3]
        loss = -(z * res.converged).sum() / batch
        record.append((res.converged.detach().clone(), z.detach().clone(), loss.item()))
        if verbose:
            print(f"iter {it}: converged {res.converged.float().mean().item():.4f}, "
                  f"mean forearm height {z[res.converged].mean().item():.4f} m, loss {loss.item():.5f}")
        if it == iters:
            break
        opt.zero_grad()
        loss.backward()
        opt.step()
        q_start = res.q.detach()  # warm start: the gradient does not depend on the start
    (ok0, z0, _), (ok1, z1, _) = record[0], record[-1]
    both = ok0 & ok1
    out = {
        "converged_before": ok0.float().mean().item(),
        "converged_after": ok1.float().mean().item(),
        "height_before": z0[both].mean().item(),
        "height_after": z1[both].mean().item(),
        "losses": [r[2] for r in record],
    }
    if verbose:
        print(f"converged fraction {out['converged_before']:.4f} -> {out['converged_after']:.4f}; "
              f"mean forearm height {out['height_before']:.4f} -> {out['height_after']:.4f} m")
    return out


if __name__ == "__main__":
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument("--batch", type=int, default=4096)
    parser.add_argument("--iters", type=int, default=5)
    parser.add_argument("--lr", type=float, default=0.05)
    parser.add_argument("--max-steps", type=int, default=400)
    args = parser.parse_args()
    run(args.batch, args.iters, args.lr, args.max_steps, verbose=True)

"""Implicit gradient of a converged IK solution with respect to the task targets (fp64 numpy).

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).

The IK step solves ``min 1/2 x^T H x + c^T x`` over the box of the limits, with
``c = sum_t alpha_t J_t^T W_t^2 e_t`` (``ik.qp_objective``).  Iterated, it stops where ``x = 0``
is the minimiser: ``c_F(q**, T) = 0`` on the free coordinates F, while the coordinates the QP
holds on a configuration limit stay put.  By the implicit function theorem
``dq**/dT = -(dc_F/dq_F)^-1 dc_F/dT``.  This module evaluates the Gauss-Newton form that the
CUDA kernel runs, ``dc/dq ~ N = sum_t alpha_t J_t^T W_t^2 J_t`` and
``dc/dT ~ sum_t alpha_t J_t^T W_t^2 de_t/dT``; the terms it drops are proportional to the task
errors at the fixed point.

Target perturbations: a frame target moves as ``T* <- T* exp(d)`` (twist ``d = [v; w]``) and
its gradient is returned in the 12 floats ``[R | p]`` as ``[1/2 R [g_w]x | R g_v]``; posture,
CoM and joint-velocity targets move coordinate-wise.
"""

import numpy as np

from . import ik
from . import kinematics as kin
from . import lie
from . import qp
from . import tasks as tk

# a pivot of the triangular factor of N_FF at most this fraction of its column's norm: not
# positive definite to fp32 accuracy (PK_STATUS_NOT_POSDEF)
PIVOT_RTOL = 1e-5


def tangent_gradient(m, q, grad_q):
    """``grad_q [nq]`` -> the tangent gradient ``[nv]``: the transpose of ``d(q (+) dq)/d dq`` at
    ``dq = 0``.  On a free-flyer root ``p += R v`` and ``quat <- quat * (w / 2, 1)``."""
    q = np.asarray(q, dtype=np.float64)
    grad_q = np.asarray(grad_q, dtype=np.float64)
    rq, rv = kin.root_dims(m)
    g = np.zeros(m.nv)
    if m.free_flyer:
        R = lie.quat_to_matrix(q[3:7])
        g[0:3] = R.T @ grad_q[0:3]
        qv, s = q[3:6], q[6]
        gqv, gqw = grad_q[3:6], grad_q[6]
        g[3:6] = 0.5 * (s * gqv + np.cross(gqv, qv) - gqw * qv)
    g[rv:] = grad_q[rq:]
    return g


def held_coordinates(m, q, tasks, dt, damping=1e-12, limits=None):
    """Boolean ``[nv]``: the coordinates the step's QP at ``q`` leaves on a configuration-limit
    bound.  ``limits`` as ``ik.solve_ik``."""
    from . import limits as lim

    if limits is None:
        limits = [("configuration", 0.5), ("velocity", None)]
    H, c, G, h, _, _ = ik.assemble(m, q, tasks, dt, damping, limits)
    held = np.zeros(m.nv, dtype=bool)
    cfg = [e for e in limits if e[0] == "configuration"]
    if not cfg or G is None:
        return held
    x = qp.solve_qp(H, c, G, h, None, None).x
    rq, rv = kin.root_dims(m)
    idx = lim.configuration_limit_indices(m)
    gain = cfg[0][1]
    q = np.asarray(q, dtype=np.float64)
    for i in idx:
        hi = gain * (m.q_max[rq + i - rv] - q[rq + i - rv])
        lo = gain * (m.q_min[rq + i - rv] - q[rq + i - rv])
        tol = 1e-9 * (1.0 + abs(x[i]))
        held[i] = abs(x[i] - hi) <= tol or abs(x[i] - lo) <= tol
    return held


def target_jacobian(m, q, fk, task):
    """``de/dT [k, n_T]`` of one task in its target coordinates (twist ``d`` for frame targets),
    or None for a task without target (LINEAR)."""
    t = task["type"]
    rq, rv = kin.root_dims(m)
    if t == "frame":
        Rf, pf = kin.frame_placement(m, fk, task["frame"])
        Rt, pt = (np.asarray(a, dtype=np.float64) for a in task["target"])
        Rbt, pbt = lie.se3_act_inv(Rf, pf, Rt, pt)
        return lie.jlog6(Rbt, pbt)  # e = log6(T_bt), T_bt <- T_bt exp(d)
    if t == "relative_frame":
        _, (Rtf, ptf) = tk._relative_transforms(m, fk, task)
        # e = log6(T_tf), T_tf <- exp(-d) T_tf
        return -lie.jlog6(Rtf, ptf) @ lie.action(*lie.se3_inv(Rtf, ptf))
    if t == "com":
        return -np.eye(3)
    if t == "posture":
        out = np.zeros((m.nv - rv, m.nq))
        out[:, rq:] = -np.eye(m.nq - rq)
        return out
    if t == "joint_velocity":
        return np.eye(m.nv - rv)
    return None


def frame_gradient_12(R_target, g_twist):
    """Twist gradient ``[g_v; g_w]`` of ``T* <- T* exp(d)`` -> the 12 floats ``[R | p]``."""
    G = np.zeros((3, 4))
    G[:, :3] = 0.5 * R_target @ lie.hat(g_twist[3:6])
    G[:, 3] = R_target @ g_twist[0:3]
    return G.reshape(12)


def normal_matrix(m, q, fk, tasks):
    """``N = sum_t alpha_t J_t^T W_t^2 J_t`` over the tasks whose error depends on q."""
    N = np.zeros((m.nv, m.nv))
    for task in tasks:
        if task["type"] == "joint_velocity":
            continue
        _, J = tk.task_error_jacobian(m, q, fk, task)
        w = tk.task_weight(task, J.shape[-2])
        N += task.get("gain", 1.0) * J.T @ (w[:, None] ** 2 * J)
    return N


def solution_vjp(m, q, tasks, dt, grad_q, damping=1e-12, limits=None, held=None):
    """Gradient of a loss with respect to each task's target at a converged ``q`` (one instance),
    ``grad_q [nq]`` the loss gradient with respect to q.  Returns ``(grads, status)``: ``grads[t]``
    in the target's own layout (12 floats ``[R | p]`` for frame targets) or None for a LINEAR
    task; ``status`` 0 or 4 (``PK_STATUS_NOT_POSDEF``, all gradients zero)."""
    q = np.asarray(q, dtype=np.float64)
    fk = kin.forward_kinematics(m, q)
    if held is None:
        held = held_coordinates(m, q, tasks, dt, damping, limits)
    free = ~held
    g = tangent_gradient(m, q, grad_q)
    N = normal_matrix(m, q, fk, tasks)[np.ix_(free, free)]
    status = 0
    y = np.zeros(m.nv)
    if N.shape[0]:
        try:
            L = np.linalg.cholesky(N)
            if np.any(np.diag(L) <= PIVOT_RTOL * np.sqrt(np.diag(N))):
                status = 4
        except np.linalg.LinAlgError:
            status = 4
        if not status:
            y[free] = np.linalg.solve(N, g[free])
    grads = []
    for task in tasks:
        dT = target_jacobian(m, q, fk, task)
        if dT is None:
            grads.append(None)
            continue
        _, J = tk.task_error_jacobian(m, q, fk, task)
        wt = tk.task_weight(task, J.shape[-2])
        w = task.get("gain", 1.0) * wt**2 * (J @ y)
        gT = -dT.T @ w
        if task["type"] in ("frame", "relative_frame"):
            gT = frame_gradient_12(np.asarray(task["target"][0], dtype=np.float64), gT)
        grads.append(gT)
    return grads, status


def fixed_point(m, q, tasks, dt=1.0, damping=1e-12, limits=None, tol=1e-12, max_steps=500):
    """Iterate the oracle step ``q <- q (+) v dt`` from ``q`` until ``|v dt| < tol``; returns
    ``(q**, |v dt| of the last step)``."""
    q = np.asarray(q, dtype=np.float64).copy()
    n = np.inf
    for _ in range(max_steps):
        v, st = ik.solve_ik(m, q, tasks, dt, damping, limits, safety_break=False)
        if st:
            raise RuntimeError(f"oracle step failed with status {st}")
        n = np.linalg.norm(v * dt)
        q = kin.integrate(m, q, v * dt)
        if n < tol:
            break
    return q, n

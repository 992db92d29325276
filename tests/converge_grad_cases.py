"""Finite-difference checks of the implicit gradient of converged IK solutions (fp64, oracle only).

``q**(T)`` is the oracle's fixed point (``oracle.implicit_grad.fixed_point``); a loss ``L = g . q**``
is differentiated with respect to one coordinate of one target block at a time: a frame target
along ``T* <- T* exp(eps e_k)`` for each twist direction k, the other targets coordinate-wise.
Besides central differences of the fixed point, ``exact_directional`` evaluates the exact implicit
derivative ``-(dc_F/dq_F)^-1 dc_F/dT`` with both Jacobians of ``c`` (``oracle.ik.qp_objective``)
taken by central differences: the form with the terms the Gauss-Newton matrix drops."""

import numpy as np

from oracle import ik as oik
from oracle import implicit_grad as ig
from oracle import kinematics as okin
from oracle import lie
from oracle import tasks as otasks

CFG_ONLY = [("configuration", 0.5)]  # no velocity bound: the oracle iteration converges fastest


def n_dirs(task):
    return 6 if task["type"] in ("frame", "relative_frame") else len(np.atleast_1d(task["target"]))


def perturb(task, k, eps):
    t = dict(task)
    if t["type"] in ("frame", "relative_frame"):
        R, p = (np.asarray(a, dtype=np.float64) for a in t["target"])
        d = np.zeros(6)
        d[k] = eps
        Rd, pd = lie.exp6(d)
        t["target"] = (R @ Rd, R @ pd + p)
    else:
        a = np.array(t["target"], dtype=np.float64)
        a[k] += eps
        t["target"] = a
    return t


def with_task(tasks, ti, task):
    return [task if j == ti else t for j, t in enumerate(tasks)]


def predicted(grad, task, k):
    """Directional derivative of L along direction k of the task's target, from its gradient
    block (a frame block through its 12 floats, which checks the [R | p] mapping too)."""
    if task["type"] in ("frame", "relative_frame"):
        R = np.asarray(task["target"][0], dtype=np.float64)
        d = np.zeros(6)
        d[k] = 1.0
        dT = np.concatenate([R @ lie.hat(d[3:]), (R @ d[:3])[:, None]], axis=1).reshape(12)
        return float(grad @ dT)
    return float(grad[k])


def richardson(f, eps):
    """Central difference of f at 0 with one Richardson step (truncation O(eps^4))."""
    d1 = (f(eps) - f(-eps)) / (2 * eps)
    d2 = (f(eps / 2) - f(-eps / 2)) / eps
    return (4 * d2 - d1) / 3


def finite_difference(m, q_star, tasks, g, ti, k, eps=2e-4, limits=CFG_ONLY):
    def L(h):
        q, _ = ig.fixed_point(m, q_star, with_task(tasks, ti, perturb(tasks[ti], k, h)), limits=limits, tol=1e-14)
        return g @ q
    return float(richardson(L, eps))


def _c(m, q, tasks):
    return oik.qp_objective(m, q, okin.forward_kinematics(m, q), tasks, 0.0)[1]


def exact_directional(m, q_star, tasks, g, ti, k, held, eps=1e-3):
    """``g_tan . dq**/dT_k`` with dc/dq and dc/dT by central differences of c."""
    nv = m.nv
    dcdq = np.zeros((nv, nv))
    for i in range(nv):
        e = np.eye(nv)[i]
        dcdq[:, i] = richardson(lambda h: _c(m, okin.integrate(m, q_star, h * e), tasks), eps)
    dcdT = richardson(lambda h: _c(m, q_star, with_task(tasks, ti, perturb(tasks[ti], k, h))), eps)
    free = ~held
    dq = np.zeros(nv)
    dq[free] = -np.linalg.solve(dcdq[np.ix_(free, free)], dcdT[free])
    return float(ig.tangent_gradient(m, q_star, g) @ dq)


def residual(m, q, tasks):
    """Largest |e_t| over the tasks whose Jacobian depends on q (frame, relative frame, CoM)."""
    fk = okin.forward_kinematics(m, q)
    r = 0.0
    for t in tasks:
        if t["type"] in ("frame", "relative_frame", "com"):
            e, _ = otasks.task_error_jacobian(m, q, fk, t)
            r = max(r, float(np.linalg.norm(e)))
    return r


def check(m, q0, tasks, seed=0, dirs=None, exact=False, limits=CFG_ONLY):
    """Fixed point from q0, then the N-form gradient (and the exact form) against finite
    differences along every target direction (or ``dirs``: a list of (task, k)).  Returns
    ``(relative error of the N form, relative error of the exact form or None, residual,
    q**, held, grads, status)``; errors are max |pred - fd| / max |fd| over the directions."""
    q_star, n = ig.fixed_point(m, q0, tasks, limits=limits, tol=1e-13)
    assert n < 1e-12, n
    g = np.random.default_rng(seed).normal(size=m.nq)
    held = ig.held_coordinates(m, q_star, tasks, 1.0, 1e-12, limits)
    grads, status = ig.solution_vjp(m, q_star, tasks, 1.0, g, limits=limits)
    if dirs is None:
        dirs = [(ti, k) for ti, t in enumerate(tasks) if grads[ti] is not None for k in range(n_dirs(t))]
    fd = np.array([finite_difference(m, q_star, tasks, g, ti, k, limits=limits) for ti, k in dirs])
    pred = np.array([predicted(grads[ti], tasks[ti], k) for ti, k in dirs])
    scale = np.abs(fd).max()
    err_n = np.abs(pred - fd).max() / scale
    err_x = None
    if exact:
        ex = np.array([exact_directional(m, q_star, tasks, g, ti, k, held) for ti, k in dirs])
        err_x = np.abs(ex - fd).max() / scale
    return err_n, err_x, residual(m, q_star, tasks), q_star, held, grads, status

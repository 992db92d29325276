"""fp64 statement of the stopping error of separate position and orientation tolerances
(``pk_converge_pose_tol_prepared``, DESIGN.md section 3.2h), from the task errors of
:func:`oracle.tasks.task_error_jacobian` and the task costs:

    frame, relative frame   err_t = max(|e[0:3] on weighed axes|, (tol / r) |e[3:6] on weighed axes|)
    CoM, linear             err_t = |e on weighed rows|
    posture                 err_t = |e|

with ``r = orientation_tol`` (``inf``: the rotation rows are not tested), and ``err = max_t err_t``
over the tasks of the stopping set, a NaN kept."""

import numpy as np

from . import kinematics as kin
from . import tasks as tk


def task_error(m, q, fk, task, tol, orientation_tol):
    """``err_t [B]`` of one task at ``q [B, nq]``."""
    e, J = tk.task_error_jacobian(m, q, fk, task)
    if task["type"] == "posture":
        return np.linalg.norm(e, axis=-1)
    w = tk.task_weight(task, J.shape[-2]) > 0.0
    if task["type"] in ("frame", "relative_frame"):
        lin = np.linalg.norm(np.where(w[:3], e[..., :3], 0.0), axis=-1)
        if not np.isfinite(orientation_tol):
            return lin
        ang = np.linalg.norm(np.where(w[3:], e[..., 3:], 0.0), axis=-1)
        return _nan_max(lin, (tol / orientation_tol) * ang)
    return np.linalg.norm(np.where(w, e, 0.0), axis=-1)


def stop_error(m, q, tasks, tol, orientation_tol):
    """``err [B]``: the largest ``err_t`` over ``tasks`` (oracle task dicts of the stopping set)."""
    q = np.asarray(q, dtype=np.float64)
    fk = kin.forward_kinematics(m, q)
    err = np.zeros(q.shape[0])
    for task in tasks:
        err = _nan_max(err, task_error(m, q, fk, task, tol, orientation_tol))
    return err


def _nan_max(a, b):
    return np.where(np.isnan(a) | np.isnan(b), np.nan, np.maximum(a, b))

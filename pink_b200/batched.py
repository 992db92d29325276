"""Prepared batched solver for hot loops.

``pink_b200.solve_ik`` re-describes the problem on every call (as the reference
rebuilds its QP every call, ``pink/solve_ik.py:261-269``).  When
the task set, costs, limits and ``dt`` stay fixed and only ``q`` and the
per-instance targets change - the closed-loop case of
``examples/arm_ur5.py:65-86`` - :class:`BatchedIK` marshals the
problem once (``pk_problem_create``) so that a step costs exactly one kernel
launch through ``pk_solve_ik_prepared``.
"""

from __future__ import annotations

import ctypes as C
import math
from typing import Iterable, NamedTuple, Optional

import torch

from . import _cabi
from .engine import _addr, _stream, get_engine
from .solve_ik import describe_problem


class RolloutTrajectory(NamedTuple):
    """Result of :meth:`BatchedIK.rollout_trajectory`.  ``q [B, nq]`` final configurations,
    ``v [B, nv]`` velocity of the last step that ran, ``status [B]`` OR over the steps that ran;
    the records (``None`` without ``record``) are step-major: ``q_traj [steps, B, nq]`` q after
    each step, ``v_traj [steps, B, nv]`` velocity of each step, ``status_traj [steps, B]`` OR of
    the statuses up to each step."""

    q: torch.Tensor
    v: torch.Tensor
    status: torch.Tensor
    q_traj: Optional[torch.Tensor]
    v_traj: Optional[torch.Tensor]
    status_traj: Optional[torch.Tensor]


class Convergence(NamedTuple):
    """Result of :meth:`BatchedIK.converge`: ``q [B, nq]`` where each instance stopped,
    ``error [B]`` its error there, ``steps [B]`` the solves that ran, ``status [B]`` the OR of
    their statuses (0 if none ran), ``converged [B]`` = ``error <= tol``.  When the call was made
    with ``targets.requires_grad`` (and grad mode on), ``q`` carries the implicit gradient with
    respect to ``targets`` (:meth:`BatchedIK.converge_vjp`); the other fields never do."""

    q: torch.Tensor
    error: torch.Tensor
    steps: torch.Tensor
    status: torch.Tensor
    converged: torch.Tensor


class MultistartConvergence(NamedTuple):
    """Result of :meth:`BatchedIK.converge_multistart`, per target: ``q [B, nq]`` the winning
    seed's configuration, ``error [B]`` its error, ``seed [B]`` (int32) its index, ``steps [B]``
    the rounds the group ran, ``status [B]`` the OR of the winner's step statuses (0 if it ran
    none), ``converged [B]`` = ``error <= tol``.  ``q`` carries a gradient as in
    :class:`Convergence`, through the winning seed."""

    q: torch.Tensor
    error: torch.Tensor
    seed: torch.Tensor
    steps: torch.Tensor
    status: torch.Tensor
    converged: torch.Tensor


class GoalsetConvergence(NamedTuple):
    """Result of :meth:`BatchedIK.converge_goalset`, per instance: ``q [B, nq]`` the winning
    member's configuration, ``error [B]`` its error, ``goal [B]`` and ``seed [B]`` (int32) the
    goal it solved toward and the seed it started from, ``steps [B]`` the rounds the group ran,
    ``status [B]`` the OR of the winner's step statuses (0 if it ran none), ``converged [B]`` =
    ``error <= tol``.  ``q`` carries a gradient as in :class:`Convergence`, to the winning goal's
    row of ``goals``."""

    q: torch.Tensor
    error: torch.Tensor
    goal: torch.Tensor
    seed: torch.Tensor
    steps: torch.Tensor
    status: torch.Tensor
    converged: torch.Tensor


SEED_COUNTS = (1, 2, 4, 8, 16, 32)


class _SolutionOfTargets(torch.autograd.Function):
    """``q*`` as a function of ``targets``: the backward is one :meth:`BatchedIK.converge_vjp`
    launch, with the rows of instances that did not converge set to zero."""

    @staticmethod
    def forward(ctx, targets, solver, q_star, ok):
        ctx.solver = solver
        ctx.save_for_backward(targets, q_star, ok)
        return q_star.view_as(q_star)

    @staticmethod
    def backward(ctx, grad_q):
        targets, q_star, ok = ctx.saved_tensors
        grad_targets, _ = ctx.solver.converge_vjp(q_star, targets.detach(), grad_q.float().contiguous())
        return torch.where(ok[:, None], grad_targets, torch.zeros_like(grad_targets)), None, None, None


def _solution_of_goals(goals, goal, solver, q_star, ok):
    """``q*`` as a function of ``goals [B, G, stride]``: :class:`_SolutionOfTargets` of the
    winning goal's row, gathered by a differentiable index, so the gradient reaches that row
    alone."""
    row = goals[torch.arange(goals.shape[0], device=goals.device), goal.long()]
    return _SolutionOfTargets.apply(row, solver, q_star, ok)


class BatchedIK:
    """``solve_ik`` with the problem description frozen.

    Per-instance targets of the tasks given at construction only fix the
    *layout* of the ``targets`` argument of :meth:`solve` (``target_layout``
    lists ``(task_index, offset, width)``); shared targets are frozen.
    """

    def __init__(self, model, tasks: Iterable, dt: float, damping: float = 1e-12, limits=None,
                 barriers=None, constraints=None, safety_break: bool = True, device=None,
                 batch_size: Optional[int] = None, collision_model=None):
        from .configuration import Configuration  # attaches the default limits to the model
        import numpy as np

        if not hasattr(model, "configuration_limit"):
            Configuration(model, None, np.zeros(model.nq))
        if limits is None:  # the same defaults as solve_ik (pink/solve_ik.py:94-105)
            limits = [model.configuration_limit, model.velocity_limit]
            if getattr(model, "floating_base_velocity_limit", None) is not None:
                limits.append(model.floating_base_velocity_limit)
        tasks = list(tasks)
        if batch_size is None:
            sizes = [d.shape[0] for d in (t._pk_describe(model)["target"] for t in tasks) if isinstance(d, torch.Tensor)]
            batch_size = sizes[0] if sizes else 1
        self.engine = get_engine(model, device)
        self.model = model
        self.tasks = tasks
        self.prob, parts, descs = describe_problem(model, batch_size, tasks, dt, damping, list(limits), safety_break,
                                                   barriers, constraints, collision_model)
        self.target_stride = int(self.prob.target_stride)
        self.target_layout = [
            (k, int(self.prob.tasks[k].target_offset), int(d["target"].shape[1]))
            for k, d in enumerate(descs) if isinstance(d["target"], torch.Tensor)
        ]
        self.nq, self.nv = self.engine.nq, self.engine.nv
        handle = C.c_void_p()
        _cabi.check(self.engine.lib.pk_problem_create(self.engine.handle, C.byref(self.prob), C.byref(handle)))
        self._handle = handle

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self.engine.lib.pk_problem_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def solve(self, q: torch.Tensor, targets: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
              status: Optional[torch.Tensor] = None):
        """``q [B, nq]``, ``targets [B, target_stride]`` (fp32, contiguous, on the
        device) -> ``(v [B, nv], status [B])``; asynchronous on the current stream."""
        eng = self.engine
        B = q.shape[0]
        if out is None:
            out = torch.empty((B, self.nv), device=eng.device, dtype=torch.float32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            _cabi.check(eng.lib.pk_solve_ik_prepared(eng.handle, self._handle, _addr(q), _addr(targets), _addr(out),
                                                     _addr(status), B, _stream(eng.device)))
        return out, status

    def solve_host(self, q: torch.Tensor, targets: Optional[torch.Tensor], out: torch.Tensor,
                   status: Optional[torch.Tensor] = None):
        """Same through host tensors (pinned for full PCIe speed): the library
        copies in, solves and copies out on the current stream."""
        eng = self.engine
        with torch.cuda.device(eng.device):
            _cabi.check(eng.lib.pk_solve_ik_prepared_host(eng.handle, self._handle, _addr(q), _addr(targets),
                                                          _addr(out), _addr(status), q.shape[0], _stream(eng.device)))
        return out, status

    def set_host_schedule(self, mode: int) -> None:
        """Schedule of :meth:`solve_host` for this model (``pk_model_set_host_schedule``): 0 staged
        uploads and downloads, 2 staged uploads + results written straight into the pinned host
        buffers, 1 zero-copy, -1 environment default."""
        _cabi.check(self.engine.lib.pk_model_set_host_schedule(self.engine.handle, int(mode)))
        self.host_schedule = int(mode)

    def tune_host_path(self, q: torch.Tensor, targets: Optional[torch.Tensor], out: torch.Tensor,
                       status: Optional[torch.Tensor] = None, calls: int = 40, candidates=(0, 2)) -> dict:
        """Start-up probe: time :meth:`solve_host` on the caller's own (pinned) buffers under each
        candidate schedule and keep the fastest.  How a platform's PCIe root complex handles the
        two directions at once differs from box to box (measured: the same code is 4 % faster
        with schedule 2 on one, 8 % slower on another), so the choice is made where the code
        runs.  Returns the measured microseconds per call by schedule; results are identical
        under every schedule."""
        import time

        timings = {}
        for mode in candidates:
            self.set_host_schedule(mode)
            for _ in range(8):
                self.solve_host(q, targets, out, status)
            torch.cuda.synchronize(self.engine.device)
            best = float("inf")
            for _ in range(3):
                t0 = time.perf_counter()
                for _ in range(calls):
                    self.solve_host(q, targets, out, status)
                torch.cuda.synchronize(self.engine.device)
                best = min(best, (time.perf_counter() - t0) / calls)
            timings[mode] = best * 1e6
        self.set_host_schedule(min(timings, key=timings.get))
        return timings

    def rollout(self, q: torch.Tensor, targets: Optional[torch.Tensor], steps: int,
                q_out: Optional[torch.Tensor] = None, v_out: Optional[torch.Tensor] = None,
                status: Optional[torch.Tensor] = None):
        """``steps`` iterations of ``v = solve_ik(q); q = q (+) v dt`` with fixed targets
        (the loop of ``examples/arm_ur5.py:65-86``); serial chains keep ``q`` on chip
        for the whole loop.  Returns ``(q_final, v_last, status)``."""
        eng = self.engine
        B = q.shape[0]
        if q_out is None:
            q_out = torch.empty_like(q)
        if v_out is None:
            v_out = torch.empty((B, self.nv), device=eng.device, dtype=torch.float32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            _cabi.check(eng.lib.pk_rollout_prepared(eng.handle, self._handle, _addr(q), _addr(targets), int(steps),
                                                    _addr(q_out), _addr(v_out), _addr(status), B, _stream(eng.device)))
        return q_out, v_out, status

    def rollout_trajectory(self, q: torch.Tensor, targets: Optional[torch.Tensor], steps: Optional[int] = None,
                           record: bool = True, q_out: Optional[torch.Tensor] = None,
                           v_out: Optional[torch.Tensor] = None,
                           status: Optional[torch.Tensor] = None) -> RolloutTrajectory:
        """``steps`` iterations of ``v = solve_ik(q, targets[s]); q = q (+) v dt`` in one launch:
        the loop of ``examples/arm_ur5.py:65-86`` with a target that moves every step.

        ``targets`` is ``[steps, B, target_stride]`` (one row per instance and step; a view is
        fine as long as ``stride(2) == 1`` and ``stride(1) == target_stride``), or ``[B,
        target_stride]`` / ``None`` with ``steps`` for the same rows every step.  With
        ``record`` the configuration, velocity and status of every step come back too.  An
        instance that fails a step (no solution, or outside its limits with ``safety_break``)
        is frozen: its q stays, its later ``v_traj`` rows are zero and ``status_traj``
        repeats.  The ``dq_prev`` words of ``AccelerationLimit`` / ``LowAccelerationTask`` are
        read from each step's row as given.  Asynchronous on the current stream; no
        allocation inside the library, so the call can be captured in a CUDA graph."""
        eng = self.engine
        B = q.shape[0]
        S = self.target_stride
        if targets is None:
            if S > 0:
                raise ValueError(f"this problem has per-instance targets ({S} floats per row): pass targets")
            if steps is None:
                raise ValueError("steps is required when targets is None")
            target_step = 0
        elif targets.dim() == 2:
            if steps is None:
                raise ValueError("steps is required with one targets row per instance")
            if tuple(targets.shape) != (B, S):
                raise ValueError(f"targets has shape {tuple(targets.shape)}, expected ({B}, {S})")
            if S > 0 and (targets.stride(1) != 1 or targets.stride(0) != S):
                raise ValueError("targets rows must be contiguous, target_stride floats apart")
            target_step = 0
        elif targets.dim() == 3:
            if steps is None:
                steps = targets.shape[0]
            if targets.shape[0] != steps:
                raise ValueError(f"targets holds {targets.shape[0]} steps, steps = {steps}")
            if tuple(targets.shape[1:]) != (B, S):
                raise ValueError(f"targets has shape {tuple(targets.shape)}, expected ({steps}, {B}, {S})")
            if S > 0 and (targets.stride(2) != 1 or targets.stride(1) != S):
                raise ValueError("targets[s] rows must be contiguous, target_stride floats apart "
                                 f"(strides {tuple(targets.stride())})")
            target_step = targets.stride(0) if steps > 1 else 0
        else:
            raise ValueError(f"targets must be [steps, B, {S}] or [B, {S}], got {tuple(targets.shape)}")
        if targets is not None and targets.dtype != torch.float32:
            raise ValueError(f"targets must be float32, got {targets.dtype}")
        steps = int(steps)
        if q_out is None:
            q_out = torch.empty_like(q)
        if v_out is None:
            v_out = torch.empty((B, self.nv), device=eng.device, dtype=torch.float32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        q_traj = v_traj = st_traj = None
        if record and steps > 0:
            q_traj = torch.empty((steps, B, self.nq), device=eng.device, dtype=torch.float32)
            v_traj = torch.empty((steps, B, self.nv), device=eng.device, dtype=torch.float32)
            st_traj = torch.empty((steps, B), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            _cabi.check(eng.lib.pk_rollout_trajectory_prepared(
                eng.handle, self._handle, _addr(q), _addr(targets), int(target_step), steps, _addr(q_out),
                _addr(v_out), _addr(status), _addr(q_traj), _addr(v_traj), _addr(st_traj), B, _stream(eng.device)))
        return RolloutTrajectory(q_out, v_out, status, q_traj, v_traj, st_traj)

    def converge(self, q: torch.Tensor, targets: Optional[torch.Tensor], tasks: Iterable, tol: float,
                 max_steps: int, q_out: Optional[torch.Tensor] = None, error: Optional[torch.Tensor] = None,
                 steps: Optional[torch.Tensor] = None, status: Optional[torch.Tensor] = None,
                 orientation_tol: Optional[float] = None) -> Convergence:
        """Solve each instance to a tolerance in one launch: the loop of the reference's
        ``examples/inverse_kinematics_ur10.py`` (``while norm(task.compute_error(c)) > thres``).

        ``err(q)`` is the largest ``|task.compute_error(q)|`` (unweighted, gain-free) over
        ``tasks``, which must be task objects given to the constructor.  For s = 0, 1, ...
        an instance stops at ``q_s`` when ``err(q_s) <= tol`` or ``s == max_steps``; otherwise
        it takes the step :meth:`rollout` takes, and stops at ``q_s`` if that step fails (no
        solution, or outside its limits with ``safety_break``).  ``targets [B,
        target_stride]`` are fixed for the whole loop; the ``dq_prev`` words of
        ``AccelerationLimit`` / ``LowAccelerationTask`` are read from the row as given.
        Barriers and constraints act in every step but are not part of the stopping test.

        Poses resolve to about 1e-7 in fp32, so a ``tol`` below about 1e-6 may run to
        ``max_steps``.  Asynchronous on the current stream; no allocation inside the library,
        so the call can be captured in a CUDA graph.  ``q_out`` may be ``q``.

        With ``targets.requires_grad`` (and grad mode on) the returned ``q`` carries the gradient
        with respect to ``targets``, one :meth:`converge_vjp` launch in the backward pass, zero
        for instances that did not converge.  Every frame, relative frame and CoM task must then
        be in ``tasks`` (so that ``tol`` bounds the gradient's error), and problems with barriers,
        constraints or ``AccelerationLimit`` are rejected (``ValueError``).

        ``orientation_tol`` selects separate position and orientation tolerances: a task's error
        then counts only the components it weighs (cost > 0), and a frame or relative-frame task's
        is ``max(|e[0:3]|, (tol / orientation_tol) |e[3:6]|)``, so ``error <= tol`` means every
        weighed translation part is within ``tol`` (metres), every weighed rotation part within
        ``orientation_tol`` (radians) and every other task within ``tol``.  ``inf`` leaves
        orientations out of the test.  A position-only task (``orientation_cost=0``) can then
        converge and be differentiated (DESIGN.md section 3.2h)."""
        eng = self.engine
        B = q.shape[0]
        mask, tol = self._stop_test(tasks, tol, max_steps)
        orientation_tol = self._orientation_tol(mask, tol, orientation_tol)
        grad = self._grad_mode(targets, mask, orientation_tol)
        if tuple(q.shape) != (B, self.nq) or q.dtype != torch.float32 or not q.is_contiguous():
            raise ValueError(f"q must be a contiguous float32 [B, {self.nq}] tensor")
        self._check_fixed_targets(targets, B)
        if q_out is None:
            q_out = torch.empty_like(q)
        if error is None:
            error = torch.empty((B,), device=eng.device, dtype=torch.float32)
        if steps is None:
            steps = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            if orientation_tol is None:
                _cabi.check(eng.lib.pk_converge_prepared(eng.handle, self._handle, _addr(q), _addr(targets), mask, tol,
                                                         int(max_steps), _addr(q_out), _addr(error), _addr(steps),
                                                         _addr(status), B, _stream(eng.device)))
            else:
                _cabi.check(eng.lib.pk_converge_pose_tol_prepared(
                    eng.handle, self._handle, _addr(q), _addr(targets), mask, tol, orientation_tol, int(max_steps),
                    _addr(q_out), _addr(error), _addr(steps), _addr(status), B, _stream(eng.device)))
        if grad:
            q_out = _SolutionOfTargets.apply(targets, self, q_out, self._solved(error, status, tol))
        return Convergence(q_out, error, steps, status, error <= tol)

    def converge_vjp(self, q_star: torch.Tensor, targets: Optional[torch.Tensor], grad_q: torch.Tensor,
                     grad_targets: Optional[torch.Tensor] = None, status: Optional[torch.Tensor] = None):
        """Gradient of a loss with respect to ``targets [B, target_stride]`` at solutions ``q_star
        [B, nq]`` of :meth:`converge` / :meth:`converge_multistart`, given ``grad_q [B, nq]``, the
        loss gradient with respect to ``q_star``: ``(grad_targets [B, target_stride], status
        [B])``.  :meth:`converge` attaches the same computation to its ``q`` when ``targets``
        requires grad.

        The loop stops where the step's linear term ``c = sum_t alpha_t J_t^T W_t^2 e_t`` vanishes
        on the coordinates it leaves off the configuration limits; the gradient is that
        condition's implicit derivative, ``dq*/dT = -N_FF^-1 dc_F/dT``, with the Gauss-Newton
        ``N = sum_t alpha_t J_t^T W_t^2 J_t``.  It does not depend on ``dt``, the damping or the
        velocity limits, and it is exact up to terms proportional to the errors of the tasks at
        ``q_star`` (bounded by ``tol`` when those tasks are in the stopping test).  Semantics:

        * Only ``targets`` is differentiated: the gradient with respect to the start is zero (the
          fixed point does not depend on it), and shared targets are constants.
        * ``grad_q`` is in q coordinates; on a free-flyer root it is mapped to the tangent space
          by the transpose of ``d(q (+) dq)/d dq`` at ``dq = 0`` (a quaternion component that only
          changes the norm is dropped).
        * A coordinate the step holds on a configuration limit does not move (``dq*_i = 0``).
        * A frame target's 12 floats ``[R | p]`` receive ``[1/2 R [g_w]x | R g_v]``, with ``(g_v,
          g_w)`` the gradient of the twist ``d`` in ``T <- T exp(d)``.  ``1/2 R [g_w]x`` is the
          tangent component, so a rotation parameterisation upstream (quaternion, 6-D,
          axis-angle) receives the exact gradient.  CoM, posture and joint-velocity targets are
          differentiated coordinate-wise; the root coordinates of a free-flyer posture target get
          zero.
        * ``status``: 0, or ``PK_STATUS_NOT_POSDEF`` (4) where ``N_FF`` is not positive definite in
          fp32 (for example a 7-joint arm with one frame task and no posture task); that row is
          zero.  Rows of instances that did not converge are the caller's to discard
          (the autograd path of :meth:`converge` zeroes them).

        Problems with barriers, equality constraints or ``AccelerationLimit`` are rejected.
        Asynchronous on the current stream; no allocation inside the library, so the call can be
        captured in a CUDA graph."""
        eng = self.engine
        B = q_star.shape[0]
        if tuple(q_star.shape) != (B, self.nq) or q_star.dtype != torch.float32 or not q_star.is_contiguous():
            raise ValueError(f"q_star must be a contiguous float32 [B, {self.nq}] tensor")
        if tuple(grad_q.shape) != (B, self.nq) or grad_q.dtype != torch.float32 or not grad_q.is_contiguous():
            raise ValueError(f"grad_q must be a contiguous float32 [B, {self.nq}] tensor")
        self._check_fixed_targets(targets, B)
        if grad_targets is None:
            grad_targets = torch.empty((B, self.target_stride), device=eng.device, dtype=torch.float32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            _cabi.check(eng.lib.pk_converge_vjp_prepared(eng.handle, self._handle, _addr(q_star), _addr(targets),
                                                         _addr(grad_q), _addr(grad_targets), _addr(status), B,
                                                         _stream(eng.device)))
        return grad_targets, status

    def _grad_mode(self, targets: Optional[torch.Tensor], mask: int, orientation_tol: Optional[float] = None) -> bool:
        """Whether :meth:`converge` / :meth:`converge_multistart` attach the gradient with respect
        to ``targets``; checks that the problem is one whose gradient error ``tol`` bounds.  With
        ``orientation_tol`` the components a task does not weigh are left untested: their zero
        weight keeps them out of the gradient, so ``orientation_tol`` must only be finite."""
        if targets is None or not (torch.is_grad_enabled() and targets.requires_grad):
            return False
        if orientation_tol is not None and not math.isfinite(orientation_tol):
            raise ValueError("gradients of converge need a finite orientation_tol, so that the test bounds every "
                             "weighed error")
        for k in range(len(self.tasks)):
            if int(self.prob.tasks[k].type) in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_RELATIVE_FRAME,
                                                _cabi.PK_TASK_COM) and not (mask >> k) & 1:
                raise ValueError(f"gradients of converge need every frame, relative frame and CoM task in the "
                                 f"stopping test: {self.tasks[k]!r} is not in tasks")
        if int(self.prob.nbarriers):
            raise ValueError("gradients of converge do not support barriers")
        if int(self.prob.nconstraints):
            raise ValueError("gradients of converge do not support equality constraints")
        if int(self.prob.acc_enabled):
            raise ValueError("gradients of converge do not support AccelerationLimit")
        return True

    def _solved(self, error: torch.Tensor, status: torch.Tensor, tol: float) -> torch.Tensor:
        """Instances whose gradient is kept: converged, with no failed step."""
        failed = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF
        if int(self.prob.safety_break):
            failed |= _cabi.PK_STATUS_OUT_OF_LIMITS
        return (error <= tol) & ((status & failed) == 0)

    def _stop_test(self, tasks: Iterable, tol: float, max_steps: int):
        """The task mask and tol of :meth:`converge` / :meth:`converge_multistart`, validated."""
        mask = 0
        for t in tasks:
            ks = [k for k, t0 in enumerate(self.tasks) if t0 is t]
            if not ks:
                raise ValueError(f"{t!r} is not one of the tasks this solver was built with")
            mask |= 1 << ks[0]
        if mask == 0:
            raise ValueError("tasks is empty: the stopping test needs at least one task")
        for k in range(len(self.tasks)):
            if (mask >> k) & 1 and int(self.prob.tasks[k].type) == _cabi.PK_TASK_JOINT_VELOCITY:
                raise ValueError(f"{self.tasks[k]!r}: the error of a joint-velocity task does not depend on q")
        tol = float(tol)
        if not (tol >= 0.0) or tol == float("inf"):
            raise ValueError(f"tol must be finite and >= 0, got {tol}")
        if int(max_steps) != max_steps or max_steps < 0:
            raise ValueError(f"max_steps must be an integer >= 0, got {max_steps}")
        return mask, tol

    def _orientation_tol(self, mask: int, tol: float, orientation_tol: Optional[float]) -> Optional[float]:
        """``orientation_tol`` of :meth:`converge` and its siblings, validated (None: the default
        test).  The separate-tolerance test checks only weighed components, so every task of the
        mask must keep one."""
        if orientation_tol is None:
            return None
        r = float(orientation_tol)
        if not (tol > 0.0):
            raise ValueError(f"tol must be finite and > 0 with orientation_tol, got {tol}")
        if not (r > 0.0):
            raise ValueError(f"orientation_tol must be > 0 (inf: orientations are not tested), got {orientation_tol}")
        for k in range(len(self.tasks)):
            if not (mask >> k) & 1:
                continue
            d = self.prob.tasks[k]
            ty = int(d.type)
            n = 1 if ty == _cabi.PK_TASK_POSTURE else 3 if ty == _cabi.PK_TASK_COM else \
                int(d.rows) if ty == _cabi.PK_TASK_LINEAR else 6
            pose = ty in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_RELATIVE_FRAME)
            if not any(float(d.cost[i]) > 0.0 and (not pose or i < 3 or math.isfinite(r)) for i in range(n)):
                raise ValueError(f"{self.tasks[k]!r} weighs no component the stopping test could check")
        return r

    def _check_fixed_targets(self, targets: Optional[torch.Tensor], B: int) -> None:
        """One fixed targets row per instance (or target), ``[B, target_stride]``."""
        S = self.target_stride
        if targets is None:
            if S > 0:
                raise ValueError(f"this problem has per-instance targets ({S} floats per row): pass targets")
        else:
            if targets.dim() != 2 or tuple(targets.shape) != (B, S):
                raise ValueError(f"targets has shape {tuple(targets.shape)}, expected ({B}, {S})")
            if S > 0 and (targets.stride(1) != 1 or targets.stride(0) != S):
                raise ValueError("targets rows must be contiguous, target_stride floats apart")
            if targets.dtype != torch.float32:
                raise ValueError(f"targets must be float32, got {targets.dtype}")

    def converge_multistart(self, q_seeds: torch.Tensor, targets: Optional[torch.Tensor], tasks: Iterable, tol: float,
                            max_steps: int, q_out: Optional[torch.Tensor] = None, error: Optional[torch.Tensor] = None,
                            seed: Optional[torch.Tensor] = None, steps: Optional[torch.Tensor] = None,
                            status: Optional[torch.Tensor] = None,
                            orientation_tol: Optional[float] = None) -> MultistartConvergence:
        """Solve each target to a tolerance from several seeds in one launch, stopping a target as
        soon as one of its seeds converges.

        ``q_seeds [B, S, nq]``: S start configurations per target (:meth:`sample_seeds` makes
        them), S one of 1, 2, 4, 8, 16, 32 (at most 8 on the tree kernel, whose S warp
        workspaces must also fit one CTA's shared memory).  ``targets [B, target_stride]``: one
        row per target, shared by its seeds.  ``tasks``, ``tol`` and ``max_steps`` as
        :meth:`converge`.  The S seeds advance in lockstep rounds: in round s every seed that
        has not failed computes ``err(q_s)``; the group stops when some seed has ``err <= tol``,
        ``s == max_steps``, or every seed has failed; otherwise every seed that has not failed
        takes the :meth:`converge` step, and a seed whose step fails keeps ``q_s`` and its error.
        The winner is the seed with the smallest error at the stopping round (NaN counts as
        +inf, ties go to the lowest index).

        With S = 1 the result equals :meth:`converge`'s.  With seed 0 the caller's start, every
        target :meth:`converge` solves from it is solved here too, in at most as many steps.
        Asynchronous on the current stream; no allocation inside the library, so the call can
        be captured in a CUDA graph.  ``q_seeds`` is only read and must not overlap ``q_out``.
        ``orientation_tol`` as in :meth:`converge`."""
        eng = self.engine
        mask, tol = self._stop_test(tasks, tol, max_steps)
        orientation_tol = self._orientation_tol(mask, tol, orientation_tol)
        grad = self._grad_mode(targets, mask, orientation_tol)
        if (q_seeds.dim() != 3 or q_seeds.shape[2] != self.nq or q_seeds.dtype != torch.float32
                or not q_seeds.is_contiguous()):
            raise ValueError(f"q_seeds must be a contiguous float32 [B, S, {self.nq}] tensor")
        B, S = int(q_seeds.shape[0]), int(q_seeds.shape[1])
        if S not in SEED_COUNTS:
            raise ValueError(f"the number of seeds must be one of {SEED_COUNTS}, got {S}")
        self._check_fixed_targets(targets, B)
        lib = eng.lib
        # the path-dependent limits on S (the tree kernel's): the library validates a call with no
        # targets without launching anything
        if orientation_tol is None:
            bad = lib.pk_converge_multistart_prepared(eng.handle, self._handle, None, S, None, mask, tol,
                                                      int(max_steps), None, None, None, None, None, 0, None)
        else:
            bad = lib.pk_converge_goalset_pose_tol_prepared(eng.handle, self._handle, None, S, None, 1, mask, tol,
                                                            orientation_tol, int(max_steps), None, None, None, None,
                                                            None, None, 0, None)
        if bad:
            raise ValueError("pink_b200: " + lib.pk_last_error().decode("utf-8", "replace"))
        if q_out is None:
            q_out = torch.empty((B, self.nq), device=eng.device, dtype=torch.float32)
        if error is None:
            error = torch.empty((B,), device=eng.device, dtype=torch.float32)
        if seed is None:
            seed = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if steps is None:
            steps = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            if orientation_tol is None:
                _cabi.check(lib.pk_converge_multistart_prepared(
                    eng.handle, self._handle, _addr(q_seeds), S, _addr(targets), mask, tol, int(max_steps),
                    _addr(q_out), _addr(error), _addr(seed), _addr(steps), _addr(status), B, _stream(eng.device)))
            else:  # multi-start is the goal-set solve with one goal
                _cabi.check(lib.pk_converge_goalset_pose_tol_prepared(
                    eng.handle, self._handle, _addr(q_seeds), S, _addr(targets), 1, mask, tol, orientation_tol,
                    int(max_steps), _addr(q_out), _addr(error), None, _addr(seed), _addr(steps), _addr(status), B,
                    _stream(eng.device)))
        if grad:
            q_out = _SolutionOfTargets.apply(targets, self, q_out, self._solved(error, status, tol))
        return MultistartConvergence(q_out, error, seed, steps, status, error <= tol)

    def converge_goalset(self, q_seeds: torch.Tensor, goals: torch.Tensor, tasks: Iterable, tol: float,
                         max_steps: int, q_out: Optional[torch.Tensor] = None, error: Optional[torch.Tensor] = None,
                         goal: Optional[torch.Tensor] = None, seed: Optional[torch.Tensor] = None,
                         steps: Optional[torch.Tensor] = None,
                         status: Optional[torch.Tensor] = None,
                         orientation_tol: Optional[float] = None) -> GoalsetConvergence:
        """Solve each instance toward the best of several goals, from several seeds, in one launch,
        stopping an instance as soon as one of its (goal, seed) members converges.

        ``q_seeds [B, S, nq]``: as in :meth:`converge_multistart`; every goal starts from the
        same S seeds.  ``goals [B, G, target_stride]``: G complete targets rows per instance (the
        layout ``target_layout`` describes), so a goal may change any per-instance target;
        shared targets stay shared.  G and S are powers of two with ``G * S`` one of 1, 2, 4, 8,
        16, 32 (at most 8 on the tree kernel, whose ``G * S`` warp workspaces must also fit one
        CTA's shared memory).  To use a goal count that is not a power of two, pad ``goals`` by
        repeating one of them: a duplicate never changes the winner, since ties go to the lower
        index.  ``tasks``, ``tol`` and ``max_steps`` as :meth:`converge`.

        Member ``j = g * S + s`` starts at ``q_seeds[b, s]`` and solves toward ``goals[b, g]``.
        The G*S members form one group of :meth:`converge_multistart`'s rule: they advance in
        lockstep rounds, the group stops when some member has ``err <= tol``, at ``max_steps``,
        or when every member has failed, and the winner is the member with the smallest error at
        the stopping round (NaN counts as +inf; ties go to the lowest ``j``: the earlier goal,
        then the earlier seed, so goals may be listed in order of preference).  The result gives
        ``goal = j // S`` and ``seed = j % S``.

        With G = 1 the result equals :meth:`converge_multistart`'s.  With S = 1, every instance
        that :meth:`converge` from ``q_seeds[:, 0]`` solves toward some goal is solved here too,
        in at most the smallest of those step counts.  With ``goals.requires_grad`` (and grad mode
        on) the returned ``q`` carries the gradient with respect to the winning goal's row
        (the other rows get zero; so do instances that did not converge), under the conditions
        of :meth:`converge`.  Asynchronous on the current stream; no allocation inside the
        library, so the call can be captured in a CUDA graph.  ``q_seeds`` is only read and must
        not overlap ``q_out``.  ``orientation_tol`` as in :meth:`converge`."""
        eng = self.engine
        mask, tol = self._stop_test(tasks, tol, max_steps)
        orientation_tol = self._orientation_tol(mask, tol, orientation_tol)
        grad = self._grad_mode(goals, mask, orientation_tol)
        if (q_seeds.dim() != 3 or q_seeds.shape[2] != self.nq or q_seeds.dtype != torch.float32
                or not q_seeds.is_contiguous()):
            raise ValueError(f"q_seeds must be a contiguous float32 [B, S, {self.nq}] tensor")
        B, S = int(q_seeds.shape[0]), int(q_seeds.shape[1])
        T = self.target_stride
        if goals is None or goals.dim() != 3 or goals.shape[0] != B or goals.shape[2] != T:
            shape = None if goals is None else tuple(goals.shape)
            raise ValueError(f"goals has shape {shape}, expected ({B}, G, {T})")
        G = int(goals.shape[1])
        if goals.dtype != torch.float32:
            raise ValueError(f"goals must be float32, got {goals.dtype}")
        if T > 0 and (goals.stride(2) != 1 or goals.stride(1) != T or goals.stride(0) != G * T):
            raise ValueError("goals rows must be contiguous, target_stride floats apart")
        if G not in SEED_COUNTS:
            raise ValueError(f"the number of goals must be one of {SEED_COUNTS} (pad by repeating a goal), got {G}")
        if S not in SEED_COUNTS:
            raise ValueError(f"the number of seeds must be one of {SEED_COUNTS}, got {S}")
        if G * S > SEED_COUNTS[-1]:
            raise ValueError(f"goals x seeds must be at most {SEED_COUNTS[-1]}, got {G} x {S}")
        lib = eng.lib
        # the path-dependent limits on G S (the tree kernel's): the library validates a call with
        # no targets without launching anything
        if orientation_tol is None:
            bad = lib.pk_converge_goalset_prepared(eng.handle, self._handle, None, S, None, G, mask, tol,
                                                   int(max_steps), None, None, None, None, None, None, 0, None)
        else:
            bad = lib.pk_converge_goalset_pose_tol_prepared(eng.handle, self._handle, None, S, None, G, mask, tol,
                                                            orientation_tol, int(max_steps), None, None, None, None,
                                                            None, None, 0, None)
        if bad:
            raise ValueError("pink_b200: " + lib.pk_last_error().decode("utf-8", "replace"))
        if q_out is None:
            q_out = torch.empty((B, self.nq), device=eng.device, dtype=torch.float32)
        if error is None:
            error = torch.empty((B,), device=eng.device, dtype=torch.float32)
        if goal is None:
            goal = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if seed is None:
            seed = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if steps is None:
            steps = torch.empty((B,), device=eng.device, dtype=torch.int32)
        if status is None:
            status = torch.empty((B,), device=eng.device, dtype=torch.int32)
        with torch.cuda.device(eng.device):
            if orientation_tol is None:
                _cabi.check(lib.pk_converge_goalset_prepared(
                    eng.handle, self._handle, _addr(q_seeds), S, _addr(goals), G, mask, tol, int(max_steps),
                    _addr(q_out), _addr(error), _addr(goal), _addr(seed), _addr(steps), _addr(status), B,
                    _stream(eng.device)))
            else:
                _cabi.check(lib.pk_converge_goalset_pose_tol_prepared(
                    eng.handle, self._handle, _addr(q_seeds), S, _addr(goals), G, mask, tol, orientation_tol,
                    int(max_steps), _addr(q_out), _addr(error), _addr(goal), _addr(seed), _addr(steps),
                    _addr(status), B, _stream(eng.device)))
        if grad:
            q_out = _solution_of_goals(goals, goal, self, q_out, self._solved(error, status, tol))
        return GoalsetConvergence(q_out, error, goal, seed, steps, status, error <= tol)

    def sample_seeds(self, q: torch.Tensor, num_seeds: int, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """Seeds for :meth:`converge_multistart`: ``q [B, nq]`` -> ``[B, num_seeds, nq]``.

        Seed 0 is ``q``.  In the other seeds, each coordinate with finite lower and upper limits
        is drawn uniformly strictly inside them; a revolute coordinate without limits (URDF
        ``continuous``) is drawn in [-pi, pi]; the other coordinates (unbounded prismatic
        joints, the free-flyer root) are copied from ``q``.  Plain torch on ``q``'s device."""
        return sample_seeds(self.model, q, num_seeds, generator)


def sample_seeds(model, q: torch.Tensor, num_seeds: int, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """:meth:`BatchedIK.sample_seeds` for a model."""
    import math

    import numpy as np

    if q.dim() != 2 or q.shape[1] != model.nq:
        raise ValueError(f"q must be a [B, {model.nq}] tensor")
    if int(num_seeds) != num_seeds or num_seeds < 1:
        raise ValueError(f"num_seeds must be an integer >= 1, got {num_seeds}")
    lo = np.array(model.lowerPositionLimit, dtype=np.float64)
    hi = np.array(model.upperPositionLimit, dtype=np.float64)
    bounded = np.isfinite(lo) & np.isfinite(hi) & (hi > lo)
    circle = np.zeros(model.nq, dtype=bool)
    for j in model.joints:
        if j.kind == "revolute" and not np.isfinite(lo[j.idx_q]) and not np.isfinite(hi[j.idx_q]):
            circle[j.idx_q] = True
    lo = np.where(circle, -math.pi, np.where(bounded, lo, 0.0))
    hi = np.where(circle, math.pi, np.where(bounded, hi, 0.0))
    B, S = q.shape[0], int(num_seeds)
    u = torch.rand((B, S - 1, model.nq), generator=generator, dtype=torch.float64, device=q.device)
    lo_t = torch.as_tensor(lo, device=q.device)
    hi_t = torch.as_tensor(hi, device=q.device)
    x = (lo_t + (hi_t - lo_t) * u).to(q.dtype)
    # strictly inside after the rounding to q's dtype
    inside_lo = torch.nextafter(lo_t.to(q.dtype), hi_t.to(q.dtype))
    inside_hi = torch.nextafter(hi_t.to(q.dtype), lo_t.to(q.dtype))
    x = torch.minimum(torch.maximum(x, inside_lo), inside_hi)
    draw = torch.as_tensor(bounded | circle, device=q.device)
    rest = torch.where(draw, x, q[:, None, :].expand(B, S - 1, model.nq))
    return torch.cat([q[:, None, :], rest], dim=1).contiguous()

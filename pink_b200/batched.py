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
    their statuses (0 if none ran), ``converged [B]`` = ``error <= tol``."""

    q: torch.Tensor
    error: torch.Tensor
    steps: torch.Tensor
    status: torch.Tensor
    converged: torch.Tensor


class MultistartConvergence(NamedTuple):
    """Result of :meth:`BatchedIK.converge_multistart`, per target: ``q [B, nq]`` the winning
    seed's configuration, ``error [B]`` its error, ``seed [B]`` (int32) its index, ``steps [B]``
    the rounds the group ran, ``status [B]`` the OR of the winner's step statuses (0 if it ran
    none), ``converged [B]`` = ``error <= tol``."""

    q: torch.Tensor
    error: torch.Tensor
    seed: torch.Tensor
    steps: torch.Tensor
    status: torch.Tensor
    converged: torch.Tensor


SEED_COUNTS = (1, 2, 4, 8, 16, 32)


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
                 steps: Optional[torch.Tensor] = None, status: Optional[torch.Tensor] = None) -> Convergence:
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
        so the call can be captured in a CUDA graph.  ``q_out`` may be ``q``."""
        eng = self.engine
        B = q.shape[0]
        mask, tol = self._stop_test(tasks, tol, max_steps)
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
            _cabi.check(eng.lib.pk_converge_prepared(eng.handle, self._handle, _addr(q), _addr(targets), mask, tol,
                                                     int(max_steps), _addr(q_out), _addr(error), _addr(steps),
                                                     _addr(status), B, _stream(eng.device)))
        return Convergence(q_out, error, steps, status, error <= tol)

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
                            status: Optional[torch.Tensor] = None) -> MultistartConvergence:
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
        be captured in a CUDA graph.  ``q_seeds`` is only read and must not overlap ``q_out``."""
        eng = self.engine
        mask, tol = self._stop_test(tasks, tol, max_steps)
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
        if lib.pk_converge_multistart_prepared(eng.handle, self._handle, None, S, None, mask, tol, int(max_steps),
                                               None, None, None, None, None, 0, None):
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
            _cabi.check(lib.pk_converge_multistart_prepared(
                eng.handle, self._handle, _addr(q_seeds), S, _addr(targets), mask, tol, int(max_steps), _addr(q_out),
                _addr(error), _addr(seed), _addr(steps), _addr(status), B, _stream(eng.device)))
        return MultistartConvergence(q_out, error, seed, steps, status, error <= tol)

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

"""Gradients of converged solutions with respect to the targets (``pk_converge_vjp_prepared``) on the
CPU build of the kernel body, and the autograd glue of ``BatchedIK.converge`` /
``converge_multistart`` driven through that build.

The body (``Generic::solution_vjp``) is compared with the fp64 oracle (oracle/implicit_grad.py)
at the same fp32 configuration cast to fp64.  Tolerance, per instance, binned by cond(N_FF)
of the oracle: |grad - ref| <= grad_rtol(cond) * max |ref| + 1e-6.  The body factorises N_FF in
square-root form, but y = N_FF^-1 g is still a solve with N_FF, so the relative error of the
gradient grows like cond(N_FF) times the fp32 rounding of the rows (the worst seen between the
GPU and the host build: 1.1e-2 at cond 9e6, a G1 instance)."""

import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ik as oik
from oracle import implicit_grad as ig
from oracle import kinematics as okin
from pink_b200 import _cabi
from tests import helpers
from tests.host_engine import host_engine  # noqa: F401  (fixture)
from tests.hostsim import HostSim
from tests import hostsim
from tests import hostsim_vjp
from tests.hostsim_vjp import HostVjp

GRAD_BINS = [(0.0, 1e4, 1e-4), (1e4, 1e6, 1e-2), (1e6, float("inf"), 1e-1)]
# a failed step: the autograd path of BatchedIK.converge zeroes these rows (safety_break is on)
FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF | _cabi.PK_STATUS_OUT_OF_LIMITS


def grad_rtol(cond):
    for lo, hi, rtol in GRAD_BINS:
        if lo <= cond < hi:
            return rtol
    raise AssertionError(f"cond(N_FF) = {cond:g}")


def oracle_rows(sc, prob, q, gq, n):
    """The oracle's gradient rows [n, target_stride], statuses and cond(N_FF) at fp32 q."""
    stride = int(prob.target_stride)
    rows, sts, conds = np.zeros((n, stride)), np.zeros(n, dtype=np.int32), np.zeros(n)
    for i in range(n):
        tasks = [oik._slice_task(t, i) for t in sc.oracle_tasks]
        qi = q[i].astype(np.float64)
        grads, sts[i] = ig.solution_vjp(sc.table, qi, tasks, sc.dt, gq[i].astype(np.float64), sc.damping,
                                        sc.oracle_limits)
        held = ig.held_coordinates(sc.table, qi, tasks, sc.dt, sc.damping, sc.oracle_limits)
        N = ig.normal_matrix(sc.table, qi, okin.forward_kinematics(sc.table, qi), tasks)[np.ix_(~held, ~held)]
        conds[i] = np.linalg.cond(N)
        for k, g in enumerate(grads):
            if g is not None and not prob.tasks[k].target_shared:
                off = int(prob.tasks[k].target_offset)
                rows[i, off:off + g.size] += g
    return rows, sts, conds


def converged_case(sc, mask, tol, max_steps, seed=0):
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    q, err, _, st = hs.converge(prob, sc.q32, targets, mask, tol, max_steps)
    gq = np.random.default_rng(seed).normal(size=q.shape).astype(np.float32)
    return hs, prob, targets, q, gq


@pytest.mark.parametrize("case", ["ur5", "chain7_posture_rows", "g1_com_relative", "tree_extras40"])
def test_body_against_oracle(case):
    if case == "ur5":
        sc, mask = helpers.ur5_scenario(16, posture_cost=1e-3), 1
    elif case == "chain7_posture_rows":
        sc, mask = helpers.chain_scenario(7, 16, two_tasks=True, posture_per_instance=True), 3
    elif case == "g1_com_relative":
        sc = helpers.humanoid_scenario("g1_description", 8, with_com=True, with_relative=True)
        mask = (1 << len(sc.tasks)) - 1 - (1 << 5)  # every task but the posture task
    else:
        sc = helpers.tree_scenario(40, 8)
        mask = (1 << len(sc.tasks)) - 1 - (1 << 3)
    hs, prob, targets, q, gq = converged_case(sc, mask, 1e-4, 60)
    gt, st = HostVjp(sc.model).converge_vjp(prob, q, targets, gq)
    ref, ref_st, cond = oracle_rows(sc, prob, q, gq, sc.B)
    assert (st == ref_st).all(), (st, ref_st)
    for i in range(sc.B):
        tol = grad_rtol(cond[i]) * np.abs(ref[i]).max() + 1e-6
        assert np.abs(gt[i] - ref[i]).max() <= tol, (i, cond[i], np.abs(gt[i] - ref[i]).max(), tol)


def test_not_positive_definite_seven_joints_one_frame_task():
    sc = helpers.chain_scenario(7, 8)
    sc.tasks, sc.oracle_tasks = sc.tasks[:1], sc.oracle_tasks[:1]
    prob, targets, _ = sc.problem()
    gq = np.ones((sc.B, sc.table.nq), dtype=np.float32)
    gt, st = HostVjp(sc.model).converge_vjp(prob, sc.q32, targets, gq)
    _, ref_st, _ = oracle_rows(sc, prob, sc.q32, gq, sc.B)
    assert (st == _cabi.PK_STATUS_NOT_POSDEF).all() and (ref_st == 4).all()
    assert not gt.any()


# ---- BatchedIK on the host build -------------------------------------------------------------


class _HostLib:
    """The entries of libpink_b200.so that BatchedIK's converge calls use, on the host builds;
    a failing entry raises with the host build's message."""

    def __init__(self, hs, hv):
        self.hs, self.hv, self.problems = hs, hv, {}

    @staticmethod
    def _p(a):
        return None if a is None else C.c_void_p(a)

    @staticmethod
    def _rc(rc, last_error):
        if rc:
            raise RuntimeError("pink_b200: " + last_error().decode())
        return 0

    def pk_problem_create(self, model, prob, handle):
        key = len(self.problems) + 1
        self.problems[key] = prob._obj
        handle._obj.value = key
        return 0

    def pk_problem_destroy(self, handle):
        pass

    def pk_converge_prepared(self, model, h, q, t, mask, tol, max_steps, q_out, err, steps, status, B, stream):
        p = self._p
        return self._rc(hostsim.lib().hs_converge(
            self.hs.handle, C.byref(self.problems[h.value]), p(q), p(t), C.c_uint32(mask), C.c_float(tol),
            C.c_int(max_steps), p(q_out), p(err), p(steps), p(status), C.c_int64(B), 0, (C.c_int * 8)()),
            hostsim.lib().hs_last_error)

    def pk_converge_multistart_prepared(self, model, h, qs, S, t, mask, tol, max_steps, q_out, err, seed, steps,
                                        status, B, stream):
        if B == 0:
            return 0
        p = self._p
        return self._rc(hostsim.lib().hs_converge_multistart(
            self.hs.handle, C.byref(self.problems[h.value]), p(qs), S, p(t), C.c_uint32(mask), C.c_float(tol),
            C.c_int(max_steps), p(q_out), p(err), p(seed), p(steps), p(status), C.c_int64(B), 0, (C.c_int * 8)()),
            hostsim.lib().hs_last_error)

    def pk_converge_vjp_prepared(self, model, h, q, t, gq, gt, status, B, stream):
        return self._rc(self.hv.converge_vjp_raw(self.problems[h.value], q, t, gq, gt, status, B),
                        hostsim_vjp.lib().hv_last_error)


class _HostBatchedEngine:
    def __init__(self, model):
        self.hs = HostSim(model)
        self.lib = _HostLib(self.hs, HostVjp(model))
        self.handle = None
        self.device = torch.device("cpu")
        self.nq, self.nv = self.hs.nq, self.hs.nv


@pytest.fixture
def host_batched(monkeypatch, host_engine):  # noqa: F811
    import pink_b200.batched as bmod

    monkeypatch.setattr(bmod, "get_engine", lambda model, device=None: _HostBatchedEngine(model))
    monkeypatch.setattr(bmod, "_stream", lambda device: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    return bmod


def _ur5_example(B, seed=0):
    from examples import arm_ur5_reach_batched as ex

    return ex.setup(B, device="cpu", seed=seed)


def test_backward_equals_converge_vjp_and_zeroes_unconverged_rows(host_batched):
    ik, task, q0, targets = _ur5_example(24)
    tg = targets.clone().requires_grad_(True)
    res = ik.converge(q0, tg, [task], 1e-5, 8)  # some instances do not converge in 8 steps
    assert res.q.grad_fn is not None
    assert all(not t.requires_grad for t in (res.error, res.steps, res.status, res.converged))
    assert 0 < int(res.converged.sum()) < 24
    W = torch.randn(res.q.shape, generator=torch.Generator().manual_seed(1))
    (res.q * W).sum().backward()
    gt, st = ik.converge_vjp(res.q.detach().contiguous(), targets, W.contiguous())
    ok = res.converged & ((res.status & FAILED) == 0)
    assert torch.equal(tg.grad[ok], gt[ok])
    assert not tg.grad[~ok].any()
    assert (st == 0).all()


def test_multistart_winner_gradient_equals_converge_vjp(host_batched):
    ik, task, q0, targets = _ur5_example(8, seed=2)
    seeds = ik.sample_seeds(q0, 4, generator=torch.Generator().manual_seed(3))
    tg = targets.clone().requires_grad_(True)
    res = ik.converge_multistart(seeds, tg, [task], 1e-5, 60)
    W = torch.randn(res.q.shape, generator=torch.Generator().manual_seed(4))
    (res.q * W).sum().backward()
    gt, _ = ik.converge_vjp(res.q.detach().contiguous(), targets, W.contiguous())
    ok = res.converged & ((res.status & FAILED) == 0)
    assert ok.any()
    assert torch.equal(tg.grad[ok], gt[ok]) and not tg.grad[~ok].any()


def test_outputs_without_gradient_are_unchanged(host_batched):
    ik, task, q0, targets = _ur5_example(16)
    plain = ik.converge(q0, targets, [task], 1e-5, 40)
    graded = ik.converge(q0, targets.clone().requires_grad_(True), [task], 1e-5, 40)
    assert plain.q.grad_fn is None
    for a, b in zip(plain, graded):
        assert torch.equal(a, b.detach())
    with torch.no_grad():
        nograd = ik.converge(q0, targets.clone().requires_grad_(True), [task], 1e-5, 40)
    assert nograd.q.grad_fn is None


def _quat_to_matrix(qt):
    x, y, z, w = (qt / qt.norm(dim=-1, keepdim=True)).unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def test_quaternion_parameterised_target_matches_finite_differences(host_batched):
    """The 12-float gradient through a quaternion -> matrix map in torch equals the finite
    differences of the oracle's fixed point with respect to the quaternion (UR5, one full-pose
    frame task: the fixed point has zero residual)."""
    from oracle import lie
    from tests import converge_grad_cases as cg

    ik, task, q0, targets = _ur5_example(4, seed=5)
    T = targets.reshape(-1, 3, 4).double()
    quat = torch.as_tensor(lie.matrix_to_quat(T[:, :, :3].numpy())).requires_grad_(True)
    p = T[:, :, 3]
    rows = torch.cat([_quat_to_matrix(quat), p[:, :, None]], dim=2).reshape(-1, 12).float().contiguous()
    res = ik.converge(q0, rows, [task], 1e-6, 300)
    assert res.converged.all()
    g = torch.randn(res.q.shape, generator=torch.Generator().manual_seed(6))
    (res.q * g).sum().backward()
    table = ik.model.table()
    f = table.frame_names.index("tool0")
    for i in range(2):
        for k in range(4):
            def L(h):
                qk = quat[i].detach().numpy().copy()
                qk[k] += h
                R = _quat_to_matrix(torch.as_tensor(qk)[None]).numpy()[0]
                otask = {"type": "frame", "frame": f, "cost": np.ones(6), "gain": 1.0, "lm_damping": 0.0,
                         "target": (R, p[i].numpy())}
                qs, _ = ig.fixed_point(table, res.q[i].detach().double().numpy(), [otask], limits=cg.CFG_ONLY,
                                       tol=1e-14)
                return g[i].double().numpy() @ qs
            fd = cg.richardson(L, 1e-4)
            assert abs(quat.grad[i, k].item() - fd) <= 2e-3 * max(1.0, abs(fd)), (i, k, quat.grad[i, k].item(), fd)


def test_gradient_mode_rejects_problems_it_cannot_bound(host_batched):
    from pink_b200 import BatchedIK, FrameTask, PostureTask
    from pink_b200.barriers import PositionBarrier
    from pink_b200.limits import AccelerationLimit, ConfigurationLimit, VelocityLimit

    ik, task, q0, targets = _ur5_example(4)
    tg = targets.clone().requires_grad_(True)
    model = ik.model
    post = PostureTask(cost=1e-3)
    post.set_target(np.zeros(model.nq))
    two = BatchedIK(model, [task, post], 1e-2, batch_size=4)
    with pytest.raises(ValueError, match="stopping test"):
        two.converge(q0, tg, [post], 1e-5, 10)
    two.converge(q0, targets, [post], 1e-5, 10)  # fine without a gradient
    from pink_b200.model import SE3

    held = FrameTask("wrist_1_link", position_cost=1.0, orientation_cost=0.0)
    held.set_target(SE3(np.eye(3), np.zeros(3)))
    cases = [
        (dict(barriers=[PositionBarrier("tool0", indices=[2], p_max=np.array([2.0]), gain=1.0)]), "barriers"),
        (dict(constraints=[held]), "constraints"),
        (dict(limits=[ConfigurationLimit(model), VelocityLimit(model), AccelerationLimit(model, np.full(model.nv, 10.0))]),
         "AccelerationLimit"),
    ]
    for kw, what in cases:
        solver = BatchedIK(model, [task], 1e-2, batch_size=4, **kw)
        with pytest.raises(ValueError, match=what):
            solver.converge(q0, tg, [task], 1e-5, 10)

"""Solve to a tolerance (``pk_converge_prepared``) on the CPU build of the kernel bodies: the
converge loop of every path (chain, tree, general in its size classes) against the same loop
written in Python with separate host ``solve_ik``, ``integrate`` and ``task_terms`` calls and
the stop rule

    for s = 0, 1, ...: stop at q_s if err(q_s) <= tol or s == max_steps; solve step s;
                       stop at q_s if the freeze rule fires; q_{s+1} = q_s (+) v dt,

and against the fp64 oracle's task errors at the returned configuration."""

import numpy as np
import pytest

from oracle import kinematics as okin
from oracle import tasks as otasks
from pink_b200 import _cabi
from tests import extras, helpers
from tests.hostsim import HostSim

FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF


def _rows(table, prob, t):
    ty = int(prob.tasks[t].type)
    if ty == _cabi.PK_TASK_POSTURE:
        return table.nv - (6 if table.free_flyer else 0)
    return 3 if ty == _cabi.PK_TASK_COM else 6


def task_error(hs, table, prob, mask, q, targets):
    """max over the tasks of mask of |e_t|_2 from the task-terms body (fp32, NaN kept)."""
    err = np.zeros(q.shape[0], dtype=np.float32)
    for t in range(int(prob.ntasks)):
        if (mask >> t) & 1:
            e, _ = hs.task_terms(prob, t, _rows(table, prob, t), q, targets)
            err = np.maximum(err, np.linalg.norm(e, axis=1))
    return err


def python_loop(hs, table, prob, q, targets, mask, tol, max_steps, dt, safety_break, path):
    """(q_out, err, steps, status, errors along the way) of separate host calls with the stop rule."""
    B = q.shape[0]
    q = q.astype(np.float32).copy()
    done = np.zeros(B, dtype=bool)
    err = np.zeros(B, dtype=np.float32)
    steps = np.zeros(B, dtype=np.int32)
    st_all = np.zeros(B, dtype=np.int32)
    history = []
    for s in range(max_steps + 1):
        e = task_error(hs, table, prob, mask, q, targets)
        history.append(np.where(done, np.nan, e))
        stop = ~done & ((e <= tol) | (s == max_steps))
        err[stop], steps[stop] = e[stop], s
        done |= stop
        if done.all():
            break
        v, st = hs.solve_ik(prob, q, targets, path=path)
        st_all[~done] |= st[~done]
        bad = (st_all & FAILED) != 0
        if safety_break:
            bad |= (st_all & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
        frozen = ~done & bad
        err[frozen], steps[frozen] = e[frozen], s + 1
        done |= frozen
        qn = hs.integrate(q, v, dt)
        q[~done] = qn[~done]
    return q, err, steps, st_all, np.array(history)


def oracle_error(sc, q_out, mask, n):
    """fp64 max over the tasks of mask of |e_t| at q_out[:n]."""
    q = q_out[:n].astype(np.float64)
    fk = okin.forward_kinematics(sc.table, q)
    from oracle import ik as oik

    err = np.zeros(n)
    for t, task in enumerate(sc.oracle_tasks):
        if (mask >> t) & 1:
            e, _ = otasks.task_error_jacobian(sc.table, q, fk, oik._slice_task_range(task, 0, n))
            err = np.maximum(err, np.linalg.norm(e, axis=-1))
    return err


def check(sc, mask, tol, max_steps, path=0, expect=None, q=None, targets=None, n_oracle=16):
    prob, tg, _ = sc.problem()
    targets = tg if targets is None else targets
    q = sc.q32 if q is None else q
    hs = HostSim(sc.model)
    q_out, err, steps, st = hs.converge(prob, q, targets, mask, tol, max_steps, path=path)
    if expect is not None:
        assert hs.selection.path == expect, hs.selection
    q_l, err_l, steps_l, st_l, _ = python_loop(hs, sc.table, prob, q, targets, mask, tol, max_steps, sc.dt,
                                               sc.safety_break, path)
    np.testing.assert_array_equal(steps, steps_l)
    np.testing.assert_array_equal(st, st_l)
    np.testing.assert_array_equal(q_out.view(np.int32), q_l.view(np.int32))
    # the kernel's error comes from its own forward kinematics: equal to the task-terms body's up to
    # fp32 pose resolution
    fin = np.isfinite(err_l)
    assert (np.isfinite(err) == fin).all()
    np.testing.assert_allclose(err[fin], err_l[fin], rtol=1e-6, atol=5e-7)
    np.testing.assert_array_equal(err <= tol, err_l <= tol)
    n = min(n_oracle, q.shape[0])
    if n:
        ok = np.isfinite(err[:n])
        np.testing.assert_allclose(err[:n][ok], oracle_error(sc, q_out, mask, n)[ok], rtol=1e-3, atol=5e-6)
    return q_out, err, steps, st


# ---- paths ---------------------------------------------------------------------------------

def test_chain_ur5_reachable():
    sc = helpers.ur5_scenario(96, "reachable", out_of_limits=3)
    q_out, err, steps, st = check(sc, 0b01, 1e-4, 60, expect="chain")
    assert (err <= 1e-4).sum() > 60
    # the three instances outside their limits stop after one step with OUT_OF_LIMITS
    assert ((st & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0).sum() == 3
    assert (steps[(st & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0] == 1).all()


def test_chain_ur5_frame_and_posture_mask():
    sc = helpers.ur5_scenario(48, "reachable")
    check(sc, 0b11, 0.5, 30, expect="chain")


def test_chain_ur5_unreachable_runs_to_max_steps():
    sc = helpers.ur5_scenario(32, "unreachable")
    _, err, steps, st = check(sc, 0b01, 1e-4, 12, expect="chain")
    alive = (st & FAILED) == 0
    assert alive.sum() > 20
    assert (steps[alive] == 12).all() and (err[alive] > 1e-4).all()


@pytest.mark.parametrize("nj,kw", [(2, {}), (4, {"two_tasks": True}), (7, {"two_tasks": True, "prismatic": (2,)})])
def test_chain_instantiations(nj, kw):
    sc = helpers.chain_scenario(nj, 40, seed=nj, **kw)
    prob, _, _ = sc.problem()
    mask = (1 << int(prob.ntasks)) - 1
    for t in range(int(prob.ntasks)):
        if int(prob.tasks[t].type) == _cabi.PK_TASK_POSTURE:
            mask &= ~(1 << t)  # frame tasks only: the max of two frame errors when there are two
    check(sc, mask, 1e-3, 25, expect="chain")


def test_tree_g1_com():
    sc = helpers.humanoid_scenario("g1_description", 24, with_com=True)
    prob, _, _ = sc.problem()
    com = [t for t in range(int(prob.ntasks)) if int(prob.tasks[t].type) == _cabi.PK_TASK_COM][0]
    check(sc, (1 << 1) | (1 << 2) | (1 << com), 2e-3, 25, expect="tree")


def test_tree_relative_frame_in_mask():
    sc = helpers.humanoid_scenario("g1_description", 16, with_com=True, with_relative=True)
    prob, _, _ = sc.problem()
    n = int(prob.ntasks)
    check(sc, (1 << (n - 1)) | (1 << (n - 2)), 2e-3, 15, expect="tree")


@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_general_path_forced(name):
    if name == "ur5":
        sc = helpers.ur5_scenario(32, "reachable", out_of_limits=2)
        mask = 0b01
    else:
        sc = helpers.humanoid_scenario("g1_description", 16, with_com=True)
        mask = 0b110
    check(sc, mask, 1e-3, 20, path=1, expect="general")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 12, True, seed=7)
    prob, _, _ = sc.problem()
    mask = 0
    for t in range(int(prob.ntasks)):
        if int(prob.tasks[t].type) in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_COM):
            mask |= 1 << t
    check(sc, mask, 1e-3, 8, expect="general", n_oracle=0)


# ---- edge cases ----------------------------------------------------------------------------

def test_tol_met_at_start_and_zero_max_steps():
    sc = helpers.ur5_scenario(16, "at_target")
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    q_out, err, steps, st = hs.converge(prob, sc.q32, targets, 0b01, 1e-4, 50)
    assert (steps == 0).all() and (st == 0).all() and (err <= 1e-4).all()
    np.testing.assert_array_equal(q_out.view(np.int32), sc.q32.view(np.int32))
    sc = helpers.ur5_scenario(16, "reachable")
    prob, targets, _ = sc.problem()
    q_out, err, steps, st = hs.converge(prob, sc.q32, targets, 0b01, 1e-4, 0)
    assert (steps == 0).all() and (st == 0).all() and (err > 1e-4).all()
    np.testing.assert_array_equal(q_out.view(np.int32), sc.q32.view(np.int32))
    np.testing.assert_allclose(err, task_error(hs, sc.table, prob, 0b01, sc.q32, targets), rtol=1e-6, atol=5e-7)


@pytest.mark.parametrize("path", [0, 1, 2])
def test_nan_target_takes_one_failed_step(path):
    sc = helpers.ur5_scenario(8, "reachable")
    prob, targets, _ = sc.problem()
    targets = targets.copy()
    targets[3, 5] = np.nan
    hs = HostSim(sc.model)
    q_out, err, steps, st = hs.converge(prob, sc.q32, targets, 0b01, 1e-4, 30, path=path)
    assert np.isnan(err[3]) and steps[3] == 1 and st[3] & FAILED
    np.testing.assert_array_equal(q_out[3].view(np.int32), sc.q32[3].view(np.int32))
    keep = np.arange(8) != 3
    assert np.isfinite(err[keep]).all() and (steps[keep] > 1).all()


@pytest.mark.parametrize("safety_break", [True, False])
def test_out_of_limits(safety_break):
    sc = helpers.ur5_scenario(24, "reachable", out_of_limits=4)
    sc.safety_break = safety_break
    _, err, steps, st = check(sc, 0b01, 1e-4, 30)
    oob = (st & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
    assert oob.sum() >= 4
    if safety_break:
        assert (steps[oob] == 1).all() and np.isfinite(err[oob]).all()
    else:  # outside the limits is not a reason to stop; an empty box (no solution) still is
        moving = oob & ((st & FAILED) == 0)
        assert moving.sum() >= 1 and (steps[moving] > 1).all()


def test_api_errors():
    sc = helpers.ur5_scenario(4, "reachable")
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    for args in ((0, 1e-3, 5), (0b100, 1e-3, 5), (0b01, -1.0, 5), (0b01, float("nan"), 5), (0b01, float("inf"), 5),
                 (0b01, 1e-3, -1)):
        with pytest.raises(RuntimeError):
            hs.converge(prob, sc.q32, targets, *args)
    with pytest.raises(RuntimeError):
        hs.converge(prob, sc.q32, None, 0b01, 1e-3, 5)


# ---- the reference's test_single_task_convergence on UR5 -------------------------------------

def test_single_task_convergence_ur5():
    """A target 0.1 m from the start pose, one FrameTask: every instance converges within the
    reference's 42 steps (tests/test_solve_ik.py, test_single_task_convergence), and the error
    decreases strictly along the loop."""
    import torch

    from pink_b200 import FrameTask
    from pink_b200.solve_ik import describe_problem

    robot, model, table = helpers.load("ur5_description")
    rng = np.random.default_rng(11)
    B = 24
    q = np.array([0.0, -1.2, 1.4, -1.7, -1.57, 0.0]) + rng.uniform(-0.1, 0.1, size=(B, table.nq))
    f = table.frame_names.index("tool0")
    R, p = okin.frame_placement(table, okin.forward_kinematics(table, q), f)
    p = p + 0.1 * R[:, :, 2]  # 0.1 m along the frame's z axis, as the reference
    T = np.concatenate([R, p[:, :, None]], axis=2).astype(np.float32)
    task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    task.set_target(torch.as_tensor(T))
    from pink_b200.configuration import Configuration

    Configuration(model, None, np.zeros(model.nq))
    dt = 5e-3
    prob, parts, _ = describe_problem(model, B, [task], dt, 1e-12, [model.configuration_limit, model.velocity_limit],
                                      True)
    targets = torch.cat([x.float() for x in parts], dim=1).numpy()
    hs = HostSim(model)
    q32 = q.astype(np.float32)
    tol = 1e-5
    q_out, err, steps, st = hs.converge(prob, q32, targets, 0b1, tol, 200)
    assert (err <= tol).all() and (steps <= 42).all() and (st == 0).all(), (err.max(), steps.max())
    _, _, steps_l, _, hist = python_loop(hs, table, prob, q32, targets, 0b1, tol, 200, dt, True, 0)
    np.testing.assert_array_equal(steps, steps_l)
    for i in range(B):
        e = hist[: steps[i] + 1, i]
        assert (np.diff(e) < 0).all(), e

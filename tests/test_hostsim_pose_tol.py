"""Separate position and orientation tolerances (``pk_converge_pose_tol_prepared`` and
``pk_converge_goalset_pose_tol_prepared``) on the CPU build of the kernel bodies: the converge
loop of every path against the same loop written in Python with separate host ``solve_ik``,
``integrate`` and ``task_terms`` calls under the stop rule

    err(q) = max over the tasks of the mask of err_t, from the rows the task weighs (cost > 0):
             frame / relative frame  max(|e[0:3]|, (tol / orientation_tol) |e[3:6]|)
             CoM, linear             |e|
             posture                 |e|

and against the fp64 restatement of ``oracle.pose_tol``."""

import numpy as np
import pytest
import torch

from oracle import ik as oik
from oracle import pose_tol as opt
from pink_b200 import FrameTask, _cabi
from tests import extras, helpers
from tests.host_engine import host_engine  # noqa: F401  (fixture)
from tests.hostsim import HostSim
from tests.hostsim_pose_tol import HostPoseTol
from tests.hostsim_vjp import HostVjp
from tests.test_hostsim_converge_grad import _ur5_example, host_batched  # noqa: F401  (fixture)
from tests.test_hostsim_goalset import stop_mask

FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF
POSE_TYPES = (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_RELATIVE_FRAME)


def _rows(table, prob, t):
    ty = int(prob.tasks[t].type)
    if ty == _cabi.PK_TASK_POSTURE:
        return table.nv - (6 if table.free_flyer else 0)
    if ty == _cabi.PK_TASK_LINEAR:
        return int(prob.tasks[t].rows)
    return 3 if ty == _cabi.PK_TASK_COM else 6


def pose_error(hs, table, prob, mask, q, targets, tol, otol):
    """err(q) of the separate tolerances from the task-terms body (fp32, NaN kept)."""
    err = np.zeros(q.shape[0], dtype=np.float32)
    for t in range(int(prob.ntasks)):
        if not (mask >> t) & 1:
            continue
        d = prob.tasks[t]
        e, _ = hs.task_terms(prob, t, _rows(table, prob, t), q, targets)
        if int(d.type) == _cabi.PK_TASK_POSTURE:
            et = np.linalg.norm(e, axis=1)
        else:
            w = np.array([float(d.cost[r]) > 0.0 for r in range(e.shape[1])])
            ew = np.where(w, e, np.float32(0.0))
            if int(d.type) in POSE_TYPES:
                lin = np.linalg.norm(ew[:, :3], axis=1)
                ang = np.linalg.norm(ew[:, 3:], axis=1) if np.isfinite(otol) else np.zeros_like(lin)
                rs = np.float32(tol) / np.float32(otol) if np.isfinite(otol) else np.float32(0.0)
                et = np.where(np.isnan(lin) | np.isnan(ang), np.nan, np.maximum(lin, rs * ang)).astype(np.float32)
            else:
                et = np.linalg.norm(ew, axis=1)
        err = np.where(np.isnan(err) | np.isnan(et), np.nan, np.maximum(err, et)).astype(np.float32)
    return err


def python_loop(hs, table, prob, q, targets, mask, tol, otol, max_steps, dt, safety_break, path):
    """(q_out, err, steps, status) of separate host calls under the separate-tolerance rule."""
    B = q.shape[0]
    q = q.astype(np.float32).copy()
    done = np.zeros(B, dtype=bool)
    err = np.zeros(B, dtype=np.float32)
    steps = np.zeros(B, dtype=np.int32)
    st_all = np.zeros(B, dtype=np.int32)
    for s in range(max_steps + 1):
        e = pose_error(hs, table, prob, mask, q, targets, tol, otol)
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
    return q, err, steps, st_all


def oracle_error(sc, q_out, mask, n, tol, otol):
    tasks = [oik._slice_task_range(t, 0, n) for k, t in enumerate(sc.oracle_tasks) if (mask >> k) & 1]
    return opt.stop_error(sc.table, q_out[:n], tasks, tol, otol)


def check(sc, mask, tol, otol, max_steps, path=0, expect=None, n_oracle=16):
    prob, targets, _ = sc.problem()
    hp = HostPoseTol(sc.model)
    q_out, err, steps, st = hp.converge(prob, sc.q32, targets, mask, tol, otol, max_steps, path=path)
    if expect is not None:
        assert hp.selection.path == expect, hp.selection
    hs = HostSim(sc.model)
    q_l, err_l, steps_l, st_l = python_loop(hs, sc.table, prob, sc.q32, targets, mask, tol, otol, max_steps, sc.dt,
                                            sc.safety_break, path)
    np.testing.assert_array_equal(steps, steps_l)
    np.testing.assert_array_equal(st, st_l)
    np.testing.assert_array_equal(q_out.view(np.int32), q_l.view(np.int32))
    fin = np.isfinite(err_l)
    assert (np.isfinite(err) == fin).all()
    np.testing.assert_allclose(err[fin], err_l[fin], rtol=1e-5, atol=5e-7)
    np.testing.assert_array_equal(err <= tol, err_l <= tol)
    n = min(n_oracle, sc.B)
    if n:
        ok = np.isfinite(err[:n])
        np.testing.assert_allclose(err[:n][ok], oracle_error(sc, q_out, mask, n, tol, otol)[ok], rtol=1e-3,
                                   atol=5e-6)
    return q_out, err, steps, st


def position_only_ur5(B, seed=0):
    """UR5 with a position-only tool task (orientation cost 0) and a posture task of cost 1e-3."""
    sc = helpers.ur5_scenario(B, "reachable", seed=seed)
    T = np.concatenate([sc.oracle_tasks[0]["target"][0], sc.oracle_tasks[0]["target"][1][:, :, None]], axis=2)
    ft = FrameTask("tool0", position_cost=1.0, orientation_cost=0.0, lm_damping=1.0)
    ft.set_target(torch.as_tensor(T.astype(np.float32)))
    sc.tasks[0] = ft
    sc.oracle_tasks[0] = dict(sc.oracle_tasks[0], cost=np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]))
    return sc


def g1_reach(B, sigma=0.15, seed=0, posture_at_start=True, posture_cost=None):
    """The G1 task set of examples/humanoid_g1_reach_batched.py: every target taken at a
    configuration that moves only the arm joints of the start (the wrists reach; the feet, the
    pelvis and the CoM hold), the posture task toward the start (``posture_at_start``) or toward
    that configuration, where every error is zero."""
    from oracle import kinematics as okin
    from pink_b200 import ComTask, PostureTask, workloads

    robot, model, table = helpers.load("g1_description")
    rng = np.random.default_rng(seed)
    q = workloads.sample_configurations(table, B, rng, near_limit_fraction=0.0)
    qt = q.copy()
    arms = [7 + i for i, n in enumerate(table.joint_names) if any(a in n for a in ("shoulder", "elbow", "wrist"))]
    qt[:, arms] = workloads.perturb_configurations(table, q, rng, sigma=sigma)[:, arms]
    tasks, otasks = [], []
    for frame, pc, oc in workloads.G1_FRAME_TASKS:
        T = helpers.frame_targets(table, qt, frame)
        t = FrameTask(frame, position_cost=pc, orientation_cost=oc)
        t.set_target(torch.as_tensor(T))
        tasks.append(t)
        T64 = T.astype(np.float64)
        otasks.append({"type": "frame", "frame": table.frame_names.index(frame), "cost": np.array(t.cost),
                       "gain": 1.0, "lm_damping": 0.0, "target": (T64[:, :, :3], T64[:, :, 3])})
    q_ref = (q if posture_at_start else qt).astype(np.float32)
    posture_cost = workloads.G1_POSTURE_COST if posture_cost is None else posture_cost
    pt = PostureTask(cost=posture_cost)
    pt.set_target(torch.as_tensor(q_ref))
    tasks.append(pt)
    otasks.append({"type": "posture", "cost": posture_cost, "gain": 1.0, "lm_damping": 0.0,
                   "target": q_ref.astype(np.float64)})
    com = okin.center_of_mass(table, okin.forward_kinematics(table, qt)).astype(np.float32)
    ct = ComTask(cost=workloads.G1_COM_COST)
    ct.set_target(torch.as_tensor(com))
    tasks.append(ct)
    otasks.append({"type": "com", "cost": np.full(3, workloads.G1_COM_COST), "gain": 1.0, "lm_damping": 0.0,
                   "target": com.astype(np.float64)})
    return helpers.Scenario("g1-reach", robot, model, table, q, tasks, otasks, 1.0 / 200.0, workloads.G1_DAMPING,
                            safety_break=False)


def all_tasks_but_posture(prob):
    return sum(1 << t for t in range(int(prob.ntasks)) if int(prob.tasks[t].type) != _cabi.PK_TASK_POSTURE)


# ---- paths ---------------------------------------------------------------------------------

@pytest.mark.parametrize("nft", [0, 1, 2])
@pytest.mark.parametrize("nj", [2, 3, 4, 5, 6, 7])
def test_chain_instantiations(nj, nft):
    # the elbow task of two_tasks weighs no y translation: an untested row
    kw = {0: {"frame_tasks": False, "posture_per_instance": True}, 1: {}, 2: {"two_tasks": True}}[nft]
    if nj in (3, 7):
        kw["prismatic"] = (1,)
    sc = helpers.chain_scenario(nj, 32, seed=nj, **kw)
    check(sc, stop_mask(sc.problem()[0]), 1e-3, 1e-2, 25, expect="chain")


def test_chain_position_only_ur5():
    sc = position_only_ur5(48)
    _, err, steps, st = check(sc, 0b01, 1e-4, 1e-3, 80, expect="chain")
    assert (err <= 1e-4).sum() >= 40 and (steps[err <= 1e-4] < 80).all()


def test_tree_g1_every_frame_task_and_com():
    sc = g1_reach(24)
    prob, _, _ = sc.problem()
    _, err, steps, _ = check(sc, all_tasks_but_posture(prob), 2e-3, 2e-2, 40, expect="tree")
    assert (err <= 2e-3).sum() >= 16 and (steps[err <= 2e-3] < 40).all()


def test_tree_relative_frame():
    sc = helpers.humanoid_scenario("g1_description", 12, with_com=True, with_relative=True)
    prob, _, _ = sc.problem()
    check(sc, all_tasks_but_posture(prob), 2e-3, 2e-2, 25, expect="tree")


@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_general_path_forced(name):
    if name == "ur5":
        sc, mask = position_only_ur5(24), 0b01
    else:
        sc = g1_reach(12)
        mask = all_tasks_but_posture(sc.problem()[0])
    check(sc, mask, 2e-3, 2e-2, 20, path=1, expect="general")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 12, True, seed=7)
    prob, _, _ = sc.problem()
    mask = 0
    for t in range(int(prob.ntasks)):
        if int(prob.tasks[t].type) in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_COM):
            mask |= 1 << t
    check(sc, mask, 1e-3, 1e-2, 8, expect="general", n_oracle=0)


# ---- what the mode is for ------------------------------------------------------------------

def test_position_only_converges_where_the_default_test_cannot():
    sc = position_only_ur5(48, seed=3)
    prob, targets, _ = sc.problem()
    _, err, steps, _ = HostPoseTol(sc.model).converge(prob, sc.q32, targets, 0b01, 1e-4, 1e-3, 100)
    _, err_d, steps_d, st_d = HostSim(sc.model).converge(prob, sc.q32, targets, 0b01, 1e-4, 100)
    ok = err <= 1e-4
    assert ok.sum() >= 40 and np.median(steps[ok]) < 50
    alive = (st_d & FAILED) == 0
    assert (steps_d[ok & alive] == 100).all() and (err_d[ok & alive] > 1e-4).all()


@pytest.mark.parametrize("path", [0, 1, 2])
def test_superset_of_the_default_test(path):
    sc = helpers.ur5_scenario(48, "reachable", seed=5)
    prob, targets, _ = sc.problem()
    tol = 1e-4
    _, err_d, steps_d, _ = HostSim(sc.model).converge(prob, sc.q32, targets, 0b01, tol, 60, path=path)
    _, err, steps, _ = HostPoseTol(sc.model).converge(prob, sc.q32, targets, 0b01, tol, tol, 60, path=path)
    old = err_d <= tol
    assert old.sum() >= 20
    assert (err[old] <= tol).all() and (steps[old] <= steps_d[old]).all()


@pytest.mark.parametrize("path", [0, 1, 2])
def test_infinite_orientation_tol_tests_translations_only(path):
    sc = helpers.ur5_scenario(32, "reachable", seed=6)
    prob, targets, _ = sc.problem()
    hp = HostPoseTol(sc.model)
    q_out, err, steps, _ = hp.converge(prob, sc.q32, targets, 0b01, 1e-3, np.inf, 0, path=path)
    fk_err = opt.stop_error(sc.table, sc.q32, [sc.oracle_tasks[0]], 1e-3, np.inf)
    np.testing.assert_allclose(err, fk_err, rtol=1e-4, atol=1e-6)
    e, _ = HostSim(sc.model).task_terms(prob, 0, 6, sc.q32, targets)
    np.testing.assert_allclose(err, np.linalg.norm(e[:, :3], axis=1), rtol=1e-5, atol=5e-7)
    assert (np.linalg.norm(e[:, 3:], axis=1) > err).any()  # the rotation parts would have decided


def test_axis_free_grasp_goal_set():
    """A grasp free about the tool axis (orientation cost [1, 1, 0]) among goals turned about that
    axis: the goal set converges and the tool z-axis ends within orientation_tol of the goal's."""
    sc = helpers.ur5_scenario(16, "reachable", seed=8)
    T = np.concatenate([sc.oracle_tasks[0]["target"][0], sc.oracle_tasks[0]["target"][1][:, :, None]], axis=2)
    ft = FrameTask("tool0", position_cost=1.0, orientation_cost=[1.0, 1.0, 0.0], lm_damping=1.0)
    ft.set_target(torch.as_tensor(T.astype(np.float32)))
    sc.tasks[0] = ft
    prob, targets, _ = sc.problem()
    G, S = 4, 2
    rng = np.random.default_rng(0)
    goals = np.repeat(targets[:, None], G, axis=1).copy()
    for g in range(G):
        a = rng.uniform(-np.pi, np.pi, size=sc.B)
        Rz = np.zeros((sc.B, 3, 3))
        Rz[:, 0, 0] = Rz[:, 1, 1] = np.cos(a)
        Rz[:, 0, 1], Rz[:, 1, 0] = -np.sin(a), np.sin(a)
        Rz[:, 2, 2] = 1.0
        R = T[:, :, :3] @ Rz
        goals[:, g, 0:12] = np.concatenate([R, T[:, :, 3:]], axis=2).reshape(sc.B, 12)
    seeds = np.stack([sc.q32, sc.q32[::-1]], axis=1)
    r = 2e-2
    q, err, goal, seed, steps, st = HostPoseTol(sc.model).converge_goalset(prob, seeds, goals, 0b01, 1e-3, r, 150)
    assert (err <= 1e-3).sum() >= 14
    from oracle import kinematics as okin

    fk = okin.forward_kinematics(sc.table, q.astype(np.float64))
    Rq, _ = okin.frame_placement(sc.table, fk, sc.table.frame_names.index("tool0"))
    Rg = goals[np.arange(sc.B), goal, 0:12].reshape(sc.B, 3, 4)[:, :, :3]
    tilt = np.arccos(np.clip(np.einsum("bi,bi->b", Rq[:, :, 2], Rg[:, :, 2]), -1.0, 1.0))
    ok = err <= 1e-3
    assert (tilt[ok] <= r * 1.01 + 1e-4).all(), tilt[ok].max()


@pytest.mark.parametrize("path", [0, 1, 2])
def test_one_goal_one_seed_equals_converge(path):
    sc = helpers.chain_scenario(6, 24, seed=4, two_tasks=True)
    prob, targets, _ = sc.problem()
    hp = HostPoseTol(sc.model)
    a = hp.converge(prob, sc.q32, targets, 0b111, 1e-3, 1e-2, 30, path=path)
    b = hp.converge_goalset(prob, sc.q32[:, None], targets[:, None], 0b111, 1e-3, 1e-2, 30, path=path)
    for x, y in zip(a, (b[0], b[1], b[4], b[5])):
        np.testing.assert_array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32))
    assert not b[2].any() and not b[3].any()


@pytest.mark.parametrize("path", [0, 1, 2])
def test_multistart_groups_against_the_group_rule(path):
    """S seeds, G goals: the winner's error is the smallest of the members' own converge, and the
    group stops no later than its fastest member."""
    sc = position_only_ur5(8, seed=9)
    prob, targets, _ = sc.problem()
    hp = HostPoseTol(sc.model)
    G, S = 2, 4
    rng = np.random.default_rng(1)
    seeds = np.repeat(sc.q32[:, None], S, axis=1) + rng.normal(scale=0.3, size=(sc.B, S, 6)).astype(np.float32)
    seeds = np.ascontiguousarray(seeds.astype(np.float32))
    goals = np.repeat(targets[:, None], G, axis=1)
    q, err, goal, seed, steps, st = hp.converge_goalset(prob, seeds, goals, 0b01, 1e-4, 1e-3, 60, path=path)
    per = [hp.converge(prob, np.ascontiguousarray(seeds[:, s]), targets, 0b01, 1e-4, 1e-3, 60, path=path)
           for s in range(S)]
    best = np.min(np.stack([p[2] for p in per]), axis=0)
    ok = err <= 1e-4
    assert ok.sum() >= 6 and (steps[ok] <= best[ok]).all()
    assert (goal == 0).all()  # duplicate goals: the earlier wins


# ---- the stop error at the rotation-angle edges ----------------------------------------------

def test_zero_steps_error_matches_the_oracle_on_the_angle_ladder():
    """err at max_steps = 0 against the separate-tolerance error of the ladder's fp64 logs (either
    log where the angle is pi), with all axes weighed and with the tool's z rotation free."""
    from tests import pose_edges as pe

    ladder = pe.Ladder()
    tol = 1e-3
    for ocost in (1.0, [1.0, 1.0, 0.0]):
        sc, k, case = pe.scenario("ur5", ladder)
        T = sc.tasks[k].transform_target_to_world
        ft = FrameTask("tool0", position_cost=1.0, orientation_cost=ocost, lm_damping=1.0)
        ft.set_target(T)
        sc.tasks[k] = ft
        prob, targets, _ = sc.problem()
        ref = pe.reference(sc, k)
        w = np.array([float(prob.tasks[k].cost[r]) > 0.0 for r in range(6)])
        for otol in (2e-2, np.inf):
            _, err, steps, _ = HostPoseTol(sc.model).converge(prob, sc.q32, targets, 1 << k, tol, otol, 0)
            assert (steps == 0).all()

            def stop(e):
                e = np.where(w, e, 0.0)
                ang = np.linalg.norm(e[:, 3:], axis=1) * (tol / otol if np.isfinite(otol) else 0.0)
                return np.maximum(np.linalg.norm(e[:, :3], axis=1), ang)

            n = stop(ref.e)
            d = np.abs(err - n)
            d = np.where(ref.two_logs, np.minimum(d, np.abs(err - stop(ref.e_alt))), d)
            assert (d <= pe.E_ATOL + pe.E_RTOL * n).all(), (ocost, otol, d.max())


# ---- argument errors -----------------------------------------------------------------------

def test_argument_errors():
    sc = position_only_ur5(4)
    prob, targets, _ = sc.problem()
    hp = HostPoseTol(sc.model)
    qs = sc.q32[:, None].copy()
    for tol, otol, msg in ((0.0, 1e-2, "tol must be finite and > 0"), (np.inf, 1e-2, "tol must be finite"),
                           (np.nan, 1e-2, "tol"), (1e-3, 0.0, "orientation_tol must be > 0"),
                           (1e-3, -1.0, "orientation_tol must be > 0"), (1e-3, np.nan, "orientation_tol must be > 0")):
        with pytest.raises(RuntimeError, match=msg):
            hp.converge(prob, sc.q32, targets, 0b01, tol, otol, 5)
        with pytest.raises(RuntimeError, match=msg):
            hp.converge_goalset(prob, qs, targets[:, None], 0b01, tol, otol, 5)
    # the position-only task keeps its translation rows; a rotation-only one has nothing left at inf
    hp.converge(prob, sc.q32, targets, 0b01, 1e-3, np.inf, 1)
    sc2 = helpers.ur5_scenario(4, "reachable")
    T = np.concatenate([sc2.oracle_tasks[0]["target"][0], sc2.oracle_tasks[0]["target"][1][:, :, None]], axis=2)
    ft = FrameTask("tool0", position_cost=0.0, orientation_cost=1.0)
    ft.set_target(torch.as_tensor(T.astype(np.float32)))
    sc2.tasks[0] = ft
    prob2, targets2, _ = sc2.problem()
    hp2 = HostPoseTol(sc2.model)
    hp2.converge(prob2, sc2.q32, targets2, 0b01, 1e-3, 1e-2, 1)
    with pytest.raises(RuntimeError, match="no weighed component"):
        hp2.converge(prob2, sc2.q32, targets2, 0b01, 1e-3, np.inf, 1)
    sc3 = helpers.ur5_scenario(4, "reachable", posture_cost=0.0)
    prob3, targets3, _ = sc3.problem()
    with pytest.raises(RuntimeError, match="no weighed component"):
        HostPoseTol(sc3.model).converge(prob3, sc3.q32, targets3, 0b10, 1e-3, 1e-2, 1)


# ---- gradients of position-only tasks --------------------------------------------------------

def test_position_only_gradient_matches_the_oracle():
    """The VJP body at solutions of the separate-tolerance loop, for a position-only task with a
    posture task: zero-cost rows enter neither N nor dc/dT, as in oracle.implicit_grad."""
    from tests.test_hostsim_converge_grad import grad_rtol, oracle_rows

    sc = position_only_ur5(12, seed=10)
    prob, targets, _ = sc.problem()
    q, err, _, st = HostPoseTol(sc.model).converge(prob, sc.q32, targets, 0b01, 1e-4, 1e-2, 200)
    ok = (err <= 1e-4) & ((st & FAILED) == 0)
    assert ok.sum() >= 8
    gq = np.random.default_rng(2).normal(size=q.shape).astype(np.float32)
    gt, gst = HostVjp(sc.model).converge_vjp(prob, q, targets, gq)
    ref, ref_st, cond = oracle_rows(sc, prob, q, gq, sc.B)
    for i in np.flatnonzero(ok):
        assert gst[i] == ref_st[i]
        bound = grad_rtol(cond[i]) * np.abs(ref[i]).max() + 1e-6
        assert np.abs(gt[i] - ref[i]).max() <= bound, (i, cond[i], np.abs(gt[i] - ref[i]).max(), bound)


# ---- BatchedIK's checks ------------------------------------------------------------------------

def test_batched_ik_argument_errors(host_batched):  # noqa: F811
    """BatchedIK rejects a bad orientation_tol before it reaches the library."""
    ik, task, q0, targets = _ur5_example(4)
    seeds = q0[:, None].contiguous()
    for tol, otol in ((0.0, 1e-2), (float("inf"), 1e-2), (float("nan"), 1e-2), (1e-3, 0.0), (1e-3, -1.0),
                      (1e-3, float("nan"))):
        with pytest.raises(ValueError, match="tol"):
            ik.converge(q0, targets, [task], tol, 5, orientation_tol=otol)
        with pytest.raises(ValueError, match="tol"):
            ik.converge_multistart(seeds, targets, [task], tol, 5, orientation_tol=otol)
        with pytest.raises(ValueError, match="tol"):
            ik.converge_goalset(seeds, targets[:, None].contiguous(), [task], tol, 5, orientation_tol=otol)
    with pytest.raises(ValueError, match="finite orientation_tol"):
        ik.converge(q0, targets.clone().requires_grad_(True), [task], 1e-3, 5, orientation_tol=float("inf"))
    ft = FrameTask("tool0", position_cost=0.0, orientation_cost=1.0)
    ft.set_target(targets.reshape(-1, 3, 4))
    ik2 = type(ik)(ik.model, [ft], 1e-2, batch_size=4)
    with pytest.raises(ValueError, match="weighs no component"):
        ik2.converge(q0, targets, [ft], 1e-3, 5, orientation_tol=float("inf"))

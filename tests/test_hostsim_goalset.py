"""Goal-set solve to a tolerance (``pk_converge_goalset_prepared``) on the CPU build of the kernel
bodies, on every path (chain, tree, general):

* with one goal, the goal-set loop (``hs_converge_goalset``, tests/hostsim_goalset) equals the
  multi-start loop (``hs_converge_multistart``) bitwise;
* with several, it equals the group rule written in Python with separate host ``solve_ik``,
  ``integrate`` and ``task_terms`` calls on the tiled ``[B*G*S, nq]`` batch, member
  ``j = g*S + s`` starting at seed s toward goal g:

      for s = 0, 1, ...: err of every member that has not failed (a failed member keeps its error);
          the group stops if some err <= tol, s == max_steps or every member has failed;
          every member that has not failed solves step s; a failing member keeps q_s;
      winner = the smallest error at the stopping round (NaN as +inf, ties to the lowest j);
      goal = winner // S, seed = winner % S;

plus the S = 1 superset of ``converge``, the edge cases of the rule, the argument checks and the
gradient glue of ``BatchedIK.converge_goalset``."""

import numpy as np
import pytest
import torch

from pink_b200 import _cabi
from pink_b200.batched import _solution_of_goals
from tests import extras, helpers
from tests.hostsim import HostSim
from tests.hostsim_goalset import HostGoalset
from tests.test_hostsim_converge import FAILED, task_error
from tests.test_hostsim_multistart import pose_mask, seeds_for, winner


def python_goalset_loop(hs, table, prob, qs, goals, mask, tol, max_steps, dt, safety_break, path):
    """(q [B, G*S, nq], err [B, G*S], steps [B], status [B, G*S]) of every member at the stopping
    round of its group, by the group rule with separate host calls."""
    B, S, nq = qs.shape
    G = goals.shape[1]
    M = G * S
    q = np.repeat(qs[:, None], G, axis=1).reshape(B * M, nq).astype(np.float32)
    t = np.repeat(goals, S, axis=1).reshape(B * M, -1).astype(np.float32)
    failed = np.zeros(B * M, dtype=bool)
    e_keep = np.zeros(B * M, dtype=np.float32)
    st_all = np.zeros(B * M, dtype=np.int32)
    done = np.zeros(B, dtype=bool)
    steps = np.zeros(B, dtype=np.int32)
    e_stop = np.zeros((B, M), dtype=np.float32)
    for s in range(max_steps + 1):
        e = np.where(failed, e_keep, task_error(hs, table, prob, mask, q, t))
        E, F = e.reshape(B, M), failed.reshape(B, M)
        stop = ~done & ((E <= tol).any(axis=1) | (s == max_steps) | F.all(axis=1))
        e_stop[stop], steps[stop] = E[stop], s
        done |= stop
        if done.all():
            break
        v, st = hs.solve_ik(prob, q, t, path=path)
        live = ~failed & ~np.repeat(done, M)
        st_all[live] |= st[live]
        bad = (st_all & FAILED) != 0
        if safety_break:
            bad |= (st_all & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
        newly = live & bad
        failed |= newly
        e_keep[newly] = e[newly]
        qn = hs.integrate(q, v, dt)
        adv = live & ~newly
        q[adv] = qn[adv]
    return q.reshape(B, M, nq), e_stop, steps, st_all.reshape(B, M)


def rolled_goals(targets, G):
    """goals[b, g] = the targets row of instance b - g: G complete, valid rows per instance."""
    return np.stack([np.roll(targets, g, axis=0) for g in range(G)], axis=1).astype(np.float32)


def check(sc, mask, tol, max_steps, G, S, path=0, expect=None, qs=None, goals=None):
    prob, targets, _ = sc.problem()
    qs = seeds_for(sc, S) if qs is None else qs
    goals = rolled_goals(targets, G) if goals is None else goals
    hs, hg = HostSim(sc.model), HostGoalset(sc.model)
    q_out, err, goal, seed, steps, st = hg.converge_goalset(prob, qs, goals, mask, tol, max_steps, path=path)
    if expect is not None:
        assert hg.selection.path == expect, hg.selection
    q_all, e_all, steps_l, st_all = python_goalset_loop(hs, sc.table, prob, qs, goals, mask, tol, max_steps, sc.dt,
                                                        sc.safety_break, path)
    np.testing.assert_array_equal(steps, steps_l)
    B = qs.shape[0]
    w = goal * S + seed
    assert ((goal >= 0) & (goal < G) & (seed >= 0) & (seed < S)).all()
    # the kernel's error comes from its own forward kinematics: where two members' errors agree
    # to that rounding, either may win
    w_l = winner(e_all)
    other = w != w_l
    np.testing.assert_allclose(e_all[np.arange(B), w][other], e_all[np.arange(B), w_l][other], rtol=1e-6, atol=5e-7)
    q_l, err_l, st_l = q_all[np.arange(B), w], e_all[np.arange(B), w], st_all[np.arange(B), w]
    np.testing.assert_array_equal(st, st_l)
    np.testing.assert_array_equal(q_out.view(np.int32), q_l.view(np.int32))
    fin = np.isfinite(err_l)
    assert (np.isfinite(err) == fin).all()
    np.testing.assert_allclose(err[fin], err_l[fin], rtol=1e-6, atol=5e-7)
    return q_out, err, goal, seed, steps, st


def stop_mask(prob):
    """The frame and CoM tasks, or the posture task of a chain without frame tasks."""
    return pose_mask(prob) or 1 << (int(prob.ntasks) - 1)


def ur5_mixed(B):
    """UR5 with G = 8 goals per instance: even goals reachable, odd goals out of reach."""
    sc = helpers.ur5_scenario(B, "reachable", out_of_limits=2)
    _, reach, _ = sc.problem()
    _, far, _ = helpers.ur5_scenario(B, "unreachable").problem()
    goals = rolled_goals(reach, 8)
    goals[:, 1::2] = rolled_goals(far, 4)
    return sc, goals


# ---- one goal is multi-start -----------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_one_goal_equals_multistart(which):
    if which == "tree":
        sc = helpers.humanoid_scenario("g1_description", 8, with_com=True)
    else:
        sc = helpers.ur5_scenario(24, "reachable", out_of_limits=2)
    prob, targets, _ = sc.problem()
    mask = pose_mask(prob)
    path = 1 if which == "general" else 0
    qs = seeds_for(sc, 4)
    hs, hg = HostSim(sc.model), HostGoalset(sc.model)
    ref = hs.converge_multistart(prob, qs, targets, mask, 1e-3, 20, path=path)
    q_out, err, goal, seed, steps, st = hg.converge_goalset(prob, qs, targets[:, None], mask, 1e-3, 20, path=path)
    assert hg.selection.path == which
    assert (goal == 0).all()
    for x, y in zip((q_out, err, seed, steps, st), ref):
        np.testing.assert_array_equal(x.view(np.int32), y.view(np.int32))


# ---- the group rule on every path ------------------------------------------------------------

@pytest.mark.parametrize("G,S", [(8, 1), (4, 2), (2, 4)])
def test_chain_ur5_mixed_goals(G, S):
    sc, goals = ur5_mixed(16)
    goals = goals[:, :G].copy()
    _, err, goal, seed, steps, _ = check(sc, 0b01, 1e-4, 30, G, S, goals=goals, expect="chain")
    assert (err <= 1e-4).sum() >= 4
    assert (goal % 2 == 0)[err <= 1e-4].all()  # the odd goals are out of reach


@pytest.mark.parametrize("nft", [0, 1, 2])
@pytest.mark.parametrize("nj", [2, 3, 4, 5, 6, 7])
def test_chain_instantiations(nj, nft):
    kw = {0: {"frame_tasks": False, "posture_per_instance": True}, 1: {}, 2: {"two_tasks": True}}[nft]
    if nj in (3, 7):
        kw["prismatic"] = (1,)
    sc = helpers.chain_scenario(nj, 8, seed=nj, **kw)
    prob, _, _ = sc.problem()
    check(sc, stop_mask(prob), 1e-3, 15, 2, 2, expect="chain")


@pytest.mark.parametrize("G,S", [(2, 1), (2, 4), (4, 2), (8, 1)])
def test_tree_g1_com(G, S):
    sc = helpers.humanoid_scenario("g1_description", 4, with_com=True)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 2e-3, 10, G, S, expect="tree")


@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_general_path_forced(name):
    if name == "ur5":
        sc = helpers.ur5_scenario(12, "reachable", out_of_limits=1)
    else:
        sc = helpers.humanoid_scenario("g1_description", 4, with_com=True)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 1e-3, 10, 2, 2, path=1, expect="general")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 4, True, seed=7)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 1e-3, 6, 2, 2, expect="general")


# ---- the S = 1 superset of converge ----------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_one_seed_superset_of_converge_toward_each_goal(which):
    if which == "chain":
        sc, goals = ur5_mixed(24)
        mask, tol, n = 0b01, 1e-4, 40
    else:
        sc = helpers.humanoid_scenario("g1_description", 6, with_com=True)
        goals = rolled_goals(sc.problem()[1], 4)
        mask, n = pose_mask(sc.problem()[0]), 20
    prob, _, _ = sc.problem()
    hs = HostSim(sc.model)
    if which == "tree":  # a tolerance that about half the (instance, goal) pairs reach
        tol = float(np.median([hs.converge(prob, sc.q32, goals[:, g], mask, 0.0, n)[1] for g in range(4)]))
    per_goal = [hs.converge(prob, sc.q32, goals[:, g], mask, tol, n) for g in range(goals.shape[1])]
    solved = np.stack([r[1] <= tol for r in per_goal], axis=1)
    first = np.min(np.where(solved, np.stack([r[2] for r in per_goal], axis=1), n + 1), axis=1)
    hg = HostGoalset(sc.model)
    _, err, goal, seed, steps, _ = hg.converge_goalset(prob, sc.q32[:, None], goals, mask, tol, n)
    some = solved.any(axis=1)
    assert some.any() and (seed == 0).all()
    assert (err[some] <= tol).all() and (steps[some] <= first[some]).all()
    # the group stops at the first round one of its goals converges: converge's step count there
    np.testing.assert_array_equal(steps[some], first[some])
    assert solved[some, goal[some]].all()


# ---- edge cases ------------------------------------------------------------------------------

@pytest.mark.parametrize("path", [0, 1, 2])
def test_zero_steps_picks_argmin_and_duplicate_goals_the_lowest(path):
    sc = helpers.ur5_scenario(16, "reachable") if path != 2 else helpers.humanoid_scenario("g1_description", 4,
                                                                                          with_com=True)
    prob, targets, _ = sc.problem()
    mask = pose_mask(prob)
    G, S = 4, 2
    qs = seeds_for(sc, S)
    goals = rolled_goals(targets, G)
    goals[:, 3] = goals[:, 1]  # goals 1 and 3 tie on every seed
    hs, hg = HostSim(sc.model), HostGoalset(sc.model)
    q_out, err, goal, seed, steps, st = hg.converge_goalset(prob, qs, goals, mask, 1e-9, 0, path=path)
    B = qs.shape[0]
    e = task_error(hs, sc.table, prob, mask, np.repeat(qs[:, None], G, axis=1).reshape(-1, sc.table.nq),
                   np.repeat(goals, S, axis=1).reshape(B * G * S, -1)).reshape(B, G * S)
    np.testing.assert_array_equal(goal * S + seed, np.argmin(e, axis=1))
    assert (goal != 3).all() and (steps == 0).all() and (st == 0).all()
    np.testing.assert_array_equal(q_out, qs[np.arange(B), seed])


@pytest.mark.parametrize("path", [0, 1, 2])
def test_nan_goal_never_wins(path):
    sc = helpers.ur5_scenario(8, "reachable") if path != 2 else helpers.humanoid_scenario("g1_description", 4,
                                                                                         with_com=True)
    prob, targets, _ = sc.problem()
    mask = pose_mask(prob)
    G, S = 4, 2
    qs = seeds_for(sc, S)
    goals = rolled_goals(targets, G)
    goals[0, 0] = np.nan  # the preferred goal of instance 0 is NaN
    goals[1, :] = np.nan  # every goal of instance 1
    hg = HostGoalset(sc.model)
    q_out, err, goal, seed, steps, st = hg.converge_goalset(prob, qs, goals, mask, 1e-3, 10, path=path)
    assert goal[0] != 0 and np.isfinite(err[0])
    assert goal[1] == 0 and seed[1] == 0 and np.isnan(err[1]) and steps[1] == 1 and st[1] & FAILED
    check(sc, mask, 1e-3, 10, G, S, path=path, qs=qs, goals=goals)


# ---- argument checks -------------------------------------------------------------------------

def test_argument_errors():
    sc = helpers.ur5_scenario(4, "reachable")
    prob, targets, _ = sc.problem()
    hg = HostGoalset(sc.model)
    qs = seeds_for(sc, 4)
    goals = rolled_goals(targets, 2)
    for args in ((0, 1e-3, 5), (0b100, 1e-3, 5), (0b01, -1.0, 5), (0b01, float("nan"), 5), (0b01, 1e-3, -1)):
        with pytest.raises(RuntimeError):
            hg.converge_goalset(prob, qs, goals, *args)
    for G in (3, 6):
        with pytest.raises(RuntimeError, match="num_goals must be 1, 2, 4, 8, 16 or 32"):
            hg.converge_goalset(prob, qs, rolled_goals(targets, G), 0b01, 1e-3, 5)
    with pytest.raises(RuntimeError, match="num_seeds must be"):
        hg.converge_goalset(prob, np.repeat(sc.q32[:, None], 3, axis=1), goals, 0b01, 1e-3, 5)
    with pytest.raises(RuntimeError, match=r"num_goals \* num_seeds must be 1, 2, 4, 8, 16 or 32"):
        hg.converge_goalset(prob, np.repeat(sc.q32[:, None], 8, axis=1), rolled_goals(targets, 8), 0b01, 1e-3,
                            5)
    hg.converge_goalset(prob, np.repeat(sc.q32[:, None], 4, axis=1), rolled_goals(targets, 8), 0b01, 1e-3, 5)
    # the tree kernel: at most 8 members, one warp each in one CTA
    sc = helpers.humanoid_scenario("g1_description", 2, with_com=True)
    prob, targets, _ = sc.problem()
    hg = HostGoalset(sc.model)
    mask = pose_mask(prob)
    with pytest.raises(RuntimeError, match=r"num_goals \* num_seeds must be at most 8 on the tree kernel"):
        hg.converge_goalset(prob, np.repeat(sc.q32[:, None], 4, axis=1), rolled_goals(targets, 4), mask, 1e-3,
                            5)
    hg.converge_goalset(prob, np.repeat(sc.q32[:, None], 2, axis=1), rolled_goals(targets, 4), mask, 1e-3, 5)


# ---- the gradient glue -----------------------------------------------------------------------

class _UnitVjp:
    """A solver whose converge_vjp maps grad_q to a row of ones times its sum."""

    def converge_vjp(self, q_star, targets, grad_q):
        return grad_q.sum(dim=1, keepdim=True).expand(-1, targets.shape[1]).clone(), None


def test_gradient_reaches_the_winning_goal_row_only():
    B, G, T, nq = 5, 4, 3, 2
    goals = torch.randn(B, G, T, requires_grad=True)
    goal = torch.tensor([0, 3, 1, 2, 3], dtype=torch.int32)
    ok = torch.tensor([True, True, False, True, True])
    q = _solution_of_goals(goals, goal, _UnitVjp(), torch.zeros(B, nq), ok)
    (2.0 * q).sum().backward()
    expect = torch.zeros(B, G, T)
    for b in range(B):
        if ok[b]:
            expect[b, goal[b]] = 2.0 * nq
    assert torch.equal(goals.grad, expect)

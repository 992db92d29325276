"""Multi-start solve to a tolerance (``pk_converge_multistart_prepared``) on the CPU build of the
kernel bodies, on every path (chain, tree, general):

* with one seed, the multi-start loop equals the converge loop (``hs_converge``) bitwise;
* with several, it equals the group rule written in Python with separate host ``solve_ik``,
  ``integrate`` and ``task_terms`` calls on the tiled ``[B*S, nq]`` batch:

      for s = 0, 1, ...: err of every seed that has not failed (a failed seed keeps its error);
          the group stops if some err <= tol, s == max_steps or every seed has failed;
          every seed that has not failed solves step s; a failing seed keeps q_s;
      winner = the smallest error at the stopping round (NaN as +inf, ties to the lowest index);

plus the edge cases of the rule, ``sample_seeds`` and the argument checks."""

import numpy as np
import pytest
import torch

from pink_b200 import _cabi
from pink_b200.batched import sample_seeds
from tests import extras, helpers
from tests.hostsim.multistart import MultistartSim
from tests.test_hostsim_converge import FAILED, task_error


def python_group_loop(hs, table, prob, qs, targets, mask, tol, max_steps, dt, safety_break, path):
    """(q [B, S, nq], err [B, S], steps [B], status [B, S]) of every seed at the stopping round of
    its group, by the group rule with separate host calls."""
    B, S, nq = qs.shape
    q = qs.reshape(B * S, nq).astype(np.float32).copy()
    t = None if targets is None else np.repeat(targets, S, axis=0)
    failed = np.zeros(B * S, dtype=bool)
    e_keep = np.zeros(B * S, dtype=np.float32)
    st_all = np.zeros(B * S, dtype=np.int32)
    done = np.zeros(B, dtype=bool)
    steps = np.zeros(B, dtype=np.int32)
    e_stop = np.zeros((B, S), dtype=np.float32)
    for s in range(max_steps + 1):
        e = np.where(failed, e_keep, task_error(hs, table, prob, mask, q, t))
        E, F = e.reshape(B, S), failed.reshape(B, S)
        stop = ~done & ((E <= tol).any(axis=1) | (s == max_steps) | F.all(axis=1))
        e_stop[stop], steps[stop] = E[stop], s
        done |= stop
        if done.all():
            break
        v, st = hs.solve_ik(prob, q, t, path=path)
        live = ~failed & ~np.repeat(done, S)
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
    return q.reshape(B, S, nq), e_stop, steps, st_all.reshape(B, S)


def winner(e_stop):
    """The first seed of the smallest error (NaN as +inf) per target."""
    return np.argmin(np.where(np.isnan(e_stop), np.inf, e_stop), axis=1).astype(np.int32)


def seeds_for(sc, S, seed=0):
    g = torch.Generator().manual_seed(seed)
    return sample_seeds(sc.model, torch.as_tensor(sc.q32), S, g).numpy()


def check(sc, mask, tol, max_steps, S, path=0, expect=None, qs=None):
    prob, targets, _ = sc.problem()
    qs = seeds_for(sc, S) if qs is None else qs
    hs = MultistartSim(sc.model)
    q_out, err, seed, steps, st = hs.converge_multistart(prob, qs, targets, mask, tol, max_steps, path=path)
    if expect is not None:
        assert hs.selection.path == expect, hs.selection
    q_all, e_all, steps_l, st_all = python_group_loop(hs, sc.table, prob, qs, targets, mask, tol, max_steps, sc.dt,
                                                      sc.safety_break, path)
    np.testing.assert_array_equal(steps, steps_l)
    # the kernel's error comes from its own forward kinematics: where two seeds' errors agree to
    # that rounding, either may win
    B = qs.shape[0]
    seed_l = winner(e_all)
    other = seed != seed_l
    np.testing.assert_allclose(e_all[np.arange(B), seed][other], e_all[np.arange(B), seed_l][other], rtol=1e-6,
                               atol=5e-7)
    q_l, err_l, st_l = q_all[np.arange(B), seed], e_all[np.arange(B), seed], st_all[np.arange(B), seed]
    np.testing.assert_array_equal(st, st_l)
    np.testing.assert_array_equal(q_out.view(np.int32), q_l.view(np.int32))
    fin = np.isfinite(err_l)
    assert (np.isfinite(err) == fin).all()
    np.testing.assert_allclose(err[fin], err_l[fin], rtol=1e-6, atol=5e-7)
    return q_out, err, seed, steps, st


def pose_mask(prob):
    mask = 0
    for t in range(int(prob.ntasks)):
        if int(prob.tasks[t].type) in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_COM):
            mask |= 1 << t
    return mask


# ---- one seed is converge --------------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_one_seed_equals_converge(which):
    if which == "tree":
        sc = helpers.humanoid_scenario("g1_description", 12, with_com=True)
    else:
        sc = helpers.ur5_scenario(40, "reachable", out_of_limits=3)
    prob, targets, _ = sc.problem()
    mask = pose_mask(prob)
    path = 1 if which == "general" else 0
    hs = MultistartSim(sc.model)
    ref = hs.converge(prob, sc.q32, targets, mask, 1e-3, 25, path=path)
    q_out, err, seed, steps, st = hs.converge_multistart(prob, sc.q32[:, None, :], targets, mask, 1e-3, 25, path=path)
    assert hs.selection.path == which
    assert (seed == 0).all()
    for x, y in zip((q_out, err, steps, st), ref):
        np.testing.assert_array_equal(x.view(np.int32), y.view(np.int32))


# ---- the group rule on every path ----------------------------------------------------------

@pytest.mark.parametrize("S", [2, 8])
def test_chain_ur5(S):
    sc = helpers.ur5_scenario(24, "reachable", out_of_limits=2)
    _, err, seed, steps, _ = check(sc, 0b01, 1e-4, 40, S, expect="chain")
    assert (err <= 1e-4).sum() > 12
    # no seed reaches an unreachable target: the group runs to max_steps, the best seed wins
    sc = helpers.ur5_scenario(16, "unreachable")
    _, err, seed, steps, _ = check(sc, 0b01, 1e-4, 8, S, expect="chain")
    assert (seed > 0).any() and (steps == 8).any()


@pytest.mark.parametrize("nj,kw", [(3, {"prismatic": (1,)}), (4, {"two_tasks": True}), (6, {})])
def test_chain_instantiations(nj, kw):
    sc = helpers.chain_scenario(nj, 12, seed=nj, **kw)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 1e-3, 20, 4, expect="chain")


def test_tree_g1_com():
    sc = helpers.humanoid_scenario("g1_description", 6, with_com=True)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 2e-3, 12, 4, expect="tree")


@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_general_path_forced(name):
    if name == "ur5":
        sc = helpers.ur5_scenario(16, "reachable", out_of_limits=1)
    else:
        sc = helpers.humanoid_scenario("g1_description", 4, with_com=True)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 1e-3, 12, 4, path=1, expect="general")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 4, True, seed=7)
    prob, _, _ = sc.problem()
    check(sc, pose_mask(prob), 1e-3, 6, 2, expect="general")


# ---- edge cases ----------------------------------------------------------------------------

@pytest.mark.parametrize("path", [0, 1])
def test_zero_steps_picks_argmin_and_duplicates_the_lowest(path):
    sc = helpers.ur5_scenario(16, "reachable")
    prob, targets, _ = sc.problem()
    qs = seeds_for(sc, 4)
    qs[:, 3] = qs[:, 1]  # seeds 1 and 3 tie
    hs = MultistartSim(sc.model)
    q_out, err, seed, steps, st = hs.converge_multistart(prob, qs, targets, 0b01, 1e-6, 0, path=path)
    e = task_error(hs, sc.table, prob, 0b01, qs.reshape(-1, sc.table.nq), np.repeat(targets, 4, axis=0)).reshape(16, 4)
    np.testing.assert_array_equal(seed, np.argmin(e, axis=1))
    assert (seed != 3).all() and (steps == 0).all() and (st == 0).all()
    np.testing.assert_array_equal(q_out, qs[np.arange(16), seed])


@pytest.mark.parametrize("path", [0, 1, 2])
def test_nan_seed_never_wins(path):
    sc = helpers.ur5_scenario(8, "reachable") if path != 2 else helpers.humanoid_scenario("g1_description", 4,
                                                                                          with_com=True)
    prob, targets, _ = sc.problem()
    mask = pose_mask(prob)
    qs = seeds_for(sc, 4)
    qs[0, 2] = np.nan  # one NaN seed in group 0
    qs[1, :] = np.nan  # group 1 all NaN
    hs = MultistartSim(sc.model)
    q_out, err, seed, steps, st = hs.converge_multistart(prob, qs, targets, mask, 1e-3, 10, path=path)
    assert seed[0] != 2 and np.isfinite(err[0])
    assert seed[1] == 0 and np.isnan(err[1]) and steps[1] == 1 and st[1] & FAILED
    assert np.isnan(q_out[1]).all()
    check(sc, mask, 1e-3, 10, 4, path=path, qs=qs)


def test_out_of_limits_seed_fails_while_its_group_goes_on():
    sc = helpers.ur5_scenario(8, "reachable")
    assert sc.safety_break
    prob, targets, _ = sc.problem()
    qs = seeds_for(sc, 2)
    qs[:, 1, 0] = 10.0  # outside the limits of joint 0
    hs = MultistartSim(sc.model)
    _, err, seed, steps, st = check(sc, 0b01, 1e-4, 20, 2, qs=qs)
    assert (seed == 0).all() and (steps > 1).any()
    assert ((st & _cabi.PK_STATUS_OUT_OF_LIMITS) == 0).all()


def test_superset_of_converge_from_seed_zero():
    sc = helpers.ur5_scenario(32, "reachable", out_of_limits=2)
    prob, targets, _ = sc.problem()
    hs = MultistartSim(sc.model)
    _, err1, steps1, _ = hs.converge(prob, sc.q32, targets, 0b01, 1e-4, 40)
    _, err, seed, steps, _ = hs.converge_multistart(prob, seeds_for(sc, 8), targets, 0b01, 1e-4, 40)
    solved = err1 <= 1e-4
    assert solved.any()
    assert (err[solved] <= 1e-4).all() and (steps[solved] <= steps1[solved]).all()


# ---- sample_seeds --------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_sample_seeds(name):
    if name == "ur5":
        sc = helpers.ur5_scenario(64, "reachable")
    else:
        sc = helpers.humanoid_scenario("g1_description", 64, with_com=True)
    model = sc.model
    q = torch.as_tensor(sc.q32)
    qs = sample_seeds(model, q, 8, torch.Generator().manual_seed(3))
    assert qs.shape == (64, 8, model.nq) and qs.dtype == torch.float32 and qs.is_contiguous()
    assert torch.equal(qs[:, 0], q)
    lo = torch.as_tensor(np.array(model.lowerPositionLimit), dtype=torch.float32)
    hi = torch.as_tensor(np.array(model.upperPositionLimit), dtype=torch.float32)
    bounded = torch.isfinite(lo) & torch.isfinite(hi)
    rest = qs[:, 1:]
    assert ((rest > lo) & (rest < hi))[..., bounded].all()
    assert not torch.equal(rest[..., bounded], q[:, None].expand_as(rest)[..., bounded])
    # everything without both limits is copied (the free flyer), or on the circle if revolute
    for j in model.joints:
        if j.kind == "free_flyer":
            assert torch.equal(rest[..., j.idx_q:j.idx_q + 7], q[:, None, j.idx_q:j.idx_q + 7].expand(64, 7, 7))
    again = sample_seeds(model, q, 8, torch.Generator().manual_seed(3))
    assert torch.equal(qs, again)


def test_sample_seeds_continuous_and_unbounded_prismatic():
    from pink_b200.model import SE3, Model

    m = Model("toy")
    m.add_joint("a", 0, SE3(), [0, 0, 1], "revolute")  # continuous
    m.add_joint("b", 1, SE3(), [1, 0, 0], "prismatic")  # unbounded
    m.add_joint("c", 2, SE3(), [0, 1, 0], "revolute", lower=-0.5, upper=0.25)
    q = torch.tensor([[5.0, 7.0, 0.0]] * 32)
    qs = sample_seeds(m, q, 16, torch.Generator().manual_seed(1))
    rest = qs[:, 1:]
    assert (rest[..., 0].abs() <= np.pi).all() and rest[..., 0].std() > 1.0
    assert (rest[..., 1] == 7.0).all()
    assert ((rest[..., 2] > -0.5) & (rest[..., 2] < 0.25)).all()


# ---- argument checks -----------------------------------------------------------------------

def test_argument_errors():
    sc = helpers.ur5_scenario(4, "reachable")
    prob, targets, _ = sc.problem()
    hs = MultistartSim(sc.model)
    qs = seeds_for(sc, 4)
    for args in ((0, 1e-3, 5), (0b100, 1e-3, 5), (0b01, -1.0, 5), (0b01, float("nan"), 5), (0b01, 1e-3, -1)):
        with pytest.raises(RuntimeError):
            hs.converge_multistart(prob, qs, targets, *args)
    with pytest.raises(RuntimeError):
        hs.converge_multistart(prob, qs, None, 0b01, 1e-3, 5)
    for S in (3, 6, 64):
        with pytest.raises(RuntimeError, match="num_seeds"):
            hs.converge_multistart(prob, np.repeat(sc.q32[:, None], S, axis=1), targets, 0b01, 1e-3, 5)
    # the tree kernel: at most 8 seeds, one warp each in one CTA
    sc = helpers.humanoid_scenario("g1_description", 2, with_com=True)
    prob, targets, _ = sc.problem()
    with pytest.raises(RuntimeError, match="at most 8"):
        hs = MultistartSim(sc.model)
        hs.converge_multistart(prob, np.repeat(sc.q32[:, None], 16, axis=1), targets, pose_mask(prob), 1e-3, 5)

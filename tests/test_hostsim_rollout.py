"""Trajectory rollouts (``pk_rollout_trajectory_prepared``) on the CPU build of the kernel
bodies: the rollout loop of every path (chain kernel, its sub-warp variant, tree kernel, general
path) against the same closed loop made of separate host ``solve_ik`` and ``integrate`` calls
with the freeze emulated:

    an instance whose statuses so far have NO_SOLUTION / NOT_POSDEF (or OUT_OF_LIMITS with
    safety_break) keeps its q, gets v = 0 and keeps its status; on the tree kernel the step
    that fails does not move q either.

The records must be bitwise equal to the loop's."""

import numpy as np
import pytest

from pink_b200 import _cabi
from tests import extras, helpers
from tests.hostsim import HostSim

FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF


def _frozen(st, safety_break):
    bad = (st & FAILED) != 0
    if safety_break:
        bad |= (st & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
    return bad


def moving_targets(sc, base, steps, amp=0.05, seed=0):
    """[steps, B, target_stride]: the rows of ``base`` plus ``amp sin(2 t + phase_i)`` (t = s dt)
    on the translation of every per-instance frame target and on every other per-instance task
    target word (the rows of tests/test_gpu_rollout_trajectory.py)."""
    prob, _, descs = sc.problem()
    B = base.shape[0]
    rng = np.random.default_rng(seed)
    phase = 2.0 * np.pi * rng.random(B)
    t = np.arange(steps) * sc.dt
    wave = (amp * np.sin(2.0 * t[:, None] + phase[None, :])).astype(np.float32)
    rows = np.repeat(base[None], steps, axis=0)
    for k, d in enumerate(descs):
        if hasattr(d["target"], "shape") and d["target"].ndim == 2:
            off, width = int(prob.tasks[k].target_offset), int(d["target"].shape[1])
            for c in ((off + 3, off + 7, off + 11) if width == 12 else range(off, off + width)):
                rows[:, :, c] += wave
    return rows


def loop(hs, prob, q0, targets, steps, dt, safety_break, path, tree):
    """(q_traj, v_traj, status_traj) of separate solve_ik + integrate calls, freeze emulated."""
    q = q0.copy()
    st_or = np.zeros(q0.shape[0], dtype=np.int32)
    qs, vs, ss = [], [], []
    for s in range(steps):
        t = targets[s] if targets is not None and targets.ndim == 3 else targets
        v, st = hs.solve_ik(prob, q, t, path=path)
        frozen = _frozen(st_or, safety_break)
        v[frozen] = 0.0
        st_or = np.where(frozen, st_or, st_or | st)
        hold = frozen | (tree & _frozen(st, safety_break))
        q = np.where(hold[:, None], q, hs.integrate(q, v, dt))
        qs.append(q)
        vs.append(v)
        ss.append(st_or.copy())
    return np.stack(qs), np.stack(vs), np.stack(ss)


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def check_consistency(res, safety_break):
    """q_traj[-1] = q, status_traj[-1] = status, v_traj[-1] = v where never frozen; status_traj
    is monotone."""
    q, v, st, q_traj, v_traj, st_traj = res
    np.testing.assert_array_equal(bits(q_traj[-1]), bits(q))
    np.testing.assert_array_equal(st_traj[-1], st)
    alive = ~_frozen(st, safety_break)
    np.testing.assert_array_equal(bits(v_traj[-1][alive]), bits(v[alive]))
    np.testing.assert_array_equal(st_traj[:-1] & st_traj[1:], st_traj[:-1])


def check(sc, steps=4, amp=0.05, path=0, expect=None, targets=None, q=None):
    """The rollout with moving targets against the loop, bitwise; returns the rollout's outputs."""
    prob, base, _ = sc.problem()
    q = sc.q32 if q is None else q
    if targets is None and base is not None:
        targets = moving_targets(sc, base, steps, amp)
    hs = HostSim(sc.model)
    res = hs.rollout(prob, q, targets, steps, path=path)
    if expect is not None:
        assert hs.selection.path == expect, hs.selection
    tree = hs.selection.path == "tree"
    q_l, v_l, s_l = loop(hs, prob, q, targets, steps, sc.dt, sc.safety_break, path, tree)
    for s in range(steps):
        np.testing.assert_array_equal(res[5][s], s_l[s], err_msg=f"status, step {s}")
        np.testing.assert_array_equal(bits(res[3][s]), bits(q_l[s]), err_msg=f"q, step {s}")
        np.testing.assert_array_equal(bits(res[4][s]), bits(v_l[s]), err_msg=f"v, step {s}")
    check_consistency(res, sc.safety_break)
    return res


# ---- chains ------------------------------------------------------------------------------

def _chain(nj, nft, B=48):
    kw = {0: {"frame_tasks": False, "posture_per_instance": True}, 1: {}, 2: {"two_tasks": True}}[nft]
    return helpers.chain_scenario(nj, B, seed=nj, prismatic=(1,) if nj % 2 else (), **kw)


@pytest.mark.parametrize("nft", [0, 1, 2])
@pytest.mark.parametrize("nj", [2, 3, 4, 5, 6, 7])
def test_chain_instantiations(nj, nft):
    sc = _chain(nj, nft)
    check(sc, steps=5, expect="chain")
    hs = HostSim(sc.model)
    prob, base, _ = sc.problem()
    hs.solve_ik(prob, sc.q32[:1], None if base is None else base[:1])
    assert (hs.selection.nj, hs.selection.nft, hs.selection.lanes) == (nj, nft, 0)


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_ur5_sub_warp_kernel(lanes):
    sc = helpers.ur5_scenario(40, "reachable", out_of_limits=3)
    res = check(sc, steps=6, amp=0.1, path=10 + lanes, expect="chain")
    assert ((res[2] & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0).sum() == 3


def test_ur5_moving_targets_change_the_rollout():
    sc = helpers.ur5_scenario(40, "reachable")
    prob, base, _ = sc.problem()
    rows = moving_targets(sc, base, 6, amp=0.1)
    res = check(sc, steps=6, targets=rows, expect="chain")
    fixed = HostSim(sc.model).rollout(prob, sc.q32, rows[0], 6)
    assert np.abs(fixed[0] - res[0]).max() > 1e-3


# ---- tree kernel and general path ----------------------------------------------------------

def test_tree_g1_com():
    sc = helpers.humanoid_scenario("g1_description", 12, with_com=True)
    check(sc, steps=4, amp=0.02, expect="tree")


def test_tree_g1_extras():
    check(extras.g1_extras(6), steps=3, amp=0.02, expect="tree")


@pytest.mark.parametrize("name", ["ur5", "g1", "g1_extras"])
def test_general_path_forced(name):
    if name == "ur5":
        sc = helpers.ur5_scenario(24, "reachable", out_of_limits=2)
    elif name == "g1":
        sc = helpers.humanoid_scenario("g1_description", 8, with_com=True)
    else:
        sc = extras.g1_extras(4)
    check(sc, steps=3, amp=0.02, path=1, expect="general")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 6, True, seed=7)
    check(sc, steps=3, amp=0.02, expect="general")
    hs = HostSim(sc.model)
    prob, base, _ = sc.problem()
    hs.solve_ik(prob, sc.q32[:1], base[:1])
    assert hs.selection.generic == (58, 64)


# ---- freeze ------------------------------------------------------------------------------

@pytest.mark.parametrize("path,expect", [(0, "chain"), (12, "chain"), (2, "tree"), (1, "general")])
def test_nan_target_freezes_one_instance(path, expect):
    sc = helpers.ur5_scenario(16, "reachable")
    prob, base, _ = sc.problem()
    K, j, s_bad = 6, 5, 2
    rows = moving_targets(sc, base, K)
    clean = check(sc, steps=K, targets=rows, path=path, expect=expect)
    poisoned = rows.copy()
    poisoned[s_bad, j, 3] = np.nan
    q, v, st, q_traj, v_traj, st_traj = check(sc, steps=K, targets=poisoned, path=path, expect=expect)
    assert not (st_traj[:s_bad, j] & FAILED).any() and (st_traj[s_bad:, j] & FAILED).all()
    assert (st_traj[s_bad:, j] == st_traj[s_bad, j]).all()
    assert (v_traj[s_bad + 1:, j] == 0).all()
    assert (bits(q_traj[s_bad + 1:, j]) == bits(q_traj[s_bad, j])).all()
    keep = np.arange(sc.B) != j
    for a, b in zip((q, v, st), clean[:3]):
        np.testing.assert_array_equal(bits(a[keep]), bits(b[keep]))
    for a, b in zip((q_traj, v_traj, st_traj), clean[3:]):
        np.testing.assert_array_equal(bits(a[:, keep]), bits(b[:, keep]))


@pytest.mark.parametrize("safety_break", [True, False])
@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_out_of_limits_start(which, safety_break):
    if which == "chain":
        sc, path = helpers.ur5_scenario(24, "reachable", out_of_limits=4), 0
    else:  # a floating base: q (+) 0 dt renormalises the quaternion, so a frozen q must not be integrated
        sc, path = helpers.humanoid_scenario("g1_description", 8, with_com=True), 0 if which == "tree" else 1
        j = sc.table.nq - 1
        sc.q32[:4, j] = sc.table.q_max[j] + 0.1
    sc.safety_break = safety_break
    q, v, st, q_traj, v_traj, st_traj = check(sc, steps=4, path=path, expect=which)
    oob = (st & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
    assert oob.sum() >= 4
    moved = (q_traj[-1] != sc.q32).any(axis=1)
    if safety_break:  # frozen from the first step on
        assert (v_traj[:, oob] == 0).all() and (bits(q_traj[:, oob]) == bits(q_traj[0, oob])).all()
    else:  # outside the limits is not a reason to stop; an empty box (no solution) still is
        going = oob & ((st & FAILED) == 0)
        assert going.sum() >= 1 and moved[going].all()


# ---- layouts -----------------------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_misaligned_step_stride_equals_contiguous(which):
    sc = helpers.ur5_scenario(24, "reachable") if which == "chain" else \
        helpers.humanoid_scenario("g1_description", 6, with_com=True)
    prob, base, _ = sc.problem()
    K = 4
    rows = moving_targets(sc, base, K)
    B, S = rows.shape[1], rows.shape[2]
    store = np.full((K, B * S + 1), np.nan, dtype=np.float32)
    view = store[:, 1:].reshape(K, B, S)  # step stride B S + 1 floats: every other step 4-byte aligned only
    view[...] = rows
    assert view.strides == ((B * S + 1) * 4, S * 4, 4) and np.shares_memory(view, store)
    hs = HostSim(sc.model)
    a = hs.rollout(prob, sc.q32, view, K)
    b = hs.rollout(prob, sc.q32, np.ascontiguousarray(view), K)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(bits(x), bits(y))


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_fixed_rows_without_records_equal_the_last_records(which):
    if which == "chain":
        sc, path = helpers.ur5_scenario(24, "reachable", out_of_limits=2), 0
    else:
        sc, path = helpers.humanoid_scenario("g1_description", 6, with_com=True), 0 if which == "tree" else 1
    prob, base, _ = sc.problem()
    hs = HostSim(sc.model)
    K = 4
    res = check(sc, steps=K, targets=base, path=path, expect=which)
    q, v, st, q_traj, v_traj, st_traj = hs.rollout(prob, sc.q32, base, K, record=False, path=path)
    assert q_traj is None and v_traj is None and st_traj is None
    for a, b in zip((q, v, st), res[:3]):
        np.testing.assert_array_equal(bits(a), bits(b))
    check_consistency((q, v, st) + res[3:], sc.safety_break)

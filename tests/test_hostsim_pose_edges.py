"""Pose errors, Jacobians and free-flyer steps at the rotation-angle edges of the fp32 SE(3) maps
(``tests/pose_edges.py``) on the CPU build of the kernel bodies: the task-terms body, every
path's converge error, every path's solve through v of an unconstrained QP, and the integrate
body; and the fp64 reference itself against mpmath.  ``tests/test_gpu_pose_edges.py`` runs the
same cases on the device."""

import numpy as np
import pytest

from tests import helpers
from tests import pose_edges as pe
from tests.hostsim import HostSim

LADDER = pe.Ladder()


# ---- the reference ---------------------------------------------------------------------------

def test_reference_against_mpmath():
    """The projected-rotation reference against a 40-digit evaluation of log6 / Jlog6 at ladder
    points on both sides of each switch, on the fp32-rounded exp6 of the case; and the other-log
    closed forms equal to the oracle's where both apply."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    idx = [i for i in range(LADDER.n) if LADDER.angle[i] in (1e-6, 0.0201, 2.001, pe.ACOS_M09 + 1e-3, 3.0,
                                                              np.pi - 1e-3, np.pi - 1e-5)][::7]
    R, p = pe._split64(pe._pose32(LADDER.R[idx], LADDER.p[idx]))
    e, Jl = pe.log6_jlog6(R, p)
    worst_e = worst_j = 0.0
    for n, i in enumerate(idx):
        e_mp, Jl_mp = _mp_log6_jlog6(mp, R[n], p[n])
        worst_e = max(worst_e, np.abs(e[n] - e_mp).max())
        worst_j = max(worst_j, np.abs(Jl[n] - Jl_mp).max() / np.abs(Jl_mp).max())
        assert np.abs(e[n] - e_mp).max() < 1e-10, (LADDER.angle[i], e[n], e_mp)
        assert np.abs(Jl[n] - Jl_mp).max() < 1e-10 * np.abs(Jl_mp).max(), LADDER.angle[i]
    print(f"[pose edges] reference against mpmath: {len(idx)} cases, |de| {worst_e:.2e}, |dJ|/max|J| {worst_j:.2e}")
    # the closed forms of the other log, fed the oracle's own log, are the oracle's maps
    Rp = pe.nearest_rotation(R)
    w, _ = pe.lie.log3(Rp)
    e2, Jl2 = pe.se3_terms_of_log(w, p)
    np.testing.assert_allclose(e2, e, rtol=0, atol=1e-11)
    np.testing.assert_allclose(Jl2, Jl, rtol=0, atol=1e-11)


def _mp_log6_jlog6(mp, R, p):
    """log6 and Jlog6 of (R, p) in mpmath: the nearest rotation, its angle from atan2(|vee|, cos)
    and axis from the largest column of R + R^T - (tr R - 1) I (well conditioned at every angle),
    then the closed forms of oracle/lie.py."""
    M = mp.matrix(R.tolist())
    U, S, V = mp.svd_r(M)
    Q = U * V
    if mp.det(Q) < 0:
        U[:, 2] = -U[:, 2]
        Q = U * V
    vee = [(Q[2, 1] - Q[1, 2]) / 2, (Q[0, 2] - Q[2, 0]) / 2, (Q[1, 0] - Q[0, 1]) / 2]
    s = mp.sqrt(sum(x * x for x in vee))
    c = (Q[0, 0] + Q[1, 1] + Q[2, 2] - 1) / 2
    th = mp.atan2(s, c)
    if th < mp.mpf("0.5"):
        k = th / s if s > 0 else mp.mpf(1)
        w = [k * x for x in vee]
    else:
        # (1 - cos) n n^T = (R + R^T)/2 - cos I
        S2 = [[(Q[i, j] + Q[j, i]) / 2 - (c if i == j else 0) for j in range(3)] for i in range(3)]
        col = max(range(3), key=lambda j: S2[j][j])
        n = [S2[i][col] for i in range(3)]
        nn = mp.sqrt(sum(x * x for x in n))
        n = [x / nn for x in n]
        if sum(n[i] * vee[i] for i in range(3)) < 0:
            n = [-x for x in n]
        w = [th * x for x in n]
    th2 = th * th
    if th == 0:
        alpha, a, adot = mp.mpf(1), mp.mpf(1) / 12, mp.mpf(1) / 360
    else:
        st, ct = mp.sin(th), mp.cos(th)
        alpha = th * st / (2 * (1 - ct))
        a = 1 / th2 - st / (2 * th * (1 - ct))
        adot = -2 / th2**2 + (1 + st / th) / (th2 * 2 * (1 - ct))
    pm = [mp.mpf(float(x)) for x in p]
    wp = sum(w[i] * pm[i] for i in range(3))
    cross = lambda u, v: [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
    wxp = cross(w, pm)
    v = [alpha * pm[i] - wxp[i] / 2 + a * wp * w[i] for i in range(3)]
    hat = lambda u: mp.matrix([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]])
    W = mp.matrix([[w[i] * w[j] for j in range(3)] for i in range(3)])
    A = a * W + (1 - th2 * a) * mp.eye(3) + hat(w) / 2
    v3 = [adot * wp * w[i] - (th2 * adot + 2 * a) * pm[i] for i in range(3)]
    C = (mp.matrix([[v3[i] * w[j] for j in range(3)] for i in range(3)])
         + a * mp.matrix([[w[i] * pm[j] for j in range(3)] for i in range(3)]) + a * wp * mp.eye(3) + hat(pm) / 2)
    Bm = C * A
    J = np.zeros((6, 6))
    for i in range(3):
        for j in range(3):
            J[i, j] = J[3 + i, 3 + j] = float(A[i, j])
            J[i, 3 + j] = float(Bm[i, j])
    return np.array([float(x) for x in v + w]), J


# ---- the kernel bodies -----------------------------------------------------------------------

@pytest.mark.parametrize("name", ["ur5", "g1-frame", "g1-relative"])
def test_task_terms(name):
    """The task-terms body (the general path's) against the reference e and J."""
    sc, k, case = pe.scenario(name, LADDER)
    prob, targets, _ = sc.problem()
    e, J = HostSim(sc.model).task_terms(prob, k, 6, sc.q32, targets)
    pe.check_terms(e, J, pe.reference(sc, k), case, LADDER, f"host task_terms {name}")


# (scenario, path of hs.converge / hs.solve_ik, selected path); path 1 = the general path
CONVERGE = [("ur5", 0, "chain"), ("chain7-two-frames", 0, "chain"), ("g1-frame", 0, "tree"),
            ("g1-relative", 0, "tree"), ("ur5", 1, "general"), ("g1-frame", 1, "general")]


@pytest.mark.parametrize("name,path,expect", CONVERGE)
def test_converge_error(name, path, expect):
    """Each path's own error: converge and one-seed multi-start with max_steps = 0 return |e|_2
    of the reference, q unchanged, steps 0."""
    sc, k, case = pe.scenario(name, LADDER)
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    ref = pe.reference(sc, k)
    q_out, err, steps, st = hs.converge(prob, sc.q32, targets, 1 << k, 0.0, 0, path=path)
    assert hs.selection.path == expect, hs.selection
    assert (steps == 0).all() and (st == 0).all()
    np.testing.assert_array_equal(q_out.view(np.int32), sc.q32.view(np.int32))
    pe.check_error_norm(err, ref, case, LADDER, f"host converge {name} {expect}")
    q_out, err, seed, steps, st = hs.converge_multistart(prob, sc.q32[:, None], targets, 1 << k, 0.0, 0, path=path)
    assert hs.selection.path == expect, hs.selection
    assert (steps == 0).all() and (st == 0).all() and (seed == 0).all()
    np.testing.assert_array_equal(q_out.view(np.int32), sc.q32.view(np.int32))
    pe.check_error_norm(err, ref, case, LADDER, f"host multistart {name} {expect}")


# (scenario, path of hs.solve_ik, selected path): 11 / 12 / 14 / 18 = PK_CHAIN_LANES 1 / 2 / 4 / 8
SOLVE = [("ur5", 0, "chain"), ("ur5", 11, "chain"), ("ur5", 12, "chain"), ("ur5", 14, "chain"),
         ("ur5", 18, "chain"), ("chain7-two-frames", 0, "chain"), ("g1-frame", 0, "tree"),
         ("g1-relative", 0, "tree"), ("ur5", 1, "general"), ("g1-frame", 1, "general"),
         ("g1-relative", 1, "general")]


@pytest.mark.parametrize("name,path,expect", SOLVE)
def test_solve_velocity(name, path, expect):
    """Each path's Jacobian through v: the minimiser of the unconstrained QP built from the
    reference e and J."""
    sc, k, case = pe.scenario(name, LADDER, for_velocity=True)
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    v, st = hs.solve_ik(prob, sc.q32, targets, path=path)
    assert hs.selection.path == expect, hs.selection
    assert (st == 0).all()
    pe.check_velocity(v, sc, k, pe.reference(sc, k), case, LADDER, f"host solve {name} path {path}")


def test_rollout_one_step_velocity():
    """The chain kernel's rollout body (one recorded step) through v."""
    sc, k, case = pe.scenario("ur5", LADDER, for_velocity=True)
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    _, v, st, _, v_traj, _ = hs.rollout(prob, sc.q32, targets, 1, record=True)
    assert hs.selection.path == "chain" and (st == 0).all()
    np.testing.assert_array_equal(v_traj[0], v)
    pe.check_velocity(v, sc, k, pe.reference(sc, k), case, LADDER, "host rollout ur5")


def test_integrate_free_flyer():
    """The integrate body on G1 at |w dt| either side of its switches, against exp6 in fp64."""
    _, model, table = helpers.load("g1_description")
    q, v, dt, angle = pe.integrate_cases(table)
    out = HostSim(model).integrate(q, v, dt)
    pe.check_integrate(out, table, q, v, dt, angle, "host integrate g1")

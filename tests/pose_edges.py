"""Pose errors, their Jacobians and free-flyer steps at the angles where the fp32 SE(3) maps of
``pink_b200/csrc/pk_math.cuh`` switch formulas: the ladder of cases and an fp64 reference that
stays accurate there.

``log3`` takes theta / sin(theta) from a series when sin < 2e-2, the rotation vector from a
Shepperd quaternion when cos <= -0.9 (theta >~ 2.69), and ``a`` / ``adot`` from a Bernoulli series
below theta = 2; ``integrate_configuration`` switches at |w dt| = 1e-2 and 1e-4.  Random targets
rarely land near these switches, and never within 1e-3 of pi.

The reference composes the relative transform in fp64 from the fp32 inputs (forward kinematics
of ``oracle.kinematics`` at the fp32 q, the fp32 target), replaces its rotation with the nearest
rotation (SVD, det +1) and then calls ``oracle.lie.log6`` / ``jlog6``.  ``oracle.lie.log3``
follows ``pin.log3``: within 1e-2 of pi it takes the axis from sqrt((R_kk - cos) / (1 - cos)),
which turns the 6e-8 rounding of an fp32 rotation into errors of order 1e-4; on the projected
rotation the same formula is within 1e-10 (``test_hostsim_pose_edges.py`` checks this against
mpmath).  At theta = pi both w and -w are logs of the rotation, so each case also carries the
reference of the other log (``*_alt``), which a check accepts where theta is within 1e-6 of pi.

TEST CODE ONLY."""

import math

import numpy as np
import torch

from oracle import kinematics as okin
from oracle import lie
from oracle import tasks as otasks
from pink_b200 import FrameTask

ACOS_M09 = math.acos(-0.9)  # cos(theta) = -0.9: the Shepperd switch of log3
ANGLES = [0.0, 1e-6, 1.01e-4, 1e-3, 0.0199, 0.0201, 1.999, 2.001, ACOS_M09 - 1e-3, ACOS_M09 + 1e-3, 3.0,
          math.pi - 1e-2, math.pi - 1e-3, math.pi - 1e-4, math.pi - 1e-5, math.pi]
N_RANDOM_AXES = 3
# x, y, z are the three Shepperd pivots; the diagonals tie them
FIXED_AXES = [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (1.0, 1.0, 1.0), (1.0, 1.0, 0.0)]
TRANSLATIONS = [0.0, 0.05, 1.0]  # m; the B block of Jlog6 scales with p
NEAR_PI = 1e-6  # within this of pi either sign of w is a valid log

# tolerances (fp32 kernel against the fp64 reference)
E_ATOL, E_RTOL = 4e-6, 1e-6  # |e - e_ref| <= E_ATOL + E_RTOL |e_ref|, per coordinate
J_RTOL = 1e-5  # |J - J_ref| <= J_RTOL max |J_ref|, per instance
P_RTOL = 5e-7  # integrate: |p - p_ref| <= P_RTOL |v_lin dt| + ulp(p), per coordinate
QUAT_ATOL = 2e-7  # integrate: quaternion up to sign


class Ladder:
    """``n`` relative poses (R, p) with the angle of each: every angle x axis x translation."""

    def __init__(self, seed=5):
        rng = np.random.default_rng(seed)
        axes = [np.asarray(a) / np.linalg.norm(a) for a in FIXED_AXES]
        axes += [a / np.linalg.norm(a) for a in rng.normal(size=(N_RANDOM_AXES, 3))]
        w, p, angle = [], [], []
        for th in ANGLES:
            for ax in axes:
                for t in TRANSLATIONS:
                    d = rng.normal(size=3)
                    w.append(th * ax)
                    p.append(t * d / np.linalg.norm(d))
                    angle.append(th)
        self.w, self.p, self.angle = np.array(w), np.array(p), np.array(angle)
        self.R = lie.exp3(self.w)
        self.n = len(angle)

    def tile(self, B):
        """Case index of each of B instances (the ladder repeated)."""
        return np.arange(B) % self.n


def nearest_rotation(R):
    U, _, Vt = np.linalg.svd(R)
    d = np.sign(np.linalg.det(U @ Vt))
    U = U.copy()
    U[..., :, 2] *= d[..., None]
    return U @ Vt


def log6_jlog6(R, p):
    """``oracle.lie.log6`` and ``jlog6`` of (R, p) with R replaced by its nearest rotation."""
    R = nearest_rotation(R)
    return lie.log6(R, p), lie.jlog6(R, p)


def _pose32(R, p):
    return np.concatenate([R, p[..., None]], axis=-1).astype(np.float32)


def _split64(T32):
    T = np.asarray(T32, dtype=np.float64)
    return T[..., :3], T[..., 3]


def se3_terms_of_log(w, p):
    """log6 and Jlog6 of (exp3(w), p) for the given rotation vector ``w`` (any of the logs of the
    rotation): the closed forms of ``oracle.lie.log6`` / ``jlog6`` with ``w`` in place of
    ``log3(R)``.  Gives the reference of the other log at theta = pi."""
    theta = np.linalg.norm(w, axis=-1)
    alpha, a = lie._alpha_beta(theta)
    wp = np.sum(w * p, axis=-1)
    e = np.concatenate([alpha[..., None] * p - 0.5 * np.cross(w, p) + (a * wp)[..., None] * w, w], axis=-1)
    t2 = theta * theta
    small = theta < 1e-4
    ts = np.where(small, 1.0, theta)
    adot = np.where(small, 1.0 / 360.0 + t2 / 7560.0,
                    -2.0 / ts**4 + (1.0 + np.sin(ts) / ts) / (ts * ts * 2.0 * (1.0 - np.cos(ts))))
    A = lie.jlog3(w, theta)
    v3 = (adot * wp)[..., None] * w - (t2 * adot + 2.0 * a)[..., None] * p
    C = (v3[..., :, None] * w[..., None, :] + a[..., None, None] * (w[..., :, None] * p[..., None, :])
         + (a * wp)[..., None, None] * np.eye(3) + 0.5 * lie.hat(p))
    J = np.zeros(A.shape[:-2] + (6, 6))
    J[..., :3, :3] = A
    J[..., :3, 3:] = C @ A
    J[..., 3:, 3:] = A
    return e, J


def other_log(w):
    """The other rotation vector of exp3(w) where theta is within NEAR_PI of pi: angle
    2 pi - theta about -axis (-w at theta = pi); w itself elsewhere."""
    th = np.linalg.norm(w, axis=-1, keepdims=True)
    return np.where(th > np.pi - NEAR_PI, w * (th - 2.0 * np.pi) / np.where(th > 0, th, 1.0), w)


class Reference:
    """fp64 e, J (and their other-log variants) of one pose task at fp32 q and fp32 targets."""

    def __init__(self, e, J, e_alt, J_alt, theta):
        self.e, self.J, self.e_alt, self.J_alt, self.theta = e, J, e_alt, J_alt, theta
        self.two_logs = theta > np.pi - NEAR_PI


def frame_reference(table, q32, frame, T32):
    """e = log6(T_f^-1 T_t), J = -Jlog6(T_t^-1 T_f) J_f (oracle/tasks.py), with the projected rotation."""
    q = np.asarray(q32, dtype=np.float32).astype(np.float64)
    fk = okin.forward_kinematics(table, q)
    Rf, pf = okin.frame_placement(table, fk, frame)
    Rt, pt = _split64(T32)
    Rbt, pbt = lie.se3_act_inv(Rf, pf, Rt, pt)
    Rbt = nearest_rotation(Rbt)
    Rtb, ptb = lie.se3_inv(Rbt, pbt)
    Jf = okin.frame_jacobian_local(table, fk, frame)
    e = lie.log6(Rbt, pbt)
    J = -lie.jlog6(Rtb, ptb) @ Jf
    w_alt = other_log(e[:, 3:])
    e_alt, _ = se3_terms_of_log(w_alt, pbt)
    _, Jl_alt = se3_terms_of_log(-w_alt, ptb)
    return Reference(e, J, e_alt, -Jl_alt @ Jf, np.linalg.norm(e[:, 3:], axis=1))


def relative_reference(table, q32, frame, root, T32):
    """e = log6(T_t^-1 T_rf), J = Jlog6(T_t^-1 T_rf) (J_f - Ad_{T_rf^-1} J_r) (oracle/tasks.py),
    with the projected rotation."""
    q = np.asarray(q32, dtype=np.float32).astype(np.float64)
    fk = okin.forward_kinematics(table, q)
    Rf, pf = okin.frame_placement(table, fk, frame)
    Rr, pr = okin.frame_placement(table, fk, root)
    Rrf, prf = lie.se3_act_inv(Rr, pr, Rf, pf)
    Rt, pt = _split64(T32)
    Rtf, ptf = lie.se3_act_inv(Rt, pt, Rrf, prf)
    Rtf = nearest_rotation(Rtf)
    Jd = okin.frame_jacobian_local(table, fk, frame) - lie.action_inverse(Rrf, prf) @ okin.frame_jacobian_local(
        table, fk, root)
    e = lie.log6(Rtf, ptf)
    J = lie.jlog6(Rtf, ptf) @ Jd
    e_alt, Jl_alt = se3_terms_of_log(other_log(e[:, 3:]), ptf)
    return Reference(e, J, e_alt, Jl_alt @ Jd, np.linalg.norm(e[:, 3:], axis=1))


# ---- targets on a scenario -------------------------------------------------------------------

def place_ladder(sc, k, ladder):
    """Replace task ``k`` of the scenario (a frame or relative-frame task) by one whose target
    puts instance i at ladder case i mod n: ``T_f^-1 T_t = (R, p)`` for a frame task,
    ``T_t^-1 T_rf = (R, p)`` for a relative-frame task.  A frame task gets costs of one on every
    axis (so that v shows its whole Jacobian).  Returns the case index of every instance."""
    table = sc.table
    ot = dict(sc.oracle_tasks[k])
    case = ladder.tile(sc.B)
    fk = okin.forward_kinematics(table, sc.q64)
    Rf, pf = okin.frame_placement(table, fk, ot["frame"])
    Rc, pc = ladder.R[case], ladder.p[case]
    if ot["type"] == "frame":
        T = _pose32(*lie.se3_mul(Rf, pf, Rc, pc))
        task = FrameTask(table.frame_names[ot["frame"]], position_cost=1.0, orientation_cost=1.0,
                         lm_damping=ot["lm_damping"], gain=ot["gain"])
        ot["cost"] = np.ones(6)
    else:
        Rr, pr = okin.frame_placement(table, fk, ot["root"])
        Rrf, prf = lie.se3_act_inv(Rr, pr, Rf, pf)
        T = _pose32(*lie.se3_mul(Rrf, prf, *lie.se3_inv(Rc, pc)))
        task = sc.tasks[k]
    task.set_target(torch.as_tensor(T))
    sc.tasks[k] = task
    ot["target"] = _split64(T)
    sc.oracle_tasks[k] = ot
    sc.limits, sc.oracle_limits = [], []  # an unconstrained QP: a bound would hide J where e / dt is large
    return case


VELOCITY_DT = 0.1
POSTURE_COST = 0.3  # of the velocity scenarios: cond(H) stays below 1e4 at every case


def scenario(name, ladder, for_velocity=False):
    """(scenario, index of the task on the ladder, case of each instance), one instance per case:
    ``ur5`` (the benchmark arm's frame task), ``chain7-two-frames`` (the tool task of a random
    7-joint chain with a second frame task), ``g1-frame`` (the right wrist of G1) and
    ``g1-relative`` (G1's wrist-to-wrist relative-frame task).

    ``for_velocity`` keeps the QP in the range where fp32 solves meet ``helpers.within_tolerance``
    (cond(H) < 1e5, helpers.PARITY_BINS, and velocities of tens of rad/s): the time step is
    VELOCITY_DT, the posture task gets cost POSTURE_COST (at a zero error the benchmark arm's
    posture cost of 1e-3 alone would bound the smallest eigenvalue), and on G1 the other frame
    tasks (foot costs of 200 next to a posture cost of 0.1 put cond(H) at 1e6..1e7) are left out
    but for the pelvis task, which holds the floating base."""
    from pink_b200 import PostureTask
    from tests import helpers

    if name == "ur5":
        sc, k = helpers.ur5_scenario(ladder.n), 0
    elif name == "chain7-two-frames":
        sc, k = helpers.chain_scenario(7, ladder.n, seed=7, two_tasks=True), 0
    else:
        sc = helpers.humanoid_scenario("g1_description", ladder.n, with_relative=True)
        k = 3 if name == "g1-frame" else len(sc.tasks) - 1  # right_wrist_yaw_link / the relative task
    if for_velocity:
        # dt = 0.1 keeps |v| = |e| / dt near pi at ~30 rad/s: the fp32 solve's absolute error scales
        # with max |v|, and the standard tolerance was stated for velocities of that order
        sc.dt = VELOCITY_DT
        # G1: the ladder task, the posture task and the pelvis task, which holds the floating base
        # (the posture task leaves it out, and a relative task does not move it)
        keep = [t for t, ot in enumerate(sc.oracle_tasks)
                if t in (0, k) or ot["type"] == "posture" or not name.startswith("g1")]
        k = keep.index(k)
        sc.tasks = [sc.tasks[t] for t in keep]
        sc.oracle_tasks = [dict(sc.oracle_tasks[t]) for t in keep]
        for t, ot in enumerate(sc.oracle_tasks):
            if ot["type"] == "posture":
                pt = PostureTask(cost=POSTURE_COST, gain=ot["gain"])
                pt.set_target(sc.tasks[t].target_q)
                sc.tasks[t] = pt
                ot["cost"] = POSTURE_COST
            elif name.startswith("g1") and t != k:  # pelvis: holds the base firmly
                ft = FrameTask("pelvis", position_cost=10.0, orientation_cost=10.0)
                ft.set_target(sc.tasks[t].transform_target_to_world)
                sc.tasks[t] = ft
                ot["cost"] = np.full(6, 10.0)
    return sc, k, place_ladder(sc, k, ladder)


def reference(sc, k, q32=None):
    """Reference of task k of the scenario at q32 (default: the scenario's q)."""
    ot = sc.oracle_tasks[k]
    q32 = sc.q32 if q32 is None else q32
    T32 = np.concatenate([ot["target"][0], ot["target"][1][..., None]], axis=-1)
    if ot["type"] == "frame":
        return frame_reference(sc.table, q32, ot["frame"], T32)
    return relative_reference(sc.table, q32, ot["frame"], ot["root"], T32)


# ---- checks ----------------------------------------------------------------------------------

def _e_err(e, e_ref):
    """Per-instance worst |e - e_ref| over its tolerance (<= 1 passes) and the worst |e - e_ref|."""
    d = np.abs(np.asarray(e, dtype=np.float64) - e_ref)
    return (d / (E_ATOL + E_RTOL * np.abs(e_ref))).max(axis=1), d.max(axis=1)


def _j_err(J, J_ref):
    scale = np.abs(J_ref).max(axis=(1, 2))
    d = np.abs(np.asarray(J, dtype=np.float64) - J_ref).max(axis=(1, 2))
    return d / (J_RTOL * scale), d / scale


def check_terms(e, J, ref, case, ladder, label):
    """e and J of one pose task against the reference (either log where theta is pi, the same
    for e and J).  Prints the worst errors per ladder angle; asserts every instance passes."""
    re, de = _e_err(e, ref.e)
    rj, dj = _j_err(J, ref.J)
    ra, dea = _e_err(e, ref.e_alt)
    rja, dja = _j_err(J, ref.J_alt)
    alt = ref.two_logs & (np.maximum(ra, rja) < np.maximum(re, rj))
    r = np.where(alt, np.maximum(ra, rja), np.maximum(re, rj))
    de, dj = np.where(alt, dea, de), np.where(alt, dja, dj)
    report(label, ladder, case, [("|de|", de), ("|dJ|/max|J|", dj)])
    bad = np.nonzero(r > 1.0)[0]
    assert bad.size == 0, (f"{label}: {bad.size} instances outside the tolerance; first {bad[:5].tolist()} "
                           f"at angles {ladder.angle[case[bad[:5]]].tolist()}, worst |de| {de.max():.3e}, "
                           f"worst |dJ|/max|J| {dj.max():.3e}")
    return alt


def check_error_norm(err, ref, case, ladder, label):
    """The converge kernels' error |e|_2 against |e_ref|_2 (either log where theta is pi)."""
    err = np.asarray(err, dtype=np.float64)
    n = np.linalg.norm(ref.e, axis=1)
    d = np.abs(err - n)
    d = np.where(ref.two_logs, np.minimum(d, np.abs(err - np.linalg.norm(ref.e_alt, axis=1))), d)
    report(label, ladder, case, [("|d err|", d)])
    bad = np.nonzero(d > E_ATOL + E_RTOL * n)[0]
    assert bad.size == 0, (f"{label}: {bad.size} errors outside the tolerance; first {bad[:5].tolist()} at angles "
                           f"{ladder.angle[case[bad[:5]]].tolist()}, worst {d.max():.3e}")


def reference_velocity(sc, k, ref, alt=None):
    """fp64 minimiser of the unconstrained QP (oracle/ik.py, oracle/tasks.py) with task k's e and J
    from ``ref`` (its other log where ``alt``) and every other task from the oracle: v = dq / dt."""
    table = sc.table
    fk = okin.forward_kinematics(table, sc.q64)
    nv = table.nv
    H = np.broadcast_to(sc.damping * np.eye(nv), (sc.B, nv, nv)).copy()
    c = np.zeros((sc.B, nv))
    for t, task in enumerate(sc.oracle_tasks):
        if t == k:
            e, J = ref.e, ref.J
            if alt is not None:
                e, J = np.where(alt[:, None], ref.e_alt, e), np.where(alt[:, None, None], ref.J_alt, J)
        else:
            e, J = otasks.task_error_jacobian(table, sc.q64, fk, task)
        w = otasks.task_weight(task, J.shape[-2])
        WJ = w[:, None] * J
        We = w * (-task.get("gain", 1.0) * e)
        mu = task.get("lm_damping", 0.0) * np.sum(We * We, axis=-1)
        H += np.swapaxes(WJ, -1, -2) @ WJ + mu[:, None, None] * np.eye(nv)
        c -= np.einsum("bk,bkn->bn", We, WJ)
    return np.linalg.solve(H, -c[..., None])[..., 0] / sc.dt, np.linalg.cond(H)


def check_velocity(v, sc, k, ref, case, ladder, label, atol=None, rtol=None):
    """v of a solve against the reference minimiser (the other log's where theta is pi and it fits
    better), within helpers.within_tolerance."""
    from tests import helpers

    atol = helpers.V_ATOL if atol is None else atol
    rtol = helpers.V_RTOL if rtol is None else rtol
    v = np.asarray(v, dtype=np.float64)
    v_ref, cond = reference_velocity(sc, k, ref)
    assert cond.max() < 1e5, f"{label}: cond(H) {cond.max():.3g} beyond the range of the standard tolerance"
    d = np.abs(v - v_ref) / (atol + rtol * np.abs(v_ref))
    if ref.two_logs.any():
        v_alt, _ = reference_velocity(sc, k, ref, alt=ref.two_logs)
        d_alt = np.abs(v - v_alt) / (atol + rtol * np.abs(v_alt))
        use = ref.two_logs & (d_alt.max(axis=1) < d.max(axis=1))
        v_ref, d = np.where(use[:, None], v_alt, v_ref), np.where(use[:, None], d_alt, d)
    dv = np.abs(v - v_ref).max(axis=1)
    report(label, ladder, case, [("|dv|", dv), ("|dv|/tol", d.max(axis=1)), ("cond(H)", cond)])
    bad = np.nonzero(d.max(axis=1) > 1.0)[0]
    assert bad.size == 0, (f"{label}: {bad.size} velocities outside the tolerance; first {bad[:5].tolist()} at "
                           f"angles {ladder.angle[case[bad[:5]]].tolist()}, worst |dv| {dv.max():.3e}")


def report(label, ladder, case, columns):
    """Prints the worst of each column per ladder angle."""
    angle = ladder.angle[case]
    head = " ".join(f"{name:>12}" for name, _ in columns)
    lines = [f"[pose edges] {label}", f"  {'theta':>20} {head}"]
    for th in ANGLES:
        m = angle == th
        if m.any():
            lines.append(f"  {th:20.15g} " + " ".join(f"{np.max(col[m]):12.3e}" for _, col in columns))
    lines.append(f"  {'all':>20} " + " ".join(f"{np.max(col):12.3e}" for _, col in columns))
    print("\n".join(lines))


# ---- free-flyer integrate --------------------------------------------------------------------

INTEGRATE_ANGLES = [0.0, 5e-5, 1.5e-4, 9.9e-3, 1.01e-2, 1.5e-2, 2.5e-2, 0.3, math.pi, 4.0, 2 * math.pi + 0.1]
INTEGRATE_DT = 5e-3


def integrate_cases(table, seed=9):
    """(q [B, nq], v [B, nv], dt, angle of each instance) on a free-flyer model: every |w dt| of
    INTEGRATE_ANGLES, base at the origin and at 100 m, translation steps of 1 m and 1 mm, input
    quaternions of norm 0.5, 1 and 2, half of them with w < 0."""
    from pink_b200 import workloads

    rng = np.random.default_rng(seed)
    rows = [(th, base, step, norm, neg) for th in INTEGRATE_ANGLES for base in (0.0, 100.0) for step in (1.0, 1e-3)
            for norm in (0.5, 1.0, 2.0) for neg in (False, True)]
    B = len(rows) * 2
    q = workloads.sample_configurations(table, B, rng)
    v = rng.normal(size=(B, table.nv)) * 0.5
    angle = np.zeros(B)
    for i in range(B):
        th, base, step, norm, neg = rows[i % len(rows)]
        u = rng.normal(size=3)
        q[i, 0:3] = base * u / np.linalg.norm(u) if base else 0.0
        quat = rng.normal(size=4)
        quat /= np.linalg.norm(quat)
        quat *= -1.0 if (quat[3] < 0) != neg else 1.0
        q[i, 3:7] = norm * quat
        a, d = rng.normal(size=3), rng.normal(size=3)
        v[i, 3:6] = th * a / np.linalg.norm(a) / INTEGRATE_DT
        v[i, 0:3] = step * d / np.linalg.norm(d) / INTEGRATE_DT
        angle[i] = th
    return q.astype(np.float32), v.astype(np.float32), INTEGRATE_DT, angle


def check_integrate(out, table, q32, v32, dt, angle, label):
    """q (+) v dt against ``oracle.kinematics.integrate`` (``oracle.lie.exp6``) in fp64 on the fp32
    inputs: the base translation within P_RTOL |v_lin dt| + ulp(p), the quaternion within QUAT_ATOL up to
    sign, the joints within an ulp of q + v dt."""
    out = np.asarray(out, dtype=np.float64)
    q, v = q32.astype(np.float64), v32.astype(np.float64)
    ref = okin.integrate(table, q, v * float(np.float32(dt)))
    # the translation step given, |v_lin dt|: near |w dt| = 2 pi the base moves far less than it
    # (V(w) has singular values down to |sin(theta / 2)| / (theta / 2)), while fp32 rounds its terms at its scale
    dp = np.linalg.norm(v[:, 0:3], axis=1) * float(np.float32(dt))
    ulp = np.spacing(np.abs(ref[:, 0:3]).astype(np.float32)).astype(np.float64)
    ep = np.abs(out[:, 0:3] - ref[:, 0:3])
    rp = (ep / (P_RTOL * dp[:, None] + ulp)).max(axis=1)
    sign = np.where(np.sum(out[:, 3:7] * ref[:, 3:7], axis=1) < 0, -1.0, 1.0)
    eq = np.abs(out[:, 3:7] - sign[:, None] * ref[:, 3:7]).max(axis=1)
    rel = np.maximum(ep - ulp, 0.0).max(axis=1) / np.maximum(dp, 1e-30)  # beyond an ulp of p, over the step
    lines = [f"[pose edges] {label}", f"  {'|w dt|':>20} {'|dp|/|step|':>12} {'|dp|/tol':>12} {'|dquat|':>12}"]
    for th in INTEGRATE_ANGLES:
        m = angle == th
        lines.append(f"  {th:20.15g} {rel[m].max():12.3e} {rp[m].max():12.3e} {eq[m].max():12.3e}")
    print("\n".join(lines))
    assert (rp <= 1.0).all(), (f"{label}: base translation off by {rel.max():.3e} of the step at |w dt| = "
                               f"{angle[np.argmax(rp)]:.6g} ({int((rp > 1).sum())} instances)")
    assert (eq <= QUAT_ATOL).all(), f"{label}: quaternion off by {eq.max():.3e} at |w dt| = {angle[np.argmax(eq)]:.6g}"
    np.testing.assert_allclose(out[:, 7:], ref[:, 7:], rtol=0, atol=2.5e-7 * max(1.0, np.abs(ref[:, 7:]).max()),
                               err_msg=label)

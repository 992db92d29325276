"""Scenarios with barriers, equality constraints, the opt-in limits and the
constant-Jacobian tasks, in product form (pink_b200 objects) and oracle form
(plain dicts), for the CPU (hostsim) and GPU parity tests."""

import numpy as np
import torch

from oracle import kinematics as okin
from pink_b200 import (ComTask, FrameTask, JointCouplingTask, LinearHolonomicTask, LowAccelerationTask, PostureTask,
                       SphereCollisionModel, workloads)
from pink_b200.barriers import BodySphericalBarrier, PositionBarrier, SelfCollisionBarrier
from pink_b200.limits import AccelerationLimit, ConfigurationLimit, FloatingBaseVelocityLimit, VelocityLimit
from tests import helpers


class ExtraScenario:
    def __init__(self, model, table, q, tasks, otasks, limits, olimits, barriers, obarriers, constraints, oconstraints,
                 dt, damping, collision_model=None, safety_break=False):
        self.model, self.table = model, table
        self.q32 = np.ascontiguousarray(q, dtype=np.float32)
        self.q64 = self.q32.astype(np.float64)
        self.tasks, self.otasks = tasks, otasks
        self.limits, self.olimits = limits, olimits
        self.barriers, self.obarriers = barriers, obarriers
        self.constraints, self.oconstraints = constraints, oconstraints
        self.dt, self.damping, self.collision_model, self.safety_break = dt, damping, collision_model, safety_break

    @property
    def B(self):
        return self.q32.shape[0]

    def problem(self):
        from pink_b200.solve_ik import describe_problem

        prob, parts, descs = describe_problem(self.model, self.B, self.tasks, self.dt, self.damping, self.limits,
                                              self.safety_break, self.barriers, self.constraints, self.collision_model)
        targets = torch.cat([p.cpu().float() for p in parts], dim=1).numpy() if parts else None
        return prob, targets, descs

    def oracle_solve(self, n=None):
        from oracle import ik as oik

        n = self.B if n is None else min(n, self.B)
        tasks = [oik._slice_task_range(t, 0, n) for t in self.otasks]
        cons = [oik._slice_task_range(t, 0, n) for t in self.oconstraints]
        return oik.solve_ik_batch(self.table, self.q64[:n], tasks, self.dt, self.damping, self.olimits,
                                  self.safety_break, self.obarriers, cons)

    def oracle_assemble(self, i):
        from oracle import ik as oik

        tasks = [oik._slice_task(t, i) for t in self.otasks]
        cons = [oik._slice_task(t, i) for t in self.oconstraints]
        return oik.assemble(self.table, self.q64[i], tasks, self.dt, self.damping, oik._slice_limits(self.olimits, i),
                            self.obarriers, cons)


def _frame_task(table, name, qt, pc, oc, **kw):
    T = helpers.frame_targets(table, qt, name)
    t = FrameTask(name, position_cost=pc, orientation_cost=oc, **kw)
    t.set_target(torch.as_tensor(T))
    T64 = T.astype(np.float64)
    o = {"type": "frame", "frame": table.frame_names.index(name), "cost": np.array(t.cost), "gain": kw.get("gain", 1.0),
         "lm_damping": kw.get("lm_damping", 0.0), "target": (T64[:, :, :3], T64[:, :, 3])}
    return t, o


def ur5_extras(B, seed=3, active=True):
    """UR5: frame + posture + low-acceleration tasks; default limits plus an
    AccelerationLimit with per-instance previous velocities; a position barrier
    that is active for most instances, a two-frame distance barrier, a sphere
    self-collision barrier; one joint-coupling equality constraint."""
    robot, model, _ = helpers.load("ur5_description")
    cm = SphereCollisionModel(model)
    for k, (joint, center, radius) in enumerate([
        ("shoulder_lift_joint", (0.0, 0.0, 0.2), 0.08), ("elbow_joint", (0.0, 0.0, 0.2), 0.07),
        ("wrist_1_joint", (0.0, 0.0, 0.0), 0.06), ("wrist_3_joint", (0.0, 0.05, 0.0), 0.05),
        ("shoulder_pan_joint", (0.0, 0.0, 0.0), 0.1),
    ]):
        cm.add_sphere(f"s{k}", model.getJointId(joint), center, radius)
    for pair in [(0, 2), (0, 3), (4, 2), (4, 3), (4, 1)]:  # non-adjacent links only
        cm.add_collision_pair(*pair)
    table = model.table()
    rng = np.random.default_rng(seed)
    q = workloads.sample_configurations(table, B, rng)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.3)
    ft, oft = _frame_task(table, "tool0", qt, 1.0, 1.0, lm_damping=1.0)
    q_ref = workloads.ur5_posture_reference(model)
    pt = PostureTask(cost=1e-3)
    pt.set_target(q_ref)
    opt = {"type": "posture", "cost": 1e-3, "gain": 1.0, "lm_damping": 0.0, "target": q_ref}
    v_prev = rng.normal(size=(B, 6)) * 0.3
    dt = workloads.UR5_DT
    lat = LowAccelerationTask(cost=0.05)
    lat.set_last_integration(torch.as_tensor(v_prev, dtype=torch.float32), dt)
    v_prev32 = v_prev.astype(np.float32).astype(np.float64)
    olat = {"type": "joint_velocity", "cost": 0.05, "gain": 1.0, "lm_damping": 0.0, "target": -(v_prev32 * dt)}
    # limits
    a_max = np.array([40.0, 40.0, 60.0, np.inf, 80.0, 80.0])
    acc = AccelerationLimit(model, a_max)
    acc.set_last_integration(torch.as_tensor(v_prev, dtype=torch.float32), dt)
    limits = [ConfigurationLimit(model), VelocityLimit(model), acc]
    dq_prev = (torch.as_tensor(v_prev, dtype=torch.float32) * dt).numpy().astype(np.float64)
    olimits = [("configuration", 0.5), ("velocity", None), ("acceleration", a_max, dq_prev)]
    # barriers: p_max just above the current tool position on x (active when the task pulls +x)
    fk = okin.forward_kinematics(table, q[0])
    f_tool = table.frame_names.index("tool0")
    p_max = np.array([0.5, 1.0]) if active else np.array([5.0, 5.0])
    pb = PositionBarrier("tool0", indices=[0, 2], p_min=np.array([-1.0, -0.6]), p_max=p_max, gain=np.array([0.5, 1.0]),
                         safe_displacement_gain=1.0)
    opb = {"type": "position", "frame": f_tool, "indices": [0, 2], "p_min": np.array([-1.0, -0.6]), "p_max": p_max,
           "gain": np.array([0.5, 1.0]), "safe_displacement_gain": 1.0}
    sb = BodySphericalBarrier(("tool0", "upper_arm_link"), d_min=0.15, gain=2.0, safe_displacement_gain=3.0)
    osb = {"type": "body_spherical", "frames": (f_tool, table.frame_names.index("upper_arm_link")), "d_min": 0.15,
           "gain": 2.0, "safe_displacement_gain": 3.0}
    cb = SelfCollisionBarrier(n_collision_pairs=3, gain=2.0, safe_displacement_gain=1.0, d_min=0.05)
    pf, pr = cm.pair_frames(), cm.pair_radii().astype(np.float64)
    ocb = {"type": "self_collision", "pairs": [(int(a), int(b), float(ra), float(rb)) for (a, b), (ra, rb) in zip(pf, pr)],
           "n_pairs": 3, "d_min": 0.05, "gain": 2.0, "safe_displacement_gain": 1.0}
    # equality constraint: wrist_1 + wrist_2 rates locked (a joint coupling on the current posture)
    A = np.zeros((1, 6))
    A[0, 3], A[0, 4] = 1.0, 1.0
    q0 = np.zeros(6)
    lc = LinearHolonomicTask(A, np.array([0.2]), q0, cost=[1.0], gain=0.002)
    olc = {"type": "linear", "A": A, "b": np.array([0.2]), "q0": q0, "cost": np.ones(1), "gain": 0.002, "lm_damping": 0.0}
    return ExtraScenario(model, table, q, [ft, pt, lat], [oft, opt, olat], limits, olimits, [pb, sb, cb], [opb, osb, ocb],
                         [lc], [olc], dt, workloads.UR5_DT and 1e-12, cm, safety_break=True)


def as_extra(sc):
    """A helpers.Scenario (tasks and limits only) in ExtraScenario form."""
    olimits = None if sc.oracle_limits is None else list(sc.oracle_limits)
    return ExtraScenario(sc.model, sc.table, sc.q32, list(sc.tasks), list(sc.oracle_tasks), list(sc.limits), olimits,
                         [], [], [], [], sc.dt, sc.damping, safety_break=sc.safety_break)


def with_shared_acceleration_limit(sc, a_max, seed=13):
    """Adds an AccelerationLimit fed ONE previous velocity ``[nv]`` shared by every instance,
    as the reference's unbatched usage does.  A shared non-zero previous displacement is not a
    per-instance box, so the chain and tree kernels decline the problem and the general path
    (ik_generic_kernel) solves it."""
    rng = np.random.default_rng(seed)
    nv = sc.table.nv
    v_prev = (rng.normal(size=nv) * 0.3).astype(np.float32)
    acc = AccelerationLimit(sc.model, a_max)
    acc.set_last_integration(v_prev, sc.dt)
    # the oracle takes dq_prev per instance: the shared row broadcast to [B, nv]
    dq_prev = (torch.as_tensor(v_prev) * sc.dt).numpy().astype(np.float64)[None].repeat(sc.B, axis=0)
    sc.limits = [lim for lim in sc.limits if not isinstance(lim, AccelerationLimit)] + [acc]
    olimits = [("configuration", 0.5), ("velocity", None)] if sc.olimits is None else \
        [lim for lim in sc.olimits if lim[0] != "acceleration"]
    sc.olimits = olimits + [("acceleration", np.asarray(a_max, dtype=np.float64), dq_prev)]
    return sc


def tree_rows_scenario(nj, B, free_flyer=False, frames=(), com=False, linear_rows=(), limits=True, seed=11):
    """Random tree (helpers.random_tree_model) with a task set of an exact task-row count K.

    ``frames`` lists ``(tip, position_cost, orientation_cost)`` on the tip frames (a zero cost
    component drops its row), ``com`` adds a CoM task (3 rows) and every entry of
    ``linear_rows`` a LinearHolonomicTask with that many rows (1..6) on random joint
    coordinates.  A posture task (no task rows) keeps H well conditioned; ``limits=False``
    leaves the box empty, so that every factorisation has all nv columns free."""
    rng = np.random.default_rng(seed)
    model = helpers.random_tree_model(nj, rng, free_flyer)
    table = model.table()
    q = workloads.sample_configurations(table, B, rng)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.15)
    tasks, otasks = [], []
    for tip, pc, oc in frames:
        t, o = _frame_task(table, f"tip{tip}", qt, pc, oc, lm_damping=0.02)
        tasks.append(t)
        otasks.append(o)
    if com:
        c = okin.center_of_mass(table, okin.forward_kinematics(table, qt)).astype(np.float32)
        ct = ComTask(cost=2.0)
        ct.set_target(torch.as_tensor(c))
        tasks.append(ct)
        otasks.append({"type": "com", "cost": np.full(3, 2.0), "gain": 1.0, "lm_damping": 0.0,
                       "target": c.astype(np.float64)})
    rv = 6 if free_flyer else 0
    for rows in linear_rows:
        A = np.zeros((rows, table.nv))
        for r in range(rows):
            cols = rv + rng.choice(table.nv - rv, size=3, replace=False)
            A[r, cols] = rng.uniform(-1.0, 1.0, size=3)
        b = rng.uniform(-0.05, 0.05, size=rows)
        tasks.append(LinearHolonomicTask(A, b, None, cost=[0.5] * rows, gain=0.5))
        otasks.append({"type": "linear", "A": A, "b": b, "q0": None, "cost": np.full(rows, 0.5), "gain": 0.5,
                       "lm_damping": 0.0})
    q_ref = q[0].copy()
    pt = PostureTask(cost=0.1)
    pt.set_target(q_ref)
    tasks.append(pt)
    otasks.append({"type": "posture", "cost": 0.1, "gain": 1.0, "lm_damping": 0.0, "target": q_ref})
    if limits:
        lims, olims = [ConfigurationLimit(model), VelocityLimit(model)], [("configuration", 0.5), ("velocity", None)]
    else:
        lims, olims = [], []
    return ExtraScenario(model, table, q, tasks, otasks, lims, olims, [], [], [], [], 1.0 / 100.0, 1e-6)


def g1_extras(B, seed=5, floating_base_limit=True):
    """G1-class humanoid (config 4 of BASELINE.json): CoM + feet + pelvis + wrist
    tasks, posture, a knee coupling task, default limits + floating-base velocity
    limit, sphere self-collision barrier (gain 20, safe displacement gain 1,
    d_min 0.05 as examples/barriers/kukas_self_collision.py:167-172)."""
    robot, model, _ = helpers.load("g1_description")
    cm = SphereCollisionModel(model)
    spheres = [("left_wrist_yaw_joint", 0.06), ("right_wrist_yaw_joint", 0.06), ("left_elbow_joint", 0.06),
               ("right_elbow_joint", 0.06), ("waist_yaw_joint", 0.13), ("left_knee_joint", 0.07),
               ("right_knee_joint", 0.07), ("left_ankle_roll_joint", 0.06), ("right_ankle_roll_joint", 0.06)]
    for k, (joint, radius) in enumerate(spheres):
        cm.add_sphere(f"s{k}", model.getJointId(joint), (0.0, 0.0, 0.0), radius)
    cm.add_all_collision_pairs()
    table = model.table()
    rng = np.random.default_rng(seed)
    q = workloads.sample_configurations(table, B, rng, near_limit_fraction=0.05)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.15)
    tasks, otasks = [], []
    for frame, pc, oc in [("pelvis", 0.0, 10.0), ("right_ankle_roll_link", [2.0, 2.0, 200.0], 10.0),
                          ("left_ankle_roll_link", [2.0, 2.0, 200.0], 10.0), ("right_wrist_yaw_link", 4.0, 0.0),
                          ("left_wrist_yaw_link", 4.0, 0.0)]:
        t, o = _frame_task(table, frame, qt, pc, oc)
        tasks.append(t)
        otasks.append(o)
    q_ref = q[0].copy()
    pt = PostureTask(cost=1e-1)
    pt.set_target(q_ref)
    tasks.append(pt)
    otasks.append({"type": "posture", "cost": 1e-1, "gain": 1.0, "lm_damping": 0.0, "target": q_ref})
    com = okin.center_of_mass(table, okin.forward_kinematics(table, qt)).astype(np.float32)
    ct = ComTask(cost=200.0)
    ct.set_target(torch.as_tensor(com))
    tasks.append(ct)
    otasks.append({"type": "com", "cost": np.full(3, 200.0), "gain": 1.0, "lm_damping": 0.0, "target": com.astype(np.float64)})

    class _Cfg:  # JointCouplingTask only needs configuration.model
        pass

    cfg = _Cfg()
    cfg.model = model
    jc = JointCouplingTask(["left_knee_joint", "left_hip_pitch_joint"], [1.0, 0.5], 100.0, cfg)
    tasks.append(jc)
    otasks.append({"type": "linear", "A": jc.A, "b": np.zeros(1), "q0": None, "cost": np.full(1, 100.0), "gain": 1.0,
                   "lm_damping": 0.0})
    fb = FloatingBaseVelocityLimit(model, "pelvis", [0.4, 0.2, np.inf], [np.inf, np.inf, 1.0])
    limits = [ConfigurationLimit(model), VelocityLimit(model), fb]
    olimits = [("configuration", 0.5), ("velocity", None),
               ("floating_base", table.frame_names.index("pelvis"), np.array([0.4, 0.2, np.inf, np.inf, np.inf, 1.0]))]
    if not floating_base_limit:  # barriers only: the warp-cooperative kernel takes the problem
        limits, olimits = limits[:2], olimits[:2]
    cb = SelfCollisionBarrier(n_collision_pairs=8, gain=20.0, safe_displacement_gain=1.0, d_min=0.05)
    pf, pr = cm.pair_frames(), cm.pair_radii().astype(np.float64)
    ocb = {"type": "self_collision", "pairs": [(int(a), int(b), float(ra), float(rb)) for (a, b), (ra, rb) in zip(pf, pr)],
           "n_pairs": 8, "d_min": 0.05, "gain": 20.0, "safe_displacement_gain": 1.0}
    return ExtraScenario(model, table, q, tasks, otasks, limits, olimits, [cb], [ocb], [], [], 1.0 / 200.0, 0.01, cm)


def tree_extras(nj, B, free_flyer, seed=7):
    """Random joint tree (prismatic joints, fixed or floating base): two frame tasks + posture,
    a position barrier near one tip, a distance barrier between two tips, equality constraints
    (a joint coupling; on floating trees of 12+ joints also a tip frame held in place) and, with a
    floating base, its velocity limit."""
    rng = np.random.default_rng(seed)
    model = helpers.random_tree_model(nj, rng, free_flyer)
    table = model.table()
    q = workloads.sample_configurations(table, B, rng)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.2)
    tasks, otasks = [], []
    for frame, pc, oc in [("tip0", 1.0, 0.5), ("tip1", 2.0, 0.0)]:
        t, o = _frame_task(table, frame, qt, pc, oc, lm_damping=0.05)
        tasks.append(t)
        otasks.append(o)
    q_ref = q[0].copy()
    pt = PostureTask(cost=0.05)
    pt.set_target(q_ref)
    tasks.append(pt)
    otasks.append({"type": "posture", "cost": 0.05, "gain": 1.0, "lm_damping": 0.0, "target": q_ref})
    limits = [ConfigurationLimit(model), VelocityLimit(model)]
    olimits = [("configuration", 0.5), ("velocity", None)]
    if free_flyer:
        base = next(f.name for f in model.frames if f.parentJoint == model.getJointId("root_joint"))
        fb = FloatingBaseVelocityLimit(model, base, [0.5, 0.5, 0.3], [1.0, np.inf, 1.0])
        limits.append(fb)
        olimits.append(("floating_base", table.frame_names.index(base), np.array([0.5, 0.5, 0.3, 1.0, np.inf, 1.0])))
    # barriers placed relative to the first instance's pose so that a good share is active
    fk = okin.forward_kinematics(table, q)
    f2, f0, f3 = (table.frame_names.index(n) for n in ("tip2", "tip0", "tip3"))
    _, p2 = okin.frame_placement(table, fk, f2)
    z_med = float(np.median(p2[:, 2]))
    pb = PositionBarrier("tip2", indices=[2], p_max=np.array([z_med + 0.02]), gain=2.0, safe_displacement_gain=1.0)
    opb = {"type": "position", "frame": f2, "indices": [2], "p_min": None, "p_max": np.array([z_med + 0.02]),
           "gain": np.array([2.0]), "safe_displacement_gain": 1.0}
    _, p0 = okin.frame_placement(table, fk, f0)
    _, p3 = okin.frame_placement(table, fk, f3)
    d_med = float(np.median(np.linalg.norm(p0 - p3, axis=1)))
    sb = BodySphericalBarrier(("tip0", "tip3"), d_min=0.8 * d_med, gain=3.0, safe_displacement_gain=0.5)
    osb = {"type": "body_spherical", "frames": (f0, f3), "d_min": 0.8 * d_med, "gain": 3.0, "safe_displacement_gain": 0.5}
    # equality constraints: a coupling of two joint coordinates and, with a floating base (full
    # row rank whatever the tree), tip3 held where it is (six rows J dq = 0).  On a fixed base
    # the tip may hang from fewer than six joints: six rows of rank < 6 with a right-hand side
    # of rounding size, which the fp64 oracle calls inconsistent and the fp32 kernels accept.
    rq, rv = (7, 6) if free_flyer else (0, 0)
    A = np.zeros((1, table.nv))
    A[0, rv + 1], A[0, rv + 2] = 1.0, -0.5
    lc = LinearHolonomicTask(A, np.zeros(1), None, cost=[1.0], gain=0.005)
    olc = {"type": "linear", "A": A, "b": np.zeros(1), "q0": None, "cost": np.ones(1), "gain": 0.005, "lm_damping": 0.0}
    constraints, oconstraints = [lc], [olc]
    if free_flyer and nj >= 12:
        hold, ohold = _frame_task(table, "tip3", q, 1.0, 1.0)
        constraints.append(hold)
        oconstraints.append(ohold)
    return ExtraScenario(model, table, q, tasks, otasks, limits, olimits, [pb, sb], [opb, osb], constraints, oconstraints,
                         1.0 / 100.0, 1e-6)

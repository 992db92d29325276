"""The implicit gradient of converged IK solutions (oracle/implicit_grad.py) in fp64, against central
finite differences of the oracle's own fixed point (stepped until |v dt| < 1e-12).

* Exactly determined task sets have a zero residual at the fixed point, where the Gauss-Newton
  form is exact: agreement to about 1e-6 relative.
* With a posture task the weighted tasks leave an O(cost^2) residual on the others (Pink sums
  tasks, it does not prioritise them); the Gauss-Newton form is then off by a multiple of that
  residual, while the exact form (dc/dq and dc/dT by central differences of c) matches the
  finite differences to 1e-8.
* A coordinate held on a configuration limit has a zero gradient row."""

import numpy as np
import pytest

from oracle import ik as oik
from oracle import implicit_grad as ig
from oracle import kinematics as okin
from pink_b200 import workloads
from tests import converge_grad_cases as cg
from tests import helpers

# |N form - finite differences| / max |finite differences| <= RESIDUAL_FACTOR * residual at the
# fixed point (measured: 6.8x on UR5 at posture cost 1e-3, at most 2.8x on the other cases)
RESIDUAL_FACTOR = 10.0


def _ur5(posture_cost, with_posture=True, seed=0):
    sc = helpers.ur5_scenario(4, posture_cost=posture_cost, seed=workloads.SEED + seed)
    tasks = [oik._slice_task(t, 0) for t in sc.oracle_tasks]
    if not with_posture:
        tasks = [t for t in tasks if t["type"] != "posture"]
    return sc.table, sc.q64[0], tasks


def _chain7(frames, posture_cost, posture_target=None, seed=3):
    rng = np.random.default_rng(seed)
    model = helpers.random_chain_model(7, rng)
    table = model.table()
    q = workloads.sample_configurations(table, 2, rng)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.2)
    tasks = []
    for name, pc, oc in frames:
        T = helpers.frame_targets(table, qt, name).astype(np.float64)
        tasks.append({"type": "frame", "frame": table.frame_names.index(name), "cost": np.array([pc] * 3 + [oc] * 3),
                      "gain": 1.0, "lm_damping": 0.0, "target": (T[0, :, :3], T[0, :, 3])})
    if posture_cost:
        # near the configuration the frame targets come from: a small residual at the fixed point
        tgt = qt[0] + rng.normal(size=table.nq) * 0.2 if posture_target is None else posture_target
        tasks.append({"type": "posture", "cost": posture_cost, "gain": 0.8, "lm_damping": 0.0, "target": tgt})
    return table, q[0], tasks, qt[0]


def test_ur5_full_pose_exactly_determined():
    table, q0, tasks = _ur5(1e-3, with_posture=False)
    err, _, res, _, _, _, status = cg.check(table, q0, tasks)
    assert status == 0 and res < 1e-12
    assert err < 1e-6, err


@pytest.mark.parametrize("posture_cost", [1e-3, 1e-1])
def test_ur5_full_pose_with_posture(posture_cost):
    table, q0, tasks = _ur5(posture_cost)
    err, err_exact, res, _, _, _, status = cg.check(table, q0, tasks, exact=True)
    assert status == 0
    assert err <= RESIDUAL_FACTOR * res, (err, res)
    assert err_exact < 1e-8, err_exact


def test_free_flyer_frame_and_com_exactly_determined():
    # 6 base + 3 joint coordinates of a serial chain, determined by a full-pose frame task on its
    # tip (6) and a CoM task (3); the base body gets a mass, otherwise moving it against the first
    # joint would change neither
    rng = np.random.default_rng(21)
    model = helpers.random_tree_model(3, rng, free_flyer=True)
    model.append_inertia(model.root_body, 2.0, np.array([0.02, -0.01, 0.03]))
    table = model.table()
    q = workloads.sample_configurations(table, 2, rng)
    qt = workloads.perturb_configurations(table, q, rng, sigma=0.2)
    T = helpers.frame_targets(table, qt, "tip2").astype(np.float64)
    com = okin.center_of_mass(table, okin.forward_kinematics(table, qt))
    tasks = [{"type": "frame", "frame": table.frame_names.index("tip2"), "cost": np.ones(6), "gain": 1.0,
              "lm_damping": 0.0, "target": (T[0, :, :3], T[0, :, 3])},
             {"type": "com", "cost": np.full(3, 2.0), "gain": 0.7, "lm_damping": 0.0, "target": com[0]}]
    q0 = workloads.perturb_configurations(table, qt, rng, sigma=0.05)[0]
    err, _, res, _, _, _, status = cg.check(table, q0, tasks, seed=1)
    assert status == 0 and res < 1e-12
    assert err < 1e-6, err


def test_chain7_two_position_tasks_and_posture():
    table, q0, tasks, _ = _chain7([("tool", 1.0, 0.0), ("elbow", 1.0, 0.0)], 0.05)
    err, err_exact, res, _, _, _, status = cg.check(table, q0, tasks, exact=True, seed=2)
    assert status == 0
    assert err <= RESIDUAL_FACTOR * res, (err, res)
    assert err_exact < 1e-8, err_exact


def test_g1_com_feet_relative_frame_posture():
    sc = helpers.humanoid_scenario("g1_description", 2, with_com=True, with_relative=True)
    keep = ("com", "relative_frame", "posture")
    feet = [sc.table.frame_names.index(n) for n in ("right_ankle_roll_link", "left_ankle_roll_link")]
    tasks = [oik._slice_task(t, 0) for t in sc.oracle_tasks
             if t["type"] in keep or (t["type"] == "frame" and t["frame"] in feet)]
    tasks = [dict(t, target=np.array(sc.q64[1])) if t["type"] == "posture" else t for t in tasks]
    # a few directions per block: each finite difference is two fixed points of a 35-coordinate model
    dirs = [(ti, k) for ti, t in enumerate(tasks) for k in (0, 2)]
    err, err_exact, res, _, _, _, status = cg.check(sc.table, sc.q64[0], tasks, seed=3, dirs=dirs, exact=True)
    assert status == 0
    assert err <= RESIDUAL_FACTOR * res, (err, res)
    assert err_exact < 1e-8, err_exact


def test_held_coordinate_has_zero_gradient():
    _, _, _, posture = _chain7([], 0.0)
    posture = posture.copy()
    table, q0, tasks, _ = _chain7([("tool", 1.0, 0.0)], 0.0)
    posture[3] = table.q_max[3] + 0.5  # beyond the limit: the joint ends on it
    tasks.append({"type": "posture", "cost": 0.3, "gain": 0.8, "lm_damping": 0.0, "target": posture})
    err, err_exact, res, q_star, held, grads, status = cg.check(table, q0, tasks, exact=True, seed=4)
    assert status == 0
    assert held[3] and held.sum() == 1
    assert abs(q_star[3] - table.q_max[3]) < 1e-12
    assert err <= RESIDUAL_FACTOR * res, (err, res)
    assert err_exact < 1e-8, err_exact
    # the held joint does not move: its posture target gets no gradient, and the finite
    # differences of that coordinate of q** vanish
    assert grads[1][3] == 0.0
    g = np.zeros(table.nq)
    g[3] = 1.0
    for ti, k in [(0, 0), (0, 2), (1, 0)]:
        assert abs(cg.finite_difference(table, q_star, tasks, g, ti, k)) < 1e-8


def test_seven_joints_one_frame_task_is_not_positive_definite():
    table, q0, tasks, _ = _chain7([("tool", 1.0, 1.0)], 0.0)
    grads, status = ig.solution_vjp(table, q0, tasks, 1.0, np.ones(table.nq), limits=cg.CFG_ONLY)
    assert status == 4
    assert not np.any(grads[0])

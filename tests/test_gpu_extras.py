"""GPU suite (`-m gpu`): barriers, equality constraints, the opt-in limits and the
constant-Jacobian tasks through the public Python API and the C-ABI, against the
fp64 oracle (the CPU twins are in test_hostsim_extras.py)."""

import numpy as np
import pytest
import torch

import pink_b200
from oracle import barriers as obar
from oracle import kinematics as okin
from pink_b200 import _cabi
from tests import extras, helpers

pytestmark = pytest.mark.gpu

DEVICE = "cuda"  # test_api_extras_host.py re-runs these bodies on the host build with DEVICE = "cpu"


def _sync():
    if DEVICE == "cuda":
        torch.cuda.synchronize()


def _cfg(sc):
    return pink_b200.Configuration(sc.model, None, torch.as_tensor(sc.q32, device=DEVICE),
                                   collision_model=sc.collision_model)


def _solve(sc):
    v, st = pink_b200.solve_ik(_cfg(sc), sc.tasks, sc.dt, solver="quadprog", damping=sc.damping, limits=sc.limits,
                               barriers=sc.barriers, constraints=sc.constraints, safety_break=sc.safety_break,
                               return_status=True)
    _sync()
    return v.cpu().numpy(), st.cpu().numpy()


def test_ur5_barriers_constraints_limits_match_oracle():
    sc = extras.ur5_extras(512)
    v, st = _solve(sc)
    v_ref, st_ref = sc.oracle_solve()
    feasible = st_ref == 0
    assert ((st & _cabi.PK_STATUS_NO_SOLUTION) != 0)[~feasible].all()
    assert (st[feasible] == 0).all() and feasible.mean() > 0.5
    ok = helpers.within_tolerance(v[feasible], v_ref[feasible])
    assert ok.all(), f"{(~ok).sum()} off, worst {np.abs(v - v_ref)[feasible].max()}"
    # the reference raises NoSolutionFound for the infeasible instances
    with pytest.raises(pink_b200.exceptions.NoSolutionFound):
        pink_b200.solve_ik(_cfg(sc), sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, barriers=sc.barriers,
                           constraints=sc.constraints, safety_break=False)


def test_g1_config4_self_collision_barrier_matches_oracle():
    """BASELINE.json config 4: G1-class humanoid, ComTask + FrameTasks + self-collision
    barrier (sphere pairs), plus floating-base limit and a joint coupling task."""
    sc = extras.g1_extras(96)
    v, st = _solve(sc)
    v_ref, st_ref = sc.oracle_solve()
    feasible = st_ref == 0
    assert feasible.mean() > 0.8 and (st[feasible] == 0).all()
    assert ((st & _cabi.PK_STATUS_NO_SOLUTION) != 0)[~feasible].all() and not feasible.all()
    ok = helpers.within_tolerance(v[feasible], v_ref[feasible])
    assert ok.all(), f"{(~ok).sum()} off, worst {np.abs(v - v_ref)[feasible].max()}"


@pytest.mark.parametrize("floating_base_limit", [False, True])
def test_gpu_agrees_with_host_build_on_the_dual_qp_path(floating_base_limit):
    from tests.hostsim import HostSim

    sc = extras.g1_extras(64, floating_base_limit=floating_base_limit)
    v, st = _solve(sc)
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v_h, st_h = hs.solve_ik(prob, sc.q32, targets)
    assert hs.used_tree  # both variants run on the warp-cooperative kernel
    np.testing.assert_array_equal(st, st_h)
    assert (st != 0).any() and (v[st != 0] == 0).all()  # infeasible instances: flagged, zero velocity
    np.testing.assert_allclose(v[st == 0], v_h[st == 0], rtol=2e-3, atol=2e-4)


def test_barrier_api_matches_oracle():
    """Barrier.compute_barrier / compute_jacobian / compute_qp_objective /
    compute_qp_inequalities (pink/barriers/barrier.py) and build_ik with barriers
    and constraints (pink/solve_ik.py:152-203)."""
    sc = extras.ur5_extras(16)
    cfg = _cfg(sc)
    dt = sc.dt
    for barrier, ob in zip(sc.barriers, sc.obarriers):
        h = barrier.compute_barrier(cfg).cpu().numpy()
        J = barrier.compute_jacobian(cfg).cpu().numpy()
        G, rhs = barrier.compute_qp_inequalities(cfg, dt)
        H, c = barrier.compute_qp_objective(cfg)
        G, rhs, H, c = (t.cpu().numpy() for t in (G, rhs, H, c))
        for i in range(16):
            fk = okin.forward_kinematics(sc.table, sc.q64[i])
            h_o = obar.barrier_value(sc.table, sc.q64[i], fk, ob)
            J_o = obar.barrier_jacobian(sc.table, sc.q64[i], fk, ob)
            G_o, rhs_o = obar.barrier_qp_inequalities(sc.table, sc.q64[i], fk, ob, dt)
            H_o, _ = obar.barrier_qp_objective(sc.table, sc.q64[i], fk, ob)
            order, order_o = np.argsort(h[i], kind="stable"), np.argsort(h_o, kind="stable")
            if ob["type"] != "self_collision":
                order = order_o = np.arange(h_o.shape[0])
            assert np.abs(h[i][order] - h_o[order_o]).max() < 2e-6
            assert np.abs(J[i][order] - J_o[order_o]).max() < 1e-5
            assert np.abs(G[i][order] - G_o[order_o]).max() < 5e-4 * (np.abs(G_o).max() + 1e-9)
            assert np.abs(rhs[i][order] - rhs_o[order_o]).max() < 5e-5
            assert np.abs(H[i] - H_o).max() < 2e-4 * (np.abs(H_o).max() + 1e-9) and not c[i].any()
    problem = pink_b200.build_ik(cfg, sc.tasks, dt, damping=sc.damping, limits=sc.limits, barriers=sc.barriers,
                                 constraints=sc.constraints)
    P, q, G, h, A, b = (None if t is None else t.cpu().numpy() for t in problem.unpack()[:6])
    for i in range(16):
        H_o, c_o, G_o, h_o, A_o, b_o = sc.oracle_assemble(i)
        assert G[i].shape == G_o.shape and h[i].shape == h_o.shape
        nb = sum(bb.dim for bb in sc.barriers[:-1])
        k = sc.barriers[-1].dim
        fixed = G_o.shape[0] - k  # everything but the closest-pair rows has a fixed order
        assert np.abs(G[i][:fixed] - G_o[:fixed]).max() < 5e-4 * np.abs(G_o).max()
        assert np.abs(h[i][:fixed] - h_o[:fixed]).max() < 5e-5
        assert np.abs(np.sort(h[i][fixed:]) - np.sort(h_o[fixed:])).max() < 5e-5
        assert np.abs(A[i] - A_o).max() < 1e-5 and np.abs(b[i] - b_o).max() < 1e-5
        assert np.abs(P[i] - H_o).max() < 2e-4 * np.abs(H_o).max()


def test_opt_in_limits_api():
    """FloatingBaseVelocityLimit / AccelerationLimit.compute_qp_inequalities."""
    sc = extras.g1_extras(8)
    cfg = _cfg(sc)
    fb = sc.limits[2]
    G, h = fb.compute_qp_inequalities(cfg, sc.dt)
    G, h = G.cpu().numpy(), h.cpu().numpy()
    assert G.shape == (8, 6, sc.table.nv) and not G[:, :, 6:].any()
    assert np.allclose(h[0], sc.dt * np.array([0.4, 0.2, 1.0, 0.4, 0.2, 1.0]))
    from oracle import limits as olim

    for i in range(8):
        fk = okin.forward_kinematics(sc.table, sc.q64[i])
        G_o, h_o = olim.floating_base_velocity_rows(sc.table, fk, sc.table.frame_names.index("pelvis"),
                                                    fb.twist_max, sc.dt)
        assert np.abs(G[i] - G_o).max() < 1e-5
    su = extras.ur5_extras(8)
    cfg = _cfg(su)
    acc = su.limits[2]
    G, h = acc.compute_qp_inequalities(cfg, su.dt)
    h = h.cpu().numpy()
    for i in range(8):
        G_o, h_o = olim.acceleration_limit_rows(su.table, su.q64[i], su.olimits[2][1], su.olimits[2][2][i], su.dt)
        assert np.array_equal(G, G_o)
        assert np.abs(h[i] - h_o).max() < 1e-6


def test_joint_coupling_tasks_on_the_tree_kernel():
    """examples/humanoid_draco3.py:94-107: JointCouplingTasks + frame + posture tasks
    (warp-cooperative kernel with constant task data in device memory)."""
    from oracle import ik as oik
    from pink_b200 import JointCouplingTask

    sc = helpers.humanoid_scenario("draco3_description", 256)
    cfg = pink_b200.Configuration(sc.model, None, torch.as_tensor(sc.q32, device=DEVICE))
    names = [n for n in sc.table.joint_names if "knee" in n or "hip_pitch" in n][:4]
    jc1 = JointCouplingTask(names[:2], [1.0, -1.0], 100.0, cfg)
    jc2 = JointCouplingTask(names[2:], [1.0, -0.5], 50.0, cfg, gain=0.7, lm_damping=1e-3)
    otasks = sc.oracle_tasks + [
        {"type": "linear", "A": jc1.A, "b": np.zeros(1), "q0": None, "cost": np.full(1, 100.0), "gain": 1.0, "lm_damping": 0.0},
        {"type": "linear", "A": jc2.A, "b": np.zeros(1), "q0": None, "cost": np.full(1, 50.0), "gain": 0.7, "lm_damping": 1e-3},
    ]
    v, st = pink_b200.solve_ik(cfg, sc.tasks + [jc1, jc2], sc.dt, damping=sc.damping, safety_break=sc.safety_break,
                               return_status=True)
    _sync()
    v, st = v.cpu().numpy(), st.cpu().numpy()
    n = 96
    v_ref, st_ref = oik.solve_ik_batch(sc.table, sc.q64[:n], [oik._slice_task_range(t, 0, n) for t in otasks], sc.dt,
                                       sc.damping, sc.oracle_limits, sc.safety_break)
    assert (st == 0).all() and (st_ref == 0).all()
    assert helpers.within_tolerance(v[:n], v_ref).all(), np.abs(v[:n] - v_ref).max()
    e, J = jc2.compute_error(cfg), jc2.compute_jacobian(cfg)
    assert tuple(e.shape) == (256, 1) and tuple(J.shape) == (256, 1, sc.table.nv)
    assert np.allclose(J[0].cpu().numpy(), jc2.A)


@pytest.mark.parametrize("floating_base_limit", [False, True])
def test_config4_full_batch_feasibility_and_sample_parity(floating_base_limit):
    """BASELINE config 4 at full size (B = 16384, G1-class + sphere self-collision
    barrier): every velocity flagged OK satisfies the dense rows and the box of its own
    QP (rows exported by pk_constraint_rows_batched), infeasible instances are flagged with
    zero velocity, and a random sample matches the oracle.  Both variants run on the
    warp-cooperative kernel (dual QP in shared memory); the floating-base limit adds its
    rows to that dual QP.  The general path's solve is tested in test_gpu_kernel_paths.py."""
    sc = extras.g1_extras(16384, floating_base_limit=floating_base_limit)
    v, st = _solve(sc)
    ok = st == 0
    assert ok.mean() > 0.95 and ((st[~ok] & _cabi.PK_STATUS_NO_SOLUTION) != 0).all() and not v[~ok].any()
    cfg = _cfg(sc)
    from pink_b200.solve_ik import _pack_problem

    prob, targets, _ = _pack_problem(cfg, sc.tasks, sc.dt, sc.damping, sc.limits, sc.safety_break, sc.barriers,
                                     sc.constraints)
    G, hG, _, _, lo, hi = (t.cpu().numpy().astype(np.float64) for t in cfg.engine.constraint_rows(prob, cfg.q_device, targets))
    x = v.astype(np.float64) * sc.dt
    rows = np.isfinite(hG)
    viol = np.where(rows, np.einsum("brn,bn->br", G, x) - hG, -np.inf).max(axis=1)
    box = np.maximum(x - hi, lo - x).max(axis=1)
    assert viol[ok].max() <= 2e-6 and box[ok].max() <= 1e-7
    rng = np.random.default_rng(0)
    pick = rng.choice(np.nonzero(ok)[0], size=48, replace=False)
    from oracle import ik as oik

    from oracle import qp as oqp

    compared = 0
    for i in pick:
        tasks = [oik._slice_task(t, i) for t in sc.otasks]
        v_ref, st_ref = oik.solve_ik(sc.table, sc.q64[i], tasks, sc.dt, sc.damping, oik._slice_limits(sc.olimits, i),
                                     sc.safety_break, sc.obarriers, [])
        assert st_ref == 0
        # Parity is only defined where the reference's own answer is stable under fp32-level
        # perturbations of its dense rows (spheres in deep penetration with an unbounded
        # floating base give QPs whose minimiser moves by 10 % for a 1e-6 change of G, h).
        H, c, Gm, hm, _, _ = sc.oracle_assemble(i)
        dense = [r for r in range(Gm.shape[0]) if np.count_nonzero(Gm[r]) != 1]
        Gp, hp = Gm.copy(), hm.copy()
        Gp[dense] *= 1.0 + 1e-6 * rng.standard_normal(Gp[dense].shape)
        hp[dense] += 1e-6 * (np.abs(hm[dense]) + 1e-3) * rng.standard_normal(len(dense))
        res = oqp.solve_qp(H, c, Gp, hp)
        if not res.found or not helpers.within_tolerance((res.x / sc.dt)[None], v_ref[None], atol=1e-4, rtol=1e-3).all():
            continue
        compared += 1
        assert helpers.within_tolerance(v[i][None], v_ref[None]).all(), (i, np.abs(v[i] - v_ref).max())
    assert compared >= 0.75 * len(pick), compared

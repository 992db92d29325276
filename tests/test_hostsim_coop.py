"""Sub-warp chain kernel body (pink_b200/csrc/pk_coop.cuh) on the host build, for every
lanes-per-instance variant L = 1, 2, 4, 8 (hostsim path 10 + L), against the fp64 oracle:
the same scenarios as the one-instance-per-thread kernel in test_hostsim_parity.py, plus
the KKT certificate at a large batch and the interior regime (loose limits, where the
solver leaves the two-slot loop for the Cholesky rounds).  The host build follows the library's
selection: L = 4 / 8 exist at <6, 1> only, so on other chains those cases run the
thread-per-instance kernel the library falls back to."""

import numpy as np
import pytest

from oracle import ik as oik
from tests import helpers
from tests.hostsim import HostSim

LANES = [1, 2, 4, 8]


@pytest.mark.parametrize("lanes", LANES)
@pytest.mark.parametrize("kind", ["reachable", "unreachable", "at_target"])
def test_ur5_matches_oracle(kind, lanes):
    sc = helpers.ur5_scenario(400, kind)
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    v_ref, st_ref = sc.oracle_solve()
    assert (st == 0).all() and (st_ref == 0).all()
    ok = helpers.within_tolerance(v, v_ref)
    if kind == "at_target":
        # noise floor of fp32 forward kinematics, see test_hostsim_parity.py
        assert ok.mean() >= 0.97
        assert helpers.within_tolerance(v, v_ref, atol=5e-3, rtol=2e-2).all()
    else:
        assert ok.all(), f"{(~ok).sum()} instances off, worst {np.abs(v - v_ref).max()}"


@pytest.mark.parametrize("lanes", [1, 2])
def test_ur5_large_batch_kkt_certificate(lanes):
    """The fp32 solution satisfies the fp64 KKT conditions of its own QP (unique minimiser)."""
    sc = helpers.ur5_scenario(20000, "reachable")
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    assert (st == 0).all()
    H, c, G, h = sc.oracle_build()
    x = v.astype(np.float64) * sc.dt
    stat, prim, lo, hi = oik.kkt_check_batch(H, c, G, h, x)
    scale = np.abs(c).max(axis=1)
    assert prim.max() <= 1e-6
    assert np.quantile(stat / scale, 0.999) <= 1e-4
    assert (stat / scale).max() <= 1e-3


@pytest.mark.parametrize("lanes", [1, 2])
def test_ill_conditioned_free_block_reaches_the_minimiser(lanes):
    """No Levenberg-Marquardt term, dt = 0.1: a handful of 40000 instances reach the rounds with a
    5-coordinate free block of cond ~1e7 whose refinement steps leave the box.  Those coordinates
    must become active (polish<activate_clamped>); clamping alone stalled at a relative
    stationarity of 2e-2 (profiles/r02i_hostsim_soak.txt is the sweep this came from)."""
    sc = helpers.ur5_scenario(40000, "reachable", seed=102, lm_damping=0.0, posture_cost=1e-3)
    sc.dt = 0.1
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    assert (st == 0).all()
    H, c, G, h = sc.oracle_build()
    stat, prim, _, _ = oik.kkt_check_batch(H, c, G, h, v.astype(np.float64) * sc.dt)
    assert prim.max() <= 1e-6
    assert (stat / np.abs(c).max(axis=1)).max() <= 1e-4


@pytest.mark.parametrize("lanes", LANES)
def test_lane_variants_agree_with_the_thread_per_instance_kernel(lanes):
    sc = helpers.ur5_scenario(1500, "reachable")
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v0, s0 = hs.solve_ik(prob, sc.q32, targets)
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    np.testing.assert_array_equal(st, s0)
    # same mathematics; joint frames re-oriented, rows summed in a different order
    np.testing.assert_allclose(v, v0, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("lanes", LANES)
def test_out_of_limits_and_safety_break(lanes):
    sc = helpers.ur5_scenario(200, "reachable", out_of_limits=7)
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    v_ref, st_ref = sc.oracle_solve()
    np.testing.assert_array_equal(st & 3, st_ref)
    assert (st == 2).sum() == 7
    assert np.abs(v[st == 2]).max() == 0.0
    assert helpers.within_tolerance(v, v_ref).all()
    sc.safety_break = False
    prob, targets, _ = sc.problem()
    v2, st2 = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    v2_ref, st2_ref = sc.oracle_solve()
    assert ((st2 & 2) != 0).sum() == 7
    np.testing.assert_array_equal((st2 & 1) != 0, st2_ref == 1)
    solved = (st2 & 1) == 0
    assert helpers.within_tolerance(v2[solved], v2_ref[solved]).all()


@pytest.mark.parametrize("lanes", LANES)
def test_no_limits_is_the_unconstrained_minimiser(lanes):
    """Infinite box: every coordinate starts free, the solve goes straight to the rounds."""
    sc = helpers.ur5_scenario(100, "reachable")
    sc.limits, sc.oracle_limits = [], []
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    H, c, G, h = sc.oracle_build()
    assert G is None
    x_ref = -np.linalg.solve(H, c[..., None])[..., 0]
    np.testing.assert_allclose(v * sc.dt, x_ref, rtol=2e-3, atol=2e-6)


@pytest.mark.parametrize("lanes", LANES)
def test_interior_regime_near_convergence(lanes):
    """Targets 1e-3 rad away: the minimiser is interior for almost every coordinate, i.e. the
    opposite of the benchmark workload (closed-loop tracking after convergence)."""
    robot, model, table = helpers.load("ur5_description")
    rng = np.random.default_rng(11)
    from pink_b200 import workloads

    q = workloads.sample_configurations(table, 300, rng, near_limit_fraction=0.0)
    qt = q + rng.normal(0.0, 1e-3, size=q.shape)
    sc = helpers.ur5_scenario(300, "reachable")
    sc.q32 = q.astype(np.float32)
    sc.q64 = sc.q32.astype(np.float64)
    T = helpers.frame_targets(table, qt, "tool0")
    sc.tasks[0].set_target(__import__("torch").as_tensor(T))
    sc.oracle_tasks[0]["target"] = (T[:, :, :3].astype(np.float64), T[:, :, 3].astype(np.float64))
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    v_ref, st_ref = sc.oracle_solve()
    assert (st == 0).all() and (st_ref == 0).all()
    assert helpers.within_tolerance(v, v_ref, atol=5e-4, rtol=5e-3).mean() >= 0.99


@pytest.mark.parametrize("lanes", LANES)
@pytest.mark.parametrize("nj,kw", [
    (2, {}), (3, {"prismatic": (1,)}), (4, {"two_tasks": True}), (5, {"shared_target": True}),
    (6, {"two_tasks": True, "prismatic": (0, 4)}), (7, {"two_tasks": True, "prismatic": (2,)}), (7, {}),
])
def test_chain_instantiations(nj, kw, lanes):
    """Every <NJ, NFT> instantiation, prismatic joints, mid-chain frames (zero columns, a
    frame whose joint lies in another lane's segment) and shared targets."""
    sc = helpers.chain_scenario(nj, 96, seed=nj, **kw)
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v, st = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    v_g, st_g = hs.solve_ik(prob, sc.q32, targets, path=1)
    np.testing.assert_array_equal(st, st_g)
    np.testing.assert_allclose(v, v_g, atol=5e-4, rtol=5e-3)
    v_ref, st_ref = sc.oracle_solve()
    np.testing.assert_array_equal(st & 3, st_ref)
    assert helpers.within_tolerance(v, v_ref, atol=5e-4, rtol=5e-3).mean() >= 0.97

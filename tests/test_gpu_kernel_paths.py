"""GPU suite (`-m gpu`): kernel paths that users reach but the scenarios of the other GPU tests
do not, run on the device branch by branch:

- A. general-path solves (``ik_generic_kernel`` at its three instantiations ``<8, 8>``,
  ``<30, 36>``, ``<58, 64>``, with the box QP ``BoxLSQ`` and with the dual QP of pk_dualqp.cuh);
- B. every factorisation size class of the tree kernel (``TreeStep::eqp``: ``eqp_cols<8|16|24|32>``,
  ``eqp_impl<false|true>``) and the tree / general-path boundary;
- C. the sub-warp chain kernel ``ik_coop_kernel<NJ, NFT, L>`` at L = 1, 2, 4, 8 lanes per instance;
- D. the recompute path of the chain kernel under programmatic dependent launch at every
  ``<NJ, NFT>``.

Every case is checked four ways: the dispatch (which kernel and branch the host build of the
same selection code picks), the fp64 oracle on a slice, the host build of the same path
(statuses bitwise equal), and the infeasible instances (``PK_STATUS_NO_SOLUTION`` with zero
velocity, where the oracle raises ``NoSolutionFound``).  Batch sizes are ragged, so that the last
CTA is partly empty.  The host halves of A, B and C also run without a GPU
(test_hostsim_kernel_paths.py)."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from pink_b200 import _cabi
from tests import extras, helpers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SOLUTION = _cabi.PK_STATUS_NO_SOLUTION
STD = (helpers.V_ATOL, helpers.V_RTOL)
LOOSE = (5e-4, 5e-3)  # the host tests' tolerance for random trees, chains and G1 with extra limits
TWIN = (2e-4, 2e-3)  # host build vs GPU, tree / general path (test_gpu_extras.py)
CHAIN_TWIN = (5e-4, 5e-3)  # host build vs GPU, chain kernels (test_gpu_parity.py)
UR5_A_MAX = np.array([40.0, 40.0, 60.0, np.inf, 80.0, 80.0])


class Case:
    """A scenario (extras.ExtraScenario) and what it must land on: ``kernel`` is "chain", "tree"
    or "general"; ``inst`` the ``ik_generic_kernel`` instantiation; ``qp`` "box" or "dual";
    ``branch`` the tree factorisation branch named by the case; ``tol`` against the oracle."""

    def __init__(self, sc, kernel, n_oracle, tol=STD, inst=None, qp=None, K=None, branch=None, min_feasible=0.5):
        self.sc, self.kernel, self.n_oracle, self.tol = sc, kernel, n_oracle, tol
        self.inst, self.qp, self.K, self.branch, self.min_feasible = inst, qp, K, branch, min_feasible


# ---- A: general-path solves ------------------------------------------------------------------

def _g1_a_max(table, a=150.0):
    return np.concatenate([np.full(6, np.inf), np.full(table.nv - 6, a)])


def general_case(name):
    if name == "ur5-box":
        sc = extras.with_shared_acceleration_limit(extras.as_extra(helpers.ur5_scenario(333, "reachable")), UR5_A_MAX)
        return Case(sc, "general", 200, inst="<8, 8>", qp="box")
    if name == "ur5-dual":
        sc = extras.with_shared_acceleration_limit(extras.ur5_extras(333), UR5_A_MAX)
        return Case(sc, "general", 200, inst="<8, 8>", qp="dual")
    if name == "g1-box":
        sc = extras.as_extra(helpers.humanoid_scenario("g1_description", 67, with_com=True))
        sc = extras.with_shared_acceleration_limit(sc, _g1_a_max(sc.table))
        return Case(sc, "general", 48, "by-condition", inst="<30, 36>", qp="box")
    if name == "g1-dual":
        # the acceleration box next to the self-collision barrier leaves about half of the QPs
        # infeasible (spheres that cannot separate within a dt^2)
        sc = extras.g1_extras(67)
        sc = extras.with_shared_acceleration_limit(sc, _g1_a_max(sc.table, 1000.0))
        return Case(sc, "general", 48, inst="<30, 36>", qp="dual", min_feasible=0.4)
    raise KeyError(name)


# tree_extras across the 32-joint boundary: 32 joints with a free-flyer is the largest model whose
# plan still fits the tree kernel's dual QP; beyond it the general path's <58, 64> takes over
TREE_EXTRAS = [(32, "tree", None), (33, "general", "<58, 64>"), (40, "general", "<58, 64>"),
               (58, "general", "<58, 64>")]


def tree_extras_case(nj):
    kernel, inst = {n: (k, i) for n, k, i in TREE_EXTRAS}[nj]
    return Case(extras.tree_extras(nj, 67, True, seed=7), kernel, 48, LOOSE, inst=inst, qp="dual")


# ---- B: tree-kernel factorisation size classes ------------------------------------------------

FULL = (1.0, 1.0)
SIZE_CLASSES = {
    # name: (joints, free-flyer, frame tasks on tips 0..3, CoM task, rows of the linear tasks, K, branch)
    "K6-nv20": (20, False, [FULL], False, (), 6, "eqp_cols<8>"),
    "K12-nv20": (20, False, [FULL, ([1.0, 1.0, 0.0], [0.0, 1.0, 1.0])], False, (2,), 12, "eqp_cols<16>"),
    "K24-nv20": (20, False, [FULL] * 4, False, (), 24, "eqp_cols<24>"),
    "K32-nv31": (31, False, [FULL] * 4, True, (5,), 32, "eqp_cols<32>"),
    "K32-nv32": (32, False, [FULL] * 4, True, (5,), 32, "eqp_impl<false>"),
    "K33-nv32": (32, False, [FULL] * 4, True, (6,), 33, "eqp_impl<true>"),
    # PK_MAX_TASKS = 12 bounds the task count: four frames and seven linear tasks reach K = 64
    "K64-nv38": (32, True, [FULL] * 4, False, (6, 6, 6, 6, 6, 6, 4), 64, "eqp_impl<true>"),
    "K65-nv38": (32, True, [FULL] * 4, False, (6, 6, 6, 6, 6, 6, 5), 65, None),
}


def size_class_case(name, limits):
    nj, ff, frames, com, linear, K, branch = SIZE_CLASSES[name]
    frames = [(k, pc, oc) for k, (pc, oc) in enumerate(frames)]
    sc = extras.tree_rows_scenario(nj, 67, ff, frames, com, linear, limits=limits, seed=11 + nj)
    if branch is None:  # one row beyond the tree kernel's 64: the general path, as the boundary twin
        return Case(sc, "general", 48, inst="<58, 64>", qp="box", K=K)
    if limits:  # velocity limits put some coordinates on a bound: nf < nv at the solution
        branch = eqp_branch(K, nj + 6 * ff - 1)
    return Case(sc, "tree", 48, K=K, branch=branch, qp="box")


def eqp_branch(K, nf):
    """TreeStep::eqp's choice for K task rows and nf free columns (pk_tree.cuh)."""
    if K <= 32 and nf <= 31:
        return "eqp_cols<%d>" % (8 if K <= 8 else 16 if K <= 16 else 24 if K <= 24 else 32)
    return "eqp_impl<true>" if K > 32 else "eqp_impl<false>"


def task_rows(prob):
    """K: rows of the non-diagonal tasks with a non-zero cost (make_tree_plan)."""
    diag = (_cabi.PK_TASK_POSTURE, _cabi.PK_TASK_JOINT_VELOCITY)
    return sum(int(np.count_nonzero(np.array(prob.tasks[t].cost))) for t in range(prob.ntasks)
               if prob.tasks[t].type not in diag)


# ---- the host half of every case: dispatch, oracle, host build -------------------------------

def agrees_with_oracle(case, v, v_ref, feasible):
    if case.tol == "by-condition":
        # G1-class weights: cond(H) of 1e6..1e7.  helpers.PARITY_BINS on a slice of a few dozen
        # instances: below cond 1e5 all inside the standard tolerance; above, its first fraction
        # inside the standard tolerance and all inside the loosest bound
        # inside the loosest bound or, along the flat directions of such an H, a minimiser as
        # good as fp32 gets: the same objective to 1e-8 relative and the rows satisfied
        sc = case.sc
        qps = [sc.oracle_assemble(i) for i in range(len(v_ref))]
        cond = np.linalg.cond(np.stack([qp[0] for qp in qps]))
        assert (cond < helpers.PARITY_BINS[-1][1]).all()
        for lo, hi, bounds in helpers.PARITY_BINS:
            m = feasible & (cond >= lo) & (cond < hi)
            if not m.any():
                continue
            (atol, rtol, need), loosest = bounds[0], bounds[-1]
            ok = helpers.within_tolerance(v[m], v_ref[m], atol=atol, rtol=rtol)
            assert ok.mean() >= need, (lo, ok.mean(), np.abs(v - v_ref)[m].max())
            for i in np.nonzero(m)[0]:
                if helpers.within_tolerance(v[i][None], v_ref[i][None], atol=loosest[0], rtol=loosest[1]).all():
                    continue
                H, c, G, h = qps[i][:4]
                x, xr = v[i].astype(np.float64) * sc.dt, v_ref[i] * sc.dt
                f, fr = 0.5 * x @ H @ x + c @ x, 0.5 * xr @ H @ xr + c @ xr
                assert lo > 0.0 and f - fr <= 1e-8 * abs(fr) and (G @ x - h).max() <= 1e-6, (i, cond[i], f - fr)
        return
    atol, rtol = case.tol
    ok = helpers.within_tolerance(v[feasible], v_ref[feasible], atol=atol, rtol=rtol)
    assert ok.all(), f"{(~ok).sum()} of {feasible.sum()} off, worst {np.abs(v - v_ref)[feasible].max()}"


def host_side(case):
    """Dispatch assertions and the host build against the oracle; returns the inputs and the
    results the GPU half is compared with."""
    from tests.hostsim import HostSim

    sc = case.sc
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    v_h, st_h = hs.solve_ik(prob, sc.q32, targets)
    landed = "chain" if hs.used_chain else "tree" if hs.used_tree else "general"
    assert landed == case.kernel, (landed, case.kernel)
    nv, nj = sc.table.nv, sc.table.njoints
    if case.inst is not None:  # launch_generic's choice
        inst = "<8, 8>" if nv <= 8 and nj <= 8 else "<30, 36>" if nv <= 36 and nj <= 30 else "<58, 64>"
        assert inst == case.inst, (inst, nv, nj)
    if case.qp is not None:
        dual = prob.nbarriers > 0 or prob.nconstraints > 0 or prob.fb_enabled
        assert ("dual" if dual else "box") == case.qp
    if case.K is not None:
        assert task_rows(prob) == case.K
        # moderate costs: cond(H) < 1e5, where the standard tolerance applies (helpers.PARITY_BINS)
        assert max(np.linalg.cond(sc.oracle_assemble(i)[0]) for i in range(case.n_oracle)) < 1e5
    n = case.n_oracle
    v_ref, st_ref = sc.oracle_solve(n)
    feasible = st_ref == 0
    assert feasible.mean() > case.min_feasible
    # infeasible instances: flagged, zero velocity (the oracle's NoSolutionFound)
    np.testing.assert_array_equal((st_h[:n] & NO_SOLUTION) != 0, st_ref == 1)
    assert not v_h[(st_h & NO_SOLUTION) != 0].any()
    assert (st_h[:n][feasible] == 0).all()
    agrees_with_oracle(case, v_h[:n], v_ref, feasible)
    if case.branch is not None:
        # every factorisation of the box-free runs has nf = nv; with limits, nf is the number of
        # coordinates strictly inside the box at the oracle's solution
        if sc.limits:
            _, _, _, _, lo, hi = hs.constraint_rows(prob, sc.q32[:n], targets[:n])
            x = v_ref * sc.dt
            nf = ((x > lo + 1e-7) & (x < hi - 1e-7)).sum(axis=1)[feasible]
        else:
            nf = np.full(int(feasible.sum()), nv)
        branches = {eqp_branch(case.K, int(f)) for f in nf}
        assert branches == {case.branch}, (case.branch, branches)
    return prob, targets, v_h, st_h, v_ref, st_ref


def _gpu_solve(sc):
    cfg = pink_b200.Configuration(sc.model, None, torch.as_tensor(sc.q32, device="cuda"),
                                  collision_model=sc.collision_model)
    v, st = pink_b200.solve_ik(cfg, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, barriers=sc.barriers,
                               constraints=sc.constraints, safety_break=sc.safety_break, return_status=True)
    torch.cuda.synchronize()
    return v.cpu().numpy(), st.cpu().numpy()


def check_on_gpu(case, twin=TWIN):
    _, _, v_h, st_h, v_ref, st_ref = host_side(case)
    v, st = _gpu_solve(case.sc)
    n = case.n_oracle
    np.testing.assert_array_equal(st, st_h)
    assert not v[(st & NO_SOLUTION) != 0].any()
    solved = st == 0
    np.testing.assert_allclose(v[solved], v_h[solved], atol=twin[0], rtol=twin[1])
    agrees_with_oracle(case, v[:n], v_ref, st_ref == 0)
    return v, st


GENERAL = ["ur5-box", "ur5-dual", "g1-box", "g1-dual"]


@pytest.mark.parametrize("name", GENERAL)
def test_general_path_solves(name):
    """ik_generic_kernel<8, 8> (UR5) and <30, 36> (G1) with a shared AccelerationLimit, box QP
    (BoxLSQ) and dual QP with its fp64 refinement (pk_dualqp.cuh, barriers + equalities)."""
    check_on_gpu(general_case(name))


@pytest.mark.parametrize("nj", [n for n, _, _ in TREE_EXTRAS])
def test_tree_extras_across_the_32_joint_boundary(nj):
    """Random floating trees with barriers, equalities and the base limit: 32 joints on the tree
    kernel's dual QP (pk_treedual.cuh), 33 / 40 / 58 on ik_generic_kernel<58, 64>'s dual QP."""
    check_on_gpu(tree_extras_case(nj))


@pytest.mark.parametrize("limits", [False, True], ids=["no-limits", "limits"])
@pytest.mark.parametrize("name", list(SIZE_CLASSES))
def test_tree_factorisation_size_classes(name, limits):
    """TreeStep::eqp at every size class: eqp_cols<8|16|24|32> (K <= 32, nf <= 31; nf = 31 puts
    the right-hand side in lane 31), eqp_impl<false> (nf = 32), eqp_impl<true> (K > 32), the
    largest K = 64 the tree kernel takes and its K = 65 twin on the general path."""
    check_on_gpu(size_class_case(name, limits))


def test_tree_rollout_with_more_than_32_task_rows():
    """ik_tree_rollout_kernel with K = 33 (eqp_impl<true>) against the same closed loop of
    separate solve + integrate calls."""
    case = size_class_case("K33-nv32", True)
    host_side(case)
    sc = case.sc
    ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, safety_break=False,
                             batch_size=sc.B)
    _, targets, _ = sc.problem()
    q0 = torch.as_tensor(sc.q32, device="cuda")
    t_d = torch.as_tensor(targets, device="cuda")
    steps = 4
    q_f, v_f, st_f = ik.rollout(q0, t_d, steps)
    q = q0.clone()
    st_or = torch.zeros(sc.B, dtype=torch.int32, device="cuda")
    for _ in range(steps):
        v, st = ik.solve(q, t_d)
        st_or |= st
        q = ik.engine.integrate(q, v, sc.dt)
    torch.cuda.synchronize()
    assert (st_or.cpu().numpy() == 0).all()
    np.testing.assert_array_equal(st_f.cpu().numpy(), st_or.cpu().numpy())
    # the integration is inlined into another kernel: the last bit may differ and ride along
    np.testing.assert_allclose(q_f.cpu().numpy(), q.cpu().numpy(), atol=2e-5)
    np.testing.assert_allclose(v_f.cpu().numpy(), v.cpu().numpy(), atol=5e-3, rtol=5e-3)


# ---- C: sub-warp chain kernel, one process per PK_CHAIN_LANES ---------------------------------

CHAINS = {
    "nj2": lambda: helpers.chain_scenario(2, 1002, seed=2),
    "nj3-prismatic": lambda: helpers.chain_scenario(3, 1003, seed=3, prismatic=(1,)),
    "nj4-two-frames": lambda: helpers.chain_scenario(4, 1004, seed=4, two_tasks=True),
    "nj5-shared-target": lambda: helpers.chain_scenario(5, 1005, seed=5, shared_target=True),
    "nj6-two-frames": lambda: helpers.chain_scenario(6, 1006, seed=6, two_tasks=True, prismatic=(0, 4)),
    "nj7-two-frames": lambda: helpers.chain_scenario(7, 1007, seed=7, two_tasks=True, prismatic=(2,)),
    "nj7": lambda: helpers.chain_scenario(7, 1007, seed=7),
    "nj4-posture-only": lambda: helpers.chain_scenario(4, 1004, seed=14, frame_tasks=False),
    "ur5-reachable": lambda: helpers.ur5_scenario(1001, "reachable"),
    "ur5-unreachable": lambda: helpers.ur5_scenario(1001, "unreachable"),
    "ur5-out-of-limits": lambda: helpers.ur5_scenario(1001, "reachable", out_of_limits=9),
}
ROLLOUT_STEPS = 4


def _nft(sc):
    return sum(type(t).__name__ == "FrameTask" for t in sc.tasks)


def coop_takes(lanes, sc):
    """Does the library run ik_coop_kernel for PK_CHAIN_LANES = lanes?  4 and 8 lanes exist for
    <6, 1> only; other shapes fall back to the thread-per-instance kernel."""
    return lanes in (1, 2) or (sc.table.njoints == 6 and _nft(sc) == 1)


def dump_chain_outputs(path, steps=ROLLOUT_STEPS):
    """Solve and rollout(steps, q_out) of every CHAINS case on cuda:0 (run in a subprocess:
    PK_CHAIN_LANES / PK_CHAIN_FORCE_RECOMPUTE are read once per process)."""
    out = {}
    for name, make in CHAINS.items():
        sc = make()
        ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                                 safety_break=sc.safety_break, device="cuda", batch_size=sc.B)
        _, targets, _ = sc.problem()
        q = torch.as_tensor(sc.q32, device="cuda")
        t = None if targets is None else torch.as_tensor(targets, device="cuda")
        v, st = ik.solve(q, t)
        q_out = torch.full_like(q, float("nan"))
        _, v_r, st_r = ik.rollout(q, t, steps, q_out=q_out)
        torch.cuda.synchronize()
        for key, val in (("v", v), ("status", st), ("q_out", q_out), ("v_roll", v_r), ("status_roll", st_r)):
            out[f"{name}/{key}"] = val.cpu().numpy()
    np.savez(path, **out)


def _run_dump(tmp_path, env_name, env_value, dump="dump_chain_outputs"):
    out = tmp_path / f"{env_name}-{env_value}.npz"
    env = dict(os.environ, **{env_name: str(env_value)})
    env.pop("PK_CHAIN_LANES" if env_name != "PK_CHAIN_LANES" else "PK_CHAIN_FORCE_RECOMPUTE", None)
    code = f"from tests.test_gpu_kernel_paths import {dump} as d; d({str(out)!r})"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, check=True, timeout=900)
    return dict(np.load(out))


def host_rollout(hs, prob, sc, targets, path, steps=ROLLOUT_STEPS):
    """The kernels' closed loop on the host build: an instance that fails a step (no solution /
    outside limits with safety_break) keeps that step's velocity and stops moving."""
    q = sc.q32.copy()
    v = np.zeros_like(q)
    st_all = np.zeros(sc.B, dtype=np.int32)
    for _ in range(steps):
        frozen = (st_all & (NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF)) != 0
        if sc.safety_break:
            frozen |= (st_all & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
        live = ~frozen
        if not live.any():
            break
        v_s, st_s = hs.solve_ik(prob, q[live], None if targets is None else targets[live], path=path)
        v[live] = v_s
        st_all[live] |= st_s & 0xFF
        q[live] = q[live] + v_s * np.float32(sc.dt)
    return q, v, st_all


def chain_host_side(name, lanes):
    """Dispatch (chain kernel; the host build runs the L-lane body) and the host build of the
    sub-warp kernel against the oracle."""
    from tests.hostsim import HostSim

    sc = CHAINS[name]()
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    hs.solve_ik(prob, sc.q32[:1], None if targets is None else targets[:1])
    assert hs.used_chain
    v_h, st_h = hs.solve_ik(prob, sc.q32, targets, path=10 + lanes)
    n = 200
    v_ref, st_ref = sc.oracle_solve(n)
    np.testing.assert_array_equal(st_h[:n] & 3, st_ref)
    assert not v_h[(st_h & 3) != 0].any()
    atol, rtol = STD if name.startswith("ur5") else LOOSE
    ok = helpers.within_tolerance(v_h[:n], v_ref, atol=atol, rtol=rtol)
    assert ok.mean() >= (1.0 if name.startswith("ur5") else 0.97), np.abs(v_h[:n] - v_ref).max()
    return sc, hs, prob, targets, v_h, st_h, v_ref, st_ref


@pytest.fixture(scope="module")
def default_chain_outputs(tmp_path_factory):
    return _run_dump(tmp_path_factory.mktemp("lanes0"), "PK_CHAIN_LANES", 0)


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_sub_warp_chain_kernel(lanes, tmp_path, default_chain_outputs):
    """ik_coop_kernel<NJ, NFT, L> (PK_CHAIN_LANES = L, group shuffles of pk_group.cuh): solve and
    a 4-step rollout with q_out against the host build of the L-lane body and the oracle; where
    the library has no L-lane variant (L = 4 / 8 off <6, 1>) bitwise equal to the default kernel."""
    got = _run_dump(tmp_path, "PK_CHAIN_LANES", lanes)
    for name in CHAINS:
        sc, hs, prob, targets, v_h, st_h, v_ref, st_ref = chain_host_side(name, lanes)
        g = {k: got[f"{name}/{k}"] for k in ("v", "status", "q_out", "v_roll", "status_roll")}
        if not coop_takes(lanes, sc):
            for k, val in g.items():
                np.testing.assert_array_equal(val, default_chain_outputs[f"{name}/{k}"], err_msg=f"{name} {k}")
            continue
        n = 200
        np.testing.assert_array_equal(g["status"], st_h, err_msg=name)
        assert not g["v"][(g["status"] & 3) != 0].any(), name
        np.testing.assert_allclose(g["v"], v_h, atol=CHAIN_TWIN[0], rtol=CHAIN_TWIN[1], err_msg=name)
        atol, rtol = STD if name.startswith("ur5") else LOOSE
        ok = helpers.within_tolerance(g["v"][:n], v_ref, atol=atol, rtol=rtol)
        assert ok.mean() >= (1.0 if name.startswith("ur5") else 0.97), (name, np.abs(g["v"][:n] - v_ref).max())
        q_h, vr_h, str_h = host_rollout(hs, prob, sc, targets, 10 + lanes)
        np.testing.assert_array_equal(g["status_roll"], str_h, err_msg=name)
        np.testing.assert_allclose(g["q_out"], q_h, atol=2e-5, err_msg=name)
        np.testing.assert_allclose(g["v_roll"], vr_h, atol=CHAIN_TWIN[0], rtol=CHAIN_TWIN[1], err_msg=name)


# ---- D: forced recompute of the PDL chain kernel at every <NJ, NFT> ---------------------------

def _recompute_cases():
    cases = {}
    for nj in range(2, 8):
        cases[f"nj{nj}-nft0"] = (lambda nj=nj: helpers.chain_scenario(nj, 515 + nj, seed=20 + nj, frame_tasks=False))
        cases[f"nj{nj}-nft1"] = (lambda nj=nj: helpers.chain_scenario(nj, 515 + nj, seed=20 + nj))
        cases[f"nj{nj}-nft2"] = (lambda nj=nj: helpers.chain_scenario(nj, 515 + nj, seed=20 + nj, two_tasks=True))
    # targets row of 12 + 6 floats: not a multiple of 4, the scalar copy of chain_copy_row
    cases["nj6-nft1-posture-rows"] = lambda: helpers.chain_scenario(6, 521, seed=26, posture_per_instance=True)
    return cases


RECOMPUTE = _recompute_cases()


def dump_recompute_outputs(path, steps=3):
    """Solve and rollout(3, q_out) of every RECOMPUTE case on cuda:0."""
    out = {}
    for name, make in RECOMPUTE.items():
        sc = make()
        ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, safety_break=True,
                                 device="cuda", batch_size=sc.B)
        _, targets, _ = sc.problem()
        q = torch.as_tensor(sc.q32, device="cuda")
        t = None if targets is None else torch.as_tensor(targets, device="cuda")
        v, st = ik.solve(q, t)
        q_out = torch.full_like(q, float("nan"))
        _, v_r, st_r = ik.rollout(q, t, steps, q_out=q_out)
        torch.cuda.synchronize()
        for key, val in (("v", v), ("status", st), ("q_out", q_out), ("v_roll", v_r), ("status_roll", st_r)):
            out[f"{name}/{key}"] = val.cpu().numpy()
    np.savez(path, **out)


def recompute_dispatch(name):
    """The case lands on the chain kernel with the NFT it names, and its targets row fits the PDL
    instantiation's copy (12 NFT + 2 NJ floats), so the PDL kernel runs it."""
    from tests.hostsim import HostSim

    sc = RECOMPUTE[name]()
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    hs.solve_ik(prob, sc.q32[:1], None if targets is None else targets[:1])
    assert hs.used_chain
    nj, nft = sc.table.njoints, _nft(sc)
    assert name.startswith(f"nj{nj}-nft{nft}")
    assert prob.target_stride <= 12 * nft + 2 * nj
    return prob


def test_forced_recompute_at_every_chain_instantiation(tmp_path):
    """PK_CHAIN_FORCE_RECOMPUTE=1 takes the post-wait recompute for every instance: NJ 2..7 x
    NFT 0 / 1 / 2 (odd NJ: scalar q loads), a targets row whose stride is not a multiple of 4
    (scalar row copy), solve and a 3-step rollout with q_out; all bitwise equal to the default."""
    for name in RECOMPUTE:
        recompute_dispatch(name)
    assert RECOMPUTE["nj6-nft1-posture-rows"]().problem()[0].target_stride % 4 != 0
    forced = _run_dump(tmp_path, "PK_CHAIN_FORCE_RECOMPUTE", 1, dump="dump_recompute_outputs")
    default = tmp_path / "default.npz"
    dump_recompute_outputs(default)
    default = dict(np.load(default))
    assert set(forced) == set(default)
    for key in sorted(default):
        np.testing.assert_array_equal(forced[key], default[key], err_msg=key)
    assert not np.isnan(default["nj7-nft2/q_out"]).any()

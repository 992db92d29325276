"""GPU suite (`-m gpu`): gradients of converged solutions with respect to the targets,
``ik_generic_solution_vjp_kernel`` through ``BatchedIK.converge_vjp`` and the autograd path of
``converge`` / ``converge_multistart``.

* The kernel against the host build of the same body at each size class of the general path
  (<8, 8> UR5, <30, 36> G1, <58, 64> a 40-joint tree): statuses bitwise, gradients to fp32
  rounding; and against the fp64 oracle on a slice (tolerance of test_hostsim_converge_grad).
* End to end on UR5 at B = 65536 with the task set of examples/arm_ur5_reach_batched.py:
  loss.backward() through converge against the oracle's gradient at the returned q.
* The directional derivative against central differences of GPU converge itself.
* The multi-start winner, and a CUDA-graph capture of converge_vjp."""

import numpy as np
import pytest
import torch

from oracle import ik as oik
from oracle import implicit_grad as ig
from oracle import kinematics as okin
from oracle import lie
from pink_b200 import BatchedIK
from tests import helpers
from tests.hostsim import HostSim
from tests.hostsim_vjp import HostVjp
from tests.test_hostsim_converge_grad import FAILED, grad_rtol, oracle_rows

pytestmark = pytest.mark.gpu



def cond_n(sc, q):
    """cond(N) of every instance over all coordinates: a bound on cond(N_FF) (a principal
    submatrix of a positive definite matrix is no worse conditioned)."""
    out = np.zeros(q.shape[0])
    for i in range(q.shape[0]):
        tasks = [oik._slice_task(t, i) for t in sc.oracle_tasks]
        qi = q[i].astype(np.float64)
        out[i] = np.linalg.cond(ig.normal_matrix(sc.table, qi, okin.forward_kinematics(sc.table, qi), tasks))
    return out


def _scenario(case):
    if case == "ur5":
        return helpers.ur5_scenario(512, posture_cost=1e-3), 1
    if case == "g1":
        sc = helpers.humanoid_scenario("g1_description", 512, with_com=True, with_relative=True)
        return sc, (1 << len(sc.tasks)) - 1 - (1 << 5)
    sc = helpers.tree_scenario(40, 256)
    return sc, (1 << len(sc.tasks)) - 1 - (1 << 3)


@pytest.mark.parametrize("case,size_class", [("ur5", (8, 8)), ("g1", (30, 36)), ("tree40", (58, 64))])
def test_kernel_against_host_build_and_oracle(case, size_class):
    sc, mask = _scenario(case)
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    q, _, _, _ = hs.converge(prob, sc.q32, targets, mask, 1e-4, 40)
    hs.solve_ik(prob, q[:1], targets[:1], path=1)
    assert hs.selection.generic == size_class
    gq = np.random.default_rng(0).normal(size=q.shape).astype(np.float32)
    gt_h, st_h = HostVjp(sc.model).converge_vjp(prob, q, targets, gq)
    ik = BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, safety_break=sc.safety_break,
                   batch_size=sc.B)
    assert ik.target_stride == targets.shape[1]
    dev = lambda a: torch.as_tensor(a, device="cuda").contiguous()  # noqa: E731
    gt, st = ik.converge_vjp(dev(q), dev(targets), dev(gq))
    gt, st = gt.cpu().numpy(), st.cpu().numpy()
    assert np.array_equal(st, st_h)
    # the device build contracts into FMAs where the host build rounds twice: the same binned
    # tolerance as against the oracle
    cond = cond_n(sc, q)
    for i in range(sc.B):
        tol = grad_rtol(cond[i]) * np.abs(gt_h[i]).max() + 1e-6
        assert np.abs(gt[i] - gt_h[i]).max() <= tol, (i, cond[i], np.abs(gt[i] - gt_h[i]).max(), tol)
    n = 8
    ref, ref_st, cond = oracle_rows(sc, prob, q[:n], gq[:n], n)
    assert np.array_equal(st[:n], ref_st)
    for i in range(n):
        tol = grad_rtol(cond[i]) * np.abs(ref[i]).max() + 1e-6
        assert np.abs(gt[i] - ref[i]).max() <= tol, (i, cond[i])


def _ur5_example(B, seed=0):
    from examples import arm_ur5_reach_batched as ex

    return ex.setup(B, device="cuda", seed=seed)


def test_end_to_end_ur5_65536_backward_against_oracle():
    ik, task, q0, targets = _ur5_example(65536)
    tg = targets.clone().requires_grad_(True)
    res = ik.converge(q0, tg, [task], 1e-5, 200)
    assert float(res.converged.float().mean()) > 0.95
    W = torch.randn(res.q.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    (res.q * W).sum().backward()
    g = tg.grad.cpu().numpy()
    ok = (res.converged & ((res.status & FAILED) == 0)).cpu().numpy()
    assert not g[~ok].any()
    table = ik.model.table()
    f = table.frame_names.index("tool0")
    q = res.q.detach().cpu().numpy().astype(np.float64)
    T = targets.cpu().numpy().reshape(-1, 3, 4).astype(np.float64)
    Wn = W.cpu().numpy().astype(np.float64)
    idx = np.nonzero(ok)[0][:64]
    for i in idx:
        task_i = {"type": "frame", "frame": f, "cost": np.ones(6), "gain": 1.0, "lm_damping": 0.0,
                  "target": (T[i, :, :3], T[i, :, 3])}
        (ref,), st = ig.solution_vjp(table, q[i], [task_i], 1e-2, Wn[i], damping=1e-8)
        N = ig.normal_matrix(table, q[i], okin.forward_kinematics(table, q[i]), [task_i])
        tol = grad_rtol(np.linalg.cond(N)) * np.abs(ref).max() + 1e-6
        assert st == 0 and np.abs(g[i] - ref).max() <= tol, (i, np.abs(g[i] - ref).max(), tol)


def test_directional_derivative_against_finite_differences_of_converge():
    """256 instances of the exactly determined UR5 problem (one full-pose frame task, zero residual
    at the fixed point), away from singular configurations.  Each converge stops within tol of
    the fixed point, |dq| <= tol / sigma_min(J), so the central difference with step h carries
    up to tol / (sigma_min h) |g| of stopping jitter, plus the fp32 floor of the step."""
    B, h, tol = 256, 1e-3, 1e-6
    ik, task, q0, targets = _ur5_example(B, seed=7)
    res = ik.converge(q0, targets, [task], tol, 400)
    q_star = res.q.clone()
    rng = np.random.default_rng(2)
    d = rng.normal(size=(B, 6))
    g = torch.randn(q_star.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    T = targets.cpu().numpy().reshape(-1, 3, 4).astype(np.float64)

    def moved(s):
        Rd, pd = lie.exp6(s * d)
        R = T[:, :, :3] @ Rd
        p = np.einsum("bij,bj->bi", T[:, :, :3], pd) + T[:, :, 3]
        return torch.as_tensor(np.concatenate([R, p[:, :, None]], axis=2).reshape(B, 12), dtype=torch.float32,
                               device="cuda").contiguous()

    rp = ik.converge(q_star, moved(h), [task], tol, 400)
    rm = ik.converge(q_star, moved(-h), [task], tol, 400)
    fd = ((rp.q - rm.q) * g).sum(1).cpu().numpy().astype(np.float64) / (2 * h)
    gt, st = ik.converge_vjp(q_star, targets, g.contiguous())
    dT = np.concatenate([T[:, :, :3] @ lie.hat(d[:, 3:]), np.einsum("bij,bj->bi", T[:, :, :3], d[:, :3])[:, :, None]],
                        axis=2).reshape(B, 12)
    pred = (gt.cpu().numpy().astype(np.float64) * dT).sum(1)
    table = ik.model.table()
    f = table.frame_names.index("tool0")
    qs = q_star.cpu().numpy().astype(np.float64)
    fk = okin.forward_kinematics(table, qs)
    sv = np.linalg.svd(okin.frame_jacobian_local(table, fk, f), compute_uv=False)
    ok = ((res.converged & rp.converged & rm.converged & (st == 0)).cpu().numpy()) & (sv[:, 0] / sv[:, -1] < 100)
    assert ok.sum() > B // 2
    gn = torch.linalg.vector_norm(g, dim=1).cpu().numpy()
    bound = 3 * tol / (sv[:, -1] * h) * gn + 1e-2 * np.abs(pred) + 1e-3 * gn
    assert (np.abs(pred - fd) <= bound)[ok].all(), np.max((np.abs(pred - fd) / bound)[ok])


def test_multistart_winner_gradient_equals_converge_vjp():
    ik, task, q0, targets = _ur5_example(4096, seed=4)
    seeds = ik.sample_seeds(q0, 4, generator=torch.Generator(device="cuda").manual_seed(5))
    tg = targets.clone().requires_grad_(True)
    res = ik.converge_multistart(seeds, tg, [task], 1e-5, 100)
    W = torch.randn(res.q.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(6))
    (res.q * W).sum().backward()
    gt, _ = ik.converge_vjp(res.q.detach().contiguous(), targets, W)
    ok = res.converged & ((res.status & FAILED) == 0)
    assert bool(ok.any())
    assert torch.equal(tg.grad[ok], gt[ok]) and not tg.grad[~ok].any()


def test_converge_vjp_in_a_cuda_graph_matches_eager():
    ik, task, q0, targets = _ur5_example(8192, seed=8)
    q_star = ik.converge(q0, targets, [task], 1e-5, 200).q.clone()
    gq = torch.randn(q_star.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(9))
    gt_e, st_e = ik.converge_vjp(q_star, targets, gq)
    gt = torch.full_like(gt_e, float("nan"))
    st = torch.full_like(st_e, -1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ik.converge_vjp(q_star, targets, gq, gt, st)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    gt.fill_(float("nan"))
    st.fill_(-1)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ik.converge_vjp(q_star, targets, gq, gt, st)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gt, gt_e) and torch.equal(st, st_e)

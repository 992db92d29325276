"""GPU suite (`-m gpu`): goal-set solve to a tolerance, ``BatchedIK.converge_goalset`` /
``pk_converge_goalset_prepared``, on every path (chain kernel, tree kernel, general path).

* Against the host build of the same bodies (``HostGoalset.converge_goalset``) on the paths of
  test_hostsim_goalset.py: ``goal``, ``seed``, ``steps`` and ``status`` equal, ``error`` within
  1e-3 relative and ``q`` within 1e-3 (1e-2 on the humanoid cases, which run far from their
  goals; the two builds round differently in every step of up to ``max_steps``).  An instance
  whose decision sits on a rounding edge may stop or pick differently; those are counted,
  printed and bounded at 2 %.
* G = 1 bitwise against ``converge_multistart``; the S = 1 superset of ``converge`` toward each
  goal at B = 8192; graph capture equal to eager; API errors.
* The autograd path against central differences of GPU ``converge_goalset`` itself, on the
  instances whose winning goal does not change under the perturbation; the example."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import kinematics as okin
from oracle import lie
from pink_b200 import _cabi
from tests import extras, helpers
from tests.test_gpu_converge import FAILED, _ik, _inputs, launches, pose_tasks
from tests.test_gpu_converge_grad import _ur5_example
from tests.test_hostsim_goalset import rolled_goals, stop_mask, ur5_mixed

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeds(ik, q0, S, seed=0):
    return ik.sample_seeds(q0, S, generator=torch.Generator(device="cuda").manual_seed(seed))


def check_against_host(sc, tasks_of, G, S, tol, max_steps, path=0, goals=None, label="", drift=1e-3):
    """converge_goalset on the GPU against HostGoalset.converge_goalset on the same inputs."""
    from tests.hostsim_goalset import HostGoalset

    prob, targets, _ = sc.problem()
    goals = rolled_goals(targets, G) if goals is None else goals
    ik = _ik(sc)
    q0, _ = _inputs(sc)
    qs = seeds(ik, q0, S)
    tasks = tasks_of(ik)
    mask = sum(1 << next(k for k, t0 in enumerate(ik.tasks) if t0 is t) for t in tasks)
    n0 = launches()
    res = ik.converge_goalset(qs, torch.as_tensor(goals, device="cuda"), tasks, tol, max_steps)
    assert launches() - n0 == 1
    q_h, e_h, g_h, s_h, n_h, st_h = HostGoalset(sc.model).converge_goalset(prob, qs.cpu().numpy(), goals, mask,
                                                                            tol, max_steps, path=path)
    q, e, g, s, n, st = (x.cpu().numpy() for x in (res.q, res.error, res.goal, res.seed, res.steps, res.status))
    same = (g == g_h) & (s == s_h) & (n == n_h) & (st == st_h)
    # a decision on a rounding edge: the winner's error within 1e-3 of tol, or of a tolerance
    # that two members could tie at
    edge = (np.abs(e_h - tol) <= 1e-3 * tol) | (np.abs(e - e_h) > 1e-3 * np.abs(e_h))
    B = q.shape[0]
    off = ~same
    print(f"[goalset {label}] B={B} G={G} S={S} converged={float((e <= tol).mean()):.4f} "
          f"goal>0={int((g > 0).sum())} differ={int(off.sum())} on_edge={int((off & edge).sum())}")
    assert off.sum() <= max(1, B // 50), (label, np.nonzero(off)[0][:8])
    fin = np.isfinite(e_h) & same
    assert (np.isfinite(e) == np.isfinite(e_h))[same].all()
    # the two builds round differently in every step, and unconverged members run up to max_steps
    np.testing.assert_allclose(e[fin], e_h[fin], rtol=drift, atol=2e-6, err_msg=label)
    np.testing.assert_allclose(q[fin], q_h[fin], rtol=0, atol=drift, err_msg=label)
    return res


# ---- against the host build ------------------------------------------------------------------

@pytest.mark.parametrize("G,S", [(8, 1), (4, 2), (2, 4)])
def test_chain_ur5_mixed_goals(G, S):
    sc, goals = ur5_mixed(256)
    res = check_against_host(sc, lambda ik: [sc.tasks[0]], G, S, 1e-4, 30, goals=goals[:, :G].copy(),
                             label=f"ur5 G={G} S={S}")
    solved = res.converged
    assert bool(solved.any()) and bool((res.goal[solved] % 2 == 0).all())


@pytest.mark.parametrize("nft", [0, 1, 2])
@pytest.mark.parametrize("nj", [2, 3, 4, 5, 6, 7])
def test_chain_instantiations(nj, nft):
    kw = {0: {"frame_tasks": False, "posture_per_instance": True}, 1: {}, 2: {"two_tasks": True}}[nft]
    if nj in (3, 7):
        kw["prismatic"] = (1,)
    sc = helpers.chain_scenario(nj, 128, seed=nj, **kw)
    mask = stop_mask(sc.problem()[0])
    check_against_host(sc, lambda ik: [t for k, t in enumerate(ik.tasks) if (mask >> k) & 1], 2, 2, 1e-3, 15,
                       label=f"chain{nj} nft={nft}")


@pytest.mark.parametrize("G,S", [(2, 4), (4, 2), (8, 1)])
def test_tree_g1_com(G, S):
    sc = helpers.humanoid_scenario("g1_description", 64, with_com=True)
    # goals of other instances, far from the start: ten steps of a 35-coordinate QR active set far
    # from convergence carry the two builds' rounding to a few 1e-3
    check_against_host(sc, pose_tasks, G, S, 2e-3, 10, label=f"g1 com G={G} S={S}", drift=1e-2)


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 32, True, seed=7)
    check_against_host(sc, pose_tasks, 2, 2, 1e-3, 6, label="tree40", drift=1e-2)


def check_forced_general():
    for name in ("ur5", "g1"):
        sc = (helpers.ur5_scenario(128, "reachable", out_of_limits=1) if name == "ur5"
              else helpers.humanoid_scenario("g1_description", 32, with_com=True))
        check_against_host(sc, pose_tasks, 2, 2, 1e-3, 10, path=1, label=f"{name} forced general")


def test_general_path_forced_ur5_g1():
    code = "from tests.test_gpu_goalset import check_forced_general as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, PK_FORCE_GENERIC="1"), check=True,
                   timeout=900)


# ---- the exact consequences ------------------------------------------------------------------

def _case(which):
    if which == "chain":
        sc = helpers.ur5_scenario(2048, "reachable", out_of_limits=3)
    elif which == "tree":
        sc = helpers.humanoid_scenario("g1_description", 128, with_com=True)
    else:
        sc = extras.tree_extras(40, 67, True, seed=7)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    return ik, q0, targets, pose_tasks(ik)


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_one_goal_equals_multistart(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 4)
    ref = ik.converge_multistart(qs, targets, tasks, 1e-3, 20)
    res = ik.converge_goalset(qs, targets[:, None], tasks, 1e-3, 20)
    torch.cuda.synchronize()
    assert (res.goal == 0).all()
    for name in ("q", "error", "seed", "steps", "status"):
        assert torch.equal(getattr(res, name), getattr(ref, name)), name


def test_one_seed_superset_of_converge_toward_each_goal_8192():
    B, G = 8192, 4
    sc, goals = ur5_mixed(B)
    ik = _ik(sc)
    q0, _ = _inputs(sc)
    goals = torch.as_tensor(goals[:, :G].copy(), device="cuda")
    task = sc.tasks[0]
    per_goal = [ik.converge(q0, goals[:, g].contiguous(), [task], 1e-4, 40) for g in range(G)]
    res = ik.converge_goalset(q0[:, None].contiguous(), goals, [task], 1e-4, 40)
    torch.cuda.synchronize()
    solved = torch.stack([r.converged for r in per_goal], dim=1)
    first = torch.where(solved, torch.stack([r.steps for r in per_goal], dim=1), 41).min(dim=1).values
    some = solved.any(dim=1)
    assert bool(some.any()) and bool((res.seed == 0).all())
    assert bool(res.converged[some].all())
    assert torch.equal(res.steps[some], first[some])
    assert bool(solved[some, res.goal[some].long()].all())
    print(f"[goalset superset] solved by converge toward some goal {some.float().mean().item():.4f}, "
          f"goal set {res.converged.float().mean().item():.4f}")


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_graph_capture_equals_eager(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 2)
    goals = torch.as_tensor(rolled_goals(targets.cpu().numpy(), 4), device="cuda")
    eager = ik.converge_goalset(qs, goals, tasks, 1e-3, 20)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ik.converge_goalset(qs, goals, tasks, 1e-3, 20)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    B = q0.shape[0]
    outs = dict(q_out=torch.empty_like(q0), error=torch.empty(B, device="cuda"))
    outs.update({k: torch.empty(B, device="cuda", dtype=torch.int32) for k in ("goal", "seed", "steps", "status")})
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ik.converge_goalset(qs, goals, tasks, 1e-3, 20, **outs)
    for x in outs.values():
        x.zero_()
    n0 = launches()
    g.replay()
    torch.cuda.synchronize()
    assert launches() == n0
    for x, y in zip(outs.values(), eager[:6]):
        assert torch.equal(x, y)


def test_api_errors():
    sc = helpers.ur5_scenario(64, "reachable")
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    frame = sc.tasks[0]
    qs = seeds(ik, q0, 4)
    goals = torch.as_tensor(rolled_goals(targets.cpu().numpy(), 2), device="cuda")
    for kw in ({"tasks": []}, {"tol": -1.0}, {"max_steps": -1}, {"q_seeds": q0}, {"q_seeds": qs.double()},
               {"goals": goals.double()}, {"goals": goals[:-1]}, {"goals": goals[:, :, :6]}, {"goals": targets},
               {"goals": None}, {"goals": goals.transpose(0, 1).contiguous().transpose(0, 1)},
               {"goals": torch.cat([goals, goals[:, :1]], dim=1)},
               {"goals": goals.repeat(1, 8, 1), "q_seeds": q0[:, None].repeat(1, 8, 1)}):
        args = dict(q_seeds=qs, goals=goals, tasks=[frame], tol=1e-3, max_steps=5)
        args.update(kw)
        with pytest.raises(ValueError):
            ik.converge_goalset(**args)
    lib = _cabi.load()
    eng = ik.engine
    q_out = torch.empty_like(q0)
    stream = torch.cuda.current_stream().cuda_stream

    def call(G=2, S=4):  # 8 instances: at most 8 x 32 of the 64 x 4 seed rows, 8 x 32 goal rows are read
        big = goals.repeat(1, 16, 1)
        return lib.pk_converge_goalset_prepared(eng.handle, ik._handle, qs.data_ptr(), S, big.data_ptr(), G, 1, 1e-3, 5,
                                                q_out.data_ptr(), None, None, None, None, None, 8, stream)

    assert call() == 0 and call(G=1) == 0 and call(G=8) == 0 and call(G=32, S=1) == 0
    for kw in ({"G": 0}, {"G": 3}, {"G": 16}, {"G": 64, "S": 1}):
        assert call(**kw) != 0, kw
    torch.cuda.synchronize()
    # the tree kernel: at most 8 members
    sc = helpers.humanoid_scenario("g1_description", 8, with_com=True)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    goals = torch.as_tensor(rolled_goals(targets.cpu().numpy(), 4), device="cuda")
    with pytest.raises(ValueError, match="at most 8"):
        ik.converge_goalset(q0[:, None].repeat(1, 4, 1).contiguous(), goals, pose_tasks(ik), 1e-3, 5)


# ---- gradients -------------------------------------------------------------------------------

def test_directional_derivative_against_finite_differences_of_goalset():
    """The exactly determined UR5 problem of test_gpu_converge_grad.py with two goals per
    instance, an out-of-reach pose first and the reachable target second.  Both rows move along
    the same twist; the autograd path's derivative (through the winner's row only) must match
    central differences of converge_goalset where the winning goal is the same at +h and -h."""
    B, h, tol = 256, 1e-3, 1e-6
    ik, task, q0, targets = _ur5_example(B, seed=7)
    far = targets.reshape(B, 3, 4).clone()
    far[:, 2, 3] += 3.0  # 3 m above the target: out of reach
    goals = torch.stack([far.reshape(B, 12), targets], dim=1).contiguous()
    gl = goals.clone().requires_grad_(True)
    res = ik.converge_goalset(q0[:, None].contiguous(), gl, [task], tol, 400)
    q_star = res.q.detach().clone()
    W = torch.randn(q_star.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    (res.q * W).sum().backward()
    assert not gl.grad[:, 0].any()
    rng = np.random.default_rng(2)
    d = rng.normal(size=(B, 6))
    T = goals.detach().cpu().numpy().reshape(B, 2, 3, 4).astype(np.float64)

    def moved(s):
        Rd, pd = lie.exp6(s * d)
        R = T[..., :3] @ Rd[:, None]
        p = np.einsum("bgij,bj->bgi", T[..., :3], pd) + T[..., 3]
        return torch.as_tensor(np.concatenate([R, p[..., None]], axis=3).reshape(B, 2, 12), dtype=torch.float32,
                               device="cuda").contiguous()

    rp = ik.converge_goalset(q_star[:, None].contiguous(), moved(h), [task], tol, 400)
    rm = ik.converge_goalset(q_star[:, None].contiguous(), moved(-h), [task], tol, 400)
    fd = ((rp.q - rm.q) * W).sum(1).cpu().numpy().astype(np.float64) / (2 * h)
    dT = np.concatenate([T[..., :3] @ lie.hat(d[:, 3:])[:, None],
                         np.einsum("bgij,bj->bgi", T[..., :3], d[:, :3])[..., None]], axis=3).reshape(B, 2, 12)
    pred = (gl.grad.cpu().numpy().astype(np.float64) * dT).sum(axis=(1, 2))
    table = ik.model.table()
    f = table.frame_names.index("tool0")
    qn = q_star.cpu().numpy().astype(np.float64)
    sv = np.linalg.svd(okin.frame_jacobian_local(table, okin.forward_kinematics(table, qn), f), compute_uv=False)
    stable = (rp.goal == res.goal) & (rm.goal == res.goal) & (res.goal == 1)
    ok = ((res.converged & rp.converged & rm.converged & stable & ((res.status & FAILED) == 0)).cpu().numpy()
          & (sv[:, 0] / sv[:, -1] < 100))
    assert ok.sum() > B // 2
    gn = torch.linalg.vector_norm(W, dim=1).cpu().numpy()
    bound = 3 * tol / (sv[:, -1] * h) * gn + 1e-2 * np.abs(pred) + 1e-3 * gn
    assert (np.abs(pred - fd) <= bound)[ok].all(), np.max((np.abs(pred - fd) / bound)[ok])


def test_winner_gradient_equals_converge_vjp_of_its_row():
    ik, task, q0, targets = _ur5_example(4096, seed=4)
    goals = torch.stack([targets.roll(1, 0), targets, targets.roll(2, 0), targets.roll(3, 0)], dim=1).contiguous()
    gl = goals.clone().requires_grad_(True)
    res = ik.converge_goalset(seeds(ik, q0, 2), gl, [task], 1e-5, 100)
    W = torch.randn(res.q.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(6))
    (res.q * W).sum().backward()
    rows = torch.arange(4096, device="cuda")
    gt, _ = ik.converge_vjp(res.q.detach().contiguous(), goals[rows, res.goal.long()].contiguous(), W)
    ok = res.converged & ((res.status & FAILED) == 0)
    assert bool(ok.any())
    assert torch.equal(gl.grad[rows, res.goal.long()][ok], gt[ok])
    others = torch.ones_like(gl.grad, dtype=torch.bool)
    others[rows, res.goal.long()] = False
    assert not gl.grad[others].any() and not gl.grad[~ok].any()


# ---- the example -----------------------------------------------------------------------------

def test_goalset_example():
    import importlib.util

    spec = importlib.util.spec_from_file_location("grasp_gs", os.path.join(ROOT, "examples",
                                                                           "arm_ur5_grasp_goalset_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    res, reachable = ex.run(batch=1024, num_seeds=4, max_steps=100, verbose=True)
    torch.cuda.synchronize()
    solved = res.converged
    assert solved.float().mean() > 0.9
    rows = torch.arange(1024, device="cuda")
    assert bool(reachable[rows, res.goal.long()][solved].all())

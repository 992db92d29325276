"""GPU suite (`-m gpu`): separate position and orientation tolerances, ``orientation_tol`` of
``BatchedIK.converge`` / ``converge_multistart`` / ``converge_goalset``
(``pk_converge_pose_tol_prepared``, ``pk_converge_goalset_pose_tol_prepared``), on every path.

* Against the host build of the same bodies (``HostPoseTol``) on the paths of
  test_hostsim_pose_tol.py: ``steps``, ``status``, ``goal`` and ``seed`` equal but for decisions
  on a rounding edge (counted, printed and bounded at 2 %), ``error`` and ``q`` within the drift
  of two builds that round differently.
* Goal sets and multi-start at several (G, S), G S = 8 on the tree; graph capture equal to eager.
* Autograd against central differences of GPU ``converge`` for a position-only UR5 task with a
  posture task and for the G1 wrists; API errors; the example."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import lie
from pink_b200 import FrameTask, PostureTask, _cabi
from tests import extras, helpers
from tests.test_gpu_converge import FAILED, _ik, _inputs, launches, pose_tasks
from tests.test_hostsim_goalset import rolled_goals, stop_mask
from tests.test_hostsim_pose_tol import all_tasks_but_posture, g1_reach, position_only_ur5

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeds(ik, q0, S, seed=0):
    return ik.sample_seeds(q0, S, generator=torch.Generator(device="cuda").manual_seed(seed))


def mask_tasks(ik, mask):
    return [t for k, t in enumerate(ik.tasks) if (mask >> k) & 1]


def compare(label, tol, host, dev, drift, err_atol=2e-6):
    """host / dev: (q, err, ints...) — the ints equal but for rounding-edge decisions."""
    q_h, e_h = host[0], host[1]
    q, e = dev[0], dev[1]
    same = np.ones(q.shape[0], dtype=bool)
    for a, b in zip(host[2:], dev[2:]):
        same &= a == b
    off = ~same
    print(f"[pose_tol {label}] B={q.shape[0]} converged={float((e <= tol).mean()):.4f} differ={int(off.sum())}")
    assert off.sum() <= max(1, q.shape[0] // 50), (label, np.nonzero(off)[0][:8])
    fin = np.isfinite(e_h) & same
    assert (np.isfinite(e) == np.isfinite(e_h))[same].all()
    np.testing.assert_allclose(e[fin], e_h[fin], rtol=drift, atol=err_atol, err_msg=label)
    np.testing.assert_allclose(q[fin], q_h[fin], rtol=0, atol=drift, err_msg=label)


def check_converge(sc, mask, tol, otol, max_steps, path=0, label="", drift=1e-3, err_atol=2e-6):
    from tests.hostsim_pose_tol import HostPoseTol

    prob, targets, _ = sc.problem()
    ik = _ik(sc)
    q0, tg = _inputs(sc)
    n0 = launches()
    res = ik.converge(q0, tg, mask_tasks(ik, mask), tol, max_steps, orientation_tol=otol)
    assert launches() - n0 == 1
    host = HostPoseTol(sc.model).converge(prob, sc.q32, targets, mask, tol, otol, max_steps, path=path)
    dev = [x.cpu().numpy() for x in (res.q, res.error, res.steps, res.status)]
    compare(label, tol, host, dev, drift, err_atol)
    return res


def check_goalset(sc, mask, G, S, tol, otol, max_steps, path=0, label="", drift=1e-3):
    from tests.hostsim_pose_tol import HostPoseTol

    prob, targets, _ = sc.problem()
    goals = rolled_goals(targets, G)
    ik = _ik(sc)
    q0, _ = _inputs(sc)
    qs = seeds(ik, q0, S)
    n0 = launches()
    res = ik.converge_goalset(qs, torch.as_tensor(goals, device="cuda"), mask_tasks(ik, mask), tol, max_steps,
                              orientation_tol=otol)
    assert launches() - n0 == 1
    q_h, e_h, g_h, s_h, n_h, st_h = HostPoseTol(sc.model).converge_goalset(prob, qs.cpu().numpy(), goals, mask, tol,
                                                                           otol, max_steps, path=path)
    dev = [x.cpu().numpy() for x in (res.q, res.error, res.goal, res.seed, res.steps, res.status)]
    compare(label, tol, (q_h, e_h, g_h, s_h, n_h, st_h), dev, drift)
    return res


# ---- against the host build ------------------------------------------------------------------

@pytest.mark.parametrize("nft", [0, 1, 2])
@pytest.mark.parametrize("nj", [2, 3, 4, 5, 6, 7])
def test_chain_instantiations(nj, nft):
    # the elbow task of two_tasks weighs no y translation: an untested row
    kw = {0: {"frame_tasks": False, "posture_per_instance": True}, 1: {}, 2: {"two_tasks": True}}[nft]
    if nj in (3, 7):
        kw["prismatic"] = (1,)
    sc = helpers.chain_scenario(nj, 256, seed=nj, **kw)
    mask = stop_mask(sc.problem()[0])
    check_converge(sc, mask, 1e-3, 1e-2, 25, label=f"chain{nj}")
    check_goalset(sc, mask, 2, 2, 1e-3, 1e-2, 15, label=f"chain{nj} G=2 S=2")


def test_chain_position_only_ur5():
    sc = position_only_ur5(2048)
    # instances that run to max_steps wander along the posture's null space: their errors agree
    # to a few 1e-5 and their q to 2e-2 between the builds
    res = check_converge(sc, 0b01, 1e-4, 1e-3, 80, label="ur5 position only", drift=2e-2, err_atol=2e-5)
    assert res.converged.float().mean() > 0.8


def test_tree_g1_every_frame_task_and_com():
    sc = g1_reach(256)
    mask = all_tasks_but_posture(sc.problem()[0])
    res = check_converge(sc, mask, 2e-3, 2e-2, 40, label="g1", drift=1e-2)
    assert res.converged.float().mean() > 0.6


def test_tree_relative_frame():
    sc = helpers.humanoid_scenario("g1_description", 64, with_com=True, with_relative=True)
    mask = all_tasks_but_posture(sc.problem()[0])
    check_converge(sc, mask, 2e-3, 2e-2, 15, label="g1 relative", drift=1e-2)


@pytest.mark.parametrize("G,S", [(1, 8), (2, 4), (4, 2), (8, 1)])
def test_tree_goalsets(G, S):
    sc = g1_reach(64)
    mask = all_tasks_but_posture(sc.problem()[0])
    check_goalset(sc, mask, G, S, 2e-3, 2e-2, 10, label=f"g1 G={G} S={S}", drift=1e-2)


@pytest.mark.parametrize("G,S", [(1, 4), (2, 2), (4, 8), (32, 1)])
def test_chain_goalsets(G, S):
    sc = position_only_ur5(256, seed=4)
    check_goalset(sc, 0b01, G, S, 1e-4, 1e-3, 40, label=f"ur5 G={G} S={S}")


def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 32, True, seed=7)
    prob = sc.problem()[0]
    mask = sum(1 << t for t in range(int(prob.ntasks))
               if int(prob.tasks[t].type) in (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_COM))
    check_converge(sc, mask, 1e-3, 1e-2, 8, label="tree40", drift=1e-2)
    check_goalset(sc, mask, 2, 2, 1e-3, 1e-2, 6, label="tree40 G=2 S=2", drift=1e-2)


def check_forced_general():
    sc = position_only_ur5(128)
    check_converge(sc, 0b01, 2e-3, 2e-2, 20, path=1, label="ur5 forced general")
    check_goalset(sc, 0b01, 2, 2, 2e-3, 2e-2, 10, path=1, label="ur5 forced general G=2 S=2")
    sc = g1_reach(32)
    mask = all_tasks_but_posture(sc.problem()[0])
    check_converge(sc, mask, 2e-3, 2e-2, 20, path=1, label="g1 forced general", drift=1e-2)


def test_general_path_forced_ur5_g1():
    code = "from tests.test_gpu_pose_tol import check_forced_general as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, PK_FORCE_GENERIC="1"), check=True,
                   timeout=900)


# ---- equalities, superset, graphs -----------------------------------------------------------

def _case(which):
    if which == "chain":
        sc = position_only_ur5(2048)
    elif which == "tree":
        sc = g1_reach(128)
    else:
        sc = extras.tree_extras(40, 67, True, seed=7)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    return ik, q0, targets, pose_tasks(ik)


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_one_goal_equals_multistart_and_one_seed_equals_converge(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 4)
    ms = ik.converge_multistart(qs, targets, tasks, 2e-3, 20, orientation_tol=2e-2)
    gs = ik.converge_goalset(qs, targets[:, None], tasks, 2e-3, 20, orientation_tol=2e-2)
    one = ik.converge_multistart(q0[:, None].contiguous(), targets, tasks, 2e-3, 20, orientation_tol=2e-2)
    cv = ik.converge(q0, targets, tasks, 2e-3, 20, orientation_tol=2e-2)
    torch.cuda.synchronize()
    assert (gs.goal == 0).all() and (one.seed == 0).all()
    for name in ("q", "error", "seed", "steps", "status"):
        assert torch.equal(getattr(gs, name), getattr(ms, name)), name
    for name in ("q", "error", "steps", "status"):
        assert torch.equal(getattr(one, name), getattr(cv, name)), name


def test_superset_of_the_default_test_8192():
    sc = helpers.ur5_scenario(8192, "reachable", seed=5)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    tol = 1e-4
    old = ik.converge(q0, targets, [sc.tasks[0]], tol, 60)
    new = ik.converge(q0, targets, [sc.tasks[0]], tol, 60, orientation_tol=tol)
    ok = old.converged
    assert ok.float().mean() > 0.5
    assert bool(new.converged[ok].all()) and bool((new.steps[ok] <= old.steps[ok]).all())


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_graph_capture_equals_eager(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 2)
    goals = torch.as_tensor(rolled_goals(targets.cpu().numpy(), 4), device="cuda")
    eager_c = ik.converge(q0, targets, tasks, 2e-3, 20, orientation_tol=2e-2)
    eager_g = ik.converge_goalset(qs, goals, tasks, 2e-3, 20, orientation_tol=2e-2)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ik.converge(q0, targets, tasks, 2e-3, 20, orientation_tol=2e-2)
        ik.converge_goalset(qs, goals, tasks, 2e-3, 20, orientation_tol=2e-2)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    B = q0.shape[0]
    oc = dict(q_out=torch.empty_like(q0), error=torch.empty(B, device="cuda"))
    oc.update({k: torch.empty(B, device="cuda", dtype=torch.int32) for k in ("steps", "status")})
    og = dict(q_out=torch.empty_like(q0), error=torch.empty(B, device="cuda"))
    og.update({k: torch.empty(B, device="cuda", dtype=torch.int32) for k in ("goal", "seed", "steps", "status")})
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ik.converge(q0, targets, tasks, 2e-3, 20, orientation_tol=2e-2, **oc)
        ik.converge_goalset(qs, goals, tasks, 2e-3, 20, orientation_tol=2e-2, **og)
    for x in list(oc.values()) + list(og.values()):
        x.zero_()
    n0 = launches()
    g.replay()
    torch.cuda.synchronize()
    assert launches() == n0
    for x, y in zip(oc.values(), eager_c[:4]):
        assert torch.equal(x, y)
    for x, y in zip(og.values(), eager_g[:6]):
        assert torch.equal(x, y)


def test_api_errors():
    sc = position_only_ur5(64)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    frame, posture = sc.tasks
    qs = seeds(ik, q0, 2)
    for tol, otol in ((0.0, 1e-2), (float("inf"), 1e-2), (1e-3, 0.0), (1e-3, -1.0), (1e-3, float("nan"))):
        with pytest.raises(ValueError):
            ik.converge(q0, targets, [frame], tol, 5, orientation_tol=otol)
        with pytest.raises(ValueError):
            ik.converge_multistart(qs, targets, [frame], tol, 5, orientation_tol=otol)
        with pytest.raises(ValueError):
            ik.converge_goalset(qs, targets[:, None], [frame], tol, 5, orientation_tol=otol)
    # a rotation-only task has nothing to test at orientation_tol = inf; so has a zero-cost posture
    ft = FrameTask("tool0", position_cost=0.0, orientation_cost=1.0)
    ft.set_target(sc.tasks[0].transform_target_to_world)
    pt = PostureTask(cost=0.0)
    pt.set_target(np.zeros(6))
    ik2 = __import__("pink_b200").BatchedIK(sc.model, [ft, pt], sc.dt, damping=sc.damping, batch_size=64)
    ik2.converge(q0, targets, [ft], 1e-3, 1, orientation_tol=1e-2)
    with pytest.raises(ValueError, match="weighs no component"):
        ik2.converge(q0, targets, [ft], 1e-3, 1, orientation_tol=float("inf"))
    with pytest.raises(ValueError, match="weighs no component"):
        ik2.converge(q0, targets, [pt], 1e-3, 1, orientation_tol=1e-2)
    # through C: the same checks in the library
    lib = _cabi.load()
    eng = ik.engine
    q_out = torch.empty_like(q0)
    stream = torch.cuda.current_stream().cuda_stream

    def call(tol, otol):
        return lib.pk_converge_pose_tol_prepared(eng.handle, ik._handle, q0.data_ptr(), targets.data_ptr(), 1, tol,
                                                 otol, 5, q_out.data_ptr(), None, None, None, 64, stream)

    assert call(1e-3, 1e-2) == 0 and call(1e-3, float("inf")) == 0
    for tol, otol in ((0.0, 1e-2), (1e-3, 0.0), (1e-3, float("nan")), (float("inf"), 1e-2)):
        assert call(tol, otol) != 0
        assert b"tol" in lib.pk_last_error()
    torch.cuda.synchronize()
    # gradients need a finite orientation_tol
    with pytest.raises(ValueError, match="finite orientation_tol"):
        ik.converge(q0, targets.clone().requires_grad_(True), [frame], 1e-3, 5, orientation_tol=float("inf"))


# ---- gradients -------------------------------------------------------------------------------

def _directional_fd(ik, tasks, q0, targets, frame_slices, tol, otol, max_steps, h=1e-3, seed=2):
    """(pred, fd, ok) of the autograd derivative of sum(q* W) along a twist of each frame target
    in frame_slices, against central differences of GPU converge started at q*."""
    B = q0.shape[0]
    tg = targets.clone().requires_grad_(True)
    res = ik.converge(q0, tg, tasks, tol, max_steps, orientation_tol=otol)
    q_star = res.q.detach().clone()
    W = torch.randn(q_star.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
    (res.q * W).sum().backward()
    rng = np.random.default_rng(seed)
    T0 = targets.cpu().numpy().astype(np.float64)
    d = {off: rng.normal(size=(B, 6)) for off in frame_slices}

    def moved(s):
        T = T0.copy()
        for off in frame_slices:
            Tf = T0[:, off:off + 12].reshape(B, 3, 4)
            Rd, pd = lie.exp6(s * d[off])
            T[:, off:off + 12] = np.concatenate([Tf[..., :3] @ Rd, (np.einsum("bij,bj->bi", Tf[..., :3], pd)
                                                                   + Tf[..., 3])[..., None]], axis=2).reshape(B, 12)
        return torch.as_tensor(T, dtype=torch.float32, device="cuda").contiguous()

    rp = ik.converge(q_star, moved(h), tasks, tol, max_steps, orientation_tol=otol)
    rm = ik.converge(q_star, moved(-h), tasks, tol, max_steps, orientation_tol=otol)
    fd = ((rp.q - rm.q) * W).sum(1).cpu().numpy().astype(np.float64) / (2 * h)
    pred = np.zeros(B)
    g = tg.grad.cpu().numpy().astype(np.float64)
    for off in frame_slices:
        Tf = T0[:, off:off + 12].reshape(B, 3, 4)
        dT = np.concatenate([Tf[..., :3] @ lie.hat(d[off][:, 3:]),
                             np.einsum("bij,bj->bi", Tf[..., :3], d[off][:, :3])[..., None]], axis=2).reshape(B, 12)
        pred += (g[:, off:off + 12] * dT).sum(1)
    ok = (res.converged & rp.converged & rm.converged & ((res.status | rp.status | rm.status) & FAILED == 0))
    gn = torch.linalg.vector_norm(W, dim=1).cpu().numpy()
    return pred, fd, ok.cpu().numpy(), gn


def ur5_position_toward(B, posture_cost=3e-3, seed=11):
    """A position-only UR5 tool task and a posture task toward the configuration the target was
    taken at.  A posture of cost 3e-3 keeps N conditioned for fp32 and holds the position error
    of a target moved by h = 1e-3 well below 3e-6, so converge can stop far below h."""
    from pink_b200 import workloads

    robot, model, table = helpers.load("ur5_description")
    rng = np.random.default_rng(seed)
    q = workloads.sample_configurations(table, B, rng)
    qt = workloads.perturb_configurations(table, q, rng)
    ft = FrameTask("tool0", position_cost=1.0, orientation_cost=0.0, lm_damping=1.0)
    ft.set_target(torch.as_tensor(helpers.frame_targets(table, qt, "tool0")))
    pt = PostureTask(cost=posture_cost)
    pt.set_target(torch.as_tensor(qt.astype(np.float32)))
    return helpers.Scenario("ur5-position", robot, model, table, q, [ft, pt], [], 1e-2, 1e-8)


def test_autograd_position_only_ur5_against_finite_differences():
    sc = ur5_position_toward(512)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    pred, fd, ok, gn = _directional_fd(ik, [sc.tasks[0]], q0, targets, [0], 3e-6, 1e-2, 400)
    assert ok.sum() > 256
    err = np.abs(pred - fd)
    bound = 5e-2 * np.abs(pred) + 2e-2 * gn
    print(f"[pose_tol grad ur5] ok={int(ok.sum())} worst |pred - fd| / bound {np.max((err / bound)[ok]):.3f}")
    assert (err <= bound)[ok].mean() > 0.9


def test_autograd_g1_wrists_against_finite_differences():
    # the posture toward the target configuration: a fixed point where every error is zero, so the
    # loop meets a tolerance far below the wrists' motion under the finite difference
    sc = g1_reach(128, posture_at_start=False, posture_cost=1e-2)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    prob = sc.problem()[0]
    stop = pose_tasks(ik)
    wrists = [int(prob.tasks[k].target_offset) for k in (3, 4)]
    pred, fd, ok, gn = _directional_fd(ik, stop, q0, targets, wrists, 1e-5, 1e-4, 400)
    assert ok.sum() > 32
    err = np.abs(pred - fd)
    bound = 5e-2 * np.abs(pred) + 2e-2 * gn
    print(f"[pose_tol grad g1] ok={int(ok.sum())} worst |pred - fd| / bound {np.max((err / bound)[ok]):.3f}")
    # the posture task alone holds 11 of the 35 coordinates, and the restarts from q* also move
    # along them, which the first-order derivative does not see: most instances agree
    assert (err <= bound)[ok].mean() > 0.6 and np.median((err / bound)[ok]) < 1.0


# ---- the example -----------------------------------------------------------------------------

def test_g1_reach_example():
    import importlib.util

    spec = importlib.util.spec_from_file_location("g1_reach", os.path.join(ROOT, "examples",
                                                                           "humanoid_g1_reach_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    res = ex.run(batch=2048, max_steps=200, verbose=True)
    torch.cuda.synchronize()
    assert res.converged.float().mean() > 0.5
    assert bool((res.steps[res.converged] < 200).all())
    # the default test cannot stop this set: its unweighed components never reach zero
    ik, stop, q0, targets = ex.setup(256)
    old = ik.converge(q0, targets, stop, ex.TOL, 50)
    assert not bool(old.converged.any())

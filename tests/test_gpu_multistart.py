"""GPU suite (`-m gpu`): multi-start solve to a tolerance, ``BatchedIK.converge_multistart`` /
``pk_converge_multistart_prepared``, on every path (chain kernel, tree kernel, general path).

The reference is one trajectory rollout of ``max_steps`` steps on the tiled ``[B*S, nq]`` seeds
with all records.  For every target, the winner's ``q`` and ``status`` must be bitwise the
rollout's after ``steps`` steps; its error must be the task-terms error there; at round
``steps`` no seed may have a smaller error; and no seed may have had an error <= tol in an
earlier round.  Errors within 1e-3 relative of ``tol`` (or of the winner's error) are left out
of the last two checks (the kernel's forward kinematics and the task-terms export round
differently); the number left out is printed.  Environment switches are read once per process,
so those cases run in a subprocess."""

import os
import subprocess
import sys

import pytest
import torch

import pink_b200
from pink_b200 import _cabi
from tests import extras, helpers
from tests.test_gpu_converge import FAILED, _ik, _inputs, launches, pose_tasks, task_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeds(ik, q0, S, seed=0):
    return ik.sample_seeds(q0, S, generator=torch.Generator(device="cuda").manual_seed(seed))


def check_against_trajectory(ik, qs, targets, tasks, tol, max_steps, label=""):
    """converge_multistart against one recorded trajectory rollout of the tiled seeds."""
    B, S, nq = qs.shape
    n0 = launches()
    res = ik.converge_multistart(qs, targets, tasks, tol, max_steps)
    assert launches() - n0 == 1
    flat = qs.reshape(B * S, nq)
    t_flat = None if targets is None else targets.repeat_interleave(S, dim=0).contiguous()
    tr = ik.rollout_trajectory(flat, t_flat, max_steps, record=True)
    torch.cuda.synchronize()
    steps = res.steps.long()
    seed = res.seed.long()
    assert (steps >= 0).all() and (steps <= max_steps).all() and (seed >= 0).all() and (seed < S).all()
    rows = torch.arange(B, device="cuda") * S + seed
    q_all = torch.cat([flat[None], tr.q_traj])  # q_all[s] = q after s steps
    st_all = torch.cat([torch.zeros_like(tr.status_traj[:1]), tr.status_traj])
    assert torch.equal(res.q, q_all[steps, rows]), label
    assert torch.equal(res.status, st_all[steps, rows]), label
    assert torch.equal(res.converged, res.error <= tol)
    e_tt = task_error(ik, tasks, res.q, targets)
    fin = torch.isfinite(e_tt)
    assert torch.equal(torch.isfinite(res.error), fin)
    torch.testing.assert_close(res.error[fin], e_tt[fin], rtol=1e-4, atol=2e-6)
    # errors of every seed at every round up to the last any group ran
    grid = torch.arange(S, device="cuda")
    skipped = 0
    e_steps = torch.full((B, S), float("nan"), device="cuda")
    for s in range(int(steps.max()) + 1):
        e = task_error(ik, tasks, q_all[s], t_flat).reshape(B, S)
        at = steps == s
        e_steps[at] = e[at]
        before = (steps > s)[:, None].expand(B, S)
        near = (e - tol).abs() <= 1e-3 * tol
        skipped += int((before & near).sum())
        bad = before & ~near & (e <= tol)
        assert not bad.any(), (label, s, torch.nonzero(bad)[:5].tolist())
    # at the stopping round no seed is better than the winner (NaN as +inf)
    key = torch.where(torch.isnan(e_steps), torch.full_like(e_steps, float("inf")), e_steps)
    kw = key[torch.arange(B, device="cuda"), seed][:, None]
    near = (key - kw).abs() <= 1e-3 * kw.abs()
    skipped_w = int((near & (grid[None] != seed[:, None])).sum())
    bad = (key < kw) & ~near
    assert not bad.any(), (label, torch.nonzero(bad)[:5].tolist())
    conv = res.converged.float().mean().item()
    print(f"[multistart {label}] B={B} S={S} converged={conv:.4f} seed>0={int((seed > 0).sum())} "
          f"max_steps_hit={int((steps == max_steps).sum())} skipped_near_tol={skipped} skipped_near_winner={skipped_w}")
    return res


def _ur5(B, kind="reachable", out_of_limits=0):
    sc = helpers.ur5_scenario(B, kind, out_of_limits=out_of_limits)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    return sc, ik, q0, targets


# ---- chains ----------------------------------------------------------------------------------

@pytest.mark.parametrize("S", [2, 8, 32])
def test_chain_ur5(S):
    sc, ik, q0, targets = _ur5(2048 // S * 2, out_of_limits=3)
    check_against_trajectory(ik, seeds(ik, q0, S), targets, [sc.tasks[0]], 1e-4, 40, f"ur5 reachable S={S}")
    sc, ik, q0, targets = _ur5(256, "unreachable")
    res = check_against_trajectory(ik, seeds(ik, q0, S), targets, [sc.tasks[0]], 1e-4, 10, f"ur5 unreachable S={S}")
    assert (res.seed > 0).any()


@pytest.mark.parametrize("nj,kw", [
    (2, {}), (3, {"prismatic": (1,)}), (4, {"two_tasks": True}), (5, {"shared_target": True}), (6, {}),
    (7, {"two_tasks": True, "prismatic": (2,)}), (3, {"frame_tasks": False}),
])
def test_chain_instantiations(nj, kw):
    sc = helpers.chain_scenario(nj, 500 + nj, seed=nj, **kw)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    tasks = pose_tasks(ik) or ik.tasks
    check_against_trajectory(ik, seeds(ik, q0, 4), targets, tasks, 1e-3, 20, f"chain{nj} {kw}")


# ---- trees -----------------------------------------------------------------------------------

@pytest.mark.parametrize("S", [2, 4, 8])
def test_tree_g1_com(S):
    sc = helpers.humanoid_scenario("g1_description", 256 // S, with_com=True)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    check_against_trajectory(ik, seeds(ik, q0, S), targets, pose_tasks(ik), 2e-3, 15, f"g1 com S={S}")


def test_tree_g1_extras_barriers():
    sc = extras.g1_extras(64)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    # seeds near the start: the self-collision barrier needs a start it can act on
    qs = q0[:, None].repeat(1, 4, 1)
    qs[:, 1:, 7:] += 0.05 * torch.randn(qs[:, 1:, 7:].shape, device="cuda", generator=torch.Generator(
        device="cuda").manual_seed(5))
    check_against_trajectory(ik, qs.contiguous(), targets, pose_tasks(ik), 2e-3, 10, "g1 extras S=4")


# ---- general path ----------------------------------------------------------------------------

def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 67, True, seed=7)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    check_against_trajectory(ik, seeds(ik, q0, 4), targets, pose_tasks(ik), 1e-3, 8, "tree40 S=4")


def check_forced_general():
    for name in ("ur5", "g1"):
        if name == "ur5":
            sc = helpers.ur5_scenario(512, "reachable", out_of_limits=3)
        else:
            sc = helpers.humanoid_scenario("g1_description", 128, with_com=True)
        ik = _ik(sc)
        q0, targets = _inputs(sc)
        tasks = [sc.tasks[0]] if name == "ur5" else pose_tasks(ik)
        check_against_trajectory(ik, seeds(ik, q0, 4), targets, tasks, 1e-3, 15, f"{name} forced general")
        one = ik.converge_multistart(q0[:, None].contiguous(), targets, tasks, 1e-3, 15)
        ref = ik.converge(q0, targets, tasks, 1e-3, 15)
        torch.cuda.synchronize()
        for name_ in ("q", "error", "steps", "status"):
            assert torch.equal(getattr(one, name_), getattr(ref, name_)), name_


def test_general_path_forced_ur5_g1():
    _in_subprocess("check_forced_general", PK_FORCE_GENERIC="1")


# ---- the exact consequences ------------------------------------------------------------------

def _case(which):
    if which == "chain":
        sc, ik, q0, targets = _ur5(2048, out_of_limits=3)
        return ik, q0, targets, [sc.tasks[0]]
    sc = (helpers.humanoid_scenario("g1_description", 128, with_com=True) if which == "tree"
          else extras.tree_extras(40, 67, True, seed=7))
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    return ik, q0, targets, pose_tasks(ik)


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_one_seed_equals_converge(which):
    ik, q0, targets, tasks = _case(which)
    one = ik.converge_multistart(q0[:, None].contiguous(), targets, tasks, 1e-3, 20)
    ref = ik.converge(q0, targets, tasks, 1e-3, 20)
    torch.cuda.synchronize()
    assert (one.seed == 0).all()
    for name in ("q", "error", "steps", "status"):
        assert torch.equal(getattr(one, name), getattr(ref, name)), name


@pytest.mark.parametrize("which", ["chain", "tree"])
def test_superset_of_converge(which):
    ik, q0, targets, tasks = _case(which)
    S = 8
    ref = ik.converge(q0, targets, tasks, 2e-3, 30)
    res = ik.converge_multistart(seeds(ik, q0, S), targets, tasks, 2e-3, 30)
    torch.cuda.synchronize()
    solved = ref.converged
    assert bool(res.converged[solved].all())
    assert bool((res.steps[solved] <= ref.steps[solved]).all())
    print(f"[multistart superset {which}] converge {solved.float().mean().item():.4f} "
          f"multistart {res.converged.float().mean().item():.4f}")


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_zero_steps_argmin_and_duplicates(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 4)
    qs[:, 3] = qs[:, 1]
    res = ik.converge_multistart(qs, targets, tasks, 0.0, 0)
    B = q0.shape[0]
    e = task_error(ik, tasks, qs.reshape(B * 4, -1), None if targets is None else targets.repeat_interleave(4, 0))
    e = e.reshape(B, 4)
    torch.cuda.synchronize()
    assert (res.steps == 0).all() and (res.status == 0).all() and (res.seed != 3).all()
    assert torch.equal(res.q, qs[torch.arange(B, device="cuda"), res.seed.long()])
    kw = e[torch.arange(B, device="cuda"), res.seed.long()][:, None]
    assert not ((e < kw) & ((e - kw).abs() > 1e-3 * kw)).any()


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_nan_seeds(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 4)
    qs[0, 2] = float("nan")
    qs[1] = float("nan")
    res = ik.converge_multistart(qs, targets, tasks, 1e-3, 10)
    torch.cuda.synchronize()
    assert int(res.seed[0]) != 2 and torch.isfinite(res.error[0])
    assert int(res.seed[1]) == 0 and torch.isnan(res.error[1]) and int(res.steps[1]) == 1
    assert int(res.status[1]) & FAILED and torch.isnan(res.q[1]).all()


def test_out_of_limits_seed_fails_while_its_group_goes_on():
    sc, ik, q0, targets = _ur5(512)
    qs = seeds(ik, q0, 2)
    qs[:, 1, 0] = 10.0
    res = check_against_trajectory(ik, qs, targets, [sc.tasks[0]], 1e-4, 30, "ur5 one seed outside")
    assert (res.seed == 0).all() and (res.steps > 1).any()
    assert ((res.status & _cabi.PK_STATUS_OUT_OF_LIMITS) == 0).all()


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_graph_capture_equals_eager(which):
    ik, q0, targets, tasks = _case(which)
    qs = seeds(ik, q0, 4)
    eager = ik.converge_multistart(qs, targets, tasks, 1e-3, 20)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ik.converge_multistart(qs, targets, tasks, 1e-3, 20)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    B = q0.shape[0]
    outs = dict(q_out=torch.empty_like(q0), error=torch.empty(B, device="cuda"),
                seed=torch.empty(B, device="cuda", dtype=torch.int32),
                steps=torch.empty(B, device="cuda", dtype=torch.int32),
                status=torch.empty(B, device="cuda", dtype=torch.int32))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ik.converge_multistart(qs, targets, tasks, 1e-3, 20, **outs)
    for x in outs.values():
        x.zero_()
    n0 = launches()
    g.replay()
    torch.cuda.synchronize()
    assert launches() == n0
    for x, y in zip(outs.values(), eager[:5]):
        assert torch.equal(x, y)


def test_api_errors():
    sc, ik, q0, targets = _ur5(64)
    frame, posture = sc.tasks
    qs = seeds(ik, q0, 4)
    stranger = pink_b200.FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    for kw in ({"tasks": []}, {"tasks": [stranger]}, {"tol": -1.0}, {"tol": float("nan")}, {"max_steps": -1},
               {"q_seeds": q0}, {"q_seeds": qs.double()}, {"q_seeds": qs[:, :3]}, {"q_seeds": q0[:, None].repeat(1, 64, 1)},
               {"targets": targets[:-1]}, {"targets": None}):
        args = dict(q_seeds=qs, targets=targets, tasks=[frame], tol=1e-3, max_steps=5)
        args.update(kw)
        with pytest.raises(ValueError):
            ik.converge_multistart(**args)
    lib = _cabi.load()
    eng = ik.engine
    q_out = torch.empty_like(q0)
    stream = torch.cuda.current_stream().cuda_stream

    def call(S=4, mask=1):  # 16 targets: at most 16 x 16 of the 64 x 4 seed rows are read
        return lib.pk_converge_multistart_prepared(eng.handle, ik._handle, qs.data_ptr(), S, targets.data_ptr(), mask,
                                                   1e-3, 5, q_out.data_ptr(), None, None, None, None, 16, stream)

    assert call() == 0 and call(S=1) == 0 and call(S=16) == 0
    for kw in ({"S": 0}, {"S": 3}, {"S": 64}, {"mask": 0}, {"mask": 4}):
        assert call(**kw) != 0, kw
    # the tree kernel: at most 8 seeds
    sc = helpers.humanoid_scenario("g1_description", 8, with_com=True)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    with pytest.raises(ValueError, match="at most 8"):
        ik.converge_multistart(q0[:, None].repeat(1, 16, 1).contiguous(), targets, pose_tasks(ik), 1e-3, 5)


# ---- the example -----------------------------------------------------------------------------

def test_multistart_example():
    import importlib.util

    spec = importlib.util.spec_from_file_location("reach_ms", os.path.join(ROOT, "examples",
                                                                           "arm_ur5_reach_multistart_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    one = ex.run(batch=1024, num_seeds=1, max_steps=100)
    eight = ex.run(batch=1024, num_seeds=8, max_steps=100)
    torch.cuda.synchronize()
    assert eight.converged.float().mean() >= one.converged.float().mean()
    assert bool(eight.converged[one.converged].all())


def _in_subprocess(fn, **env):
    code = f"from tests.test_gpu_multistart import {fn} as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, **env), check=True, timeout=900)

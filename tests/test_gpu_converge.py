"""GPU suite (`-m gpu`): solve to a tolerance, ``BatchedIK.converge`` /
``pk_converge_prepared``, on every path (chain kernel, tree kernel, general path).

The reference is one trajectory rollout of ``max_steps`` steps on the same inputs with all
records: an instance that stopped after ``steps`` solves must sit bitwise where the rollout was
after that many steps, with the same status; its returned error must be the task-terms error
there; and every configuration it passed through before must have had an error above ``tol``.
Instances whose error comes within 1e-3 relative of ``tol`` are left out of that last check
(the kernel's forward kinematics and the task-terms export round differently); the number left
out is printed.  Environment switches are read once per process, so those cases run in a
subprocess."""

import importlib.util
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
FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF
ERROR_TYPES = (_cabi.PK_TASK_FRAME, _cabi.PK_TASK_RELATIVE_FRAME, _cabi.PK_TASK_COM)


def _ik(sc):
    return pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                               barriers=getattr(sc, "barriers", None), constraints=getattr(sc, "constraints", None),
                               safety_break=sc.safety_break, batch_size=sc.B,
                               collision_model=getattr(sc, "collision_model", None))


def _inputs(sc):
    _, targets, _ = sc.problem()
    q0 = torch.as_tensor(sc.q32, device="cuda")
    return q0, None if targets is None else torch.as_tensor(targets, device="cuda").contiguous()


def pose_tasks(ik):
    """The frame, relative-frame and CoM tasks of the solver."""
    return [t for k, t in enumerate(ik.tasks) if int(ik.prob.tasks[k].type) in ERROR_TYPES]


def task_error(ik, tasks, q, targets):
    """max over tasks of |e_t|_2 from pk_task_terms_batched (NaN kept)."""
    err = torch.zeros(q.shape[0], device="cuda")
    for t in tasks:
        k = next(k for k, t0 in enumerate(ik.tasks) if t0 is t)
        ty = int(ik.prob.tasks[k].type)
        rows = ik.nv - (6 if ik.nq != ik.nv else 0) if ty == _cabi.PK_TASK_POSTURE else (3 if ty == _cabi.PK_TASK_COM else 6)
        e, _ = ik.engine.task_terms(ik.prob, k, rows, q, targets)
        err = torch.maximum(err, torch.linalg.vector_norm(e, dim=1))
    return err


def launches():
    return _cabi.load().pk_launch_count()


def check_against_trajectory(ik, q0, targets, tasks, tol, max_steps, label=""):
    """converge against one recorded trajectory rollout of max_steps steps; returns the result."""
    n0 = launches()
    res = ik.converge(q0, targets, tasks, tol, max_steps)
    assert launches() - n0 == 1
    tr = ik.rollout_trajectory(q0, targets, max_steps, record=True)
    torch.cuda.synchronize()
    B = q0.shape[0]
    rows = torch.arange(B, device="cuda")
    steps = res.steps.long()
    assert (steps >= 0).all() and (steps <= max_steps).all()
    q_all = torch.cat([q0[None], tr.q_traj])  # q_all[s] = q after s steps
    st_all = torch.cat([torch.zeros_like(tr.status_traj[:1]), tr.status_traj])
    assert torch.equal(res.q, q_all[steps, rows]), label
    assert torch.equal(res.status, st_all[steps, rows]), label
    assert torch.equal(res.converged, res.error <= tol)
    # the returned error is the task-terms error where the instance stopped
    e_tt = task_error(ik, tasks, res.q, targets)
    fin = torch.isfinite(e_tt)
    assert torch.equal(torch.isfinite(res.error), fin)
    np.testing.assert_allclose(res.error[fin].cpu().numpy(), e_tt[fin].cpu().numpy(), rtol=1e-4, atol=2e-6,
                               err_msg=label)
    # every configuration passed through before stopping had an error above tol
    skipped = 0
    for s in range(max_steps):
        before = steps > s  # q_all[s] was left by a solve
        if not before.any():
            break
        e = task_error(ik, tasks, q_all[s], targets)
        near = (e - tol).abs() <= 1e-3 * tol
        skipped += int((before & near).sum())
        bad = before & ~near & ~(e > tol)
        assert not bad.any(), (label, s, torch.nonzero(bad)[:5].flatten().tolist())
    print(f"[converge {label}] B={B} converged={int(res.converged.sum())} max_steps_hit="
          f"{int((steps == max_steps).sum())} skipped_near_tol={skipped}")
    return res


def _ur5(B=4096, kind="reachable", out_of_limits=3):
    sc = helpers.ur5_scenario(B, kind, out_of_limits=out_of_limits)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    return sc, ik, q0, targets


# ---- chains ----------------------------------------------------------------------------------

def test_chain_ur5_reachable_and_unreachable():
    sc, ik, q0, targets = _ur5()
    res = check_against_trajectory(ik, q0, targets, [sc.tasks[0]], 1e-4, 60, "ur5 reachable")
    assert res.converged.float().mean() > 0.6
    oob = (res.status & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
    assert int(oob.sum()) == 3 and (res.steps[oob] == 1).all()
    sc, ik, q0, targets = _ur5(kind="unreachable", out_of_limits=0)
    res = check_against_trajectory(ik, q0, targets, [sc.tasks[0]], 1e-4, 15, "ur5 unreachable")
    alive = (res.status & FAILED) == 0
    assert (res.steps[alive] == 15).all() and (res.error[alive] > 1e-4).all()
    # frame and posture together: the max of the two
    sc, ik, q0, targets = _ur5(1024, out_of_limits=0)
    check_against_trajectory(ik, q0, targets, sc.tasks, 0.3, 30, "ur5 frame+posture")


@pytest.mark.parametrize("nj,kw", [
    (2, {}), (3, {"prismatic": (1,)}), (4, {"two_tasks": True}), (5, {"shared_target": True}), (6, {}),
    (7, {"two_tasks": True, "prismatic": (2,)}), (3, {"frame_tasks": False}),
])
def test_chain_instantiations(nj, kw):
    sc = helpers.chain_scenario(nj, 1000 + nj, seed=nj, **kw)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    tasks = pose_tasks(ik) or ik.tasks  # no frame task: the posture task
    check_against_trajectory(ik, q0, targets, tasks, 1e-3, 25, f"chain{nj} {kw}")


def check_lanes_equal_default():
    """PK_CHAIN_LANES selects the solve entries' sub-warp variant only: converge always runs the
    thread-per-instance kernel, so its outputs equal those of a process without the switch."""
    sc, ik, q0, targets = _ur5(3001)
    res = ik.converge(q0, targets, [sc.tasks[0]], 1e-4, 40)
    torch.cuda.synchronize()
    path = os.environ["PK_CONVERGE_OUT"]
    if os.path.exists(path):
        ref = torch.load(path)
        for name in ("q", "error", "steps", "status"):
            assert torch.equal(getattr(res, name).cpu(), ref[name]), name
    else:
        torch.save({name: getattr(res, name).cpu() for name in ("q", "error", "steps", "status")}, path)


def test_chain_lanes_switch_has_no_effect(tmp_path):
    out = str(tmp_path / "converge.pt")
    _in_subprocess("check_lanes_equal_default", PK_CONVERGE_OUT=out)
    _in_subprocess("check_lanes_equal_default", PK_CONVERGE_OUT=out, PK_CHAIN_LANES="2")


# ---- trees -----------------------------------------------------------------------------------

def test_tree_g1_com():
    sc = helpers.humanoid_scenario("g1_description", 1000, with_com=True)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    check_against_trajectory(ik, q0, targets, pose_tasks(ik), 2e-3, 25, "g1 com")


def test_tree_g1_extras_barriers():
    sc = extras.g1_extras(192)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    check_against_trajectory(ik, q0, targets, pose_tasks(ik), 2e-3, 12, "g1 extras")


# ---- general path ----------------------------------------------------------------------------

def test_general_path_tree_extras_40_joints():
    sc = extras.tree_extras(40, 67, True, seed=7)
    ik = _ik(sc)
    q0, targets = _inputs(sc)
    check_against_trajectory(ik, q0, targets, pose_tasks(ik), 1e-3, 8, "tree40")


def check_forced_general():
    from tests.hostsim import HostSim

    for name in ("ur5", "g1"):
        if name == "ur5":
            sc = helpers.ur5_scenario(2001, "reachable", out_of_limits=3)
        else:
            sc = helpers.humanoid_scenario("g1_description", 1001, with_com=True)
        prob, targets, _ = sc.problem()
        hs = HostSim(sc.model)
        hs.solve_ik(prob, sc.q32[:1], None if targets is None else targets[:1], path=1)
        assert hs.selection.path == "general", hs.selection
        ik = _ik(sc)
        q0, targets = _inputs(sc)
        tasks = [sc.tasks[0]] if name == "ur5" else pose_tasks(ik)
        check_against_trajectory(ik, q0, targets, tasks, 1e-3, 20, f"{name} forced general")


def test_general_path_forced_ur5_g1():
    _in_subprocess("check_forced_general", PK_FORCE_GENERIC="1")


# ---- freeze, graphs, errors ------------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_nan_target_freezes_one_instance(which):
    if which == "chain":
        sc, ik, q0, targets = _ur5(2048)
        tasks = [sc.tasks[0]]
    else:
        sc = helpers.humanoid_scenario("g1_description", 256, with_com=True)
        ik = _ik(sc)
        q0, targets = _inputs(sc)
        tasks = pose_tasks(ik)
    j = 77
    clean = ik.converge(q0, targets, tasks, 1e-3, 30)
    poisoned = targets.clone()
    poisoned[j, 3] = float("nan")
    res = ik.converge(q0, poisoned, tasks, 1e-3, 30)
    torch.cuda.synchronize()
    assert torch.isnan(res.error[j]) and not bool(res.converged[j])
    assert int(res.steps[j]) == 1 and int(res.status[j]) & FAILED
    assert torch.equal(res.q[j], q0[j])
    keep = torch.arange(q0.shape[0], device="cuda") != j
    for name in ("q", "error", "steps", "status"):
        assert torch.equal(getattr(res, name)[keep], getattr(clean, name)[keep]), name


@pytest.mark.parametrize("which", ["chain", "tree", "general"])
def test_graph_capture_equals_eager(which):
    if which == "chain":
        sc, ik, q0, targets = _ur5(4096)
        tasks = [sc.tasks[0]]
    else:
        sc = (helpers.humanoid_scenario("g1_description", 128, with_com=True) if which == "tree"
              else extras.tree_extras(40, 67, True, seed=7))
        ik = _ik(sc)
        q0, targets = _inputs(sc)
        tasks = pose_tasks(ik)
    eager = ik.converge(q0, targets, tasks, 1e-3, 20)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ik.converge(q0, targets, tasks, 1e-3, 20)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    q_out = torch.empty_like(q0)
    err = torch.empty(q0.shape[0], device="cuda")
    steps = torch.empty(q0.shape[0], device="cuda", dtype=torch.int32)
    status = torch.empty_like(steps)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ik.converge(q0, targets, tasks, 1e-3, 20, q_out=q_out, error=err, steps=steps, status=status)
    for x in (q_out, err, steps, status):
        x.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip((q_out, err, steps, status), eager):
        assert torch.equal(x, y)


def test_q_out_may_alias_q():
    sc, ik, q0, targets = _ur5(1000)
    ref = ik.converge(q0, targets, [sc.tasks[0]], 1e-4, 30)
    q = q0.clone()
    res = ik.converge(q, targets, [sc.tasks[0]], 1e-4, 30, q_out=q)
    torch.cuda.synchronize()
    assert res.q.data_ptr() == q.data_ptr() and torch.equal(q, ref.q)


def test_api_errors():
    sc, ik, q0, targets = _ur5(256, out_of_limits=0)
    frame, posture = sc.tasks
    stranger = pink_b200.FrameTask("tool0", position_cost=1.0, orientation_cost=1.0)
    for kw in ({"tasks": []}, {"tasks": [stranger]}, {"tol": -1.0}, {"tol": float("nan")}, {"tol": float("inf")},
               {"max_steps": -1}, {"max_steps": 2.5}, {"targets": targets[:-1]}, {"targets": targets.double()},
               {"targets": None}):
        args = dict(q=q0, targets=targets, tasks=[frame], tol=1e-3, max_steps=5)
        args.update(kw)
        with pytest.raises(ValueError):
            ik.converge(**args)
    lib = _cabi.load()
    eng = ik.engine
    q_out = torch.empty_like(q0)
    stream = torch.cuda.current_stream().cuda_stream

    def call(mask=1, tol=1e-3, max_steps=5, q_out_ptr=q_out.data_ptr(), t_ptr=targets.data_ptr()):
        return lib.pk_converge_prepared(eng.handle, ik._handle, q0.data_ptr(), t_ptr, mask, tol, max_steps, q_out_ptr,
                                        None, None, None, sc.B, stream)

    assert call() == 0 and call(mask=3) == 0 and call(max_steps=0) == 0
    for kw in ({"mask": 0}, {"mask": 4}, {"tol": -1e-3}, {"tol": float("nan")}, {"max_steps": -1},
               {"q_out_ptr": None}, {"t_ptr": None}):
        assert call(**kw) != 0, kw
        with pytest.raises(RuntimeError):
            _cabi.check(call(**kw))
    # a joint-velocity task cannot be in the mask
    damp = pink_b200.DampingTask(cost=1e-3)
    ik2 = pink_b200.BatchedIK(sc.model, [frame, damp], sc.dt, damping=sc.damping, limits=sc.limits, batch_size=sc.B)
    with pytest.raises(ValueError):
        ik2.converge(q0, targets, [damp], 1e-3, 5)
    assert lib.pk_converge_prepared(eng.handle, ik2._handle, q0.data_ptr(), targets.data_ptr(), 2, 1e-3, 5,
                                    q_out.data_ptr(), None, None, None, sc.B, stream) != 0


# ---- the example -----------------------------------------------------------------------------

def test_reach_example():
    spec = importlib.util.spec_from_file_location("arm_ur5_reach_batched",
                                                  os.path.join(ROOT, "examples", "arm_ur5_reach_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    ik, task, q0, targets = ex.setup(4096)
    res = check_against_trajectory(ik, q0, targets, [task], ex.TOL, 200, "reach example")
    again = ex.run(batch=4096, max_steps=200)
    torch.cuda.synchronize()
    assert torch.equal(again.q, res.q) and torch.equal(again.steps, res.steps)
    assert res.converged.float().mean() > 0.9


def _in_subprocess(fn, **env):
    code = f"from tests.test_gpu_converge import {fn} as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, **env), check=True, timeout=900)

"""GPU suite (`-m gpu`): trajectory rollouts, ``BatchedIK.rollout_trajectory`` /
``pk_rollout_trajectory_prepared``: the targets of step s feed step s, and the configuration,
velocity and status of every step come back, in one launch on every path (chain kernel, its
sub-warp variant, tree kernel, general path).

The reference is the same closed loop made of separate ``solve`` and ``integrate`` calls with
the freeze emulated (an instance that failed a step gets v = 0 and keeps its status from then
on), and for UR5 the fp64 oracle.  Environment switches are read once per process, so those
cases run in a subprocess."""

import importlib.util
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from oracle import ik as oik
from oracle import kinematics as okin
from pink_b200 import _cabi
from tests import extras, helpers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAILED = _cabi.PK_STATUS_NO_SOLUTION | _cabi.PK_STATUS_NOT_POSDEF


def _ik(sc):
    return pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                               barriers=getattr(sc, "barriers", None), constraints=getattr(sc, "constraints", None),
                               safety_break=sc.safety_break, batch_size=sc.B,
                               collision_model=getattr(sc, "collision_model", None))


def _inputs(sc):
    _, targets, _ = sc.problem()
    q0 = torch.as_tensor(sc.q32, device="cuda")
    return q0, None if targets is None else torch.as_tensor(targets, device="cuda")


def moving_targets(ik, base, steps, dt, amp=0.05, seed=0):
    """[steps, B, target_stride]: the rows of ``base`` plus the arm_ur5 sinusoid
    ``amp sin(2 t + phase_i)`` (t = s dt, one phase per instance) on the translation of every
    per-instance frame target and on every other per-instance task target word."""
    B = base.shape[0]
    g = torch.Generator().manual_seed(seed)
    phase = 2.0 * math.pi * torch.rand(B, generator=g, dtype=torch.float64)
    t = torch.arange(steps, dtype=torch.float64) * dt
    wave = (amp * torch.sin(2.0 * t[:, None] + phase[None, :])).float()
    rows = base.cpu().unsqueeze(0).repeat(steps, 1, 1)
    for _, off, width in ik.target_layout:
        for c in ((off + 3, off + 7, off + 11) if width == 12 else range(off, off + width)):
            rows[:, :, c] += wave
    return rows.to("cuda")


def _frozen(st_or, safety_break):
    bad = (st_or & FAILED) != 0
    if safety_break:
        bad |= (st_or & _cabi.PK_STATUS_OUT_OF_LIMITS) != 0
    return bad


def loop(ik, q0, targets, steps, dt, safety_break):
    """(q_traj, v_traj, status_traj) of separate solve + integrate calls, freeze emulated."""
    q = q0.clone()
    st_or = torch.zeros(q0.shape[0], dtype=torch.int32, device="cuda")
    qs, vs, ss = [], [], []
    for s in range(steps):
        t = targets[s] if targets is not None and targets.dim() == 3 else targets
        v, st = ik.solve(q, t)
        frozen = _frozen(st_or, safety_break)
        v = torch.where(frozen[:, None], torch.zeros_like(v), v)
        st_or = st_or | torch.where(frozen, torch.zeros_like(st), st)
        q = ik.engine.integrate(q, v, dt)
        qs.append(q)
        vs.append(v)
        ss.append(st_or.clone())
    return torch.stack(qs), torch.stack(vs), torch.stack(ss)


def launches():
    return _cabi.load().pk_launch_count()


def check_consistency(res, safety_break):
    """q_traj[-1] = q, status_traj[-1] = status, v_traj[-1] = v where never frozen (bitwise);
    status_traj is monotone."""
    assert torch.equal(res.q_traj[-1], res.q) and torch.equal(res.status_traj[-1], res.status)
    alive = ~_frozen(res.status, safety_break)
    assert torch.equal(res.v_traj[-1][alive], res.v[alive])
    st = res.status_traj
    assert torch.equal(st[:-1] & st[1:], st[:-1])


def check_against_loop(ik, q0, targets, steps, dt, safety_break, q_atol=2e-5, v_tol=None, st_mask=-1,
                       one_launch=True):
    n0 = launches()
    res = ik.rollout_trajectory(q0, targets, steps)
    if one_launch:
        assert launches() - n0 == 1
    q_l, v_l, s_l = loop(ik, q0, targets, steps, dt, safety_break)
    torch.cuda.synchronize()
    check_consistency(res, safety_break)
    np.testing.assert_array_equal(res.status_traj.cpu().numpy() & st_mask, s_l.cpu().numpy() & st_mask)
    for s in range(steps):
        np.testing.assert_allclose(res.q_traj[s].cpu().numpy(), q_l[s].cpu().numpy(), atol=q_atol, err_msg=f"step {s}")
        if v_tol is not None:
            np.testing.assert_allclose(res.v_traj[s].cpu().numpy(), v_l[s].cpu().numpy(), atol=v_tol, rtol=v_tol,
                                       err_msg=f"step {s}")
    return res


def _ur5(B=4096):
    sc = helpers.ur5_scenario(B, "reachable", out_of_limits=3)
    ik = _ik(sc)
    q0, base = _inputs(sc)
    return sc, ik, q0, base


# ---- 1. moving targets on the chain kernel -------------------------------------------------

def test_moving_targets_chain_against_loop_and_oracle():
    sc, ik, q0, base = _ur5()
    K = 12
    rows = moving_targets(ik, base, K, sc.dt, amp=0.1)
    res = check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, v_tol=5e-3)
    assert (res.status & _cabi.PK_STATUS_OUT_OF_LIMITS).sum() > 0  # the three instances outside the limits froze
    # a rollout that read the first row at every step lands elsewhere
    fixed = ik.rollout_trajectory(q0, rows[0], K)
    assert (fixed.q - res.q).abs().max() > 1e-3
    # oracle closed loop with the same per-step targets
    n = 24
    q_o = sc.q64[:n].copy()
    alive = np.ones(n, dtype=bool)
    q_traj = res.q_traj.cpu().numpy()
    for s in range(K):
        tasks = [oik._slice_task_range(t, 0, n) for t in sc.oracle_tasks]
        T = rows[s, :n].cpu().numpy().astype(np.float64).reshape(n, 3, 4)
        tasks[0] = dict(tasks[0], target=(T[:, :, :3], T[:, :, 3]))
        v_o, st_o = oik.solve_ik_batch(sc.table, q_o, tasks, sc.dt, sc.damping)
        alive &= st_o == 0
        q_o = np.where(alive[:, None], okin.integrate(sc.table, q_o, v_o * sc.dt), q_o)
        np.testing.assert_allclose(q_traj[s, :n], q_o, atol=2e-4, err_msg=f"step {s}")


# ---- 2. consistency, and fixed targets equal the fixed-target rollout ----------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_fixed_targets_equal_rollout(which):
    if which == "chain":
        sc, ik, q0, base = _ur5()
        K = 6
    else:
        sc = helpers.humanoid_scenario("g1_description", 192, with_com=True)
        ik = _ik(sc)
        q0, base = _inputs(sc)
        K = 4
    q_r, v_r, st_r = ik.rollout(q0, base, K)
    for record in (False, True):
        res = ik.rollout_trajectory(q0, base, K, record=record)
        torch.cuda.synchronize()
        assert torch.equal(res.q, q_r) and torch.equal(res.v, v_r) and torch.equal(res.status, st_r), record
        assert (res.q_traj is None) == (not record)
        if record:
            check_consistency(res, sc.safety_break)


# ---- 3. every <NJ, NFT> chain instantiation ------------------------------------------------

@pytest.mark.parametrize("nj,kw", [
    (2, {}), (3, {"prismatic": (1,)}), (4, {"two_tasks": True}), (5, {"shared_target": True}),
    (7, {"two_tasks": True, "prismatic": (2,)}), (7, {}),
])
def test_chain_instantiations_against_loop(nj, kw):
    sc = helpers.chain_scenario(nj, 1000 + nj, seed=nj, **kw)
    ik = _ik(sc)
    q0, base = _inputs(sc)
    K = 5
    rows = None if base is None else moving_targets(ik, base, K, sc.dt, amp=0.05, seed=nj)
    check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, v_tol=5e-3)


# ---- 4. tree kernel --------------------------------------------------------------------------

def test_tree_g1_com_against_loop():
    sc = helpers.humanoid_scenario("g1_description", 192, with_com=True)
    ik = _ik(sc)
    q0, base = _inputs(sc)
    K = 5
    rows = moving_targets(ik, base, K, sc.dt, amp=0.02)
    check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, v_tol=5e-3, st_mask=FAILED)


def test_tree_g1_extras_against_loop_and_freeze():
    sc = extras.g1_extras(96)
    ik = _ik(sc)
    q0, base = _inputs(sc)
    K = 3
    rows = moving_targets(ik, base, K, sc.dt, amp=0.02)
    res = check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, q_atol=1e-4, st_mask=FAILED)
    check_frozen_rows(res)


def check_frozen_rows(res):
    """Every instance that fails a step: from that step on q_traj is constant and v_traj is 0;
    status_traj repeats after it."""
    st = res.status_traj.cpu().numpy()
    q, v = res.q_traj.cpu().numpy(), res.v_traj.cpu().numpy()
    bad = np.nonzero(st[-1] & FAILED)[0]
    assert bad.size > 0
    for i in bad:
        s0 = int(np.argmax(st[:, i] & FAILED != 0))
        assert (v[s0 + 1:, i] == 0).all() and (st[s0:, i] == st[s0, i]).all()
        assert (q[s0:, i] == q[s0, i]).all()


# ---- 5. general path -----------------------------------------------------------------------

def check_general(scs=("ur5", "g1")):
    """The general path in one launch (ik_generic_rollout_kernel) against the loop; statuses bitwise."""
    from tests.hostsim import HostSim

    for name in scs:
        if name == "ur5":
            sc = helpers.ur5_scenario(3001, "reachable", out_of_limits=3)
        elif name == "g1":
            sc = helpers.humanoid_scenario("g1_description", 1001, with_com=True)
        elif name == "g1_extras":
            sc = extras.g1_extras(96)
        else:
            sc = extras.tree_extras(40, 67, True, seed=7)
        prob, targets, _ = sc.problem()
        hs = HostSim(sc.model)
        hs.solve_ik(prob, sc.q32[:1], None if targets is None else targets[:1],
                    path=1 if os.environ.get("PK_FORCE_GENERIC") == "1" else 0)
        assert hs.selection.path == "general", (name, hs.selection)
        ik = _ik(sc)
        q0, base = _inputs(sc)
        K = 4
        rows = moving_targets(ik, base, K, sc.dt, amp=0.02)
        res = check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, q_atol=5e-5)
        if name in ("g1_extras", "tree40"):
            check_frozen_rows(res)


def test_general_path_tree_extras_40_joints():
    check_general(("tree40",))


def test_general_path_forced_ur5_g1_and_barriers():
    _in_subprocess("check_general", PK_FORCE_GENERIC="1")


def check_general_forced_barriers():
    check_general(("g1_extras",))


def test_general_path_forced_freeze_on_infeasible_barrier():
    _in_subprocess("check_general_forced_barriers", PK_FORCE_GENERIC="1")


# ---- 6. freeze -----------------------------------------------------------------------------

def test_nan_target_freezes_one_instance_chain():
    sc, ik, q0, base = _ur5(2048)
    K, j, s_bad = 8, 77, 3
    rows = moving_targets(ik, base, K, sc.dt, amp=0.05).contiguous()
    clean = ik.rollout_trajectory(q0, rows, K)
    poisoned = rows.clone()
    poisoned[s_bad, j, 3] = float("nan")
    res = ik.rollout_trajectory(q0, poisoned, K)
    torch.cuda.synchronize()
    st = res.status_traj[:, j].cpu().numpy()
    assert not (st[:s_bad] & FAILED).any() and (st[s_bad:] & _cabi.PK_STATUS_NO_SOLUTION).all()
    assert (st[s_bad:] == st[s_bad]).all()
    assert (res.v_traj[s_bad:, j] == 0).all()
    assert (res.q_traj[s_bad:, j] == res.q_traj[s_bad - 1, j]).all()
    keep = torch.arange(sc.B, device="cuda") != j
    for name in ("q", "v", "status"):
        assert torch.equal(getattr(res, name)[keep], getattr(clean, name)[keep]), name
    for name in ("q_traj", "v_traj", "status_traj"):
        assert torch.equal(getattr(res, name)[:, keep], getattr(clean, name)[:, keep]), name


# ---- 7. misaligned step stride -------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_misaligned_step_stride_equals_contiguous(which):
    if which == "chain":
        sc, ik, q0, base = _ur5(3000)
    else:
        sc = helpers.humanoid_scenario("g1_description", 130, with_com=True)
        ik = _ik(sc)
        q0, base = _inputs(sc)
    K = 4
    rows = moving_targets(ik, base, K, sc.dt)
    B, S = rows.shape[1], rows.shape[2]
    store = torch.full((K, B * S + 1), float("nan"), device="cuda")
    view = store[:, 1:].view(K, B, S)  # step stride B S + 1 floats: every other row 4-byte aligned only
    view.copy_(rows)
    assert view.stride() == (B * S + 1, S, 1)
    a = ik.rollout_trajectory(q0, view, K)
    b = ik.rollout_trajectory(q0, view.contiguous(), K)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- 8. sub-warp chain kernel --------------------------------------------------------------

def check_lanes():
    sc, ik, q0, base = _ur5(3001)
    K = 6
    rows = moving_targets(ik, base, K, sc.dt, amp=0.1)
    check_against_loop(ik, q0, rows, K, sc.dt, sc.safety_break, v_tol=5e-3)


def test_sub_warp_kernel_two_lanes_against_loop():
    _in_subprocess("check_lanes", PK_CHAIN_LANES="2")


# ---- 9. graph capture ----------------------------------------------------------------------

@pytest.mark.parametrize("which", ["chain", "tree"])
def test_graph_capture_equals_eager(which):
    if which == "chain":
        sc, ik, q0, base = _ur5(4096)
    else:
        sc = helpers.humanoid_scenario("g1_description", 128, with_com=True)
        ik = _ik(sc)
        q0, base = _inputs(sc)
    K = 5
    rows = moving_targets(ik, base, K, sc.dt)
    eager = ik.rollout_trajectory(q0, rows, K)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ik.rollout_trajectory(q0, rows, K)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = ik.rollout_trajectory(q0, rows, K)
    for x in captured:
        x.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(captured, eager):
        assert torch.equal(x, y)


# ---- 10. API errors ------------------------------------------------------------------------

def test_api_errors():
    sc, ik, q0, base = _ur5(256)
    K = 3
    rows = moving_targets(ik, base, K, sc.dt)
    with pytest.raises(ValueError):
        ik.rollout_trajectory(q0, rows[:, :-1], K)  # batch mismatch
    with pytest.raises(ValueError):
        ik.rollout_trajectory(q0, rows, K + 1)  # steps mismatch
    with pytest.raises(ValueError):
        ik.rollout_trajectory(q0, base)  # fixed rows without steps
    wide = torch.zeros((K, sc.B, ik.target_stride + 4), device="cuda")
    with pytest.raises(ValueError):
        ik.rollout_trajectory(q0, wide[:, :, :ik.target_stride], K)  # stride(1) != target_stride
    lib = _cabi.load()
    eng = ik.engine
    q_out = torch.empty_like(q0)
    v = torch.empty((sc.B, ik.nv), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    step = rows.stride(0)

    def call(n_steps=K, v_ptr=v.data_ptr(), target_step=step):
        return lib.pk_rollout_trajectory_prepared(eng.handle, ik._handle, q0.data_ptr(), rows.data_ptr(), target_step,
                                                  n_steps, q_out.data_ptr(), v_ptr, None, None, None, None, sc.B,
                                                  stream)

    assert call() == 0
    for kw in ({"n_steps": 0}, {"v_ptr": None}, {"target_step": -1}):
        assert call(**kw) != 0, kw
        with pytest.raises(RuntimeError):
            _cabi.check(call(**kw))


# ---- 11. the fused example -----------------------------------------------------------------

def test_fused_example_equals_step_by_step():
    spec = importlib.util.spec_from_file_location("arm_ur5_batched", os.path.join(ROOT, "examples", "arm_ur5_batched.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    err_f, q_f = ex.run(batch=4096, steps=20, fused=True)
    err_s, q_s = ex.run(batch=4096, steps=20, fused=False)
    torch.cuda.synchronize()
    np.testing.assert_allclose(q_f.cpu().numpy(), q_s.cpu().numpy(), atol=2e-5)
    np.testing.assert_allclose(err_f.cpu().numpy(), err_s.cpu().numpy(), atol=5e-5)


def _in_subprocess(fn, **env):
    code = f"from tests.test_gpu_rollout_trajectory import {fn} as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, **env), check=True, timeout=900)

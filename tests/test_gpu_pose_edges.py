"""GPU suite (`-m gpu`): pose errors, Jacobians and free-flyer steps at the rotation-angle edges
of the fp32 SE(3) maps (``tests/pose_edges.py``) on every kernel path, through the library's
entry points: ``pk_task_terms_batched`` (the general path's body); each path's own error
(converge and one-seed multi-start with max_steps = 0); each path's Jacobian through v of an
unconstrained QP (solve on the PDL chain kernel, a recorded one-step rollout on the plain chain
kernel, the sub-warp chain kernels, the tree kernel, the general path); and the integrate
kernel.  Environment switches are read once per process, so those cases run in a subprocess.
The worst errors per ladder angle are printed."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from tests import helpers
from tests import pose_edges as pe

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LADDER = pe.Ladder()


def _setup(name, for_velocity=False):
    sc, k, case = pe.scenario(name, LADDER, for_velocity=for_velocity)
    ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                             safety_break=sc.safety_break, batch_size=sc.B)
    _, targets, _ = sc.problem()
    q = torch.as_tensor(sc.q32, device="cuda")
    return sc, k, case, ik, q, torch.as_tensor(targets, device="cuda").contiguous()


def _np(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def check_terms(name):
    sc, k, case, ik, q, targets = _setup(name)
    e, J = ik.engine.task_terms(ik.prob, k, 6, q, targets)
    pe.check_terms(_np(e), _np(J), pe.reference(sc, k), case, LADDER, f"gpu task_terms {name}")


def check_errors(name, label):
    sc, k, case, ik, q, targets = _setup(name)
    ref = pe.reference(sc, k)
    res = ik.converge(q, targets, [sc.tasks[k]], 0.0, 0)
    assert (_np(res.steps) == 0).all() and (_np(res.status) == 0).all()
    assert torch.equal(res.q, q)
    pe.check_error_norm(_np(res.error), ref, case, LADDER, f"gpu converge {name} {label}")
    res = ik.converge_multistart(q[:, None].contiguous(), targets, [sc.tasks[k]], 0.0, 0)
    assert (_np(res.steps) == 0).all() and (_np(res.status) == 0).all() and (_np(res.seed) == 0).all()
    assert torch.equal(res.q, q)
    pe.check_error_norm(_np(res.error), ref, case, LADDER, f"gpu multistart {name} {label}")


def check_solve(name, label):
    sc, k, case, ik, q, targets = _setup(name, for_velocity=True)
    v, st = ik.solve(q, targets)
    assert (_np(st) == 0).all()
    pe.check_velocity(_np(v), sc, k, pe.reference(sc, k), case, LADDER, f"gpu solve {name} {label}")


def _host_selection(name, path=0):
    from tests.hostsim import HostSim

    sc, _, _ = pe.scenario(name, LADDER, for_velocity=True)
    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    hs.solve_ik(prob, sc.q32[:1], targets[:1], path=path)
    return hs.selection


# ---- in this process -------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["ur5", "g1-frame", "g1-relative"])
def test_task_terms(name):
    check_terms(name)


@pytest.mark.parametrize("name,expect", [("ur5", "chain"), ("chain7-two-frames", "chain"), ("g1-frame", "tree"),
                                         ("g1-relative", "tree")])
def test_converge_error(name, expect):
    """Chain converge kernel at <6, 1> and <7, 2>, tree converge kernel, and their multi-start kernels."""
    assert _host_selection(name).path == expect
    check_errors(name, expect)


@pytest.mark.parametrize("name,expect", [("ur5", "chain"), ("chain7-two-frames", "chain"), ("g1-frame", "tree"),
                                         ("g1-relative", "tree")])
def test_solve_velocity(name, expect):
    """solve: the PDL chain kernel on UR5, the chain kernel at <7, 2>, the tree kernel on G1."""
    sel = _host_selection(name)
    assert sel.path == expect
    if name == "ur5":
        assert sel.pdl_row_fits
    check_solve(name, expect)


def test_rollout_one_step_velocity():
    """A recorded one-step trajectory rollout runs the plain chain kernel instantiation."""
    sc, k, case, ik, q, targets = _setup("ur5", for_velocity=True)
    tr = ik.rollout_trajectory(q, targets, 1, record=True)
    assert (_np(tr.status_traj) == 0).all()
    pe.check_velocity(_np(tr.v_traj[0]), sc, k, pe.reference(sc, k), case, LADDER, "gpu rollout ur5")


def test_integrate_free_flyer():
    _, model, table = helpers.load("g1_description")
    q, v, dt, angle = pe.integrate_cases(table)
    eng = pink_b200.engine.get_engine(model, "cuda")
    out = eng.integrate(torch.as_tensor(q, device="cuda"), torch.as_tensor(v, device="cuda"), dt)
    pe.check_integrate(_np(out), table, q, v, dt, angle, "gpu integrate g1")


# ---- one process per switch ------------------------------------------------------------------

def check_lanes():
    """solve on the sub-warp chain kernel PK_CHAIN_LANES selects (UR5: <6, 1>)."""
    lanes = int(os.environ["PK_CHAIN_LANES"])
    assert _host_selection("ur5", 10 + lanes).lanes in (lanes, 0)
    check_solve("ur5", f"lanes {lanes}")


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_sub_warp_chain_kernel(lanes):
    _in_subprocess("check_lanes", PK_CHAIN_LANES=str(lanes))


def check_general():
    """PK_FORCE_GENERIC=1: solve, converge and multi-start on the general path."""
    for name in ("ur5", "g1-frame", "g1-relative"):
        assert _host_selection(name, 1).path == "general"
        check_solve(name, "general")
        check_errors(name, "general")


def test_general_path_forced():
    _in_subprocess("check_general", PK_FORCE_GENERIC="1")


def _in_subprocess(fn, **env):
    code = f"from tests.test_gpu_pose_edges import {fn} as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, **env), check=True, timeout=900)

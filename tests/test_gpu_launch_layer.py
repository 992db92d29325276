"""GPU suite (`-m gpu`): the launch layer of the CUDA library around the kernels.

- The host-buffer entry ``pk_solve_ik_prepared_host`` under its three schedules (0 staged uploads
  and downloads, 1 zero-copy, 2 staged uploads with the kernels writing into the pinned host
  buffers), and with ``PK_HOST_DUPLEX=1`` (chunks round-robin over three streams), is bitwise equal
  to the device entry.  UR5 at B = 70001 is three chunks of the default 32768 rows, the last one
  ragged; G1 (tree kernel) at B = 40000 is two.
- ``pk_rollout_prepared`` on the general path (``PK_FORCE_GENERIC=1``: separate solve and
  integrate launches) is bitwise equal to the same solve + integrate calls made one by one.

Environment switches are read once per process, so those cases run in a subprocess."""

import os
import subprocess
import sys

import pytest
import torch

import pink_b200
from pink_b200 import _cabi
from tests import helpers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(sc, kernel, path=0):
    """BatchedIK of the scenario and its per-instance targets, after checking which kernel the
    library selects (its host build, ``path`` as in HostSim.solve_ik)."""
    from tests.hostsim import HostSim

    prob, targets, _ = sc.problem()
    hs = HostSim(sc.model)
    hs.solve_ik(prob, sc.q32[:1], targets[:1], path=path)
    assert hs.selection.path == kernel, (sc.name, hs.selection)
    ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                             safety_break=sc.safety_break, batch_size=sc.B)
    return ik, targets


def check_host_schedules():
    """solve_host under schedules 0, 1 and 2 against solve, bit for bit."""
    for sc, kernel in ((helpers.ur5_scenario(70001, "reachable"), "chain"),
                       (helpers.humanoid_scenario("g1_description", 40000, with_com=True), "tree")):
        ik, targets = _run(sc, kernel)
        v_d, st_d = ik.solve(torch.as_tensor(sc.q32, device="cuda"), torch.as_tensor(targets, device="cuda"))
        v_d, st_d = v_d.cpu(), st_d.cpu()
        q_h, t_h = torch.as_tensor(sc.q32).pin_memory(), torch.as_tensor(targets).pin_memory()
        try:
            for mode in (0, 1, 2):
                ik.set_host_schedule(mode)
                v_h = torch.full((sc.B, ik.nv), float("nan")).pin_memory()
                st_h = torch.full((sc.B,), -1, dtype=torch.int32).pin_memory()
                ik.solve_host(q_h, t_h, v_h, st_h)
                torch.cuda.synchronize()
                assert torch.equal(v_h, v_d) and torch.equal(st_h, st_d), (sc.name, mode)
        finally:
            ik.set_host_schedule(-1)


def check_general_rollout(steps=4):
    """pk_rollout_prepared with PK_FORCE_GENERIC=1 in the environment: 2 launches per step."""
    lib = _cabi.load()
    for sc in (helpers.ur5_scenario(3001, "reachable"), helpers.humanoid_scenario("g1_description", 1001, with_com=True)):
        ik, targets = _run(sc, "general", path=1)
        q0 = torch.as_tensor(sc.q32, device="cuda")
        t = torch.as_tensor(targets, device="cuda")
        n0 = lib.pk_launch_count()
        q_f, v_f, st_f = ik.rollout(q0, t, steps)
        assert lib.pk_launch_count() - n0 == 2 * steps, sc.name
        q = q0.clone()
        for _ in range(steps):
            v, st = ik.solve(q, t)
            q = ik.engine.integrate(q, v, sc.dt)
        torch.cuda.synchronize()
        assert torch.equal(q_f, q) and torch.equal(v_f, v) and torch.equal(st_f, st), sc.name


def _in_subprocess(fn, **env):
    code = f"from tests.test_gpu_launch_layer import {fn} as f; f()"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, **env), check=True, timeout=900)


def test_host_entry_equals_device_entry_under_every_schedule():
    check_host_schedules()


def test_host_entry_equals_device_entry_with_duplex_streams():
    _in_subprocess("check_host_schedules", PK_HOST_DUPLEX="1")


def test_general_path_rollout_equals_solve_and_integrate_calls():
    _in_subprocess("check_general_rollout", PK_FORCE_GENERIC="1")

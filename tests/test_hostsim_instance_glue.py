"""The per-instance glue around the rollout and converge loops (the kernels' ``*_instance``
bodies) on the CPU build: ``converge`` with ``q_out`` aliasing ``q``, the optional outputs left
null, and the tree kernel's converge workspace, where the step's ``v`` sits after the plan's
words (``converge_tree_layout``)."""

import ctypes as C

import numpy as np
import pytest

from tests import helpers
from tests.hostsim import HostSim, _p, lib

# (scenario, path, task mask, expected selection): every path of the converge and rollout bodies
CASES = {
    "chain": (lambda: helpers.ur5_scenario(24, "reachable", out_of_limits=2), 0, 0b01, "chain"),
    "sub_warp_2": (lambda: helpers.ur5_scenario(24, "reachable", out_of_limits=2), 12, 0b01, "chain"),
    "tree_on_chain": (lambda: helpers.ur5_scenario(24, "reachable", out_of_limits=2), 2, 0b01, "tree"),
    "general": (lambda: helpers.ur5_scenario(24, "reachable", out_of_limits=2), 1, 0b01, "general"),
    "tree_g1": (lambda: helpers.humanoid_scenario("g1_description", 8, with_com=True), 0, 0b110, "tree"),
}
CONVERGE_CASES = [c for c in CASES if c != "sub_warp_2"]  # converge always runs the thread-per-instance chain kernel


def _converge_raw(hs, prob, q, targets, mask, tol, max_steps, q_out, err, steps, status, path):
    sel = (C.c_int * 8)()
    hs._chk(lib().hs_converge(hs.handle, C.byref(prob), _p(q), _p(targets), C.c_uint32(mask), C.c_float(tol),
                              C.c_int(max_steps), _p(q_out), _p(err), _p(steps), _p(status), C.c_int64(q.shape[0]),
                              path, sel))


def _rollout_raw(hs, prob, q, targets, n_steps, q_out, v, status, path):
    sel = (C.c_int * 8)()
    hs._chk(lib().hs_rollout(hs.handle, C.byref(prob), _p(q), _p(targets), C.c_int64(0), n_steps, _p(q_out), _p(v),
                             _p(status), None, None, None, C.c_int64(q.shape[0]), path, sel))


def _setup(case):
    make, path, mask, expect = CASES[case]
    sc = make()
    prob, targets, _ = sc.problem()
    return sc, prob, np.ascontiguousarray(targets, dtype=np.float32), path, mask, expect


@pytest.mark.parametrize("case", CONVERGE_CASES)
def test_converge_q_out_aliasing_q(case):
    sc, prob, targets, path, mask, expect = _setup(case)
    hs = HostSim(sc.model)
    q_ref, err_ref, steps_ref, st_ref = hs.converge(prob, sc.q32, targets, mask, 1e-4, 20, path=path)
    assert hs.selection.path == expect
    q = sc.q32.astype(np.float32).copy()
    B = q.shape[0]
    err, steps, st = np.zeros(B, np.float32), np.zeros(B, np.int32), np.zeros(B, np.int32)
    _converge_raw(hs, prob, q, targets, mask, 1e-4, 20, q, err, steps, st, path)
    np.testing.assert_array_equal(q.view(np.int32), q_ref.view(np.int32))
    np.testing.assert_array_equal(err.view(np.int32), err_ref.view(np.int32))
    np.testing.assert_array_equal(steps, steps_ref)
    np.testing.assert_array_equal(st, st_ref)


@pytest.mark.parametrize("case", CONVERGE_CASES)
def test_converge_optional_outputs_null(case):
    sc, prob, targets, path, mask, _ = _setup(case)
    hs = HostSim(sc.model)
    q_ref, _, _, _ = hs.converge(prob, sc.q32, targets, mask, 1e-4, 20, path=path)
    q_out = np.zeros_like(q_ref)
    _converge_raw(hs, prob, sc.q32.astype(np.float32), targets, mask, 1e-4, 20, q_out, None, None, None, path)
    np.testing.assert_array_equal(q_out.view(np.int32), q_ref.view(np.int32))


@pytest.mark.parametrize("case", list(CASES))
def test_rollout_status_null(case):
    sc, prob, targets, path, _, expect = _setup(case)
    hs = HostSim(sc.model)
    q_ref, v_ref, _, _, _, _ = hs.rollout(prob, sc.q32, targets, 6, record=False, path=path)
    assert hs.selection.path == expect
    q_out = np.zeros_like(q_ref)
    v = np.zeros_like(v_ref)
    _rollout_raw(hs, prob, sc.q32.astype(np.float32), targets, 6, q_out, v, None, path)
    np.testing.assert_array_equal(q_out.view(np.int32), q_ref.view(np.int32))
    np.testing.assert_array_equal(v.view(np.int32), v_ref.view(np.int32))


@pytest.mark.parametrize("case", ["tree_on_chain", "tree_g1"])
def test_tree_converge_workspace_matches_rollout(case):
    """With tol = 0 an instance that neither converges nor fails takes max_steps steps, each the
    rollout's step: the converge loop keeps v in the warp's workspace, the rollout in the v row,
    so equal results mean the step's v and the plan's words do not overlap."""
    sc, prob, targets, path, mask, _ = _setup(case)
    hs = HostSim(sc.model)
    n = 5
    q_c, _, steps, st = hs.converge(prob, sc.q32, targets, mask, 0.0, n, path=path)
    assert hs.selection.path == "tree"
    q_r, _, st_r, _, _, _ = hs.rollout(prob, sc.q32, targets, n, record=False, path=path)
    full = steps == n
    assert full.sum() >= q_c.shape[0] // 2
    np.testing.assert_array_equal(q_c[full].view(np.int32), q_r[full].view(np.int32))
    np.testing.assert_array_equal(st[full], st_r[full])

"""The PDL instantiation of the chain kernel lets its lowest-index CTAs prefetch the whole grid's q
and targets rows into L2 (PK_CHAIN_L2_PREFETCH, on by default).  A prefetch is a hint: with it on
and off every output must be bitwise the same, whatever the batch size (one CTA, partial CTAs, one
wave with spare slots, more than one wave), the alignment and length of the targets rows, and
whatever ran before the launch: back-to-back graph launches, a launch reading the previous one's
v as its q, and a foreign kernel that lets its dependents start and writes the targets later.
Each setting runs in its own process (the switch is read once per process)."""

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MULTI_WAVE_B = 140000  # 1094 CTAs of 128 threads: more than the 528 an H100 holds at once


def _ik(sc):
    return pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                               safety_break=sc.safety_break, device="cuda", batch_size=sc.B)


def _solve_case(out, name, sc, offset=0):
    from tests.test_gpu_chain_pdl_staging import _offset_view

    ik = _ik(sc)
    _, targets, _ = sc.problem()
    t = _offset_view(torch.as_tensor(targets, device="cuda"), offset)
    q = torch.as_tensor(sc.q32, device="cuda")
    v, st = ik.solve(q, t)
    q_r, v_r, st_r = ik.rollout(q, t, 3)
    torch.cuda.synchronize()
    for key, val in (("v", v), ("status", st), ("q_roll", q_r), ("v_roll", v_r), ("status_roll", st_r)):
        out[f"{name}/{key}"] = val.cpu().numpy()


def _graph_case(out, B=65536, launches=8, nbuf=4):
    """back-to-back graph launches over rotating input sets, then a chain in which call k + 1
    reads call k's v as its q; both against the same calls made one at a time"""
    sc = helpers.ur5_scenario(B, "reachable")
    ik = _ik(sc)
    _, targets, _ = sc.problem()
    rng = np.random.default_rng(3)
    q0 = torch.as_tensor(sc.q32, device="cuda")
    t0 = torch.as_tensor(targets, device="cuda")
    qs = [q0 + torch.as_tensor(rng.normal(size=sc.q32.shape) * 0.01, dtype=torch.float32, device="cuda")
          for _ in range(nbuf)]
    ts = [t0.clone() for _ in range(nbuf)]
    for k, t in enumerate(ts):
        t.view(-1, 12)[:, 3:12:4] += 0.01 * k
    vs = [torch.empty_like(q0) for _ in range(launches)]
    ss = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(launches)]
    vc = [torch.empty_like(q0) for _ in range(launches)]
    sv = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(launches)]

    def calls():
        for k in range(launches):
            ik.solve(qs[k % nbuf], ts[k % nbuf], vs[k], ss[k])
        for k in range(launches):
            ik.solve(q0 if k == 0 else vc[k - 1], t0, vc[k], sv[k])

    calls()  # warm-up, outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            calls()
    torch.cuda.current_stream().wait_stream(side)
    for x in vs + vc:
        x.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    graph = [x.cpu().numpy() for x in vs + ss + vc + sv]
    for x in vs + vc:
        x.fill_(float("nan"))
    for k in range(launches):  # one at a time
        ik.solve(qs[k % nbuf], ts[k % nbuf], vs[k], ss[k])
        torch.cuda.synchronize()
    for k in range(launches):
        ik.solve(q0 if k == 0 else vc[k - 1], t0, vc[k], sv[k])
        torch.cuda.synchronize()
    single = [x.cpu().numpy() for x in vs + ss + vc + sv]
    for k, (a, b) in enumerate(zip(graph, single)):
        out[f"graph/{k}"] = a
        out[f"single/{k}"] = b


def _late_writer_case(out, offset):
    """a foreign kernel triggers its dependents at once and writes the targets 200 us later"""
    from tests.test_gpu_chain_pdl_staging import _late_writer, _offset_view

    lib = _late_writer()
    sc = helpers.ur5_scenario(65536, "reachable")
    ik = _ik(sc)
    q = torch.as_tensor(sc.q32, device="cuda")
    _, targets, _ = sc.problem()
    new = torch.as_tensor(targets, device="cuda")
    old = new.clone()
    old.view(-1, 12)[:, 3:12:4] += 0.05
    v_new, s_new = ik.solve(q, new)
    v_old, _ = ik.solve(q, old)
    t = _offset_view(old, offset)
    stream = torch.cuda.current_stream()
    assert lib.launch_late_writer(t.data_ptr(), new.data_ptr(), new.numel(), 200_000, stream.cuda_stream) == 0
    v, s = ik.solve(q, t)
    torch.cuda.synchronize()
    name = f"late{offset}"
    for key, val in (("v", v), ("status", s), ("v_new", v_new), ("status_new", s_new), ("v_old", v_old)):
        out[f"{name}/{key}"] = val.cpu().numpy()


def _chain(nj, B, two_tasks, acceleration):
    from tests.test_gpu_chain_pdl_staging import _chain as staging_chain

    return staging_chain(nj, B, two_tasks, acceleration)[0]


SOLVE_CASES = {
    **{f"ur5-B{B}": (lambda B=B: helpers.ur5_scenario(B, "reachable", out_of_limits=min(B, 3)), 0)
       for B in (1, 127, 129, 4096, 65536, MULTI_WAVE_B)},
    **{f"ur5-B65536-offset{o}": (lambda: helpers.ur5_scenario(65536, "reachable"), o) for o in (1, 2, 3)},
    "nj6-stride18-B65536": (lambda: _chain(6, 65536, False, False), 0),          # 18 words
    "nj5-dq_prev-stride22-B4099": (lambda: _chain(5, 4099, False, True), 1),   # 22 words
    "nj7-nft2-dq_prev-stride38-B65536": (lambda: _chain(7, 65536, True, True), 0),  # chain_row_words(7, 2)
    "nj7-nft2-dq_prev-stride38-B333": (lambda: _chain(7, 333, True, True), 3),
}


def dump_outputs(path):
    """Every case on cuda:0 in this process's PK_CHAIN_L2_PREFETCH setting, saved to `path`."""
    out = {}
    for name, (make, offset) in SOLVE_CASES.items():
        _solve_case(out, name, make(), offset)
    _graph_case(out)
    for offset in (0, 1):
        _late_writer_case(out, offset)
    np.savez(path, **out)


def _run_dump(tmp_path, value):
    out = tmp_path / f"prefetch-{value}.npz"
    env = dict(os.environ, PK_CHAIN_L2_PREFETCH=str(value))
    env.pop("PK_CHAIN_FORCE_RECOMPUTE", None)
    code = f"from tests.test_gpu_chain_l2_prefetch import dump_outputs as d; d({str(out)!r})"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, check=True, timeout=1200)
    return dict(np.load(out))


@pytest.fixture(scope="module")
def outputs(tmp_path_factory):
    return {value: _run_dump(tmp_path_factory.mktemp(f"l2pf{value}"), value) for value in (0, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SOLVE_CASES))
def test_prefetch_on_and_off_bitwise_equal(name, outputs):
    off, on = outputs[0], outputs[1]
    for key in ("v", "status", "q_roll", "v_roll", "status_roll"):
        k = f"{name}/{key}"
        np.testing.assert_array_equal(on[k], off[k], err_msg=k)
    assert np.isfinite(on[f"{name}/v"]).all()


@pytest.mark.gpu
def test_graph_launches_and_v_as_next_q(outputs):
    """graph replays equal the same calls made one at a time, and the two settings equal each other"""
    off, on = outputs[0], outputs[1]
    keys = [k for k in on if k.startswith("graph/")]
    assert keys
    for k in keys:
        s = k.replace("graph/", "single/")
        np.testing.assert_array_equal(on[k], on[s], err_msg=k)
        np.testing.assert_array_equal(on[k], off[k], err_msg=k)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
def test_targets_written_after_the_predecessor_triggers(offset, outputs):
    """the launch after a late writer returns the new targets' results with the prefetch on and off"""
    for value in (0, 1):
        o = outputs[value]
        name = f"late{offset}"
        assert (o[f"{name}/v_new"] != o[f"{name}/v_old"]).any(axis=1).sum() > 1000
        np.testing.assert_array_equal(o[f"{name}/v"], o[f"{name}/v_new"], err_msg=f"prefetch {value}")
        np.testing.assert_array_equal(o[f"{name}/status"], o[f"{name}/status_new"], err_msg=f"prefetch {value}")


RULE_SHIM = r"""
#include "@CSRC@/pk_select.hpp"
extern "C" int chain_l2_prefetch_ctas(int64_t grid, int64_t resident, int64_t input_bytes, int64_t l2_bytes) {
  return pk::chain_l2_prefetch_ctas(grid, resident, input_bytes, l2_bytes);
}
"""


def test_prefetch_cta_rule(tmp_path):
    """pk::chain_l2_prefetch_ctas (pk_select.hpp) compiled for the host: the CTAs that prefetch a
    launch's inputs"""
    src, so = tmp_path / "rule.cpp", tmp_path / "rule.so"
    src.write_text(RULE_SHIM.replace("@CSRC@", os.path.join(ROOT, "pink_b200", "csrc")))
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                           str(src)])
    f = C.CDLL(str(so)).chain_l2_prefetch_ctas
    f.restype = C.c_int
    f.argtypes = [C.c_int64] * 4
    l2 = 50 * 2**20
    ur5 = 65536 * 4 * (6 + 12)  # bench.py's launch: 4.5 MiB of q and targets
    assert f(512, 528, ur5, l2) == 16  # one wave with 16 spare slots (H100: 132 SMs x 4)
    assert f(500, 528, ur5, l2) == 28
    assert f(100, 528, ur5 // 5, l2) == 32  # many spare slots: at most 32
    assert f(4, 528, 512 * 72, l2) == 4  # at most the grid
    assert f(1, 528, 72, l2) == 1
    assert f(528, 528, ur5, l2) == 1  # an exactly full wave
    assert f(529, 528, ur5, l2) == 0  # more than one wave
    assert f(1094, 528, 140000 * 72, l2) == 0
    assert f(512, 528, l2 // 4, l2) == 16  # inputs of a quarter of the L2
    assert f(512, 528, l2 // 4 + 1, l2) == 0  # more: no prefetch
    assert f(512, 0, ur5, l2) == 0  # occupancy unknown
    assert f(0, 528, 0, l2) == 0

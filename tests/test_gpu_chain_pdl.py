"""Chain kernel under programmatic dependent launch: consecutive launches on one stream overlap,
and an instance whose q or targets a predecessor wrote after the launch began is recomputed from
the final values.  Every result must be bitwise equal to the same calls with a synchronize after
each."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from tests import helpers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0.75  # inside the UR5 joint limits: a stale read gives a plausible, wrong answer


def _ik(sc):
    return pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits, safety_break=True,
                               device="cuda", batch_size=sc.B)


def _inputs(sc):
    _, targets, _ = sc.problem()
    return torch.as_tensor(sc.q32, device="cuda"), torch.as_tensor(targets, device="cuda")


def _graphed(fn):
    """fn() captured once in a CUDA graph, then replayed once"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        fn()  # warm-up outside the capture
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=side):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()


def _np(ts):
    return [t.cpu().numpy().copy() for t in ts]


def test_back_to_back_launches_equal_synchronized_launches():
    sc = helpers.ur5_scenario(65536, "reachable")
    ik = _ik(sc)
    q, t = _inputs(sc)
    K, NBUF = 8, 3
    qs = [q + 0.01 * b for b in range(NBUF)]
    vs = [torch.empty((sc.B, 6), device="cuda") for _ in range(K)]
    ss = [torch.empty((sc.B,), dtype=torch.int32, device="cuda") for _ in range(K)]

    def run(sync):
        for k in range(K):
            ik.solve(qs[k % NBUF], t, vs[k], ss[k])
            if sync:
                torch.cuda.synchronize()

    run(True)
    v_ref, s_ref = _np(vs), _np(ss)
    for v in vs:
        v.fill_(SENTINEL)
    _graphed(lambda: run(False))
    for k in range(K):
        np.testing.assert_array_equal(vs[k].cpu().numpy(), v_ref[k])
        np.testing.assert_array_equal(ss[k].cpu().numpy(), s_ref[k])


@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("call", ["solve", "rollout"])
def test_output_of_one_call_is_input_of_the_next(call, mode):
    """x[k + 1] = f(x[k]): the next launch starts before its q is written (x[k + 1] holds a
    sentinel until then), so it must notice and recompute"""
    sc = helpers.ur5_scenario(65536, "reachable")
    ik = _ik(sc)
    q, t = _inputs(sc)
    N = 4
    xs = [q.clone()] + [torch.empty_like(q) for _ in range(N)]
    ss = [torch.empty((sc.B,), dtype=torch.int32, device="cuda") for _ in range(N)]
    v_last = torch.empty_like(q)

    def run(sync):
        for x in xs[1:]:
            x.fill_(SENTINEL)
        for k in range(N):
            if call == "solve":
                ik.solve(xs[k], t, xs[k + 1], ss[k])
            else:
                ik.rollout(xs[k], t, 3, q_out=xs[k + 1], v_out=v_last, status=ss[k])
            if sync:
                torch.cuda.synchronize()

    run(True)
    x_ref, s_ref = _np(xs), _np(ss)
    if mode == "eager":
        run(False)
        torch.cuda.synchronize()
    else:
        _graphed(lambda: run(False))
    for k in range(N):
        np.testing.assert_array_equal(xs[k + 1].cpu().numpy(), x_ref[k + 1])
        np.testing.assert_array_equal(ss[k].cpu().numpy(), s_ref[k])
    assert not np.any(x_ref[N] == SENTINEL)


def _benchmark_workload_outputs():
    sc = helpers.ur5_scenario(65536, "reachable")
    ik = _ik(sc)
    q, t = _inputs(sc)
    v, s = ik.solve(q, t)
    return v.cpu().numpy(), s.cpu().numpy()


def dump_benchmark_workload_outputs(path):
    v, s = _benchmark_workload_outputs()
    np.savez(path, v=v, status=s)


def test_forced_recompute_gives_the_same_outputs(tmp_path):
    """PK_CHAIN_FORCE_RECOMPUTE=1 (read once per process, hence the subprocess) takes the
    recompute path for every instance"""
    out = tmp_path / "forced.npz"
    env = dict(os.environ, PK_CHAIN_FORCE_RECOMPUTE="1")
    code = f"from tests.test_gpu_chain_pdl import dump_benchmark_workload_outputs as d; d({str(out)!r})"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, check=True, timeout=600)
    forced = np.load(out)
    v, s = _benchmark_workload_outputs()
    np.testing.assert_array_equal(forced["v"], v)
    np.testing.assert_array_equal(forced["status"], s)

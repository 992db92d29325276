"""The PDL instantiation of the chain kernel stages each instance's targets row in shared memory
before griddepcontrol.wait and re-reads it from L2 after.  Every layout of the row that takes a
different copy path must give bitwise the results of the plain instantiation: 16-byte and 4-byte
copies, rows that end mid-vector, the longest row the instantiation accepts, partial warps and
CTAs.  A predecessor that writes the targets after it lets the launch start must be caught by
the re-read."""

import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import pink_b200
from pink_b200.limits import AccelerationLimit
from tests import helpers

pytestmark = pytest.mark.gpu


def _ik(sc):
    return pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                               safety_break=sc.safety_break, device="cuda", batch_size=sc.B)


def _offset_view(t, words):
    """t's values in a fresh buffer that starts `words` floats past a 16-byte boundary"""
    buf = torch.zeros(t.numel() + 4, dtype=torch.float32, device="cuda")
    assert buf.data_ptr() % 16 == 0
    view = buf[words:words + t.numel()].view(t.shape)
    view.copy_(t)
    return view


def _pdl_equals_plain(ik, q, targets, steps=3):
    """rollout launches the PDL instantiation; a recording trajectory launches the plain one"""
    q_p, v_p, s_p = ik.rollout(q, targets, steps)
    res = ik.rollout_trajectory(q, targets, steps, record=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(v_p.cpu().numpy(), res.v.cpu().numpy())
    np.testing.assert_array_equal(q_p.cpu().numpy(), res.q.cpu().numpy())
    np.testing.assert_array_equal(s_p.cpu().numpy(), res.status.cpu().numpy())
    return v_p


def _chain(nj, B, two_tasks, acceleration, seed=5):
    """random chain, posture target per instance, optionally dq_prev per instance: a targets row
    of 12 NFT + NJ (+ NJ) words"""
    sc = helpers.chain_scenario(nj, B, seed=seed, two_tasks=two_tasks, posture_per_instance=True)
    if acceleration:
        rng = np.random.default_rng(seed)
        acc = AccelerationLimit(sc.model, np.full(nj, 30.0))
        acc.set_last_integration(torch.as_tensor(rng.normal(size=(B, nj)) * 0.3, dtype=torch.float32), sc.dt)
        sc.limits = list(sc.limits) + [acc]
    ik = _ik(sc)
    assert ik.target_stride == 12 * (2 if two_tasks else 1) + nj * (2 if acceleration else 1)
    return sc, ik


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_ur5_rows_at_every_base_alignment(offset):
    """stride 12: 128-bit copies from a 16-byte aligned base, 4-byte copies otherwise; B = 1000
    ends in a partial warp and a partial CTA"""
    sc = helpers.ur5_scenario(1000, "reachable", out_of_limits=3)
    ik = _ik(sc)
    _, targets, _ = sc.problem()
    t = _offset_view(torch.as_tensor(targets, device="cuda"), offset)
    assert (t.data_ptr() % 16 == 0) == (offset == 0)
    v = _pdl_equals_plain(ik, torch.as_tensor(sc.q32, device="cuda"), t)
    assert np.isfinite(v.cpu().numpy()).all()


@pytest.mark.parametrize("nj,two_tasks,acceleration,B", [
    (6, False, False, 4099),   # 18 words: ends mid-vector
    (5, False, True, 777),     # 22 words, dq_prev words
    (7, True, True, 333),      # 38 words = chain_row_words(7, 2): the longest row, NFT = 2
    (4, True, False, 65),      # 28 words, NFT = 2
])
@pytest.mark.parametrize("offset", [0, 1])
def test_chain_rows_with_posture_and_dq_prev(nj, two_tasks, acceleration, B, offset):
    """frame targets, posture and dq_prev words in one row, as the problem lays it out"""
    sc, ik = _chain(nj, B, two_tasks, acceleration)
    _, targets, _ = sc.problem()
    assert targets.shape == (B, ik.target_stride)
    t = _offset_view(torch.as_tensor(targets, device="cuda"), offset)
    _pdl_equals_plain(ik, torch.as_tensor(sc.q32, device="cuda"), t)


LATE_WRITER = r"""
#include <cstdint>
// Lets its dependents start at once, waits `ns`, then writes dst = src: a dependent that read
// dst before its griddepcontrol.wait saw the old values.
__global__ void late_writer(float* dst, const float* src, int64_t n, unsigned long long ns) {
  asm volatile("griddepcontrol.launch_dependents;");
  unsigned long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  do {
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  } while (t - t0 < ns);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = src[i];
}
extern "C" int launch_late_writer(float* dst, const float* src, long long n, unsigned long long ns, void* stream) {
  late_writer<<<16, 256, 0, (cudaStream_t)stream>>>(dst, src, n, ns);
  return (int)cudaGetLastError();
}
"""


def _late_writer():
    import ctypes

    d = tempfile.mkdtemp(prefix="pk_late_writer_")
    src, so = os.path.join(d, "w.cu"), os.path.join(d, "w.so")
    with open(src, "w") as fh:
        fh.write(LATE_WRITER)
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-Xcompiler", "-fPIC",
                           "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.launch_late_writer.restype = ctypes.c_int
    lib.launch_late_writer.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_ulonglong,
                                       ctypes.c_void_p]
    return lib


@pytest.mark.parametrize("offset", [0, 1])
def test_targets_written_after_the_predecessor_triggers(offset):
    """A foreign kernel triggers its dependents first and writes the targets 200 us later: the
    launch after it must give the results of the new targets, bitwise."""
    lib = _late_writer()
    sc = helpers.ur5_scenario(65536, "reachable")
    ik = _ik(sc)
    q = torch.as_tensor(sc.q32, device="cuda")
    _, targets, _ = sc.problem()
    new = torch.as_tensor(targets, device="cuda")
    old = new.clone()
    old.view(-1, 12)[:, 3:12:4] += 0.05  # every translation moved
    v_new, s_new = ik.solve(q, new)
    v_old, _ = ik.solve(q, old)
    torch.cuda.synchronize()
    # instances at their velocity bounds keep their v: enough others change for a stale read to show
    assert (v_new != v_old).any(dim=1).sum() > 1000
    t = _offset_view(old, offset)
    stream = torch.cuda.current_stream()
    rc = lib.launch_late_writer(t.data_ptr(), new.data_ptr(), new.numel(), 200_000, stream.cuda_stream)
    assert rc == 0
    v, s = ik.solve(q, t)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(t.cpu().numpy(), new.cpu().numpy())
    np.testing.assert_array_equal(v.cpu().numpy(), v_new.cpu().numpy())
    np.testing.assert_array_equal(s.cpu().numpy(), s_new.cpu().numpy())

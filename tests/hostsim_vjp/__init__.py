"""ctypes wrapper of ``libpk_hostsim_vjp.so``: the gradient body of ``pk_converge_vjp_prepared``
(``Generic::solution_vjp``) compiled for the host CPU (see hostsim_vjp.cpp), with the same build
variants as ``tests/hostsim``: ``PK_HOSTSIM_SANITIZE=1`` (AddressSanitizer + UBSan) and
``PK_HOSTSIM_FMA=1`` (a*b + c contracted into FMAs, as nvcc does).

TEST HARNESS ONLY.  The product package never imports this module."""

import ctypes as C
import os
import subprocess

import numpy as np

from pink_b200 import _cabi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SANITIZE = os.environ.get("PK_HOSTSIM_SANITIZE", "0") == "1"
_FMA = os.environ.get("PK_HOSTSIM_FMA", "0") == "1"
_SO = os.path.join(_HERE, "libpk_hostsim_vjp_asan.so" if _SANITIZE else
                   "libpk_hostsim_vjp_fma.so" if _FMA else "libpk_hostsim_vjp.so")
_SRC = os.path.join(_HERE, "hostsim_vjp.cpp")
_CSRC = os.path.join(_HERE, "..", "..", "pink_b200", "csrc")
_lib = None


def build(force: bool = False) -> str:
    srcs = [_SRC] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [
        os.path.join(_HERE, "..", "..", "include", "pink_b200.h")
    ]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs)
    if force or stale:
        extra = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer"] if _SANITIZE else ["-O2"]
        subprocess.check_call(
            ["g++", *extra, "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas",
             *(["-ffp-contract=fast", "-mfma"] if _FMA else ["-ffp-contract=off"]), "-o", _SO, _SRC]
        )
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.hv_last_error.restype = C.c_char_p
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    return a[None] if a.ndim == 1 else a


class HostVjp:
    """Runs the gradient body on the CPU for one model."""

    def __init__(self, model):
        self.table = model.table()
        self.holder = _cabi.ModelDescHolder(self.table)
        self.handle = C.c_void_p()
        self._chk(lib().hv_model_create(C.byref(self.holder.desc), C.byref(self.handle)))
        self.nq, self.nv = self.table.nq, self.table.nv

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().hv_model_destroy(self.handle)
                self.handle = None
        except Exception:  # interpreter shutdown
            pass

    @staticmethod
    def _chk(rc):
        if rc:
            raise RuntimeError(lib().hv_last_error().decode())

    def converge_vjp(self, prob, q_star, targets, grad_q):
        """``(grad_targets [B, target_stride], status [B])`` at converged solutions ``q_star``."""
        q = _f32(q_star)
        B = q.shape[0]
        t = None if targets is None else _f32(targets)
        gq = _f32(grad_q)
        gt = np.zeros((B, int(prob.target_stride)), dtype=np.float32)
        st = np.zeros(B, dtype=np.int32)
        self._chk(lib().hv_converge_vjp(self.handle, C.byref(prob), _p(q), _p(t), _p(gq), _p(gt), _p(st),
                                        C.c_int64(B)))
        return gt, st

    def converge_vjp_raw(self, prob, q_star, targets, grad_q, grad_targets, status, B):
        """The same on raw addresses (ints or None), as the CUDA library's entry takes them."""
        p = lambda a: None if a is None else C.c_void_p(a)  # noqa: E731
        return lib().hv_converge_vjp(self.handle, C.byref(prob), p(q_star), p(targets), p(grad_q), p(grad_targets),
                                     p(status), C.c_int64(B))

"""ctypes wrapper of ``libpk_hostsim_kinematics.so``: the bodies of ``pk_frame_placements_batched``
and ``pk_frame_placements_vjp_batched`` (``pink_b200/csrc/pk_kinematics.cuh``) compiled for the host
CPU (see hostsim_kinematics.cpp), with the same build variants as ``tests/hostsim``:
``PK_HOSTSIM_SANITIZE=1`` (AddressSanitizer + UBSan) and ``PK_HOSTSIM_FMA=1`` (a*b + c contracted
into FMAs, as nvcc does).

TEST HARNESS ONLY.  The product package never imports this module."""

import ctypes as C
import os
import subprocess

import numpy as np

from pink_b200 import _cabi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SANITIZE = os.environ.get("PK_HOSTSIM_SANITIZE", "0") == "1"
_FMA = os.environ.get("PK_HOSTSIM_FMA", "0") == "1"
_SO = os.path.join(_HERE, "libpk_hostsim_kinematics_asan.so" if _SANITIZE else
                   "libpk_hostsim_kinematics_fma.so" if _FMA else "libpk_hostsim_kinematics.so")
_SRC = os.path.join(_HERE, "hostsim_kinematics.cpp")
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
        _lib.hk_last_error.restype = C.c_char_p
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    return a[None] if a.ndim == 1 else a


class HostKinematics:
    """Runs the forward-kinematics bodies on the CPU for one model."""

    def __init__(self, model):
        self.table = model.table()
        self.holder = _cabi.ModelDescHolder(self.table)
        self.handle = C.c_void_p()
        self._chk(lib().hk_model_create(C.byref(self.holder.desc), C.byref(self.handle)))
        self.nq, self.nv = self.table.nq, self.table.nv

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().hk_model_destroy(self.handle)
                self.handle = None
        except Exception:  # interpreter shutdown
            pass

    @staticmethod
    def _chk(rc):
        if rc:
            raise RuntimeError(lib().hk_last_error().decode())

    def frame_placements(self, frames, q, com=False):
        """``(oMf [B, F, 3, 4], com [B, 3] or None)`` of frame indices ``frames`` at ``q [B, nq]``."""
        q = _f32(q)
        B = q.shape[0]
        f = np.ascontiguousarray(frames, dtype=np.int32)
        oMf = np.zeros((B, f.size, 3, 4), dtype=np.float32)
        c = np.zeros((B, 3), dtype=np.float32) if com else None
        self._chk(lib().hk_frame_placements(self.handle, _p(f), C.c_int32(f.size), _p(q), _p(oMf), _p(c),
                                            C.c_int64(B)))
        return oMf, c

    def frame_placements_vjp(self, frames, q, grad_oMf=None, grad_com=None):
        """``grad_q [B, nq]`` from ``grad_oMf [B, F, 3, 4]`` and ``grad_com [B, 3]`` (each or None)."""
        q = _f32(q)
        B = q.shape[0]
        f = np.ascontiguousarray(frames, dtype=np.int32)
        gF = None if grad_oMf is None else np.ascontiguousarray(grad_oMf, dtype=np.float32)
        gc = None if grad_com is None else np.ascontiguousarray(grad_com, dtype=np.float32)
        gq = np.full((B, self.nq), np.nan, dtype=np.float32)
        self._chk(lib().hk_frame_placements_vjp(self.handle, _p(f), C.c_int32(f.size), _p(q), _p(gF), _p(gc), _p(gq),
                                                C.c_int64(B)))
        return gq

    def frame_placements_raw(self, frames, num_frames, q, oMf, com, B):
        """``hk_frame_placements`` on raw addresses (ints or None), for the argument checks."""
        p = lambda a: None if a is None else C.c_void_p(a)  # noqa: E731
        return lib().hk_frame_placements(self.handle, p(frames), C.c_int32(num_frames), p(q), p(oMf), p(com),
                                         C.c_int64(B))

    def frame_placements_vjp_raw(self, frames, num_frames, q, grad_oMf, grad_com, grad_q, B):
        """``hk_frame_placements_vjp`` on raw addresses (ints or None), for the argument checks."""
        p = lambda a: None if a is None else C.c_void_p(a)  # noqa: E731
        return lib().hk_frame_placements_vjp(self.handle, p(frames), C.c_int32(num_frames), p(q), p(grad_oMf),
                                             p(grad_com), p(grad_q), C.c_int64(B))

"""ctypes wrapper of ``libpk_hostsim_pose_tol.so``: the host build of the kernel bodies
(``tests/hostsim``) plus ``hs_converge_pose_tol`` and ``hs_converge_goalset_pose_tol``, the
separate-tolerance solves of ``pk_converge_pose_tol_prepared`` and
``pk_converge_goalset_pose_tol_prepared`` (see hostsim_pose_tol.cpp), with the same build
variants: ``PK_HOSTSIM_SANITIZE=1`` (AddressSanitizer + UBSan) and ``PK_HOSTSIM_FMA=1`` (a*b + c
contracted into FMAs, as nvcc does).

TEST HARNESS ONLY.  The product package never imports this module."""

import ctypes as C
import os
import subprocess

import numpy as np

from pink_b200 import _cabi
from tests.hostsim import _p, _selection

_HERE = os.path.dirname(os.path.abspath(__file__))
_SANITIZE = os.environ.get("PK_HOSTSIM_SANITIZE", "0") == "1"
_FMA = os.environ.get("PK_HOSTSIM_FMA", "0") == "1"
_SO = os.path.join(_HERE, "libpk_hostsim_pose_tol_asan.so" if _SANITIZE else
                   "libpk_hostsim_pose_tol_fma.so" if _FMA else "libpk_hostsim_pose_tol.so")
_SRC = os.path.join(_HERE, "hostsim_pose_tol.cpp")
_CSRC = os.path.join(_HERE, "..", "..", "pink_b200", "csrc")
_lib = None


def build(force: bool = False) -> str:
    srcs = [_SRC, os.path.join(_HERE, "..", "hostsim", "hostsim.cpp")] + [
        os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [os.path.join(_HERE, "..", "..", "include", "pink_b200.h")]
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
        _lib.hs_last_error.restype = C.c_char_p
    return _lib


class HostPoseTol:
    """Runs the separate-tolerance solves on the CPU for one model."""

    def __init__(self, model):
        self.table = model.table()
        self.holder = _cabi.ModelDescHolder(self.table)
        self.handle = C.c_void_p()
        self._chk(lib().hs_model_create(C.byref(self.holder.desc), C.byref(self.handle)))

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().hs_model_destroy(self.handle)
                self.handle = None
        except Exception:  # interpreter shutdown
            pass

    def _chk(self, rc):
        if rc:
            raise RuntimeError(lib().hs_last_error().decode())

    def converge(self, prob, q, targets, mask, tol, orientation_tol, max_steps, path=0):
        """Solve to separate tolerances (hs_converge_pose_tol): ``(q_out, err, steps, status)``;
        ``path`` as ``HostSim.converge``, ``self.selection`` the kernel selection the loop ran."""
        q = np.ascontiguousarray(np.asarray(q, dtype=np.float32))
        B = q.shape[0]
        tg = None if targets is None else np.ascontiguousarray(np.asarray(targets, dtype=np.float32))
        q_out = np.zeros_like(q)
        err = np.zeros(B, dtype=np.float32)
        steps, st = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        self._chk(lib().hs_converge_pose_tol(self.handle, C.byref(prob), _p(q), _p(tg), C.c_uint32(mask),
                                             C.c_float(tol), C.c_float(orientation_tol), C.c_int(max_steps),
                                             _p(q_out), _p(err), _p(steps), _p(st), C.c_int64(B), path, sel))
        self.selection = _selection(sel)
        return q_out, err, steps, st

    def converge_goalset(self, prob, q_seeds, goals, mask, tol, orientation_tol, max_steps, path=0):
        """Goal-set solve to separate tolerances (hs_converge_goalset_pose_tol): ``q_seeds [B, S,
        nq]``, ``goals [B, G, target_stride]`` -> ``(q_out, err, goal, seed, steps, status)``."""
        qs = np.ascontiguousarray(np.asarray(q_seeds, dtype=np.float32))
        B, S, nq = qs.shape
        g = np.ascontiguousarray(np.asarray(goals, dtype=np.float32))
        G = g.shape[1]
        q_out = np.zeros((B, nq), dtype=np.float32)
        err = np.zeros(B, dtype=np.float32)
        goal, seed, steps, st = (np.zeros(B, dtype=np.int32) for _ in range(4))
        sel = (C.c_int * 8)()
        self._chk(lib().hs_converge_goalset_pose_tol(
            self.handle, C.byref(prob), _p(qs), S, _p(g), G, C.c_uint32(mask), C.c_float(tol),
            C.c_float(orientation_tol), C.c_int(max_steps), _p(q_out), _p(err), _p(goal), _p(seed), _p(steps), _p(st),
            C.c_int64(B), path, sel))
        self.selection = _selection(sel)
        return q_out, err, goal, seed, steps, st

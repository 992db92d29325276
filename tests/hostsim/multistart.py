"""ctypes wrapper of ``libpk_hostsim_multistart.so``: the multi-start loop
(``pk_converge_multistart_prepared``) over the kernel bodies compiled for the host CPU (see
multistart.cpp), with the build switches of :mod:`tests.hostsim` (``PK_HOSTSIM_SANITIZE``,
``PK_HOSTSIM_FMA``).

TEST HARNESS ONLY, like :mod:`tests.hostsim`: the product package never imports it.
"""

import ctypes as C
import os
import subprocess

import numpy as np

from tests import hostsim
from tests.hostsim import Selection, _p
from tests.hostsim.converge import ConvergeSim

_SO = os.path.join(hostsim._HERE, "libpk_hostsim_multistart_asan.so" if hostsim._SANITIZE
                   else "libpk_hostsim_multistart_fma.so" if hostsim._FMA else "libpk_hostsim_multistart.so")
_SRC = os.path.join(hostsim._HERE, "multistart.cpp")
_lib = None


def build(force: bool = False) -> str:
    srcs = [_SRC] + [os.path.join(hostsim._CSRC, f) for f in os.listdir(hostsim._CSRC)] + [
        os.path.join(hostsim._HERE, "..", "..", "include", "pink_b200.h")
    ]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs)
    if force or stale:
        extra = (["-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer"] if hostsim._SANITIZE
                 else ["-O2"])
        subprocess.check_call(
            ["g++", *extra, "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas",
             *(["-ffp-contract=fast", "-mfma"] if hostsim._FMA else ["-ffp-contract=off"]), "-o", _SO, _SRC]
        )
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.hs_multistart_last_error.restype = C.c_char_p
    return _lib


class MultistartSim(ConvergeSim):
    """:class:`ConvergeSim` plus the multi-start loop."""

    def converge_multistart(self, prob, q_seeds, targets, mask, tol, max_steps, path=0):
        """Multi-start solve to a tolerance (hs_converge_multistart): ``q_seeds [B, S, nq]`` ->
        ``(q_out, err, seed, steps, status)``; ``path`` as :meth:`HostSim.solve_ik` (0: the
        library's selection, 1: the general path, 2: the tree kernel)."""
        qs = self._f32(q_seeds)
        B, S, nq = qs.shape
        t = None if targets is None else self._f32(targets)
        q_out = np.zeros((B, nq), dtype=np.float32)
        err = np.zeros(B, dtype=np.float32)
        seed = np.zeros(B, dtype=np.int32)
        steps = np.zeros(B, dtype=np.int32)
        st = np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        rc = lib().hs_converge_multistart(C.byref(self.holder.desc), C.byref(prob), _p(qs), S, _p(t),
                                          C.c_uint32(mask), C.c_float(tol), C.c_int(max_steps), _p(q_out), _p(err),
                                          _p(seed), _p(steps), _p(st), C.c_int64(B), path, sel)
        if rc:
            raise RuntimeError(lib().hs_multistart_last_error().decode())
        self.selection = Selection(("chain", "tree", "general")[sel[0]], sel[1], sel[2], (sel[3], sel[4]), sel[5],
                                   bool(sel[6]), sel[7])
        return q_out, err, seed, steps, st

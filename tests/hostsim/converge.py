"""ctypes wrapper of ``libpk_hostsim_converge.so``: the converge loops of the kernel bodies
(``pk_converge_prepared``) compiled for the host CPU (see converge.cpp), with the build
switches of :mod:`tests.hostsim` (``PK_HOSTSIM_SANITIZE``, ``PK_HOSTSIM_FMA``).

TEST HARNESS ONLY, like :mod:`tests.hostsim`: the product package never imports it.
"""

import ctypes as C
import os
import subprocess

import numpy as np

from tests import hostsim
from tests.hostsim import HostSim, Selection, _p

_SO = os.path.join(hostsim._HERE, "libpk_hostsim_converge_asan.so" if hostsim._SANITIZE
                   else "libpk_hostsim_converge_fma.so" if hostsim._FMA else "libpk_hostsim_converge.so")
_SRC = os.path.join(hostsim._HERE, "converge.cpp")
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
        _lib.hs_converge_last_error.restype = C.c_char_p
    return _lib


class ConvergeSim(HostSim):
    """:class:`HostSim` plus the converge loops."""

    def converge(self, prob, q, targets, mask, tol, max_steps, path=0):
        """Solve to a tolerance with the converge loop of the selected body (hs_converge):
        ``(q_out, err, steps, status)``; ``path`` as :meth:`HostSim.solve_ik`, and
        ``self.selection`` the kernel selection the loop ran."""
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        q_out = np.zeros_like(q)
        err = np.zeros(B, dtype=np.float32)
        steps = np.zeros(B, dtype=np.int32)
        st = np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        rc = lib().hs_converge(C.byref(self.holder.desc), C.byref(prob), _p(q), _p(t), C.c_uint32(mask),
                               C.c_float(tol), C.c_int(max_steps), _p(q_out), _p(err), _p(steps), _p(st),
                               C.c_int64(B), path, sel)
        if rc:
            raise RuntimeError(lib().hs_converge_last_error().decode())
        self.selection = Selection(("chain", "tree", "general")[sel[0]], sel[1], sel[2], (sel[3], sel[4]), sel[5],
                                   bool(sel[6]), sel[7])
        return q_out, err, steps, st

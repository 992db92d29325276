"""ctypes wrapper of ``libpk_hostsim.so``: the kernel bodies of
``pink_b200/csrc`` compiled for the host CPU (see hostsim.cpp).  Each entry makes the problem,
runs the library's kernel selection and loops over the instances with the body the selection
names: the per-instance bodies the kernels call (indexing, loads, rollout / converge loop,
stores), the step bodies for the chain solve and the general path, and the two-pass rounds of
multi-start.

TEST HARNESS ONLY.  The product package never imports this module; it exists
so that the CPU test-suite can run the kernels' exact fp32 arithmetic against
the fp64 oracle without a GPU.
"""

import ctypes as C
import os
import subprocess
from collections import namedtuple

import numpy as np

from pink_b200 import _cabi

_HERE = os.path.dirname(os.path.abspath(__file__))
# PK_HOSTSIM_SANITIZE=1: AddressSanitizer + UBSan build of the same sources (run the suite
# with LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0)
_SANITIZE = os.environ.get("PK_HOSTSIM_SANITIZE", "0") == "1"
# PK_HOSTSIM_FMA=1: a*b + c contracted into FMAs, as nvcc does for the device build (a second
# rounding pattern of the same source; `PK_HOSTSIM_FMA=1 python -m pytest tests -m "not gpu"`)
_FMA = os.environ.get("PK_HOSTSIM_FMA", "0") == "1"
_SO = os.path.join(_HERE, "libpk_hostsim_asan.so" if _SANITIZE else "libpk_hostsim_fma.so" if _FMA else "libpk_hostsim.so")
_SRC = os.path.join(_HERE, "hostsim.cpp")
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
        _lib.hs_last_error.restype = C.c_char_p
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# The CUDA library's kernel selection for a problem (pk_select.hpp): path "chain" / "tree" /
# "general"; the chain kernels' <NJ, NFT>; generic = <NJMAX, NVMAX> of ik_generic_kernel; lanes per
# instance of the sub-warp chain kernel (0: ik_chain_kernel); pdl_row_fits: the targets row fits the
# PDL chain kernel's copy; K: task rows of the tree plan.
Selection = namedtuple("Selection", "path nj nft generic lanes pdl_row_fits K")


def _selection(sel):
    return Selection(("chain", "tree", "general")[sel[0]], sel[1], sel[2], (sel[3], sel[4]), sel[5], bool(sel[6]),
                     sel[7])


class HostSim:
    """Runs the kernel bodies on the CPU for one model."""

    def __init__(self, model):
        self.table = model.table()
        self.holder = _cabi.ModelDescHolder(self.table)
        self.handle = C.c_void_p()
        rc = lib().hs_model_create(C.byref(self.holder.desc), C.byref(self.handle))
        if rc:
            raise RuntimeError(lib().hs_last_error().decode())
        self.nq, self.nv, self.nframes = self.table.nq, self.table.nv, self.table.nframes

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

    @staticmethod
    def _f32(a, cols=None):
        a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
        if a.ndim == 1:
            a = a[None]
        return a

    def solve_ik(self, prob, q, targets=None, general_path=False, path=None):
        """path: see hs_solve_ik; ``self.selection`` is the kernel selection the body ran."""
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        v = np.zeros((B, self.nv), dtype=np.float32)
        st = np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        self._chk(lib().hs_solve_ik(self.handle, C.byref(prob), _p(q), _p(t), _p(v), _p(st),
                                    C.c_int64(B), (1 if general_path else 0) if path is None else path, sel))
        self.selection = _selection(sel)
        return v, st

    def rollout(self, prob, q, targets, n_steps, target_step=None, record=True, path=0):
        """Trajectory rollout with the loop of the selected body (hs_rollout): ``targets`` is
        ``[n_steps, B, stride]`` (step s at ``target_step`` floats from step 0; default: its stride)
        or ``[B, stride]`` (the same rows every step, ``target_step`` 0).  Returns ``(q, v, status,
        q_traj, v_traj, status_traj)``, the records None unless ``record``; ``path`` as
        :meth:`solve_ik`."""
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else np.asarray(targets, dtype=np.float32)
        if t is not None and t.ndim < 3:
            t = self._f32(t)
        if target_step is None:
            target_step = t.strides[0] // 4 if t is not None and t.ndim == 3 else 0
        q_out = np.zeros_like(q)
        v = np.zeros((B, self.nv), dtype=np.float32)
        st = np.zeros(B, dtype=np.int32)
        rec = ((np.zeros((n_steps, B, self.nq), dtype=np.float32), np.zeros((n_steps, B, self.nv), dtype=np.float32),
                np.zeros((n_steps, B), dtype=np.int32)) if record else (None, None, None))
        sel = (C.c_int * 8)()
        self._chk(lib().hs_rollout(self.handle, C.byref(prob), _p(q), _p(t), C.c_int64(target_step), n_steps,
                                   _p(q_out), _p(v), _p(st), *map(_p, rec), C.c_int64(B), path, sel))
        self.selection = _selection(sel)
        return (q_out, v, st) + rec

    def converge(self, prob, q, targets, mask, tol, max_steps, path=0):
        """Solve to a tolerance with the converge loop of the selected body (hs_converge):
        ``(q_out, err, steps, status)``; ``path`` as :meth:`solve_ik`, and ``self.selection``
        the kernel selection the loop ran."""
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        q_out = np.zeros_like(q)
        err = np.zeros(B, dtype=np.float32)
        steps = np.zeros(B, dtype=np.int32)
        st = np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        self._chk(lib().hs_converge(self.handle, C.byref(prob), _p(q), _p(t), C.c_uint32(mask), C.c_float(tol),
                                    C.c_int(max_steps), _p(q_out), _p(err), _p(steps), _p(st), C.c_int64(B), path,
                                    sel))
        self.selection = _selection(sel)
        return q_out, err, steps, st

    def converge_multistart(self, prob, q_seeds, targets, mask, tol, max_steps, path=0):
        """Multi-start solve to a tolerance (hs_converge_multistart): ``q_seeds [B, S, nq]`` ->
        ``(q_out, err, seed, steps, status)``; ``path`` as :meth:`solve_ik` (0: the library's
        selection, 1: the general path, 2: the tree kernel)."""
        qs = self._f32(q_seeds)
        B, S, nq = qs.shape
        t = None if targets is None else self._f32(targets)
        q_out = np.zeros((B, nq), dtype=np.float32)
        err = np.zeros(B, dtype=np.float32)
        seed = np.zeros(B, dtype=np.int32)
        steps = np.zeros(B, dtype=np.int32)
        st = np.zeros(B, dtype=np.int32)
        sel = (C.c_int * 8)()
        self._chk(lib().hs_converge_multistart(self.handle, C.byref(prob), _p(qs), S, _p(t), C.c_uint32(mask),
                                               C.c_float(tol), C.c_int(max_steps), _p(q_out), _p(err), _p(seed),
                                               _p(steps), _p(st), C.c_int64(B), path, sel))
        self.selection = _selection(sel)
        return q_out, err, seed, steps, st

    @property
    def used_chain(self):
        return self.selection.path == "chain"

    @property
    def used_tree(self):
        return self.selection.path == "tree"

    def build_ik(self, prob, q, targets=None):
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        H = np.zeros((B, self.nv, self.nv), dtype=np.float32)
        c = np.zeros((B, self.nv), dtype=np.float32)
        h = np.zeros((B, 4, self.nv), dtype=np.float32)
        self._chk(lib().hs_build_ik(self.handle, C.byref(prob), _p(q), _p(t), _p(H), _p(c), _p(h), C.c_int64(B)))
        return H, c, h

    def constraint_rows(self, prob, q, targets=None):
        """(G, hG, E, f, lo, hi) of every instance (pk_constraint_rows_batched)."""
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        G = np.zeros((B, _cabi.PK_MAX_INEQ_ROWS, self.nv), dtype=np.float32)
        hG = np.zeros((B, _cabi.PK_MAX_INEQ_ROWS), dtype=np.float32)
        E = np.zeros((B, _cabi.PK_MAX_EQ_ROWS, self.nv), dtype=np.float32)
        f = np.zeros((B, _cabi.PK_MAX_EQ_ROWS), dtype=np.float32)
        lo = np.zeros((B, self.nv), dtype=np.float32)
        hi = np.zeros((B, self.nv), dtype=np.float32)
        self._chk(lib().hs_constraint_rows(self.handle, C.byref(prob), _p(q), _p(t), _p(G), _p(hG), _p(E), _p(f),
                                           _p(lo), _p(hi), C.c_int64(B)))
        return G, hG, E, f, lo, hi

    def task_terms(self, prob, task_index, k, q, targets=None):
        q = self._f32(q)
        B = q.shape[0]
        t = None if targets is None else self._f32(targets)
        e = np.zeros((B, k), dtype=np.float32)
        J = np.zeros((B, k, self.nv), dtype=np.float32)
        self._chk(lib().hs_task_terms(self.handle, C.byref(prob), task_index, _p(q), _p(t), _p(e), _p(J), C.c_int64(B)))
        return e, J

    def forward_kinematics(self, q):
        q = self._f32(q)
        B = q.shape[0]
        oMf = np.zeros((B, self.nframes, 3, 4), dtype=np.float32)
        com = np.zeros((B, 3), dtype=np.float32)
        self._chk(lib().hs_forward_kinematics(self.handle, _p(q), _p(oMf), _p(com), C.c_int64(B)))
        return oMf, com

    def integrate(self, q, v, dt):
        q, v = self._f32(q), self._f32(v)
        out = np.zeros_like(q)
        self._chk(lib().hs_integrate(self.handle, _p(q), _p(v), C.c_float(dt), _p(out), C.c_int64(q.shape[0])))
        return out

    def frame_jacobian(self, frame, q):
        q = self._f32(q)
        B = q.shape[0]
        J = np.zeros((B, 6, self.nv), dtype=np.float32)
        self._chk(lib().hs_frame_jacobian(self.handle, frame, _p(q), _p(J), C.c_int64(B)))
        return J

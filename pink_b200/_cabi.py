"""ctypes binding of ``include/pink_b200.h`` (the C-ABI of the CUDA library).

This is the only place the shared library is loaded.  There is no CPU
fallback: if ``libpink_b200.so`` is missing, or no CUDA device is usable, every
compute entry point raises.
"""

from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

PK_MAX_JOINTS = 58
PK_MAX_NV = 64
PK_MAX_FRAMES = 256
PK_MAX_TASKS = 12
PK_MAX_SHARED = 192
PK_MAX_INEQ_ROWS = 24
PK_MAX_EQ_ROWS = 12
PK_MAX_BARRIERS = 8
PK_MAX_CONSTRAINTS = 4
PK_MAX_PAIRS = 256
PK_MAX_PEERS = 16
PK_IPC_HANDLE_BYTES = 64
PK_PEER_FLAG_WORDS = 48
PK_ABI_VERSION = 3

PK_STATUS_NO_SOLUTION = 1
PK_STATUS_OUT_OF_LIMITS = 2
PK_STATUS_NOT_POSDEF = 4
PK_STATUS_ITER_LIMIT = 8

PK_TASK_FRAME, PK_TASK_RELATIVE_FRAME, PK_TASK_POSTURE, PK_TASK_COM, PK_TASK_JOINT_VELOCITY, PK_TASK_LINEAR = 0, 1, 2, 3, 4, 5
PK_BARRIER_POSITION, PK_BARRIER_BODY_SPHERICAL, PK_BARRIER_SELF_COLLISION = 0, 1, 2
PK_GAINFN_IDENTITY, PK_GAINFN_SATURATING = 0, 1

_LIB_NAME = "libpink_b200.so"
_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


class PkModelDesc(C.Structure):
    _fields_ = [
        ("njoints", C.c_int32),
        ("free_flyer", C.c_int32),
        ("nq", C.c_int32),
        ("nv", C.c_int32),
        ("parent", C.POINTER(C.c_int32)),
        ("jtype", C.POINTER(C.c_int32)),
        ("joint_placement", C.POINTER(C.c_double)),
        ("axis", C.POINTER(C.c_double)),
        ("nframes", C.c_int32),
        ("frame_body", C.POINTER(C.c_int32)),
        ("frame_placement", C.POINTER(C.c_double)),
        ("mass", C.POINTER(C.c_double)),
        ("com", C.POINTER(C.c_double)),
    ]


class PkTaskDesc(C.Structure):
    _fields_ = [
        ("type", C.c_int32),
        ("frame", C.c_int32),
        ("root", C.c_int32),
        ("target_offset", C.c_int32),
        ("target_shared", C.c_int32),
        ("cost", C.c_float * 6),
        ("gain", C.c_float),
        ("lm_damping", C.c_float),
        ("rows", C.c_int32),
        ("data_offset", C.c_int32),
    ]


class PkBarrierDesc(C.Structure):
    _fields_ = [
        ("type", C.c_int32),
        ("frame", C.c_int32),
        ("frame2", C.c_int32),
        ("dim", C.c_int32),
        ("nidx", C.c_int32),
        ("indices", C.c_int32 * 3),
        ("has_min", C.c_int32),
        ("has_max", C.c_int32),
        ("p_min", C.c_float * 3),
        ("p_max", C.c_float * 3),
        ("gain", C.c_float * 6),
        ("d_min", C.c_float),
        ("safe_displacement_gain", C.c_float),
        ("gain_function", C.c_int32),
        ("npairs", C.c_int32),
        ("pair_offset", C.c_int32),
        ("data_offset", C.c_int32),
    ]


class PkProblemDesc(C.Structure):
    _fields_ = [
        ("ntasks", C.c_int32),
        ("tasks", PkTaskDesc * PK_MAX_TASKS),
        ("dt", C.c_float),
        ("damping", C.c_float),
        ("target_stride", C.c_int32),
        ("safety_break", C.c_int32),
        ("cfg_gain", C.c_float),
        ("cfg_lo", C.c_float * PK_MAX_NV),
        ("cfg_hi", C.c_float * PK_MAX_NV),
        ("vel", C.c_float * PK_MAX_NV),
        ("chk_lo", C.c_float * PK_MAX_NV),
        ("chk_hi", C.c_float * PK_MAX_NV),
        ("shared", C.c_float * PK_MAX_SHARED),
        ("nbarriers", C.c_int32),
        ("barriers", PkBarrierDesc * PK_MAX_BARRIERS),
        ("nconstraints", C.c_int32),
        ("constraints", PkTaskDesc * PK_MAX_CONSTRAINTS),
        ("fb_enabled", C.c_int32),
        ("fb_frame", C.c_int32),
        ("fb_max", C.c_float * 6),
        ("acc_enabled", C.c_int32),
        ("acc_prev_offset", C.c_int32),
        ("acc_prev_shared", C.c_int32),
        ("acc_max", C.c_float * PK_MAX_NV),
        ("acc_qlo", C.c_float * PK_MAX_NV),
        ("acc_qhi", C.c_float * PK_MAX_NV),
        ("extra", C.POINTER(C.c_float)),
        ("n_extra", C.c_int32),
        ("pairs", C.POINTER(C.c_int32)),
        ("n_pairs", C.c_int32),
    ]


def _dptr(a: np.ndarray, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


class ModelDescHolder:
    """Owns the numpy arrays a ``PkModelDesc`` points into."""

    def __init__(self, table):
        nj = int(table.njoints)
        self.parent = np.ascontiguousarray(table.parent, dtype=np.int32)
        self.jtype = np.ascontiguousarray(table.jtype, dtype=np.int32)
        jp = np.concatenate([np.asarray(table.joint_R).reshape(nj, 3, 3), np.asarray(table.joint_p).reshape(nj, 3, 1)], axis=2)
        self.joint_placement = np.ascontiguousarray(jp.reshape(-1), dtype=np.float64)
        self.axis = np.ascontiguousarray(np.asarray(table.axis).reshape(-1), dtype=np.float64)
        nf = int(table.nframes)
        self.frame_body = np.ascontiguousarray(table.frame_body, dtype=np.int32)
        fp = np.concatenate([np.asarray(table.frame_R).reshape(nf, 3, 3), np.asarray(table.frame_p).reshape(nf, 3, 1)], axis=2)
        self.frame_placement = np.ascontiguousarray(fp.reshape(-1), dtype=np.float64)
        self.mass = np.ascontiguousarray(table.mass, dtype=np.float64)
        self.com = np.ascontiguousarray(np.asarray(table.com).reshape(-1), dtype=np.float64)
        d = PkModelDesc()
        d.njoints = nj
        d.free_flyer = 1 if table.free_flyer else 0
        d.nq = int(table.nq)
        d.nv = int(table.nv)
        d.parent = _dptr(self.parent, C.c_int32)
        d.jtype = _dptr(self.jtype, C.c_int32)
        d.joint_placement = _dptr(self.joint_placement, C.c_double)
        d.axis = _dptr(self.axis, C.c_double)
        d.nframes = nf
        d.frame_body = _dptr(self.frame_body, C.c_int32)
        d.frame_placement = _dptr(self.frame_placement, C.c_double)
        d.mass = _dptr(self.mass, C.c_double)
        d.com = _dptr(self.com, C.c_double)
        self.desc = d


_lib: Optional[C.CDLL] = None

_FP = C.c_void_p  # device / host buffers are passed as raw addresses


def declare(lib: C.CDLL, prefix: str = "pk_") -> None:
    """Attach argument / return types of the exported symbols."""
    if prefix != "pk_":
        return
    lib.pk_abi_version.restype = C.c_int
    lib.pk_last_error.restype = C.c_char_p
    lib.pk_launch_count.restype = C.c_int64
    lib.pk_model_create.argtypes = [C.POINTER(PkModelDesc), C.c_int, C.POINTER(C.c_void_p)]
    lib.pk_model_destroy.argtypes = [C.c_void_p]
    lib.pk_model_destroy.restype = None
    lib.pk_model_set_host_schedule.argtypes = [C.c_void_p, C.c_int]
    lib.pk_solve_ik_batched.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_solve_ik_batched_host.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_problem_create.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), C.POINTER(C.c_void_p)]
    lib.pk_problem_destroy.argtypes = [C.c_void_p]
    lib.pk_problem_destroy.restype = None
    lib.pk_solve_ik_prepared.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_solve_ik_prepared_host.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_rollout_prepared.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, C.c_int32, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_rollout_trajectory_prepared.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, C.c_int64, C.c_int32, _FP, _FP, _FP,
                                                   _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_converge_prepared.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, C.c_uint32, C.c_float, C.c_int32, _FP, _FP,
                                         _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_build_ik_batched.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), _FP, _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_constraint_rows_batched.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), _FP, _FP, _FP, _FP, _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_task_terms_batched.argtypes = [C.c_void_p, C.POINTER(PkProblemDesc), C.c_int32, _FP, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_forward_kinematics_batched.argtypes = [C.c_void_p, _FP, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_frame_jacobian_batched.argtypes = [C.c_void_p, C.c_int32, _FP, _FP, C.c_int64, C.c_void_p]
    lib.pk_integrate_batched.argtypes = [C.c_void_p, _FP, _FP, C.c_float, _FP, C.c_int64, C.c_void_p]
    lib.pk_peer_alloc.argtypes = [C.c_int, C.c_int64, C.POINTER(C.c_void_p), C.c_char_p]
    lib.pk_peer_open.argtypes = [C.c_int, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.pk_peer_close.argtypes = [C.c_int, C.c_void_p]
    lib.pk_peer_free.argtypes = [C.c_int, C.c_void_p]
    lib.pk_solve_ik_prepared_gather.argtypes = [C.c_void_p, C.c_void_p, _FP, _FP, _FP, _FP, C.c_int64,
                                                C.POINTER(C.c_void_p), C.c_int32, C.c_int64,
                                                C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_void_p]
    lib.pk_peer_sync.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p]


EXPORTED_SYMBOLS = [
    "pk_abi_version",
    "pk_struct_size",
    "pk_last_error",
    "pk_launch_count",
    "pk_model_create",
    "pk_model_destroy",
    "pk_model_set_host_schedule",
    "pk_solve_ik_batched",
    "pk_solve_ik_batched_host",
    "pk_problem_create",
    "pk_problem_destroy",
    "pk_solve_ik_prepared",
    "pk_solve_ik_prepared_host",
    "pk_rollout_prepared",
    "pk_rollout_trajectory_prepared",
    "pk_converge_prepared",
    "pk_build_ik_batched",
    "pk_constraint_rows_batched",
    "pk_task_terms_batched",
    "pk_forward_kinematics_batched",
    "pk_frame_jacobian_batched",
    "pk_integrate_batched",
    "pk_peer_alloc",
    "pk_peer_open",
    "pk_peer_close",
    "pk_peer_free",
    "pk_solve_ik_prepared_gather",
    "pk_peer_sync",
]


def library_path() -> str:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load ``libpink_b200.so`` (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError(
                f"{_LIB_NAME} not found at {_LIB_PATH}: build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` "
                "(pink_b200 has no CPU fallback)"
            )
        lib = C.CDLL(_LIB_PATH)
        declare(lib)
        if lib.pk_abi_version() != PK_ABI_VERSION:
            raise RuntimeError("libpink_b200.so ABI version mismatch; rebuild")
        for which, struct in enumerate((PkModelDesc, PkTaskDesc, PkBarrierDesc, PkProblemDesc)):
            if lib.pk_struct_size(which) != C.sizeof(struct):
                raise RuntimeError(f"libpink_b200.so: layout of {struct.__name__} differs from the binding; rebuild")
        _lib = lib
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("pink_b200: " + load().pk_last_error().decode("utf-8", "replace"))

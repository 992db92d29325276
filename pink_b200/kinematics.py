"""Differentiable batched forward kinematics: placements of selected frames and the CoM, with a
gradient in q behind ``torch.autograd`` (``pk_frame_placements_batched`` and
``pk_frame_placements_vjp_batched``, DESIGN.md section 3.2i).

    from pink_b200 import kinematics
    fp = kinematics.frame_placements(model, q, ["tool0", "forearm_link"], com=True)
    fp.oMf   # [B, F, 3, 4]
    fp.com   # [B, 3] (None without com=True)

The gradient is in q coordinates, the form :meth:`BatchedIK.converge_vjp` takes, so a loss of
``frame_placements(model, converge(...).q, ...)`` backpropagates to the targets of ``converge``."""

from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Sequence, Union

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _cabi
from .engine import _addr, _stream, get_engine
from .exceptions import FrameNotFound


class FramePlacements(NamedTuple):
    """``oMf [B, F, 3, 4]``: ``[R | p]`` of each requested frame in the world; ``com [B, 3]`` or
    None."""

    oMf: torch.Tensor
    com: Optional[torch.Tensor]


def _frame_indices(model, frames: Sequence[Union[str, int]]) -> np.ndarray:
    out = []
    for f in frames:
        if isinstance(f, str):
            if not model.existFrame(f):
                raise FrameNotFound(f, model.frames)
            out.append(model.getFrameId(f))
        else:
            k = int(f)
            if not 0 <= k < len(model.frames):
                raise ValueError(f"frame index {k} out of range [0, {len(model.frames)})")
            out.append(k)
    if len(out) > _cabi.PK_MAX_FRAMES:
        raise ValueError(f"at most {_cabi.PK_MAX_FRAMES} frames per call, got {len(out)}")
    return np.ascontiguousarray(out, dtype=np.int32)


def _forward(eng, frames: np.ndarray, q: torch.Tensor, com: bool):
    B = q.shape[0]
    oMf = torch.empty((B, frames.size, 3, 4), device=eng.device, dtype=torch.float32)
    c = torch.empty((B, 3), device=eng.device, dtype=torch.float32) if com else None
    with torch.cuda.device(eng.device):
        _cabi.check(eng.lib.pk_frame_placements_batched(eng.handle, frames.ctypes.data_as(C.c_void_p), frames.size,
                                                        _addr(q), _addr(oMf), _addr(c), B, _stream(eng.device)))
    return oMf, c


def frame_placements_vjp(model, q: torch.Tensor, frames: Sequence[Union[str, int]],
                         grad_oMf: Optional[torch.Tensor] = None, grad_com: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``grad_q [B, nq] = (d (oMf, com) / d q)^T (grad_oMf, grad_com)`` in one launch: the explicit
    form of the backward of :func:`frame_placements`.  ``grad_oMf [B, F, 3, 4]`` and ``grad_com
    [B, 3]`` may each be None (that term is zero).  On a free-flyer root the quaternion gets the
    gradient of the normalised map, so its component along the quaternion is zero."""
    q = _check_q(model, q)
    eng = get_engine(model, q.device)
    f = _frame_indices(model, frames)
    B = q.shape[0]

    def rows(t, shape, what):
        if t is None:
            return None
        if tuple(t.shape) != shape:
            raise ValueError(f"{what} has shape {tuple(t.shape)}, expected {shape}")
        return t.detach().to(device=eng.device, dtype=torch.float32).contiguous()

    gF = rows(grad_oMf, (B, f.size, 3, 4), "grad_oMf")
    gc = rows(grad_com, (B, 3), "grad_com")
    gq = torch.empty((B, eng.nq), device=eng.device, dtype=torch.float32)
    with torch.cuda.device(eng.device):
        _cabi.check(eng.lib.pk_frame_placements_vjp_batched(eng.handle, f.ctypes.data_as(C.c_void_p), f.size, _addr(q),
                                                            _addr(gF), _addr(gc), _addr(gq), B, _stream(eng.device)))
    return gq


class _FramePlacementsOfQ(torch.autograd.Function):
    """``(oMf, com)`` as a function of ``q``: the backward is one ``pk_frame_placements_vjp_batched``
    launch; an output that received no gradient is passed as NULL."""

    @staticmethod
    def forward(ctx, q, model, frames, com):
        ctx.set_materialize_grads(False)
        ctx.model, ctx.frames, ctx.com = model, frames, com
        qd = q.detach()
        ctx.save_for_backward(qd)
        oMf, c = _forward(get_engine(model, q.device), frames, qd, com)
        return (oMf, c) if com else oMf

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        (q,) = ctx.saved_tensors
        grad_oMf = grads[0]
        grad_com = grads[1] if ctx.com else None
        if grad_oMf is None and grad_com is None:
            return None, None, None, None
        return frame_placements_vjp(ctx.model, q, ctx.frames, grad_oMf, grad_com), None, None, None


def _check_q(model, q) -> torch.Tensor:
    if not isinstance(q, torch.Tensor):
        raise ValueError("q must be a torch.Tensor")
    if q.dtype != torch.float32:
        raise ValueError(f"q must be float32, got {q.dtype}")
    if q.dim() != 2 or q.shape[1] != model.nq:
        raise ValueError(f"q has shape {tuple(q.shape)}, expected [B, {model.nq}]")
    if not q.is_cuda:
        raise ValueError("q must be on a CUDA device")
    return q.contiguous()


def frame_placements(model, q: torch.Tensor, frames: Sequence[Union[str, int]], com: bool = False) -> FramePlacements:
    """World placements of ``frames`` (names or indices; repeats allowed) and, with ``com=True``,
    the centre of mass, at ``q [B, nq]`` (float32, on a CUDA device): one launch.  The values are
    bitwise those of ``Configuration.get_transform_frame_to_world`` / ``get_center_of_mass``.

    When grad mode is on and ``q.requires_grad``, both outputs carry one autograd node whose
    backward is a single :func:`frame_placements_vjp` launch (double backward is not supported);
    otherwise no node is created.  Unknown names raise ``FrameNotFound``; a CoM request on a model
    of total mass 0 raises ``RuntimeError``.  Asynchronous on the current stream, no allocation
    inside the library, so the call can be captured in a CUDA graph."""
    qc = _check_q(model, q)
    f = _frame_indices(model, frames)
    if torch.is_grad_enabled() and q.requires_grad:
        out = _FramePlacementsOfQ.apply(qc, model, f, bool(com))
        return FramePlacements(*out) if com else FramePlacements(out, None)
    return FramePlacements(*_forward(get_engine(model, q.device), f, qc.detach(), bool(com)))

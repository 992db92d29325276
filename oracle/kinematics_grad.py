"""Gradient of frame placements and the CoM with respect to q, in fp64 (the oracle of
``pk_frame_placements_vjp_batched``).

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  Written from the formulas of DESIGN.md
section 3.2i, independently of the C++ body; model tables as in ``oracle/kinematics.py``."""

import numpy as np

from .kinematics import _body_placement, forward_kinematics, frame_placement, root_dims


def frame_placements_vjp(m, q, frames, G, g_com=None):
    """Gradient in q coordinates of ``L = sum_k <G[k], oMf[frames[k]]> + g_com . com``
    (``pk_frame_placements_vjp_batched``, DESIGN.md section 3.2i): ``q [..., nq]``, ``G [..., F, 3, 4]``
    (or None) with ``[G_R | g_p]`` per frame, ``g_com [..., 3]`` (or None) -> ``[..., nq]``.

    A reverse sweep over the tree: every frame contributes the world force ``g_p`` and the moment
    about the origin ``vee(G_R R^T - R G_R^T) + p x g_p``, the CoM gradient the force ``(m_b / M) g_com``
    at each body's CoM; the pairs are summed over subtrees and joint ``j`` gets ``a_j . (N - o_j x F)``
    (revolute) or ``a_j . F`` (prismatic).  On a free-flyer the translation gets the total force and
    the quaternion the derivative of the normalised rotation map (no radial component)."""
    q = np.asarray(q, dtype=np.float64)
    batch = q.shape[:-1]
    fk = forward_kinematics(m, q)
    R_root, p_root, R, p = fk
    nj = m.njoints
    rq, _ = root_dims(m)
    F = np.zeros(batch + (nj + 1, 3))  # index body + 1: the root body, then the joints
    N = np.zeros(batch + (nj + 1, 3))

    def moving(body):
        return body >= 0 or (body == -1 and m.free_flyer)

    if G is not None:
        G = np.asarray(G, dtype=np.float64)
        for k, f in enumerate(frames):
            body = int(m.frame_body[f])
            if not moving(body):
                continue
            Rf, pf = frame_placement(m, fk, f)
            GR, gp = G[..., k, :, :3], G[..., k, :, 3]
            S = GR @ np.swapaxes(Rf, -1, -2)
            A = S - np.swapaxes(S, -1, -2)
            F[..., body + 1, :] += gp
            N[..., body + 1, :] += np.stack([A[..., 2, 1], A[..., 0, 2], A[..., 1, 0]], axis=-1) + np.cross(pf, gp)
    if g_com is not None:
        g_com = np.asarray(g_com, dtype=np.float64)
        mass = np.asarray(m.mass, dtype=np.float64)
        for b in range(-1, nj):
            if mass[b + 1] == 0.0 or not moving(b):
                continue
            Rb, pb = _body_placement(m, fk, b)
            x = pb + np.einsum("...ij,j->...i", Rb, np.asarray(m.com[b + 1], dtype=np.float64))
            f = (mass[b + 1] / mass.sum()) * g_com
            F[..., b + 1, :] += f
            N[..., b + 1, :] += np.cross(x, f)
    out = np.zeros(batch + (m.nq,))
    for j in range(nj - 1, -1, -1):
        a = np.einsum("...ij,j->...i", R[..., j, :, :], np.asarray(m.axis[j], dtype=np.float64))
        Fj, Nj = F[..., j + 1, :], N[..., j + 1, :]
        if int(m.jtype[j]) == 0:
            out[..., rq + j] = np.sum(a * (Nj - np.cross(p[..., j, :], Fj)), axis=-1)
        else:
            out[..., rq + j] = np.sum(a * Fj, axis=-1)
        par = int(m.parent[j])
        F[..., par + 1, :] += Fj
        N[..., par + 1, :] += Nj
    if m.free_flyer:
        Fr, Nr = F[..., 0, :], N[..., 0, :]
        out[..., 0:3] = Fr
        # dR = [dw]x R with dw = 2 (w dv - dw_s v + v x dv) for the unit quaternion (v, w); chain
        # through u = quat / |quat|: du = (I - u u^T) dquat / |quat|
        tau = Nr - np.cross(p_root, Fr)
        quat = q[..., 3:7]
        n = np.linalg.norm(quat, axis=-1, keepdims=True)
        u = quat / n
        v, w = u[..., :3], u[..., 3:4]
        g_u = np.concatenate([2.0 * (w * tau + np.cross(tau, v)), -2.0 * np.sum(tau * v, axis=-1, keepdims=True)],
                             axis=-1)
        g_u = g_u - np.sum(g_u * u, axis=-1, keepdims=True) * u
        out[..., 3:7] = g_u / n
    return out

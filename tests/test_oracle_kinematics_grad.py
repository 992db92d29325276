"""The fp64 oracle of the frame-placement gradient (``oracle.kinematics_grad.frame_placements_vjp``)
against central differences of the oracle's forward kinematics, to 1e-7 of the gradient's
largest entry: UR5 with a frame on the fixed base, a chain with prismatic joints, a free-flyer
tree at quaternion norms 0.7, 1.0 and 1.3, G1 with the CoM, and a repeated frame."""

import numpy as np
import pytest

from oracle import kinematics as okin
from oracle import kinematics_grad as okg
from pink_b200 import workloads
from tests import helpers


def loss(m, q, frames, G, g_com):
    """``sum_k <G[k], oMf[frames[k]]> + g_com . com`` at ``q [B, nq]`` (fp64)."""
    fk = okin.forward_kinematics(m, q)
    out = np.zeros(q.shape[:-1])
    for k, f in enumerate(frames):
        R, p = okin.frame_placement(m, fk, f)
        out += np.sum(G[..., k, :, :3] * R, axis=(-2, -1)) + np.sum(G[..., k, :, 3] * p, axis=-1)
    if g_com is not None:
        out += np.sum(g_com * okin.center_of_mass(m, fk), axis=-1)
    return out


def central_differences(m, q, frames, G, g_com, h=1e-6):
    g = np.zeros_like(q)
    for i in range(m.nq):
        d = np.zeros(m.nq)
        d[i] = h
        g[..., i] = (loss(m, q + d, frames, G, g_com) - loss(m, q - d, frames, G, g_com)) / (2 * h)
    return g


def check(m, q, frames, com=False, seed=0):
    rng = np.random.default_rng(seed)
    B = q.shape[0]
    G = rng.normal(size=(B, len(frames), 3, 4))
    g_com = rng.normal(size=(B, 3)) if com else None
    g = okg.frame_placements_vjp(m, q, frames, G, g_com)
    fd = central_differences(m, q, frames, G, g_com)
    scale = np.abs(fd).max(axis=-1, keepdims=True)
    assert (np.abs(g - fd) <= 1e-7 * scale + 1e-12).all(), np.max(np.abs(g - fd) / scale)
    return g


def test_ur5_frames_and_a_frame_on_the_fixed_base():
    _, model, m = helpers.load("ur5_description")
    q = workloads.sample_configurations(m, 16, np.random.default_rng(1))
    base = m.frame_names.index("base_link")
    assert int(m.frame_body[base]) < 0
    frames = [m.frame_names.index(n) for n in ("tool0", "forearm_link", "wrist_2_link")] + [base]
    check(m, q, frames)
    # the base frame alone: it does not move, its gradient is zero
    G = np.random.default_rng(2).normal(size=(16, 1, 3, 4))
    assert not okg.frame_placements_vjp(m, q, [base], G).any()


def test_chain_with_prismatic_joints():
    rng = np.random.default_rng(3)
    m = helpers.random_chain_model(7, rng, prismatic=(2, 5)).table()
    q = workloads.sample_configurations(m, 16, rng)
    check(m, q, [m.frame_names.index("tool"), m.frame_names.index("elbow")], com=True)


@pytest.mark.parametrize("norm", [0.7, 1.0, 1.3])
def test_free_flyer_tree_at_quaternion_norms(norm):
    rng = np.random.default_rng(4)
    m = helpers.random_tree_model(40, rng, free_flyer=True).table()
    q = workloads.sample_configurations(m, 8, rng)
    q[:, 3:7] *= norm / np.linalg.norm(q[:, 3:7], axis=1, keepdims=True)
    frames = [m.frame_names.index(f"tip{k}") for k in range(4)]
    g = check(m, q, frames, com=True)
    radial = np.sum(g[:, 3:7] * q[:, 3:7], axis=1)
    assert (np.abs(radial) <= 1e-12 * np.abs(g).max(axis=1)).all()


def test_g1_with_the_com():
    _, model, m = helpers.load("g1_description")
    q = workloads.sample_configurations(m, 8, np.random.default_rng(5))
    frames = [m.frame_names.index(n) for n in ("left_ankle_roll_link", "right_ankle_roll_link", "pelvis")]
    check(m, q, frames, com=True)
    check(m, q, [], com=True, seed=1)


def test_a_repeated_frame_gets_the_sum_of_its_gradients():
    _, model, m = helpers.load("ur5_description")
    q = workloads.sample_configurations(m, 8, np.random.default_rng(6))
    f = m.frame_names.index("tool0")
    rng = np.random.default_rng(7)
    G = rng.normal(size=(8, 2, 3, 4))
    both = okg.frame_placements_vjp(m, q, [f, f], G)
    one = okg.frame_placements_vjp(m, q, [f], G[:, :1]) + okg.frame_placements_vjp(m, q, [f], G[:, 1:])
    np.testing.assert_allclose(both, one, rtol=1e-13, atol=1e-13)
    check(m, q, [f, f])

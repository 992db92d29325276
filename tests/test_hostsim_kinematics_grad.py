"""Host build of the differentiable forward kinematics (pk_kinematics.cuh through
tests/hostsim_kinematics): the placements and CoM against the fp64 oracle, the reverse sweep against
``oracle.kinematics_grad.frame_placements_vjp`` at each size class of the general path, and the argument
checks of ``pk_frame_placements_batched`` / ``pk_frame_placements_vjp_batched``.  Also run with
``PK_HOSTSIM_FMA=1`` and under ``PK_HOSTSIM_SANITIZE=1``."""

import numpy as np
import pytest

from oracle import kinematics as okin
from oracle import kinematics_grad as okg
from pink_b200 import workloads
from tests import helpers
from tests.hostsim_kinematics import HostKinematics


def case(name):
    """``(model, table, frames, com, q [B, nq])`` at one size class: <8, 8> UR5, <30, 36> G1,
    <58, 64> a 40-joint free-flyer tree."""
    rng = np.random.default_rng(11)
    if name == "ur5":
        _, model, m = helpers.load("ur5_description")
        frames = [m.frame_names.index(n) for n in ("tool0", "forearm_link", "upper_arm_link", "base_link", "tool0")]
        com = False
    elif name == "g1":
        _, model, m = helpers.load("g1_description")
        frames = [m.frame_names.index(n) for n in ("left_ankle_roll_link", "right_ankle_roll_link", "left_wrist_yaw_link",
                                                   "right_wrist_yaw_link", "pelvis")]
        com = True
    else:
        model = helpers.random_tree_model(40, rng, free_flyer=True)
        m = model.table()
        frames = [m.frame_names.index(f"tip{k}") for k in range(4)]
        com = True
    q = workloads.sample_configurations(m, 64, rng)
    if m.free_flyer:
        q[:, 3:7] *= rng.uniform(0.7, 1.3, size=(64, 1))
    return model, m, frames, com, q.astype(np.float32)


def oracle_forward(m, q, frames):
    fk = okin.forward_kinematics(m, q.astype(np.float64))
    oMf = np.stack([np.concatenate([R, p[..., None]], axis=-1) for R, p in (okin.frame_placement(m, fk, f)
                                                                              for f in frames)], axis=1)
    return oMf, okin.center_of_mass(m, fk)


def within(g, g_ref):
    """|g - g_ref| <= 1e-4 max|g_ref| + 1e-6, row by row."""
    bound = 1e-4 * np.abs(g_ref).max(axis=1, keepdims=True) + 1e-6
    return np.abs(g - g_ref) <= bound


@pytest.mark.parametrize("name", ["ur5", "g1", "tree40"])
def test_forward_against_the_oracle(name):
    model, m, frames, com, q = case(name)
    oMf, c = HostKinematics(model).frame_placements(frames, q, com=com)
    ref, c_ref = oracle_forward(m, q, frames)
    np.testing.assert_allclose(oMf, ref, atol=2e-5)
    if com:
        np.testing.assert_allclose(c, c_ref, atol=2e-5)


@pytest.mark.parametrize("name", ["ur5", "g1", "tree40"])
@pytest.mark.parametrize("terms", ["frames", "com", "both"])
def test_vjp_against_the_oracle(name, terms):
    model, m, frames, com, q = case(name)
    if terms != "frames" and not com:
        pytest.skip("no CoM term on this case")
    rng = np.random.default_rng(12)
    G = rng.normal(size=(q.shape[0], len(frames), 3, 4)).astype(np.float32) if terms != "com" else None
    gc = rng.normal(size=(q.shape[0], 3)).astype(np.float32) if terms != "frames" else None
    g = HostKinematics(model).frame_placements_vjp(frames, q, G, gc)
    g_ref = okg.frame_placements_vjp(m, q.astype(np.float64), frames, None if G is None else G.astype(np.float64),
                                      None if gc is None else gc.astype(np.float64))
    assert np.isfinite(g).all()
    ok = within(g, g_ref)
    assert ok.all(), np.max(np.abs(g - g_ref) / (np.abs(g_ref).max(axis=1, keepdims=True) + 1e-30))
    if m.free_flyer:
        radial = np.sum(g[:, 3:7] * q[:, 3:7], axis=1)
        assert (np.abs(radial) <= 1e-5 * np.abs(g).max(axis=1)).all()


def test_no_terms_and_fixed_frames_give_zero():
    model, m, _, _, q = case("ur5")
    hv = HostKinematics(model)
    assert not hv.frame_placements_vjp([], q).any()
    base = m.frame_names.index("base_link")
    G = np.ones((q.shape[0], 1, 3, 4), dtype=np.float32)
    assert not hv.frame_placements_vjp([base], q, G).any()


def test_repeated_frame_gets_the_sum():
    model, m, _, _, q = case("ur5")
    hv = HostKinematics(model)
    f = m.frame_names.index("tool0")
    G = np.random.default_rng(13).normal(size=(q.shape[0], 2, 3, 4)).astype(np.float32)
    both = hv.frame_placements_vjp([f, f], q, G)
    one = hv.frame_placements_vjp([f], q, G[:, :1]) + hv.frame_placements_vjp([f], q, G[:, 1:])
    np.testing.assert_allclose(both, one, rtol=1e-5, atol=1e-5)
    oMf, _ = hv.frame_placements([f, f], q)
    assert np.array_equal(oMf[:, 0], oMf[:, 1])


def test_argument_errors():
    model, m, _, _, q = case("ur5")
    hv = HostKinematics(model)
    with pytest.raises(RuntimeError, match="out of range"):
        hv.frame_placements([m.nframes], q)
    with pytest.raises(RuntimeError, match="out of range"):
        hv.frame_placements_vjp([-1], q, np.zeros((q.shape[0], 1, 3, 4), np.float32))
    frames = np.zeros(1, dtype=np.int32)
    qa = q.ctypes.data
    with pytest.raises(RuntimeError, match="num_frames"):
        hv._chk(hv.frame_placements_raw(frames.ctypes.data, -1, qa, None, None, 1))
    with pytest.raises(RuntimeError, match="num_frames"):
        hv._chk(hv.frame_placements_raw(frames.ctypes.data, 257, qa, None, None, 1))
    with pytest.raises(RuntimeError, match="null frames"):
        hv._chk(hv.frame_placements_raw(None, 1, qa, None, None, 1))
    with pytest.raises(RuntimeError, match="null grad_q"):
        hv._chk(hv.frame_placements_vjp_raw(frames.ctypes.data, 1, qa, None, None, None, 1))
    # B = 0 needs no buffers
    assert hv.frame_placements_vjp_raw(frames.ctypes.data, 1, None, None, None, None, 0) == 0
    # a model of total mass 0 has no CoM to differentiate
    hv0 = HostKinematics(massless_model())
    hq = np.zeros((1, 2), np.float32)
    with pytest.raises(RuntimeError, match="total mass is 0"):
        hv0.frame_placements([0], hq, com=True)
    with pytest.raises(RuntimeError, match="total mass is 0"):
        hv0.frame_placements_vjp([0], hq, None, np.zeros((1, 3), np.float32))
    hv0.frame_placements([0], hq)


def massless_model():
    """Two revolute joints and a frame, no inertias."""
    from pink_b200.model import Model, SE3

    model = Model("massless")
    j = model.add_joint("a", 0, SE3(np.eye(3), np.zeros(3)), np.array([0.0, 0.0, 1.0]), kind="revolute", lower=-1.0,
                        upper=1.0, velocity=1.0)
    j = model.add_joint("b", j, SE3(np.eye(3), np.array([0.1, 0.0, 0.0])), np.array([0.0, 1.0, 0.0]),
                        kind="revolute", lower=-1.0, upper=1.0, velocity=1.0)
    model.add_frame("tip", j, SE3(np.eye(3), np.array([0.1, 0.0, 0.0])))
    assert np.asarray(model.table().mass).sum() == 0.0
    return model

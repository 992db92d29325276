"""GPU suite (`-m gpu`): differentiable forward kinematics, ``frame_placements_kernel`` and
``frame_placements_vjp_kernel`` through ``pink_b200.kinematics``.

* The kernels against the host build of the same bodies at each size class of the general path
  (<8, 8> UR5, <30, 36> G1, <58, 64> a 40-joint free-flyer tree) and against the fp64 oracle.
* The forward bitwise equal to the rows of ``pk_forward_kinematics_batched``, to
  ``Configuration.get_transform_frame_to_world`` and to ``get_center_of_mass``.
* The autograd backward equal to an explicit VJP launch; directional derivatives against central
  differences of the GPU forward.
* ``targets -> converge -> frame_placements -> loss`` against central differences of the whole
  GPU pipeline, on the exactly determined UR5 problem.
* UR5 at B = 65536 and G1 at B = 16384 against the oracle on a slice; CUDA-graph capture; B = 0,
  the error paths, no autograd node without a gradient request; the example."""

import numpy as np
import pytest
import torch

import pink_b200 as pink
from oracle import kinematics as okin
from oracle import kinematics_grad as okg
from oracle import lie
from pink_b200 import kinematics
from pink_b200.exceptions import FrameNotFound
from tests import helpers
from tests.hostsim_kinematics import HostKinematics
from tests.test_hostsim_kinematics_grad import case, massless_model, oracle_forward, within

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator("cuda").manual_seed(seed)


@pytest.mark.parametrize("name", ["ur5", "g1", "tree40"])
def test_kernels_against_host_build_and_oracle(name):
    model, m, frames, com, q = case(name)
    hv = HostKinematics(model)
    qd = torch.as_tensor(q, device="cuda")
    fp = kinematics.frame_placements(model, qd, frames, com=com)
    oMf_h, c_h = hv.frame_placements(frames, q, com=com)
    np.testing.assert_allclose(fp.oMf.cpu().numpy(), oMf_h, atol=2e-6)
    ref, c_ref = oracle_forward(m, q, frames)
    np.testing.assert_allclose(fp.oMf.cpu().numpy(), ref, atol=2e-5)
    if com:
        np.testing.assert_allclose(fp.com.cpu().numpy(), c_h, atol=2e-6)
        np.testing.assert_allclose(fp.com.cpu().numpy(), c_ref, atol=2e-5)
    rng = np.random.default_rng(21)
    G = rng.normal(size=(q.shape[0], len(frames), 3, 4)).astype(np.float32)
    gc = rng.normal(size=(q.shape[0], 3)).astype(np.float32) if com else None
    g = kinematics.frame_placements_vjp(model, qd, frames, torch.as_tensor(G, device="cuda"),
                                        None if gc is None else torch.as_tensor(gc, device="cuda")).cpu().numpy()
    g_h = hv.frame_placements_vjp(frames, q, G, gc)
    assert within(g, g_h).all()
    g_ref = okg.frame_placements_vjp(m, q.astype(np.float64), frames, G.astype(np.float64),
                                      None if gc is None else gc.astype(np.float64))
    assert within(g, g_ref).all()


@pytest.mark.parametrize("name", ["ur5", "g1"])
def test_forward_is_bitwise_the_existing_kinematics(name):
    model, m, frames, com, q = case(name)
    qd = torch.as_tensor(q, device="cuda")
    fp = kinematics.frame_placements(model, qd, frames, com=com)
    conf = pink.Configuration(model, model.createData(), qd)
    eng = conf.engine
    oMf_all, com_all = eng.forward_kinematics(qd, want_com=True)
    assert torch.equal(fp.oMf, oMf_all[:, frames])
    for k, f in enumerate(frames):
        assert torch.equal(fp.oMf[:, k], conf.get_transform_frame_to_world(m.frame_names[f]))
    if com:
        assert torch.equal(fp.com, com_all)
        assert torch.equal(fp.com, conf.get_center_of_mass())


@pytest.mark.parametrize("name", ["ur5", "g1", "tree40"])
def test_autograd_equals_explicit_vjp_and_outputs_do_not_depend_on_grad_mode(name):
    model, m, frames, com, q = case(name)
    qd = torch.as_tensor(q, device="cuda")
    plain = kinematics.frame_placements(model, qd, frames, com=com)
    assert plain.oMf.grad_fn is None
    qg = qd.clone().requires_grad_(True)
    fp = kinematics.frame_placements(model, qg, frames, com=com)
    assert fp.oMf.grad_fn is not None
    assert torch.equal(fp.oMf.detach(), plain.oMf)
    W = torch.randn(fp.oMf.shape, device="cuda", generator=_gen(1))
    Wc = torch.randn((q.shape[0], 3), device="cuda", generator=_gen(2))
    loss = (fp.oMf * W).sum() + ((fp.com * Wc).sum() if com else 0.0)
    loss.backward()
    explicit = kinematics.frame_placements_vjp(model, qd, frames, W, Wc if com else None)
    assert torch.equal(qg.grad, explicit)
    # an output that receives no gradient is passed as NULL: the CoM alone
    if com:
        qc = qd.clone().requires_grad_(True)
        fp = kinematics.frame_placements(model, qc, frames, com=True)
        (fp.com * Wc).sum().backward()
        assert torch.equal(qc.grad, kinematics.frame_placements_vjp(model, qd, frames, None, Wc))
    with torch.no_grad():
        assert kinematics.frame_placements(model, qg, frames).oMf.grad_fn is None


@pytest.mark.parametrize("name", ["ur5", "g1", "tree40"])
def test_directional_derivatives_against_central_differences_of_the_gpu_forward(name):
    model, m, frames, com, q = case(name)
    qd = torch.as_tensor(q, device="cuda", dtype=torch.float32)
    W = torch.randn((q.shape[0], len(frames), 3, 4), device="cuda", generator=_gen(3))
    Wc = torch.randn((q.shape[0], 3), device="cuda", generator=_gen(4)) if com else None

    def L(qq):
        fp = kinematics.frame_placements(model, qq, frames, com=com)
        out = (fp.oMf.double() * W.double()).sum((1, 2, 3))
        return out + ((fp.com.double() * Wc.double()).sum(1) if com else 0.0)

    d = torch.randn(qd.shape, device="cuda", generator=_gen(5))
    h = 1e-2
    fd = (L(qd + h * d) - L(qd - h * d)) / (2 * h)
    g = kinematics.frame_placements_vjp(model, qd, frames, W, Wc)
    pred = (g.double() * d.double()).sum(1)
    gn = torch.linalg.vector_norm(g.double(), dim=1) * torch.linalg.vector_norm(d.double(), dim=1)
    # O(h^2) truncation plus the fp32 rounding of the forward over 2h
    assert (torch.abs(pred - fd) <= 2e-3 * gn + 1e-3).all(), torch.max(torch.abs(pred - fd) / (gn + 1e-9)).item()


def test_converge_then_frame_placements_against_central_differences_of_the_pipeline():
    """The exactly determined UR5 problem of test_gpu_converge_grad: a loss of the forearm's pose
    and the tool's position at q*, differentiated to the targets through both kernels."""
    from examples import arm_ur5_reach_batched as ex

    B, h, tol = 256, 1e-3, 1e-6
    ik, task, q0, targets = ex.setup(B, device="cuda", seed=7)
    model = ik.model
    frames = ["forearm_link", "tool0"]
    res = ik.converge(q0, targets, [task], tol, 400)
    q_star = res.q.clone()
    W = torch.randn((B, 2, 3, 4), device="cuda", generator=_gen(6))
    tg = targets.clone().requires_grad_(True)
    r = ik.converge(q_star, tg, [task], tol, 400)
    loss = (kinematics.frame_placements(model, r.q, frames).oMf * W).sum()
    loss.backward()
    gt = tg.grad.cpu().numpy().astype(np.float64)
    rng = np.random.default_rng(2)
    d = rng.normal(size=(B, 6))
    T = targets.cpu().numpy().reshape(-1, 3, 4).astype(np.float64)

    def moved(s):
        Rd, pd = lie.exp6(s * d)
        R = T[:, :, :3] @ Rd
        p = np.einsum("bij,bj->bi", T[:, :, :3], pd) + T[:, :, 3]
        return torch.as_tensor(np.concatenate([R, p[:, :, None]], axis=2).reshape(B, 12), dtype=torch.float32,
                               device="cuda").contiguous()

    rp = ik.converge(q_star, moved(h), [task], tol, 400)
    rm = ik.converge(q_star, moved(-h), [task], tol, 400)
    Lp = (kinematics.frame_placements(model, rp.q, frames).oMf * W).double().sum((1, 2, 3))
    Lm = (kinematics.frame_placements(model, rm.q, frames).oMf * W).double().sum((1, 2, 3))
    fd = ((Lp - Lm) / (2 * h)).cpu().numpy()
    dT = np.concatenate([T[:, :, :3] @ lie.hat(d[:, 3:]), np.einsum("bij,bj->bi", T[:, :, :3], d[:, :3])[:, :, None]],
                        axis=2).reshape(B, 12)
    pred = (gt * dT).sum(1)
    table = model.table()
    f = table.frame_names.index("tool0")
    qs = q_star.cpu().numpy().astype(np.float64)
    sv = np.linalg.svd(okin.frame_jacobian_local(table, okin.forward_kinematics(table, qs), f), compute_uv=False)
    ok = (res.converged & r.converged & rp.converged & rm.converged).cpu().numpy() & (sv[:, 0] / sv[:, -1] < 100)
    assert ok.sum() > B // 2
    gq = kinematics.frame_placements_vjp(model, q_star, frames, W).cpu().numpy()
    gn = np.linalg.norm(gq, axis=1)
    bound = 3 * tol / (sv[:, -1] * h) * gn + 1e-2 * np.abs(pred) + 1e-3 * gn
    assert (np.abs(pred - fd) <= bound)[ok].all(), np.max((np.abs(pred - fd) / bound)[ok])


@pytest.mark.parametrize("robot,B,frames,com", [
    ("ur5_description", 65536, ["tool0"], False),
    ("g1_description", 16384, ["left_ankle_roll_link", "right_ankle_roll_link", "left_wrist_yaw_link",
                                "right_wrist_yaw_link", "pelvis"], True),
])
def test_full_batches_against_the_oracle_on_a_slice(robot, B, frames, com):
    _, model, m = helpers.load(robot)
    from pink_b200 import workloads

    q = workloads.sample_configurations(m, B, np.random.default_rng(31)).astype(np.float32)
    qd = torch.as_tensor(q, device="cuda").requires_grad_(True)
    fp = kinematics.frame_placements(model, qd, frames, com=com)
    W = torch.randn(fp.oMf.shape, device="cuda", generator=_gen(7))
    Wc = torch.randn((B, 3), device="cuda", generator=_gen(8))
    ((fp.oMf * W).sum() + ((fp.com * Wc).sum() if com else 0.0)).backward()
    idx = np.r_[0:64, B - 64:B]
    fi = [m.frame_names.index(n) for n in frames]
    ref, c_ref = oracle_forward(m, q[idx], fi)
    np.testing.assert_allclose(fp.oMf.detach().cpu().numpy()[idx], ref, atol=2e-5)
    if com:
        np.testing.assert_allclose(fp.com.detach().cpu().numpy()[idx], c_ref, atol=2e-5)
    g_ref = okg.frame_placements_vjp(m, q[idx].astype(np.float64), fi, W.cpu().numpy()[idx].astype(np.float64),
                                      Wc.cpu().numpy()[idx].astype(np.float64) if com else None)
    assert within(qd.grad.cpu().numpy()[idx], g_ref).all()


def test_cuda_graph_capture_equals_eager():
    model, m, frames, com, q = case("g1")
    qd = torch.as_tensor(q, device="cuda")
    W = torch.randn((q.shape[0], len(frames), 3, 4), device="cuda", generator=_gen(9))
    Wc = torch.randn((q.shape[0], 3), device="cuda", generator=_gen(10))
    eager = kinematics.frame_placements(model, qd, frames, com=True)
    eager_g = kinematics.frame_placements_vjp(model, qd, frames, W, Wc)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture
        kinematics.frame_placements(model, qd, frames, com=True)
        kinematics.frame_placements_vjp(model, qd, frames, W, Wc)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fp = kinematics.frame_placements(model, qd, frames, com=True)
        g = kinematics.frame_placements_vjp(model, qd, frames, W, Wc)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(fp.oMf, eager.oMf) and torch.equal(fp.com, eager.com) and torch.equal(g, eager_g)


def test_empty_batch_errors_and_no_node_without_grad():
    model, m, frames, com, q = case("ur5")
    qd = torch.as_tensor(q, device="cuda")
    e = kinematics.frame_placements(model, qd[:0], frames)
    assert e.oMf.shape == (0, len(frames), 3, 4)
    assert kinematics.frame_placements_vjp(model, qd[:0], frames, torch.zeros((0, len(frames), 3, 4),
                                                                              device="cuda")).shape == (0, m.nq)
    assert kinematics.frame_placements(model, qd, []).oMf.shape == (q.shape[0], 0, 3, 4)
    assert not kinematics.frame_placements_vjp(model, qd, []).any()
    with pytest.raises(FrameNotFound):
        kinematics.frame_placements(model, qd, ["no_such_frame"])
    with pytest.raises(ValueError):
        kinematics.frame_placements(model, qd, [m.nframes])
    with pytest.raises(ValueError):
        kinematics.frame_placements(model, qd.double(), frames)
    with pytest.raises(ValueError):
        kinematics.frame_placements(model, qd.cpu(), frames)
    with pytest.raises(ValueError):
        kinematics.frame_placements(model, qd[:, :3], frames)
    with pytest.raises(ValueError):
        kinematics.frame_placements(model, qd[0], frames)
    with pytest.raises(ValueError):
        kinematics.frame_placements_vjp(model, qd, frames, torch.zeros((1, 1, 3, 4), device="cuda"))
    mm = massless_model()
    q0 = torch.zeros((4, 2), device="cuda")
    with pytest.raises(RuntimeError, match="total mass is 0"):
        kinematics.frame_placements(mm, q0, ["tip"], com=True)
    with pytest.raises(RuntimeError, match="total mass is 0"):
        kinematics.frame_placements_vjp(mm, q0, ["tip"], None, torch.zeros((4, 3), device="cuda"))
    # the C entries' own checks
    import ctypes as C

    from pink_b200 import _cabi

    eng = pink.Configuration(model, model.createData(), qd).engine
    f = np.zeros(2, dtype=np.int32)
    f[1] = m.nframes
    out = torch.empty((q.shape[0], 2, 3, 4), device="cuda")
    gq = torch.empty_like(qd)
    lib, fa = eng.lib, f.ctypes.data_as(C.c_void_p)
    assert lib.pk_frame_placements_batched(eng.handle, fa, 2, qd.data_ptr(), out.data_ptr(), None, q.shape[0], None)
    assert b"out of range" in lib.pk_last_error()
    assert lib.pk_frame_placements_batched(eng.handle, fa, _cabi.PK_MAX_FRAMES + 1, qd.data_ptr(), out.data_ptr(),
                                           None, q.shape[0], None)
    assert lib.pk_frame_placements_vjp_batched(eng.handle, fa, 1, qd.data_ptr(), out.data_ptr(), None, None,
                                               q.shape[0], None)
    assert b"null grad_q" in lib.pk_last_error()
    assert lib.pk_frame_placements_vjp_batched(eng.handle, fa, 1, None, None, None, None, 0, None) == 0
    assert lib.pk_frame_placements_vjp_batched(eng.handle, fa, 1, qd.data_ptr(), out.data_ptr(), None, gq.data_ptr(),
                                               q.shape[0], None) == 0


def test_example_loss_decreases_and_converged_fraction_holds():
    from examples import arm_ur5_grasp_angle_grad_batched as ex

    out = ex.run(batch=2048, iters=5)
    assert out["losses"][-1] < out["losses"][0]
    assert out["height_after"] > out["height_before"]
    assert out["converged_after"] >= out["converged_before"] - 0.01
    assert out["converged_before"] > 0.5

"""ik_chain_kernel has an instantiation for arm-shaped problems (at least one frame task, every joint
revolute, every frame task on the last joint, no AccelerationLimit: ChainParams::arm), picked at
launch.  It only drops work whose outcome that shape fixes, so v, the rolled-out q and status must be
bitwise those of the general instantiation, which PK_CHAIN_FORCE_GENERAL=1 forces (read once per
process, hence one subprocess per setting).  A problem outside the shape must keep the general
instantiation: a frame on an inner body run through the arm instantiation would get Jacobian
columns for the joints past it, so its results would differ."""

import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pink_b200
from pink_b200 import FrameTask, PostureTask, workloads
from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inner_frame(B):
    """UR5 with its frame task on wrist_2_link (joint 4 of 0..5): outside the arm shape"""
    robot, model, table = helpers.load("ur5_description")
    rng = np.random.default_rng(workloads.SEED)
    q = workloads.sample_configurations(table, B, rng)
    T = helpers.frame_targets(table, workloads.perturb_configurations(table, q, rng), "wrist_2_link")
    ft = FrameTask("wrist_2_link", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    ft.set_target(torch.as_tensor(T))
    pt = PostureTask(cost=1e-3)
    pt.set_target(workloads.ur5_posture_reference(model))
    return helpers.Scenario("ur5-inner-frame", robot, model, table, q, [ft, pt], [], workloads.UR5_DT,
                            workloads.UR5_DAMPING)


CASES = {
    "reachable-1": lambda: helpers.ur5_scenario(1, "reachable"),
    "reachable-127": lambda: helpers.ur5_scenario(127, "reachable"),
    "reachable-65536": lambda: helpers.ur5_scenario(65536, "reachable"),
    "unreachable-127": lambda: helpers.ur5_scenario(127, "unreachable"),
    "unreachable-65536": lambda: helpers.ur5_scenario(65536, "unreachable"),
    "out-of-limits-127": lambda: helpers.ur5_scenario(127, "reachable", out_of_limits=20),
    "out-of-limits-65536": lambda: helpers.ur5_scenario(65536, "reachable", out_of_limits=500),
    "inner-frame-127": lambda: _inner_frame(127),
    "inner-frame-65536": lambda: _inner_frame(65536),
}


def dump_outputs(path):
    out = {}
    for name, make in CASES.items():
        sc = make()
        ik = pink_b200.BatchedIK(sc.model, sc.tasks, sc.dt, damping=sc.damping, limits=sc.limits,
                                 safety_break=sc.safety_break, device="cuda", batch_size=sc.B)
        _, targets, _ = sc.problem()
        t = torch.as_tensor(targets, device="cuda")
        q = torch.as_tensor(sc.q32, device="cuda")
        v, st = ik.solve(q, t)
        q_r, v_r, st_r = ik.rollout(q, t, 4)
        torch.cuda.synchronize()
        for key, val in (("v", v), ("status", st), ("q_roll", q_r), ("v_roll", v_r), ("status_roll", st_r)):
            out[f"{name}/{key}"] = val.cpu().numpy()
    np.savez(path, **out)


def _run_dump(tmp_path, force_general):
    out = tmp_path / f"general-{force_general}.npz"
    env = dict(os.environ, PK_CHAIN_FORCE_GENERAL=str(force_general))
    for name in ("PK_CHAIN_FORCE_RECOMPUTE", "PK_CHAIN_LANES"):
        env.pop(name, None)
    code = f"from tests.test_gpu_chain_shape import dump_outputs as d; d({str(out)!r})"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, check=True, timeout=1200)
    return dict(np.load(out))


@pytest.fixture(scope="module")
def outputs(tmp_path_factory):
    return {f: _run_dump(tmp_path_factory.mktemp(f"shape{f}"), f) for f in (0, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_arm_instantiation_bitwise_equal_to_general(name, outputs):
    picked, general = outputs[0], outputs[1]
    for key in ("v", "status", "q_roll", "v_roll", "status_roll"):
        k = f"{name}/{key}"
        a, b = picked[k], general[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        assert a.tobytes() == b.tobytes(), k
    if name.startswith("out-of-limits"):
        assert (picked[f"{name}/status"] != 0).any()
    else:
        assert np.isfinite(picked[f"{name}/v"]).all()

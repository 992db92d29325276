"""pink_b200: batched differential inverse kinematics on H100 (sm_90a).

Drop-in surface of Pink (``pink/__init__.py``): ``solve_ik``,
``build_ik``, ``Configuration``, ``tasks.*``, ``limits.*``, exceptions - with a
leading batch dimension on ``q`` / targets / ``v``.  All arithmetic of the path
runs in hand-written CUDA kernels behind the C-ABI of ``include/pink_b200.h``;
there is no CPU fallback.
"""

from . import barriers, kinematics, limits, tasks
from .batched import BatchedIK
from .collision import SphereCollisionModel
from .configuration import Configuration
from .exceptions import PinkError
from .model import JointModelFreeFlyer, Model, RobotWrapper, load_urdf
from .solve_ik import Problem, build_ik, solve_ik
from .spatial import SE3
from .tasks import (ComTask, DampingTask, FrameTask, JointCouplingTask, JointVelocityTask, LinearHolonomicTask,
                    LowAccelerationTask, PostureTask, RelativeFrameTask, Task)
from .utils import custom_configuration_vector

__version__ = "0.1.0"

__all__ = [
    "BatchedIK",
    "ComTask",
    "Configuration",
    "DampingTask",
    "FrameTask",
    "JointCouplingTask",
    "JointModelFreeFlyer",
    "JointVelocityTask",
    "LinearHolonomicTask",
    "LowAccelerationTask",
    "Model",
    "PinkError",
    "PostureTask",
    "Problem",
    "RelativeFrameTask",
    "RobotWrapper",
    "SE3",
    "SphereCollisionModel",
    "Task",
    "build_ik",
    "kinematics",
    "custom_configuration_vector",
    "load_urdf",
    "solve_ik",
]

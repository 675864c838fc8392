from .base_task import BaseTask  # noqa: F401
from .humanoid_smpl_im import HumanoidSMPLIM  # noqa: F401
from .humanoid_smpl_im_vis import HumanoidSMPLIMVis  # noqa: F401
from .humanoid_smpl_im_mvae import HumanoidSMPLIMMVAE, HumanoidSMPLIMMVAEDual  # noqa: F401
from .physics_mvae_controller import PhysicsMVAEController, PhysicsMVAEControllerDual, SyntheticMotionPlayer  # noqa: F401
from .mvae_controller_vis import MVAEControllerVis, MVAEControllerVisDual  # noqa: F401
from .vec_task import VecTask, VecTaskPython, VecTaskPythonWrapper  # noqa: F401
from .parse_task import parse_task  # noqa: F401

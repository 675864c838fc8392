"""parse_task mirror (embodied_pose/utils/parse_task.py:19-42): same signature and error behaviour."""
from .humanoid_smpl_im import HumanoidSMPLIM
from .humanoid_smpl_im_vis import HumanoidSMPLIMVis
from .humanoid_smpl_im_mvae import HumanoidSMPLIMMVAE, HumanoidSMPLIMMVAEDual
from .mvae_controller_vis import MVAEControllerVis, MVAEControllerVisDual
from .physics_mvae_controller import PhysicsMVAEController, PhysicsMVAEControllerDual
from .vec_task import VecTaskPythonWrapper

TASKS = {"HumanoidSMPLIM": HumanoidSMPLIM, "HumanoidSMPLIMVis": HumanoidSMPLIMVis, "HumanoidSMPLIMMVAE": HumanoidSMPLIMMVAE,
         "HumanoidSMPLIMMVAEDual": HumanoidSMPLIMMVAEDual,
         "PhysicsMVAEController": PhysicsMVAEController, "PhysicsMVAEControllerDual": PhysicsMVAEControllerDual,
         "MVAEControllerVis": MVAEControllerVis, "MVAEControllerVisDual": MVAEControllerVisDual}


def warn_task_name():
    raise Exception("Unrecognized task!\nTask should be one of: [" + ", ".join(TASKS) + "]")


def parse_task(args, cfg, cfg_train, sim_params):
    device_id = args.device_id
    rl_device = args.rl_device
    cfg["seed"] = cfg_train.get("seed", -1)
    cfg_task = cfg["env"]
    cfg_task["seed"] = cfg["seed"]
    cfg['args'] = args
    try:
        cls = TASKS[args.task]
    except KeyError:
        warn_task_name()
    task = cls(cfg=cfg, sim_params=sim_params, physics_engine=args.physics_engine, device_type=args.device,
               device_id=device_id, headless=args.headless)
    env = VecTaskPythonWrapper(task, rl_device, cfg_train.get("clip_observations", 5.0), cfg_train.get("clip_actions", 1.0))
    return task, env

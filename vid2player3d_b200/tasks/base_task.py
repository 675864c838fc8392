"""BaseTask mirror: the buffer / step contract of the reference
(embodied_pose/env/tasks/base_task.py:28-124 buffers :62-74, step :147-165).

`create_sim` / `prepare_sim` are stubbed: there is no Isaac Gym sim object; the subclass
builds a native b200env handle instead.  Viewer, camera sensors and domain randomisation are
out of scope (SURVEY.md 2 row 1)."""
import torch


class BaseTask:
    def __init__(self, cfg, enable_camera_sensors=False):
        self.device_type = cfg.get("device_type", "cuda")
        self.device_id = cfg.get("device_id", 0)
        if self.device_type not in ("cuda", "GPU"):
            raise RuntimeError("the environment runs on a CUDA device only (no CPU pipeline); "
                               f"got device_type={self.device_type!r}")
        self.device = "cuda:" + str(self.device_id)
        self.headless = cfg["headless"]
        self.graphics_device_id = -1
        self.num_envs = cfg["env"]["numEnvs"]

        self.create_sim()  # subclass: builds the native env (replaces gym.create_sim + prepare_sim :48-49)

        self.num_obs = cfg["env"]["numObservations"]
        self.num_states = cfg["env"].get("numStates", 0)
        self.num_actions = cfg["env"]["numActions"]
        self.control_freq_inv = cfg["env"].get("controlFrequencyInv", 1)

        dev = self.device
        self.obs_buf = torch.zeros((self.num_envs, self.num_obs), device=dev, dtype=torch.float)
        self.states_buf = torch.zeros((self.num_envs, self.num_states), device=dev, dtype=torch.float)
        self.rew_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.float)
        self.reset_buf = torch.ones(self.num_envs, device=dev, dtype=torch.long)
        self.progress_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.long)
        self.randomize_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.long)
        self.extras = {}
        self.viewer = None
        self.enable_viewer_sync = True

    def create_sim(self):
        raise NotImplementedError

    def get_states(self):
        return self.states_buf

    def render(self, sync_frame_time=False):
        return  # headless only

    def step(self, actions):
        raise NotImplementedError

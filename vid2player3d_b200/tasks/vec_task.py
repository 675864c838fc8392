"""VecTask / VecTaskPython / VecTaskPythonWrapper mirrors - the rl_games-facing adapter
(embodied_pose/env/tasks/vec_task.py:16-63,120-138; vec_task_wrappers.py:22-28)."""
import numpy as np
import torch


class _Box:  # gym.spaces.Box stand-in (gym is not a dependency of the hot path)
    def __init__(self, low, high):
        self.low, self.high, self.shape, self.dtype = low, high, low.shape, np.float32


class VecTask:
    def __init__(self, task, rl_device, clip_observations=5.0, clip_actions=1.0):
        self.task = task
        self.num_environments = task.num_envs
        self.num_agents = 1
        self.num_observations = task.num_obs
        self.num_states = task.num_states
        self.num_actions = task.num_actions
        self.obs_space = _Box(np.ones(self.num_obs) * -np.inf, np.ones(self.num_obs) * np.inf)
        self.state_space = _Box(np.ones(self.num_states) * -np.inf, np.ones(self.num_states) * np.inf)
        self.act_space = _Box(np.ones(self.num_actions) * -1., np.ones(self.num_actions) * 1.)
        self.clip_obs = clip_observations
        self.clip_actions = clip_actions
        self.rl_device = rl_device

    def step(self, actions):
        raise NotImplementedError

    def reset(self):
        raise NotImplementedError

    def get_number_of_agents(self):
        return self.num_agents

    @property
    def observation_space(self):
        return self.obs_space

    @property
    def action_space(self):
        return self.act_space

    @property
    def num_envs(self):
        return self.num_environments

    @property
    def num_acts(self):
        return self.num_actions

    @property
    def num_obs(self):
        return self.num_observations


class VecTaskPython(VecTask):
    def get_state(self):
        return torch.clamp(self.task.states_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)

    def step(self, actions):
        if getattr(self, "_graph", None) is not None:
            if actions.data_ptr() != self._graph_actions.data_ptr():
                self._graph_actions.copy_(actions)
            self._graph.replay()
            return self._graph_obs, self.task.rew_buf, self.task.reset_buf, self.task.extras
        actions_tensor = torch.clamp(actions, -self.clip_actions, self.clip_actions)
        self.task.step(actions_tensor)
        return (torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device),
                self.task.rew_buf.to(self.rl_device), self.task.reset_buf.to(self.rl_device), self.task.extras)

    def enable_cuda_graph(self, actions=None, warmup=3, reset_graph=False):
        """Addition (not in the reference): capture `clamp(actions) -> task.step -> clamp(obs)` - 1 memset + 5 kernels - into
        one CUDA graph; `step()` then costs one graph launch on the host instead of ~8 launches through PyTorch and ctypes.
        `actions`: the device tensor the caller will keep passing (its storage becomes the graph's input; any other tensor is
        copied into it first).  The returned observation tensor is a fixed buffer, overwritten by the next step (the reference
        returns a fresh clamp() result; rl_games copies it into its own rollout storage before stepping again).
        Valid while rl_device == the task's device and the task's step makes no host synchronisation (true for the env step).
        The warm-up runs a few real env steps: call it before the reset() that starts a rollout.
        reset_graph=True (tasks with `reset_masked`, e.g. HumanoidSMPLIM): also capture `task.reset_masked(mask of the finished envs)
        -> clamp(obs)` as a second graph, which `reset_done()` replays (with cfg.env.transform_specs only under
        cfg.env.b200_device_transforms, which applies them in the window launch; otherwise that reset stays eager)."""
        assert str(self.rl_device) == str(self.task.device), "graph capture needs rl_device == sim device"
        dev = self.task.device
        self._graph = None
        self._graph_actions = actions if actions is not None else torch.zeros(self.task.num_envs, self.task.num_actions, device=dev)
        assert self._graph_actions.is_cuda and self._graph_actions.is_contiguous() and self._graph_actions.dtype == torch.float32
        self._graph_obs = torch.empty_like(self.task.obs_buf)
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):          # also runs the one-time setup of the native step (function attributes, scratch)
                self.task.step(torch.clamp(self._graph_actions, -self.clip_actions, self.clip_actions))
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.task.step(torch.clamp(self._graph_actions, -self.clip_actions, self.clip_actions))
            torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs, out=self._graph_obs)
        self._graph = g
        if reset_graph:
            self._reset_obs = torch.empty_like(self.task.obs_buf)
            self._reset_obs_in_graph = self.task._capture_reset_graph(
                lambda: torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs, out=self._reset_obs))
        return self._graph_actions

    def reset(self):
        actions = 0.01 * (1 - 2 * torch.rand([self.task.num_envs, self.task.num_actions], dtype=torch.float32,
                                             device=self.rl_device))
        self.task.step(actions)
        return torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)


class VecTaskPythonWrapper(VecTaskPython):
    def __init__(self, task, rl_device, clip_observations=5.0, clip_actions=1.0):
        super().__init__(task, rl_device, clip_observations, clip_actions)

    def reset(self, env_ids=None):
        self.task.reset(env_ids)
        return torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)

    def reset_done(self):
        """Addition: `reset(reset_buf.nonzero())` from the device flags (task.reset_done: no host synchronisation unless the task has
        cfg.env.transform_specs without cfg.env.b200_device_transforms).  Returns the clamped observations in a fixed buffer, overwritten by the next reset_done(); with
        enable_cuda_graph(reset_graph=True) the reset and the clamp are one graph replay after the mask launch."""
        self.task.reset_done()
        if not getattr(self, "_reset_obs_in_graph", False):
            if getattr(self, "_reset_obs", None) is None:
                self._reset_obs = torch.empty_like(self.task.obs_buf)
            torch.clamp(self.task.obs_buf, -self.clip_obs, self.clip_obs, out=self._reset_obs)
        return self._reset_obs

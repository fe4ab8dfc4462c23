"""Env runtime with the reference's surface (`isaacgymenvs/tasks/base/vec_task.py`): the same
constructor arguments, buffers, spaces and step()/reset()/reset_done() contracts, but the work
between "actions in" and "obs/rew/reset out" is ONE fused CUDA launch through the C ABI
(include/b200gym.h b2g_task_step) instead of pre_physics_step -> gym.simulate ->
post_physics_step with O(100) torch kernels (SURVEY.md 3.2).
"""
import abc
from typing import Any, Dict, Tuple

import numpy as np
import torch

from ... import engine

try:                                     # gym==0.23.1 in the reference (vec_task.py:34-35)
    from gym import spaces               # noqa: F401
except Exception:                        # not installed here: the minimal Box the callers read
    class _Box:
        def __init__(self, low, high, dtype=np.float32):
            self.low = np.asarray(low, dtype=dtype)
            self.high = np.asarray(high, dtype=dtype)
            self.shape = self.low.shape
            self.dtype = np.dtype(dtype)

        def sample(self):
            lo = np.where(np.isfinite(self.low), self.low, -1.0)
            hi = np.where(np.isfinite(self.high), self.high, 1.0)
            return np.random.uniform(lo, hi).astype(self.dtype)

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

        def __repr__(self):
            return f"Box({self.shape}, {self.dtype})"

    class spaces:                        # noqa: N801
        Box = _Box


class Env(abc.ABC):
    """vec_task.py:67-204 (device parsing, spaces, clip ranges)."""

    def __init__(self, config: Dict[str, Any], rl_device: str, sim_device: str, graphics_device_id: int, headless: bool):
        split_device = sim_device.split(":")
        self.device_type = split_device[0]
        self.device_id = int(split_device[1]) if len(split_device) > 1 else 0
        self.device = "cpu"
        if config["sim"]["use_gpu_pipeline"]:
            if self.device_type.lower() in ("cuda", "gpu"):
                self.device = "cuda" + ":" + str(self.device_id)
            else:
                print("GPU Pipeline can only be used with GPU simulation. Forcing CPU Pipeline.")
                config["sim"]["use_gpu_pipeline"] = False
        self.rl_device = rl_device
        self.headless = headless
        enable_camera_sensors = config["env"].get("enableCameraSensors", False)
        self.graphics_device_id = graphics_device_id
        if enable_camera_sensors is False and self.headless is True:
            self.graphics_device_id = -1
        self.num_environments = config["env"]["numEnvs"]
        self.num_agents = config["env"].get("numAgents", 1)
        self.num_observations = config["env"].get("numObservations", 0)
        self.num_states = config["env"].get("numStates", 0)
        self.obs_space = spaces.Box(np.ones(self.num_obs) * -np.inf, np.ones(self.num_obs) * np.inf)
        self.state_space = spaces.Box(np.ones(self.num_states) * -np.inf, np.ones(self.num_states) * np.inf)
        self.num_actions = config["env"]["numActions"]
        self.control_freq_inv = config["env"].get("controlFrequencyInv", 1)
        self.act_space = spaces.Box(np.ones(self.num_actions) * -1., np.ones(self.num_actions) * 1.)
        self.clip_obs = config["env"].get("clipObservations", np.inf)
        self.clip_actions = config["env"].get("clipActions", np.inf)
        self.total_train_env_frames: int = 0
        self.control_steps: int = 0
        self.render_fps: int = config["env"].get("renderFPS", -1)
        self.last_frame_time: float = 0.0
        self.record_frames: bool = False

    @abc.abstractmethod
    def allocate_buffers(self):
        """Create torch buffers for observations, rewards, actions dones and any additional data."""

    @abc.abstractmethod
    def step(self, actions: torch.Tensor) -> Tuple[Dict[str, torch.Tensor], torch.Tensor, torch.Tensor, Dict[str, Any]]:
        """Step the physics of the environment."""

    @abc.abstractmethod
    def reset(self) -> Dict[str, torch.Tensor]:
        """Reset the environment."""

    @abc.abstractmethod
    def reset_idx(self, env_ids: torch.Tensor):
        """Reset environments having the provided indices."""

    @property
    def observation_space(self):
        return self.obs_space

    @property
    def action_space(self):
        return self.act_space

    @property
    def num_envs(self) -> int:
        return self.num_environments

    @property
    def num_acts(self) -> int:
        return self.num_actions

    @property
    def num_obs(self) -> int:
        return self.num_observations

    def set_train_info(self, env_frames, *args, **kwargs):
        self.total_train_env_frames = env_frames

    def get_env_state(self):
        return None

    def set_env_state(self, env_state):
        pass


class VecTask(Env):
    """vec_task.py:207-455.  Subclasses describe the asset and the task scalars
    (`_build_model`, `_task_params`); the per-step hooks of the reference (pre_physics_step,
    post_physics_step, compute_observations, compute_reward, reset_idx) are fused in the engine."""

    metadata = {"render.modes": ["human", "rgb_array"], "video.frames_per_second": 24}

    def __init__(self, config, rl_device, sim_device, graphics_device_id, headless,
                 virtual_screen_capture: bool = False, force_render: bool = False):
        self.cfg = config
        super().__init__(config, rl_device, sim_device, graphics_device_id, headless)
        self.virtual_screen_capture = virtual_screen_capture
        self.force_render = force_render
        if self.cfg["physics_engine"] not in ("physx", "flex"):
            raise ValueError(f"Invalid physics engine backend: {self.cfg['physics_engine']}")
        sim_cfg = self.cfg["sim"]
        self.dt: float = sim_cfg["dt"]
        self.viewer = None
        self.first_randomization = True
        self.dr_randomizations = {}
        # domain randomisation: observation / action noise only (utils/dr.py); physical parameters raise
        self.randomizer = None
        task_cfg = self.cfg.get("task", {}) if isinstance(self.cfg, dict) else {}
        self.physical_randomizer = None
        if task_cfg.get("randomize", False):
            from ...utils.dr import Randomizer
            self.randomizer = Randomizer(task_cfg.get("randomization_params", {}))
        if self.device == "cpu":
            raise engine.EngineError(
                "sim_device=cpu / pipeline=cpu: the CUDA-native stepper has no CPU path (north_star: no CPU "
                "fallback); the CPU restatement lives in oracle/ and is only driven by tests and bench.py")
        self.seed = int(self.cfg.get("seed", 42)) if isinstance(self.cfg, dict) else 42
        self.env_id_offset = int(self.cfg.get("env_id_offset", 0))
        # create envs, sim (create_sim + prepare_sim, vec_task.py:259-263)
        self.sim_initialized = False
        self.create_sim()
        self.sim_initialized = True
        self.obs_dict = {}
        self.allocate_buffers()
        self._bind_task()
        ap = task_cfg.get("randomization_params", {}).get("actor_params") if task_cfg.get("randomize", False) else None
        if ap:      # physical domain randomisation: per-env parameter tensors read by the step kernel (utils/dr.py)
            from ...utils.dr import PhysicalRandomizer
            self.physical_randomizer = PhysicalRandomizer(ap, self.model, self.num_envs, self.device,
                                                          task_cfg["randomization_params"].get("frequency", 1))
            self.physical_randomizer.apply(0, self.randomize_buf, self.reset_buf)
            for slot, t in self.physical_randomizer.tensors(engine).items():
                self.sim._bind(slot, t)

    # ---- vec_task.py:301-324
    def allocate_buffers(self):
        dev = self.device
        self.obs_buf = torch.zeros((self.num_envs, self.num_obs), device=dev, dtype=torch.float)
        self.states_buf = torch.zeros((self.num_envs, self.num_states), device=dev, dtype=torch.float)
        self.rew_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.float)
        self.reset_buf = torch.ones(self.num_envs, device=dev, dtype=torch.long)
        self.timeout_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.bool)
        self.progress_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.long)
        self.randomize_buf = torch.zeros(self.num_envs, device=dev, dtype=torch.long)
        self.actions = torch.zeros((self.num_envs, self.num_actions), device=dev, dtype=torch.float)
        self.reset_count = torch.zeros(self.num_envs, device=dev, dtype=torch.int32)
        # clamp(obs, +-clip_obs) is a separate tensor only when the clip is finite (vec_task.py:402)
        self.obs_clipped = self.obs_buf if not np.isfinite(self.clip_obs) else torch.zeros_like(self.obs_buf)
        self._obs_engine = self.obs_buf            # the tensor bound to the engine (obs_buf may be rebound by observation noise)
        self.extras = {}

    def create_sim(self):
        """gym.create_sim + ground + envs + prepare_sim -> one engine.Sim of num_envs actors."""
        model = self._build_model()
        sim_cfg = self.cfg["sim"]
        plane = self.cfg["env"].get("plane", {})
        self.model = model
        self.sim = engine.Sim(model, self.num_envs, dt=sim_cfg["dt"], substeps=sim_cfg["substeps"],
                              gravity=tuple(sim_cfg["gravity"]), ground_mu=plane.get("dynamicFriction", 1.0),
                              device=self.device)
        return self.sim

    @abc.abstractmethod
    def _build_model(self):
        """asset -> importer Model (gym.load_asset + create_asset_force_sensor)."""

    @abc.abstractmethod
    def _task_params(self) -> engine.CTaskParams:
        """scalars of the fused task kernel."""

    def _task_buffers(self) -> dict:
        return {}

    def _bind_task(self):
        E = engine
        bufs = {E.T_ACTIONS: self.actions, E.T_OBS: self._obs_engine, E.T_REW: self.rew_buf, E.T_RESET: self.reset_buf,
                E.T_PROGRESS: self.progress_buf, E.T_TIMEOUT: self.timeout_buf.view(torch.uint8),
                E.T_RESET_COUNT: self.reset_count, E.T_OBS_CLIPPED: self.obs_clipped}
        bufs.update(self._task_buffers())
        p = self._task_params()
        p.num_obs, p.num_actions = self.num_obs, self.num_actions
        p.control_freq_inv = int(self.control_freq_inv)
        p.clip_actions = float(min(self.clip_actions, 3e38))
        p.clip_obs = float(min(self.clip_obs, 3e38))
        p.seed = self.seed
        p.env_id_offset = self.env_id_offset
        self.sim.set_task(p, bufs)
        # what step() hands back when nothing has to be converted (rl_device == sim device, no observation noise, no
        # asymmetric states): the same tensor objects every step, as the reference returns its own buffers
        # (vec_task.py:402-408 -- `.to(rl_device)` of a tensor already there is the tensor itself)
        self._same_device = torch.device(self.rl_device) == torch.device(self.device)
        self._torch_device = torch.device(self.device)
        self.extras["time_outs"] = self.timeout_buf
        self.obs_dict["obs"] = self.obs_clipped
        self._step_ret = (self.obs_dict, self.rew_buf, self.reset_buf, self.extras)

    def get_state(self):
        return torch.clamp(self.states_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)

    # ---- vec_task.py:360-408
    def step(self, actions: torch.Tensor) -> Tuple[Dict[str, torch.Tensor], torch.Tensor, torch.Tensor, Dict[str, Any]]:
        if self.physical_randomizer is not None:   # apply_randomizations for the envs this step is about to reset (vec_task.py:631-637)
            self.physical_randomizer.apply(self.control_steps * max(int(self.control_freq_inv), 1), self.randomize_buf, self.reset_buf)
            self.randomize_buf += 1
        if self.randomizer is not None:         # apply_randomizations, vec_task.py:610-718 (non-physical part)
            if self.randomizer.update(self.control_steps * max(int(self.control_freq_inv), 1)):
                for key, model in self.randomizer.models.items():
                    self.dr_randomizations[key] = {"noise_lambda": model}
        if self.dr_randomizations.get('actions', None):
            actions = self.dr_randomizations['actions']['noise_lambda'](actions)
        a = actions
        if a.dtype is not torch.float32 or a.device != self._torch_device or not a.is_contiguous():
            a = a.to(device=self.device, dtype=torch.float32).contiguous()
        self.sim.task_step(a)                   # clamp + pre_physics + simulate + post_physics + timeout + clip
        self.control_steps += 1
        self._fill_extras()
        if self._same_device and self.num_states == 0 and not self.dr_randomizations.get('observations', None):
            self.extras["time_outs"] = self.timeout_buf      # the buffers themselves: `.to()` of a tensor already there
            self.obs_dict["obs"] = self.obs_clipped
            return self._step_ret
        self.extras["time_outs"] = self.timeout_buf.to(self.rl_device)
        if self.dr_randomizations.get('observations', None):
            # vec_task.py:397-402: noise on the observation, then the clamp.  The engine keeps writing the tensor it is
            # bound to (_obs_engine); obs_buf is the noisy copy the caller sees
            self.obs_buf = self.dr_randomizations['observations']['noise_lambda'](self._obs_engine)
            self.obs_dict["obs"] = torch.clamp(self.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)
        else:
            self.obs_dict["obs"] = self.obs_clipped.to(self.rl_device)
        if self.num_states > 0:
            self.obs_dict["states"] = self.get_state()
        return self.obs_dict, self.rew_buf.to(self.rl_device), self.reset_buf.to(self.rl_device), self.extras

    def rollout(self, actions: torch.Tensor):
        """K steps whose actions are all known up front (K, num_envs, num_actions) -- an open-loop rollout such as the
        reference's README loop under random actions (README.md:39-51).  Equivalent to
            for k in range(K): obs[k], rew[k], reset[k], info = self.step(actions[k]); time_outs[k] = info["time_outs"]
        and returns the stacked (obs, rew, reset, time_outs).  Ant runs the K steps in one launch (b2g_task_rollout)."""
        if self.randomizer is not None or self.dr_randomizations or self.physical_randomizer is not None:
            raise engine.EngineError("rollout: domain randomisation is configured; use step()")
        a = actions.to(device=self.device, dtype=torch.float32).contiguous()
        K = a.shape[0]
        dev = self.device
        obs = torch.empty((K, self.num_envs, self.num_obs), device=dev); rew = torch.empty((K, self.num_envs), device=dev)
        reset = torch.empty((K, self.num_envs), device=dev, dtype=torch.long); tout = torch.empty((K, self.num_envs), device=dev, dtype=torch.uint8)
        self.sim.task_rollout(a, obs, rew, reset, tout)
        self.control_steps += K
        self._fill_extras()
        return obs.to(self.rl_device), rew.to(self.rl_device), reset.to(self.rl_device), tout.bool().to(self.rl_device)

    def step_host(self, h_actions, h_obs, h_rew, h_reset, h_timeout=None):
        """rl_device='cpu' fast path: the same step with host (pinned) buffers through
        b2g_task_step_host -- H2D actions, fused step, D2H obs/rew/reset, stream sync.  It runs none of step()'s
        randomisation hooks, so it refuses to run with them configured rather than silently skipping the noise."""
        if self.randomizer is not None or self.dr_randomizations or self.physical_randomizer is not None:
            raise engine.EngineError("step_host: domain randomisation is configured; use step() (the noise lambdas run on device tensors)")
        self.sim.task_step_host(h_actions, h_obs, h_rew, h_reset, h_timeout)
        self.control_steps += 1

    def _fill_extras(self):
        pass

    def zero_actions(self) -> torch.Tensor:
        return torch.zeros([self.num_envs, self.num_actions], dtype=torch.float32, device=self.rl_device)

    def reset_idx(self, env_idx):
        """Flag environments for reset; the fused step performs the reset (it is the first thing
        post_physics_step does for flagged envs, ant.py:291-293)."""
        self.reset_buf[env_idx] = 1

    def reset(self):
        """vec_task.py:426-438: returns the (initially zero) observation buffer, no sim work."""
        self.obs_dict["obs"] = torch.clamp(self.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)
        if self.num_states > 0:
            self.obs_dict["states"] = self.get_state()
        return self.obs_dict

    def reset_done(self):
        """vec_task.py:440-455: reset_idx(nonzero(reset_buf)) right at the call (one small launch, b2g_reset_flagged),
        then the clamped observation buffer -- the reference's order of events."""
        done_env_ids = self.reset_buf.nonzero(as_tuple=False).flatten()
        if len(done_env_ids) > 0:
            self.sim.reset_flagged()
        self.obs_dict["obs"] = torch.clamp(self.obs_buf, -self.clip_obs, self.clip_obs).to(self.rl_device)
        if self.num_states > 0:
            self.obs_dict["states"] = self.get_state()
        return self.obs_dict, done_env_ids

    def render(self, mode="rgb_array"):
        return None

    def get_number_of_agents(self):
        return self.num_agents

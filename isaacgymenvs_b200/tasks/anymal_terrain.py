"""AnymalTerrain with the reference class's surface (`isaacgymenvs/tasks/anymal_terrain.py`); the
per-step work runs as two fused kernels (csrc/b2g_anymal.cuh)."""
import copy
import numpy as np
import torch

from .. import engine
from ..assets import load_asset_file
from ..importer.model import BuildOptions, DRIVE_EFFORT, enable_self_collision
from ..terrain import Terrain
from .base.vec_task import VecTask
from .locomotion import _asset_root

SUM_KEYS = ("lin_vel_xy", "lin_vel_z", "ang_vel_z", "ang_vel_xy", "orient", "torques", "joint_acc", "base_height",
            "air_time", "collision", "stumble", "action_rate", "hip")          # anymal_terrain.py:144-146


class AnymalTerrain(VecTask):
    def __init__(self, cfg, rl_device, sim_device, graphics_device_id, headless, virtual_screen_capture=False,
                 force_render=False):
        self.cfg = cfg
        e, learn = cfg["env"], cfg["env"]["learn"]
        self.height_samples = None
        self.custom_origins = False
        self.init_done = False
        self.lin_vel_scale = learn["linearVelocityScale"]; self.ang_vel_scale = learn["angularVelocityScale"]
        self.dof_pos_scale = learn["dofPositionScale"]; self.dof_vel_scale = learn["dofVelocityScale"]
        self.height_meas_scale = learn["heightMeasurementScale"]
        self.action_scale = e["control"]["actionScale"]
        names = [("termination", "terminalReward"), ("lin_vel_xy", "linearVelocityXYRewardScale"),
                 ("lin_vel_z", "linearVelocityZRewardScale"), ("ang_vel_z", "angularVelocityZRewardScale"),
                 ("ang_vel_xy", "angularVelocityXYRewardScale"), ("orient", "orientationRewardScale"),
                 ("torque", "torqueRewardScale"), ("joint_acc", "jointAccRewardScale"), ("base_height", "baseHeightRewardScale"),
                 ("air_time", "feetAirTimeRewardScale"), ("collision", "kneeCollisionRewardScale"),
                 ("stumble", "feetStumbleRewardScale"), ("action_rate", "actionRateRewardScale"), ("hip", "hipRewardScale")]
        self.rew_scales = {k: learn[y] for k, y in names}
        self._rew_order = [k for k, _ in names]
        r = e["randomCommandVelocityRanges"]
        self.command_x_range, self.command_y_range, self.command_yaw_range = r["linear_x"], r["linear_y"], r["yaw"]
        b = e["baseInitState"]
        self.base_init_state_list = b["pos"] + b["rot"] + b["vLinear"] + b["vAngular"]
        self.named_default_joint_angles = e["defaultJointAngles"]
        self.decimation = e["control"]["decimation"]
        self.dt = self.decimation * cfg["sim"]["dt"]                                   # :95
        self.max_episode_length_s = learn["episodeLength_s"]
        self.max_episode_length = int(self.max_episode_length_s / self.dt + 0.5)
        self.push_interval = int(learn["pushInterval_s"] / self.dt + 0.5)
        self.allow_knee_contacts = learn["allowKneeContacts"]
        self.Kp, self.Kd = e["control"]["stiffness"], e["control"]["damping"]
        self.curriculum = e["terrain"]["curriculum"]
        for k in self.rew_scales:
            self.rew_scales[k] *= self.dt                                              # :104-105
        self.up_axis_idx = 2
        # test hook: no gym.simulate at all (decimation and control_freq_inv forced to 0 for the kernels) while every
        # dt-derived constant keeps its value -- pins the non-physics part of the step against the reference's methods
        self._skip_physics = bool(e.get("skipPhysics", False))
        if self._skip_physics:
            e["controlFrequencyInv"] = 0
        super().__init__(config=cfg, rl_device=rl_device, sim_device=sim_device, graphics_device_id=graphics_device_id,
                         headless=headless, virtual_screen_capture=virtual_screen_capture, force_render=force_render)
        self.dt = self.decimation * cfg["sim"]["dt"]     # VecTask.__init__ set the sim dt; the task uses the control dt
        self.init_done = True

    # ---- create_sim / _create_envs (:152-292)
    def _build_model(self):
        e = self.cfg["env"]
        opts = BuildOptions(collapse_fixed_joints=True, replace_cylinder_with_capsule=True, density=0.001,
                            fix_base_link=e["urdfAsset"]["fixBaseLink"], default_dof_drive_mode=DRIVE_EFFORT)
        model = copy.deepcopy(load_asset_file(_asset_root(), e["urdfAsset"]["file"], opts))
        # anymal_terrain.py:282 create_actor(..., i, 0, 0): collision filter 0 = the legs collide with each other and the base
        # (env.selfCollision: True = as the reference, on the four-chain kernels; default False = without it, announced by a warning)
        if e.get("selfCollision", False):
            enable_self_collision(model)
        else:
            engine.warn_self_collision("AnymalTerrain", "anymal_terrain.py:282 create_actor(..., i, 0, 0); set env.selfCollision=True to model it")
        self.num_dof, self.num_bodies = model.ndof, model.nb
        self.dof_names = list(model.dof_names)
        body_names = list(model.body_names)
        self._feet = [i for i, s in enumerate(body_names) if e["urdfAsset"]["footName"] in s]
        self._knees = [i for i, s in enumerate(body_names) if e["urdfAsset"]["kneeName"] in s]
        self._base = body_names.index("base")
        return model

    def create_sim(self):
        e, dev = self.cfg["env"], self.device
        tcfg = e["terrain"]
        model = self.model = self._build_model()
        sim_cfg = self.cfg["sim"]
        gen = torch.Generator().manual_seed(self.seed)
        hf_kw = {}
        terrain_type = tcfg["terrainType"]
        if terrain_type == "trimesh":
            self.terrain = Terrain(tcfg, num_robots=self.num_envs, seed=self.seed)
            self.custom_origins = True
            hf_kw = dict(hfield=self.terrain.heightsamples, hf_horizontal_scale=self.terrain.horizontal_scale,
                         hf_vertical_scale=self.terrain.vertical_scale,
                         hf_origin=(-self.terrain.border_size, -self.terrain.border_size))      # tm_params.transform.p (:200-201)
        elif terrain_type != "plane":
            raise ValueError(f"terrainType {terrain_type!r} has no ground (anymal_terrain.py:155-160)")
        self.sim = engine.Sim(model, self.num_envs, dt=sim_cfg["dt"], substeps=sim_cfg["substeps"],
                              gravity=tuple(sim_cfg["gravity"]), ground_mu=tcfg["dynamicFriction"], device=dev, **hf_kw)
        sim, N, A = self.sim, self.num_envs, self.num_dof
        if terrain_type == "trimesh":
            self.height_samples = torch.tensor(self.terrain.heightsamples).view(self.terrain.tot_rows, self.terrain.tot_cols).to(dev)
        # friction buckets (:235-281): env i takes bucket i % 100
        fr = e["learn"]["frictionRange"]
        buckets = (fr[1] - fr[0]) * torch.rand(100, generator=gen) + fr[0]
        self.env_friction = buckets[torch.arange(N) % 100].to(dev).contiguous()
        # env origins / terrain curriculum state (:255-263)
        self.env_origins = torch.zeros(N, 3, device=dev)
        if not self.curriculum:
            tcfg["maxInitMapLevel"] = tcfg["numLevels"] - 1
        self.terrain_levels = torch.randint(0, tcfg["maxInitMapLevel"] + 1, (N,), generator=gen).to(dev)
        self.terrain_types = torch.randint(0, tcfg["numTerrains"], (N,), generator=gen).to(dev)
        if self.custom_origins:
            self.terrain_origins = torch.from_numpy(self.terrain.env_origins).to(dev).to(torch.float).contiguous()
            self.env_origins[:] = self.terrain_origins[self.terrain_levels, self.terrain_types]
        else:
            self.terrain_origins = torch.zeros(1, 1, 3, device=dev)
        self.base_init_state = torch.tensor(self.base_init_state_list, dtype=torch.float, device=dev)
        self.feet_indices = torch.tensor(self._feet, dtype=torch.long, device=dev)
        self.knee_indices = torch.tensor(self._knees, dtype=torch.long, device=dev)
        self.base_index = self._base
        # tensors (:110-150)
        self.root_states = sim.root_state
        self.dof_state = sim.dof_state
        self.dof_pos = self.dof_state.view(N, A, 2)[..., 0]
        self.dof_vel = self.dof_state.view(N, A, 2)[..., 1]
        self.contact_forces = sim.acquire(engine.T_NET_CONTACT).view(N, -1, 3)
        self.common_step_counter = 0
        self.commands = torch.zeros(N, 4, device=dev)
        self.commands_scale = torch.tensor([self.lin_vel_scale, self.lin_vel_scale, self.ang_vel_scale], device=dev)
        self.gravity_vec = torch.tensor([0.0, 0.0, -1.0], device=dev).repeat((N, 1))
        self.forward_vec = torch.tensor([1.0, 0.0, 0.0], device=dev).repeat((N, 1))
        self.torques = torch.zeros(N, A, device=dev)
        self.last_actions = torch.zeros(N, A, device=dev)
        self.feet_air_time = torch.zeros(N, 4, device=dev)
        self.last_dof_vel = torch.zeros(N, A, device=dev)
        self.default_dof_pos = torch.zeros(N, A, device=dev)
        for i, name in enumerate(self.dof_names):
            self.default_dof_pos[:, i] = self.named_default_joint_angles[name]
        self._episode_sums = torch.zeros(13, N, device=dev)
        self.episode_sums = {k: self._episode_sums[i] for i, k in enumerate(SUM_KEYS)}
        self._base_scratch = torch.zeros(N, 12, device=dev)
        self._reduce = torch.zeros(1024 + 48, device=dev)
        self._reduce[1024 + 32] = float(self.terrain_levels.sum().item())          # running sum of terrain_levels, kept by the reset kernel
        self._reduce[1024 + 29] = float(self.terrain_levels.float().mean().item())
        self.measured_heights = None
        # initial reset of every env (:148, init_done False -> no curriculum move); host-side, one-off
        u = lambda lo, hi, *shape: ((hi - lo) * torch.rand(*shape, generator=gen) + lo).to(dev)
        self.dof_pos[:] = self.default_dof_pos * u(0.5, 1.5, N, A)
        self.dof_vel[:] = u(-0.1, 0.1, N, A)
        self.root_states[:] = self.base_init_state
        if self.custom_origins:
            self.root_states[:, :3] += self.env_origins
            self.root_states[:, :2] += u(-0.5, 0.5, N, 2)
        self.commands[:, 0] = u(self.command_x_range[0], self.command_x_range[1], N)
        self.commands[:, 1] = u(self.command_y_range[0], self.command_y_range[1], N)
        self.commands[:, 3] = u(self.command_yaw_range[0], self.command_yaw_range[1], N)
        self.commands *= (torch.norm(self.commands[:, :2], dim=1) > 0.25).unsqueeze(1)
        return self.sim

    def allocate_buffers(self):
        super().allocate_buffers()
        self.noise_scale_vec = self._get_noise_scale_vec(self.cfg)

    def _get_noise_scale_vec(self, cfg):       # :174-186
        learn = cfg["env"]["learn"]
        v = torch.zeros(self.num_obs, device=self.device)
        self.add_noise = learn["addNoise"]
        nl = learn["noiseLevel"]
        v[:3] = learn["linearVelocityNoise"] * nl * self.lin_vel_scale
        v[3:6] = learn["angularVelocityNoise"] * nl * self.ang_vel_scale
        v[6:9] = learn["gravityNoise"] * nl
        v[12:24] = learn["dofPositionNoise"] * nl * self.dof_pos_scale
        v[24:36] = learn["dofVelocityNoise"] * nl * self.dof_vel_scale
        v[36:176] = learn["heightMeasurementNoise"] * nl * self.height_meas_scale
        return v

    def _task_buffers(self):
        E = engine
        b = {E.T_COMMANDS: self.commands, E.T_LAST_ACTIONS: self.last_actions, E.T_LAST_DOF_VEL: self.last_dof_vel,
             E.T_FEET_AIR_TIME: self.feet_air_time, E.T_TORQUES: self.torques, E.T_EPISODE_SUMS: self._episode_sums,
             E.T_NOISE_SCALE: self.noise_scale_vec, E.T_BASE_SCRATCH: self._base_scratch, E.T_REDUCE_SCRATCH: self._reduce,
             E.T_ENV_FRICTION: self.env_friction}
        if self.custom_origins:
            b.update({E.T_TERRAIN_LEVELS: self.terrain_levels, E.T_TERRAIN_TYPES: self.terrain_types,
                      E.T_ENV_ORIGINS: self.env_origins, E.T_TERRAIN_ORIGINS: self.terrain_origins})
        return b

    def _task_params(self):
        e, learn = self.cfg["env"], self.cfg["env"]["learn"]
        p = engine.CAnymalParams()
        p.decimation = 0 if self._skip_physics else int(self.decimation)
        p.max_episode_length, p.push_interval = int(self.max_episode_length), int(self.push_interval)
        p.push_robots, p.add_noise = int(bool(learn["pushRobots"])), int(bool(learn["addNoise"]))
        p.curriculum, p.allow_knee_contacts = int(bool(self.curriculum)), int(bool(self.allow_knee_contacts))
        p.custom_origins = int(self.custom_origins)
        p.kp, p.kd, p.action_scale, p.torque_limit = float(self.Kp), float(self.Kd), float(self.action_scale), 80.0   # :443-444
        for i in range(self.num_dof):
            p.default_dof_pos[i] = float(self.default_dof_pos[0, i])
        p.lin_vel_scale, p.ang_vel_scale = float(self.lin_vel_scale), float(self.ang_vel_scale)
        p.dof_pos_scale, p.dof_vel_scale = float(self.dof_pos_scale), float(self.dof_vel_scale)
        p.height_meas_scale = float(self.height_meas_scale)
        for i, k in enumerate(self._rew_order):
            p.rew_scales[i] = float(self.rew_scales[k])
        p.dt, p.max_episode_length_s = float(self.decimation * self.cfg["sim"]["dt"]), float(self.max_episode_length_s)
        p.command_x = (engine.C.c_float * 2)(*self.command_x_range)
        p.command_y = (engine.C.c_float * 2)(*self.command_y_range)
        p.command_yaw = (engine.C.c_float * 2)(*self.command_yaw_range)
        p.base_init_state = (engine.C.c_float * 13)(*self.base_init_state_list)
        if self.custom_origins:
            t = self.terrain
            p.border_size, p.terrain_hscale, p.terrain_vscale = float(t.border_size), float(t.horizontal_scale), float(t.vertical_scale)
            p.env_length, p.hs_rows, p.hs_cols = float(t.env_length), int(t.tot_rows), int(t.tot_cols)
            p.env_rows, p.env_cols = int(t.env_rows), int(t.env_cols)
        p.base_body = int(self._base)
        p.knee_bodies = (engine.C.c_int32 * 4)(*self._knees)
        p.feet_bodies = (engine.C.c_int32 * 4)(*self._feet)
        return p

    def _fill_extras(self):
        # reset_idx fills extras["episode"] for the envs reset this step (:420-425): the reset kernel's last warp writes the
        # means into the scratch tensor; the dict holds views of it, built once (no torch kernels on the step path)
        if "episode" not in self.extras:
            means = self._reduce[1024 + 16:1024 + 30]
            self.extras["episode"] = {"rew_" + k: means[i] for i, k in enumerate(SUM_KEYS)}
            self.extras["episode"]["terrain_level"] = means[13]
        self.common_step_counter += 1

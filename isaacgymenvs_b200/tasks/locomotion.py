"""Ant and Humanoid with the reference classes' constructor surface and public tensors
(`isaacgymenvs/tasks/ant.py`, `tasks/humanoid.py`); per-step work is the fused engine kernel."""
import copy
import os
import numpy as np
import torch

from .. import engine
from ..assets import load_asset_file
from ..importer.model import BuildOptions, enable_self_collision
from .base.vec_task import VecTask

_ASSET_ROOT_CANDIDATES = [os.environ.get("B2G_ASSET_ROOT", "")]


def _asset_root():
    for c in _ASSET_ROOT_CANDIDATES:
        if c and os.path.isdir(c):
            return c
    return "<compiled>"


class _Locomotion(VecTask):
    HUMANOID = False
    NUM_OBS = 0
    NUM_ACT = 0
    START_HEIGHT = 0.0
    DEFAULT_ASSET = ""
    ALIVE = 0.0

    def __init__(self, cfg, rl_device, sim_device, graphics_device_id, headless, virtual_screen_capture=False,
                 force_render=False):
        self.cfg = cfg
        e = cfg["env"]
        self.max_episode_length = e["episodeLength"]
        self.randomize = cfg["task"]["randomize"]
        self.dof_vel_scale = e["dofVelocityScale"]
        self.angular_velocity_scale = e.get("angularVelocityScale", 0.1)
        self.contact_force_scale = e["contactForceScale"]
        self.power_scale = e["powerScale"]
        self.heading_weight = e["headingWeight"]
        self.up_weight = e["upWeight"]
        self.actions_cost_scale = e["actionsCost"]
        self.energy_cost_scale = e["energyCost"]
        self.joints_at_limit_cost_scale = e["jointsAtLimitCost"]
        self.death_cost = e["deathCost"]
        self.termination_height = e["terminationHeight"]
        self.plane_static_friction = e["plane"]["staticFriction"]
        self.plane_dynamic_friction = e["plane"]["dynamicFriction"]
        self.plane_restitution = e["plane"]["restitution"]
        # randomize: the base class applies the noise and binds the per-env physical parameters (and the Humanoid's gravity)
        cfg["env"]["numObservations"] = self.NUM_OBS
        cfg["env"]["numActions"] = self.NUM_ACT
        self.up_axis_idx = 2
        super().__init__(config=cfg, rl_device=rl_device, sim_device=sim_device, graphics_device_id=graphics_device_id,
                         headless=headless, virtual_screen_capture=virtual_screen_capture, force_render=force_render)

    # ---- ant.py:135-212 / humanoid.py:133-218
    def _build_model(self):
        asset_file = self.cfg["env"].get("asset", {}).get("assetFileName", self.DEFAULT_ASSET)
        opts = BuildOptions(angular_damping=0.01 if self.HUMANOID else 0.0,
                            max_angular_velocity=100.0 if self.HUMANOID else 64.0)     # humanoid.py:153-154, ant.py:151
        model = copy.deepcopy(load_asset_file(_asset_root(), asset_file, opts))
        if self.HUMANOID:
            # humanoid.py:194 create_actor(..., i, 0, 0): collision filter 0 = the links collide with each other
            # (env.selfCollision: True = as the reference; default False = the faster step without it, announced by a warning)
            if self.cfg["env"].get("selfCollision", False):
                enable_self_collision(model)
            else:
                engine.warn_self_collision("Humanoid", "humanoid.py:194 create_actor(..., i, 0, 0); set env.selfCollision=True to model it")
            feet = [model.body_names.index("right_foot"), model.body_names.index("left_foot")]   # humanoid.py:164-168
        else:
            feet = [i for i, n in enumerate(model.body_names) if "foot" in n]                   # ant.py:167-178
        model.sensor_body = np.array(feet, dtype=np.int32)
        model.sensor_pos = np.zeros((len(feet), 3)); model.sensor_quat = np.tile([0, 0, 0, 1.0], (len(feet), 1))
        self.num_dof = model.ndof
        self.num_bodies = model.nb
        # motor_effort in ACTUATOR file order (ant.py:155-157, humanoid.py:160-161; SURVEY.md 3.3)
        self.motor_efforts_np = np.asarray(model.actuator_gear, dtype=np.float32)
        lo, hi = model.lower[1:], model.upper[1:]
        self.dof_limits_lower_np = np.minimum(lo, hi).astype(np.float32)                         # ant.py:199-207
        self.dof_limits_upper_np = np.maximum(lo, hi).astype(np.float32)
        return model

    def create_sim(self):
        sim = super().create_sim()
        dev = self.device
        # create_actor(start_pose) (ant.py:163-164,190): root at the start height, identity rotation
        sim.root_state[:, 2] = self.START_HEIGHT
        self.start_rotation = torch.tensor([0.0, 0.0, 0.0, 1.0], device=dev)
        # public tensor views (ant.py:78-95)
        self.root_states = sim.root_state
        self.initial_root_states = self.root_states.clone()
        self.initial_root_states[:, 7:13] = 0
        self.dof_state = sim.dof_state
        self.dof_pos = self.dof_state.view(self.num_envs, self.num_dof, 2)[..., 0]
        self.dof_vel = self.dof_state.view(self.num_envs, self.num_dof, 2)[..., 1]
        self.vec_sensor_tensor = sim.acquire(engine.T_FORCE_SENSOR).view(self.num_envs, -1)
        if self.HUMANOID:
            self.dof_force_tensor = sim.acquire(engine.T_DOF_FORCE).view(self.num_envs, self.num_dof)
        self.dof_limits_lower = torch.tensor(self.dof_limits_lower_np, device=dev)
        self.dof_limits_upper = torch.tensor(self.dof_limits_upper_np, device=dev)
        zero = torch.zeros_like(self.dof_limits_lower)
        init = torch.where(self.dof_limits_lower > 0, self.dof_limits_lower,
                           torch.where(self.dof_limits_upper < 0, self.dof_limits_upper, zero))      # ant.py:96-99
        self.initial_dof_pos = init.unsqueeze(0).repeat(self.num_envs, 1)
        self.initial_dof_vel = torch.zeros_like(self.initial_dof_pos)
        self.dof_pos[:] = self.initial_dof_pos
        if self.HUMANOID:
            self.motor_efforts = torch.tensor(self.motor_efforts_np, device=dev)
            self.max_motor_effort = float(self.motor_efforts_np.max())
        else:
            self.joint_gears = torch.tensor(self.motor_efforts_np, device=dev)
        # ant.py:102-114
        self.up_vec = torch.tensor([0.0, 0.0, 1.0], device=dev).repeat((self.num_envs, 1))
        self.heading_vec = torch.tensor([1.0, 0.0, 0.0], device=dev).repeat((self.num_envs, 1))
        self.inv_start_rot = torch.tensor([-0.0, -0.0, -0.0, 1.0], device=dev).repeat((self.num_envs, 1))
        self.basis_vec0 = self.heading_vec.clone()
        self.basis_vec1 = self.up_vec.clone()
        self.targets = torch.tensor([1000.0, 0.0, 0.0], device=dev).repeat((self.num_envs, 1))
        self.target_dirs = torch.tensor([1.0, 0.0, 0.0], device=dev).repeat((self.num_envs, 1))
        self.potentials = torch.tensor([-1000. / self.dt], device=dev, dtype=torch.float).repeat(self.num_envs)
        self.prev_potentials = self.potentials.clone()
        return sim

    def _task_buffers(self):
        E = engine
        return {E.T_POTENTIALS: self.potentials, E.T_PREV_POTENTIALS: self.prev_potentials, E.T_UP_VEC: self.up_vec,
                E.T_HEADING_VEC: self.heading_vec, E.T_INITIAL_ROOT: self.initial_root_states}

    def _task_params(self):
        p = engine.CTaskParams()
        p.task = engine.TASK_HUMANOID if self.HUMANOID else engine.TASK_ANT
        p.max_episode_length = float(self.max_episode_length)
        p.power_scale = float(self.power_scale)
        nd = self.num_dof
        for i in range(nd):
            p.joint_gears[i] = float(self.motor_efforts_np[i])
            p.motor_efforts[i] = float(self.motor_efforts_np[i])
            p.dof_limits_lower[i] = float(self.dof_limits_lower_np[i])
            p.dof_limits_upper[i] = float(self.dof_limits_upper_np[i])
            p.initial_dof_pos[i] = float(self.initial_dof_pos[0, i])
        p.max_motor_effort = float(self.motor_efforts_np.max())
        p.dof_vel_scale = float(self.dof_vel_scale)
        p.contact_force_scale = float(self.contact_force_scale)
        p.angular_velocity_scale = float(self.angular_velocity_scale)
        p.heading_weight, p.up_weight = float(self.heading_weight), float(self.up_weight)
        p.actions_cost_scale, p.energy_cost_scale = float(self.actions_cost_scale), float(self.energy_cost_scale)
        p.joints_at_limit_cost_scale = float(self.joints_at_limit_cost_scale)
        p.death_cost, p.termination_height = float(self.death_cost), float(self.termination_height)
        p.alive_reward = float(self.ALIVE)
        p.reset_pos_noise, p.reset_vel_noise = 0.2, 0.1          # ant.py:257-258
        p.dt = float(self.dt)
        p.target = (engine.C.c_float * 3)(1000.0, 0.0, 0.0)
        return p

    def _fill_extras(self):
        if 'true_objective' not in self.extras:                  # ant.py:245-250; a view of the bound root tensor: set once
            self.extras['true_objective'] = self.root_states[:, 7]


class Ant(_Locomotion):
    NUM_OBS, NUM_ACT, START_HEIGHT, DEFAULT_ASSET, ALIVE = 60, 8, 0.44, "mjcf/nv_ant.xml", 0.5


class Humanoid(_Locomotion):
    HUMANOID = True
    NUM_OBS, NUM_ACT, START_HEIGHT, DEFAULT_ASSET, ALIVE = 108, 21, 1.34, "mjcf/nv_humanoid.xml", 2.0

    # domain randomisation (task.randomize): the Humanoid step kernels read a bound gravity vector
    dr_gravity = True

    def _randomize_this_step(self):
        # humanoid.py:255-256: apply_randomizations runs inside reset_idx, on steps where some env resets
        return bool(self.reset_buf.any())

    def _fill_extras(self):
        pass

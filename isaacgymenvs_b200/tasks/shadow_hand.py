"""ShadowHand with the reference class's surface (`isaacgymenvs/tasks/shadow_hand.py`): three actors per env (hand,
object, goal marker), the same public tensors, one fused kernel per step (csrc/b2g_hand.cuh)."""
import copy
import numpy as np
import torch

from .. import engine
from ..assets import load_asset_file
from ..importer.model import BuildOptions
from .base.vec_task import VecTask
from .locomotion import _asset_root

FINGERTIPS = ["robot0:ffdistal", "robot0:mfdistal", "robot0:rfdistal", "robot0:lfdistal", "robot0:thdistal"]   # shadow_hand.py:120
RELEVANT_TENDONS = ["robot0:T_FFJ1c", "robot0:T_MFJ1c", "robot0:T_RFJ1c", "robot0:T_LFJ1c"]                    # shadow_hand.py:258
NUM_OBS = {"openai": 42, "full_no_vel": 77, "full": 157, "full_state": 211}                                     # shadow_hand.py:108-113


def object_shape(model):
    """(half extents, rounding radius) of the free object's contact shape -- a rounded box (include/b200gym.h b2g_model_ext):
    box -> its half sizes; capsule (pen.xml:19) -> a segment along z + its radius; sphere -> a point + radius; a prolate
    spheroid (egg.xml:10, size 0.03 0.03 0.04) -> the capsule with the same equatorial radius and polar extent."""
    from ..importer.model import GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX, GEOM_ELLIPSOID
    if len(model.geom_type) != 1:
        raise NotImplementedError("the free object must be a single collision primitive")
    t, sz = int(model.geom_type[0]), [float(v) for v in np.asarray(model.geom_size)[0]]
    if t == GEOM_BOX:
        return sz[:3], 0.0
    if t == GEOM_CAPSULE:
        return [0.0, 0.0, sz[1]], sz[0]
    if t == GEOM_SPHERE:
        return [0.0, 0.0, 0.0], sz[0]
    if t == GEOM_ELLIPSOID and abs(sz[0] - sz[1]) < 1e-9 and sz[2] >= sz[0]:
        return [0.0, 0.0, sz[2] - sz[0]], sz[0]
    raise NotImplementedError("free object shape: box, capsule, sphere or a prolate spheroid along z")


class ShadowHand(VecTask):
    def __init__(self, cfg, rl_device, sim_device, graphics_device_id, headless, virtual_screen_capture=False,
                 force_render=False):
        self.cfg = cfg
        e = cfg["env"]
        self.randomize = cfg["task"]["randomize"]
        # randomize: the base class applies the noise, gravity and the hand / object actor_params (utils/dr.py), on the steps
        # that reset some env (reset_idx calls apply_randomizations, shadow_hand.py:604-607,670-682)
        self.dist_reward_scale = e["distRewardScale"]; self.rot_reward_scale = e["rotRewardScale"]
        self.action_penalty_scale = e["actionPenaltyScale"]; self.success_tolerance = e["successTolerance"]
        self.reach_goal_bonus = e["reachGoalBonus"]; self.fall_dist = e["fallDistance"]; self.fall_penalty = e["fallPenalty"]
        self.rot_eps = e["rotEps"]
        self.vel_obs_scale = 0.2; self.force_torque_obs_scale = 10.0                                            # shadow_hand.py:62-63
        self.reset_position_noise = e["resetPositionNoise"]; self.reset_rotation_noise = e["resetRotationNoise"]
        self.reset_dof_pos_noise = e["resetDofPosRandomInterval"]; self.reset_dof_vel_noise = e["resetDofVelRandomInterval"]
        self.force_scale = e.get("forceScale", 0.0)                                                             # shadow_hand.py:69-72
        self.force_prob_range = e.get("forceProbRange", [0.001, 0.1])
        self.force_decay = e.get("forceDecay", 0.99)
        self.force_decay_interval = e.get("forceDecayInterval", 0.08)
        self.shadow_hand_dof_speed_scale = e["dofSpeedScale"]; self.use_relative_control = e["useRelativeControl"]
        self.act_moving_average = e["actionsMovingAverage"]
        self.max_episode_length = e["episodeLength"]
        self.reset_time = e.get("resetTime", -1.0)
        self.print_success_stat = e["printNumSuccesses"]
        self.max_consecutive_successes = e["maxConsecutiveSuccesses"]
        self.av_factor = e.get("averFactor", 0.1)
        self.object_type = e["objectType"]
        assert self.object_type in ["block", "egg", "pen"]                                                      # shadow_hand.py:87
        self.ignore_z = (self.object_type == "pen")                                                             # :89
        self.obs_type = e["observationType"]
        if self.obs_type not in NUM_OBS:
            raise Exception("Unknown type of observations!\\nobservationType should be one of: [openai, full_no_vel, full, full_state]")
        self.asymmetric_obs = bool(e["asymmetric_observations"])
        self.fingertips = list(FINGERTIPS); self.num_fingertips = 5
        cfg["env"]["numObservations"] = NUM_OBS[self.obs_type]
        cfg["env"]["numStates"] = 211 if self.asymmetric_obs else 0                                            # shadow_hand.py:126-128
        cfg["env"]["numActions"] = 20
        self.up_axis, self.up_axis_idx = "z", 2
        super().__init__(config=cfg, rl_device=rl_device, sim_device=sim_device, graphics_device_id=graphics_device_id,
                         headless=headless, virtual_screen_capture=virtual_screen_capture, force_render=force_render)
        if self.reset_time > 0.0:                                                                              # shadow_hand.py:147-151
            self.max_episode_length = int(round(self.reset_time / (self.control_freq_inv * self.dt)))
            self._bind_task()

    # ---- shadow_hand.py:225-300
    def _build_model(self):
        a = self.cfg["env"].get("asset", {})
        opts = BuildOptions(fix_base_link=True, collapse_fixed_joints=True, disable_gravity=True, angular_damping=0.01,
                            capsule_mid_spheres=1)
        model = copy.deepcopy(load_asset_file(_asset_root(), a.get("assetFileName", "mjcf/open_ai_assets/hand/shadow_hand.xml"), opts))
        engine.warn_self_collision("ShadowHand", "shadow_hand.py:359 create_actor(..., i, -1, 0): the MJCF's own contact pairs, finger vs finger")
        obj_file = {"block": a.get("assetFileNameBlock", "urdf/objects/cube_multicolor.urdf"),                  # :91-99
                    "egg": a.get("assetFileNameEgg", "mjcf/open_ai_assets/hand/egg.xml"),
                    "pen": a.get("assetFileNamePen", "mjcf/open_ai_assets/hand/pen.xml")}[self.object_type]
        cube = load_asset_file(_asset_root(), obj_file, BuildOptions())
        self.fingertip_handles_np = np.array([model.body_names.index(n) for n in self.fingertips], dtype=np.int32)
        model.sensor_body = self.fingertip_handles_np.copy()                                                   # :292-296
        model.sensor_pos = np.zeros((5, 3)); model.sensor_quat = np.tile([0, 0, 0, 1.0], (5, 1))
        self.num_shadow_hand_dofs = self.num_dof = model.ndof
        self.num_shadow_hand_bodies = model.nb
        names = list(model.dof_names)
        self.actuated_dof_indices_np = np.array([names.index(j) for j in model.actuator_joint], dtype=np.int32)  # :268-269
        self.object_model = cube
        half, rnd = object_shape(cube)
        self._obj = dict(mass=float(cube.mass[0]), inertia=[float(cube.inertia[0][k]) for k in range(3)], half=half, round=rnd,
                         mu=1.0, gravity_on=1,
                         # object_asset_options = gymapi.AssetOptions() (shadow_hand.py:279): the defaults angular_damping 0.5, linear 0
                         # and max_angular_velocity 64 rad/s
                         angular_damping=0.5, linear_damping=0.0, max_angular_velocity=64.0)
        self._tendons = [t for t in model.tendons if t["name"] in RELEVANT_TENDONS]                             # :255-266
        return model

    def create_sim(self):
        model = self._build_model()
        sim_cfg = self.cfg["sim"]
        self.model = model
        self.tendon_damping = 0.1                                                                              # t_damping, shadow_hand.py:257
        ext = engine.pack_model_ext(model, obj=self._obj, actors_per_env=3, tendons=self._tendons, tendon_k=30.0, tendon_d=self.tendon_damping)
        self.sim = sim = engine.Sim(model, self.num_envs, dt=sim_cfg["dt"], substeps=sim_cfg["substeps"],
                                    gravity=tuple(sim_cfg["gravity"]), ground_mu=1.0, device=self.device, ext=ext)
        dev, N = self.device, self.num_envs
        # start poses, shadow_hand.py:299-317
        hand_p = np.array([0.0, 0.0, 0.5]); hand_q = np.asarray(model.default_root_quat, dtype=np.float64)
        obj_p = hand_p + np.array([0.0, -0.39, 0.02 if self.object_type == "pen" else 0.10])               # :312-318
        self.goal_displacement_tensor = torch.tensor([-0.2, -0.06, 0.12], device=dev)
        rs = sim.root_state.view(N, 3, 13)
        rs[:, :, 6] = 1.0
        rs[:, 0, 0:3] = torch.tensor(hand_p, dtype=torch.float32, device=dev)
        rs[:, 0, 3:7] = torch.tensor(hand_q, dtype=torch.float32, device=dev)
        rs[:, 1, 0:3] = torch.tensor(obj_p, dtype=torch.float32, device=dev)
        goal_p = torch.tensor(obj_p, dtype=torch.float32, device=dev) + self.goal_displacement_tensor
        goal_p[2] -= 0.04
        rs[:, 2, 0:3] = goal_p
        self.root_state_tensor = sim.root_state                                                                # (N*3, 13), :183
        self.hand_indices = torch.arange(0, 3 * N, 3, device=dev)
        self.object_indices = self.hand_indices + 1
        self.goal_object_indices = self.hand_indices + 2
        self.hand_start_states = rs[:, 0].clone()
        self.object_init_state = rs[:, 1].clone()                                                              # :398
        self.goal_states = self.object_init_state.clone()
        self.goal_states[:, 2] -= 0.04                                                                         # :399-401
        self.goal_init_state = self.goal_states.clone()
        self.initial_root_states = torch.stack([self.hand_start_states, self.object_init_state, self.goal_init_state], 1).reshape(3 * N, 13).contiguous()
        # tensors of __init__, shadow_hand.py:157-200
        self.dof_state = sim.dof_state
        self.shadow_hand_dof_state = self.dof_state.view(N, -1, 2)[:, :self.num_shadow_hand_dofs]
        self.shadow_hand_dof_pos = self.shadow_hand_dof_state[..., 0]
        self.shadow_hand_dof_vel = self.shadow_hand_dof_state[..., 1]
        self.vec_sensor_tensor = sim.acquire(engine.T_FORCE_SENSOR).view(N, 30)
        self.dof_force_tensor = sim.acquire(engine.T_DOF_FORCE).view(N, self.num_shadow_hand_dofs)
        self.num_bodies = model.nb + 2
        self.num_dofs = self.num_shadow_hand_dofs
        self.cur_targets = sim.dof_target
        self.prev_targets = torch.zeros((N, self.num_dofs), dtype=torch.float, device=dev)
        self.actuated_dof_indices = torch.tensor(self.actuated_dof_indices_np, dtype=torch.long, device=dev)
        self.shadow_hand_dof_lower_limits = torch.tensor(model.lower[1:], dtype=torch.float, device=dev)
        self.shadow_hand_dof_upper_limits = torch.tensor(model.upper[1:], dtype=torch.float, device=dev)
        self.shadow_hand_dof_default_pos = torch.zeros(self.num_dofs, dtype=torch.float, device=dev)
        self.shadow_hand_dof_default_vel = torch.zeros(self.num_dofs, dtype=torch.float, device=dev)
        self.fingertip_handles = torch.tensor(self.fingertip_handles_np, dtype=torch.long, device=dev)
        self.reset_goal_buf = torch.ones(N, device=dev, dtype=torch.long)                                      # reset_buf.clone(), :192
        self.successes = torch.zeros(N, dtype=torch.float, device=dev)
        self._cons = torch.zeros(4, dtype=torch.float, device=dev)
        self.consecutive_successes = self._cons[0:1]
        self.goal_reset_count = torch.zeros(N, dtype=torch.int32, device=dev)
        self.object_rb_masses = torch.tensor([self._obj["mass"]], dtype=torch.float, device=dev)
        # random forces on the object (shadow_hand.py:196-201).  The reference keeps rb_forces (N, bodies, 3) of which only the
        # object's row is ever non-zero; the engine's tensor is that row (N, 3), in the object's frame (LOCAL_SPACE, :708)
        self.force_decay = torch.tensor(self.force_decay, dtype=torch.float, device=dev)
        self.force_prob_range = torch.tensor(self.force_prob_range, dtype=torch.float, device=dev)
        self.random_force_prob = torch.exp((torch.log(self.force_prob_range[0]) - torch.log(self.force_prob_range[1]))
                                           * torch.rand(N, device=dev) + torch.log(self.force_prob_range[1])).contiguous()
        self.object_rb_forces = torch.zeros((N, 3), dtype=torch.float, device=dev)
        self.object_rb_handles = torch.tensor([model.nb], dtype=torch.long, device=dev)
        self.total_successes = 0; self.total_resets = 0
        return sim

    # ---- domain randomisation (task.randomize): the hand and object kernels read per-env object, tendon and gravity parameters
    dr_gravity = True

    def _dr_actors(self):
        return dict(actors={"hand": "articulation", "object": "object"}, obj=self._obj,
                    tendon_damping=[self.tendon_damping] * len(self._tendons))

    def _randomize_this_step(self):
        return bool(self.reset_buf.any())

    @property
    def rigid_body_states(self):
        """(N, bodies, 13) like gym.refresh_rigid_body_state_tensor + the view of shadow_hand.py:180 (computed on demand)."""
        return self.sim.refresh_rigid_body_state().view(self.num_envs, -1, 13)

    @property
    def rb_forces(self):
        """(N, bodies, 3) as shadow_hand.py:201 holds it: zero except the object's row (a copy; the engine owns object_rb_forces)."""
        f = torch.zeros((self.num_envs, self.num_bodies, 3), dtype=torch.float, device=self.device)
        f[:, self.model.nb] = self.object_rb_forces
        return f

    @property
    def object_pos(self):
        return self.root_state_tensor[self.object_indices, 0:3]

    @property
    def object_rot(self):
        return self.root_state_tensor[self.object_indices, 3:7]

    @property
    def goal_pos(self):
        return self.goal_states[:, 0:3]

    @property
    def goal_rot(self):
        return self.goal_states[:, 3:7]

    def _task_buffers(self):
        E = engine
        extra = {E.T_STATES: self.states_buf} if self.asymmetric_obs else {}
        return {**extra, E.T_INITIAL_ROOT: self.initial_root_states, E.T_GOAL_STATES: self.goal_states, E.T_PREV_TARGETS: self.prev_targets,
                E.T_SUCCESSES: self.successes, E.T_CONSECUTIVE_SUCCESSES: self._cons, E.T_RESET_GOAL: self.reset_goal_buf,
                E.T_GOAL_RESET_COUNT: self.goal_reset_count, E.T_OBJ_FORCE: self.object_rb_forces,
                E.T_RANDOM_FORCE_PROB: self.random_force_prob}

    def _task_params(self):
        p = engine.CHandParams()
        p.obs_type = engine.HAND_OBS[self.obs_type]
        p.num_states = int(self.num_states)
        p.max_episode_length = float(self.max_episode_length)
        p.use_relative_control = int(bool(self.use_relative_control))
        p.max_consecutive_successes = int(self.max_consecutive_successes)
        p.dof_speed_scale = float(self.shadow_hand_dof_speed_scale)
        p.act_moving_average = float(self.act_moving_average)
        p.dt = float(self.dt)
        p.dist_reward_scale, p.rot_reward_scale, p.rot_eps = float(self.dist_reward_scale), float(self.rot_reward_scale), float(self.rot_eps)
        # compute_hand_reward doubles the tolerance when ignore_z_rot (the pen), shadow_hand.py:758-759
        p.action_penalty_scale, p.success_tolerance = float(self.action_penalty_scale), float(self.success_tolerance) * (2.0 if self.ignore_z else 1.0)
        p.reach_goal_bonus, p.fall_dist, p.fall_penalty = float(self.reach_goal_bonus), float(self.fall_dist), float(self.fall_penalty)
        p.av_factor = float(self.av_factor)
        p.vel_obs_scale, p.force_torque_obs_scale = float(self.vel_obs_scale), float(self.force_torque_obs_scale)
        p.reset_position_noise = float(self.reset_position_noise)
        p.reset_dof_pos_noise, p.reset_dof_vel_noise = float(self.reset_dof_pos_noise), float(self.reset_dof_vel_noise)
        p.goal_displacement = (engine.C.c_float * 3)(-0.2, -0.06, 0.12)
        for k, d in enumerate(self.actuated_dof_indices_np):
            p.actuated_dof[k] = int(d)
        lo, hi = self.model.lower[1:], self.model.upper[1:]
        for d in range(self.num_dofs):
            p.dof_lower[d], p.dof_upper[d] = float(lo[d]), float(hi[d])
            p.dof_default_pos[d] = 0.0; p.dof_default_vel[d] = 0.0
        for f in range(5):
            p.fingertip_body[f] = int(self.fingertip_handles_np[f])
        # random object forces (:700-709): the constants in the float32 arithmetic of the reference's tensors
        p.object_is_pen = int(self.object_type == "pen")            # reset_idx poses the pen with randomize_rotation_pen (:626-629)
        p.force_scale = float(self.force_scale)
        p.force_decay_factor = float(torch.pow(self.force_decay, self.dt / self.force_decay_interval))
        p.force_logp_span = float(torch.log(self.force_prob_range[0]) - torch.log(self.force_prob_range[1]))
        p.force_logp1 = float(torch.log(self.force_prob_range[1]))
        return p

    def _fill_extras(self):
        self.extras['consecutive_successes'] = self.consecutive_successes.mean()                                # shadow_hand.py:424

"""ctypes binding of libb200gym.so (include/b200gym.h) -- the only way the Python side reaches the
CUDA engine.  torch is used for device memory and streams only: every tensor handed out by `Sim`
is a torch tensor whose storage the engine reads/writes in place (the reference's
`gymtorch.wrap_tensor` contract, tasks/ant.py:78-95).

There is no CPU fallback: if the library is missing or no CUDA device is present, construction
raises (b2g_create returns B2G_E_CUDA).
"""
import ctypes as C
import os
import numpy as np
import torch

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
MAXL = 32

# tensor slots (mirror of the enum in include/b200gym.h)
(T_ROOT_STATE, T_DOF_STATE, T_DOF_ACTUATION, T_DOF_TARGET, T_RIGID_BODY_STATE, T_FORCE_SENSOR, T_DOF_FORCE,
 T_NET_CONTACT, T_ACTIONS, T_OBS, T_REW, T_RESET, T_PROGRESS, T_TIMEOUT, T_POTENTIALS, T_PREV_POTENTIALS,
 T_UP_VEC, T_HEADING_VEC, T_INITIAL_ROOT, T_RESET_COUNT, T_OBS_CLIPPED, T_COMMANDS, T_LAST_ACTIONS, T_LAST_DOF_VEL,
 T_FEET_AIR_TIME, T_TORQUES, T_EPISODE_SUMS, T_TERRAIN_LEVELS, T_TERRAIN_TYPES, T_ENV_ORIGINS, T_TERRAIN_ORIGINS,
 T_NOISE_SCALE, T_BASE_SCRATCH, T_REDUCE_SCRATCH, T_ENV_FRICTION, T_GOAL_STATES, T_PREV_TARGETS, T_SUCCESSES,
 T_CONSECUTIVE_SUCCESSES, T_RESET_GOAL, T_GOAL_RESET_COUNT, T_STATES, T_ENV_MASS_SCALE, T_ENV_DOF_PROPS,
 T_JACOBIAN, T_MASS_MATRIX, T_OBJ_FORCE, T_RANDOM_FORCE_PROB, T_ENV_OBJ_PROPS, T_ENV_TENDON_DAMPING, T_GRAVITY) = range(51)
TASK_NONE, TASK_CARTPOLE, TASK_ANT, TASK_HUMANOID, TASK_ANYMAL_TERRAIN, TASK_SHADOW_HAND = 0, 1, 2, 3, 4, 5
HAND_OBS = {"openai": 0, "full_no_vel": 1, "full": 2, "full_state": 3}


class CHandParams(C.Structure):
    _fields_ = [("num_obs", C.c_int32), ("num_actions", C.c_int32), ("obs_type", C.c_int32), ("control_freq_inv", C.c_int32),
                ("clip_actions", C.c_float), ("clip_obs", C.c_float), ("max_episode_length", C.c_float),
                ("use_relative_control", C.c_int32), ("max_consecutive_successes", C.c_int32),
                ("dof_speed_scale", C.c_float), ("act_moving_average", C.c_float), ("dt", C.c_float),
                ("dist_reward_scale", C.c_float), ("rot_reward_scale", C.c_float), ("rot_eps", C.c_float),
                ("action_penalty_scale", C.c_float), ("success_tolerance", C.c_float), ("reach_goal_bonus", C.c_float),
                ("fall_dist", C.c_float), ("fall_penalty", C.c_float), ("av_factor", C.c_float),
                ("vel_obs_scale", C.c_float), ("force_torque_obs_scale", C.c_float),
                ("reset_position_noise", C.c_float), ("reset_dof_pos_noise", C.c_float), ("reset_dof_vel_noise", C.c_float),
                ("goal_displacement", C.c_float * 3), ("actuated_dof", C.c_int32 * 32),
                ("dof_lower", C.c_float * 32), ("dof_upper", C.c_float * 32), ("dof_default_pos", C.c_float * 32),
                ("dof_default_vel", C.c_float * 32), ("fingertip_body", C.c_int32 * 5), ("num_states", C.c_int32),
                ("seed", C.c_uint64), ("env_id_offset", C.c_int32), ("pad1", C.c_int32),
                ("force_scale", C.c_float), ("force_decay_factor", C.c_float), ("force_logp_span", C.c_float), ("force_logp1", C.c_float),
                ("object_is_pen", C.c_int32), ("pad2", C.c_int32)]


class CAnymalParams(C.Structure):
    _fields_ = [("num_obs", C.c_int32), ("num_actions", C.c_int32), ("decimation", C.c_int32), ("control_freq_inv", C.c_int32),
                ("clip_actions", C.c_float), ("clip_obs", C.c_float), ("max_episode_length", C.c_int32),
                ("push_interval", C.c_int32), ("push_robots", C.c_int32), ("add_noise", C.c_int32), ("curriculum", C.c_int32),
                ("allow_knee_contacts", C.c_int32), ("custom_origins", C.c_int32), ("pad0", C.c_int32),
                ("kp", C.c_float), ("kd", C.c_float), ("action_scale", C.c_float), ("torque_limit", C.c_float),
                ("default_dof_pos", C.c_float * 32), ("lin_vel_scale", C.c_float), ("ang_vel_scale", C.c_float),
                ("dof_pos_scale", C.c_float), ("dof_vel_scale", C.c_float), ("height_meas_scale", C.c_float),
                ("rew_scales", C.c_float * 14), ("dt", C.c_float), ("max_episode_length_s", C.c_float),
                ("command_x", C.c_float * 2), ("command_y", C.c_float * 2), ("command_yaw", C.c_float * 2),
                ("base_init_state", C.c_float * 13), ("border_size", C.c_float), ("terrain_hscale", C.c_float),
                ("terrain_vscale", C.c_float), ("env_length", C.c_float), ("hs_rows", C.c_int32), ("hs_cols", C.c_int32),
                ("env_rows", C.c_int32), ("env_cols", C.c_int32), ("base_body", C.c_int32), ("knee_bodies", C.c_int32 * 4),
                ("feet_bodies", C.c_int32 * 4), ("pad1", C.c_int32), ("seed", C.c_uint64), ("env_id_offset", C.c_int32),
                ("pad2", C.c_int32)]


class CModel(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("nl", "ncp", "nb", "nsens", "root_fixed", "gravity_on")] + \
               [(n, C.c_void_p) for n in ("parent", "jtype", "limited", "drive_mode", "cp_link", "cp_body", "body_link",
                                          "sensor_body", "axis", "lpos", "lquat", "mass", "com", "inertia", "armature",
                                          "damping", "stiffness", "lower", "upper", "effort", "kp", "kd", "limit_k",
                                          "limit_d", "cp_pos", "cp_radius", "cp_mu", "body_pos", "body_quat")] + \
               [("contact_kn", C.c_float), ("contact_cn", C.c_float), ("contact_vs", C.c_float),
                ("angular_damping", C.c_float), ("linear_damping", C.c_float), ("max_angular_velocity", C.c_float),
                ("self_collide", C.c_int32), ("pad_self", C.c_int32), ("self_pairs", C.c_void_p),
                ("self_kn", C.c_float), ("self_cn", C.c_float), ("self_mu", C.c_float), ("pad_self2", C.c_float)]


class CModelExt(C.Structure):
    _fields_ = [("actors_per_env", C.c_int32), ("obj_actor", C.c_int32), ("obj_gravity_on", C.c_int32), ("pad0", C.c_int32),
                ("obj_mass", C.c_float), ("obj_inertia", C.c_float * 3), ("obj_half", C.c_float * 3),
                ("obj_kn", C.c_float), ("obj_cn", C.c_float), ("obj_mu", C.c_float),
                ("nbox", C.c_int32), ("box_link", C.c_int32 * 4), ("box_pos", (C.c_float * 3) * 4),
                ("box_quat", (C.c_float * 4) * 4), ("box_half", (C.c_float * 3) * 4),
                ("nten", C.c_int32), ("ten_dof", (C.c_int32 * 2) * 4), ("ten_coef", (C.c_float * 2) * 4),
                ("ten_range", (C.c_float * 2) * 4), ("ten_k", C.c_float), ("ten_d", C.c_float),
                ("obj_angular_damping", C.c_float), ("obj_linear_damping", C.c_float),
                ("obj_round", C.c_float), ("obj_max_angular_velocity", C.c_float)]


def object_contact_gains(mass):
    """Penalty gains of every contact of the free object (DESIGN.md "free object"): the object is light, so the
    gains scale with ITS mass; critically damped for the two-body reduced mass."""
    kn = 10000.0 * mass
    return kn, 2.0 * float(np.sqrt(kn * mass / 4.0))


def pack_model_ext(model, obj=None, actors_per_env=1, tendons=None, tendon_k=0.0, tendon_d=0.0):
    """obj: dict(mass, inertia(3), half(3), mu, gravity_on[, round]) of the free (rounded) box (actor 1), or None."""
    ex = CModelExt()
    ex.actors_per_env = int(actors_per_env)
    ex.obj_actor = -1
    if obj is not None:
        ex.obj_actor, ex.obj_gravity_on = 1, int(obj.get("gravity_on", 1))
        ex.obj_mass = float(obj["mass"])
        ex.obj_angular_damping, ex.obj_linear_damping = float(obj.get("angular_damping", 0.0)), float(obj.get("linear_damping", 0.0))
        ex.obj_inertia = (C.c_float * 3)(*obj["inertia"]); ex.obj_half = (C.c_float * 3)(*obj["half"])
        ex.obj_round = float(obj.get("round", 0.0))
        ex.obj_max_angular_velocity = float(obj.get("max_angular_velocity", 64.0))       # gymapi.AssetOptions default
        kn, cn = object_contact_gains(ex.obj_mass)
        ex.obj_kn, ex.obj_cn, ex.obj_mu = kn, cn, float(obj.get("mu", 1.0))
        bl = getattr(model, "box_link", None)
        ex.nbox = 0 if bl is None else len(bl)
        for b in range(ex.nbox):
            ex.box_link[b] = int(model.box_link[b])
            for c in range(3):
                ex.box_pos[b][c] = float(model.box_pos[b][c]); ex.box_half[b][c] = float(model.box_half[b][c])
            for c in range(4):
                ex.box_quat[b][c] = float(model.box_quat[b][c])
    dn = list(model.dof_names)
    ix = lambda d: int(d) if isinstance(d, (int, np.integer)) else dn.index(d)
    ex.nten = len(tendons or [])
    for t, td in enumerate(tendons or []):
        for k in range(2):
            ex.ten_dof[t][k] = ix(td["dofs"][k]); ex.ten_coef[t][k] = float(td["coefs"][k]); ex.ten_range[t][k] = float(td["range"][k])
    ex.ten_k, ex.ten_d = float(tendon_k), float(tendon_d)
    return ex


class CSimParams(C.Structure):
    _fields_ = [("dt", C.c_float), ("substeps", C.c_int32), ("gravity", C.c_float * 3), ("hf_samples", C.c_void_p),
                ("hf_nx", C.c_int32), ("hf_ny", C.c_int32), ("hf_horizontal_scale", C.c_float),
                ("hf_vertical_scale", C.c_float), ("hf_origin_x", C.c_float), ("hf_origin_y", C.c_float),
                ("ground_friction", C.c_float), ("pad_", C.c_float)]


class CTaskParams(C.Structure):
    _fields_ = [("task", C.c_int32), ("num_obs", C.c_int32), ("num_actions", C.c_int32), ("control_freq_inv", C.c_int32),
                ("clip_actions", C.c_float), ("clip_obs", C.c_float), ("max_episode_length", C.c_float),
                ("power_scale", C.c_float), ("joint_gears", C.c_float * MAXL), ("motor_efforts", C.c_float * MAXL),
                ("max_motor_effort", C.c_float), ("dof_limits_lower", C.c_float * MAXL),
                ("dof_limits_upper", C.c_float * MAXL), ("initial_dof_pos", C.c_float * MAXL),
                ("dof_vel_scale", C.c_float), ("contact_force_scale", C.c_float), ("angular_velocity_scale", C.c_float),
                ("heading_weight", C.c_float), ("up_weight", C.c_float), ("actions_cost_scale", C.c_float),
                ("energy_cost_scale", C.c_float), ("joints_at_limit_cost_scale", C.c_float), ("death_cost", C.c_float),
                ("termination_height", C.c_float), ("alive_reward", C.c_float), ("reset_pos_noise", C.c_float),
                ("reset_vel_noise", C.c_float), ("dt", C.c_float), ("target", C.c_float * 3),
                ("max_push_effort", C.c_float), ("reset_dist", C.c_float), ("seed", C.c_uint64),
                ("env_id_offset", C.c_int32), ("pad_", C.c_int32)]


_lib = None


def lib():
    """Load (building if necessary) the CUDA library.  Fails loudly when it cannot be had."""
    global _lib
    if _lib is None:
        path = os.environ.get("B2G_LIB", "")          # experiment hook: an alternative build of the same ABI
        if not path:
            path = os.path.join(_HERE, "libb200gym.so")
            if not os.path.exists(path) or _build.needs_build():
                _build.build()
        _lib = C.CDLL(path)
        _lib.b2g_last_error.restype = C.c_char_p
        _lib.b2g_launch_count.restype = C.c_int64
        _lib.b2g_launch_count.argtypes = [C.c_void_p]
        for fn in ("b2g_plan", "b2g_create", "b2g_create_ext", "b2g_destroy", "b2g_bind", "b2g_simulate", "b2g_refresh_rigid_body_state",
                   "b2g_set_task", "b2g_set_anymal_task", "b2g_set_hand_task", "b2g_task_step", "b2g_task_step_host", "b2g_reset_flagged", "b2g_task_rollout",
                   "b2g_kin_shape", "b2g_refresh_kinematic_tensors"):
            getattr(_lib, fn).restype = C.c_int
    return _lib


EXPORTS = ("b2g_plan", "b2g_create", "b2g_create_ext", "b2g_destroy", "b2g_bind", "b2g_simulate", "b2g_refresh_rigid_body_state", "b2g_set_task",
           "b2g_set_anymal_task", "b2g_set_hand_task", "b2g_task_step", "b2g_task_step_host", "b2g_launch_count", "b2g_last_error", "b2g_version",
           "b2g_quad_chain_length", "b2g_reset_flagged", "b2g_task_rollout", "b2g_kin_shape", "b2g_refresh_kinematic_tensors")


class EngineError(RuntimeError):
    pass


class UnmodelledPhysicsWarning(UserWarning):
    """A physical effect the reference configuration switches on is not part of this engine's model."""


_warned = set()


def warn_self_collision(what, where):
    """The reference enables self-collision for this actor (create_actor(..., collision_filter=0) or the asset's own
    filter); the engine tests contact spheres against the ground / height field and the one free object only -- links of
    one articulation can pass through each other.  Said once per actor kind, never silently dropped."""
    import warnings
    if what in _warned:
        return
    _warned.add(what)
    warnings.warn(f"{what}: the reference enables self-collision here ({where}); this engine does not model link-link contact "
                  "within an articulation (DESIGN.md section 7) -- limbs may interpenetrate", UnmodelledPhysicsWarning, stacklevel=3)


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
if _raw_stream is None:                                     # older torch: the public (slower) accessor
    def _raw_stream(index):
        return torch.cuda.current_stream(index).cuda_stream


def _check(rc, what):
    if rc != 0:
        raise EngineError(f"{what} failed ({rc}): {lib().b2g_last_error().decode()}")


def pack_model(model, ground_mu=1.0):
    """importer Model -> (b2g_model struct, keep-alive arrays).  Friction: PhysX default combine
    mode averages the two materials (ground plane params: tasks/ant.py:128-133)."""
    keep = {}

    def arr(name, a, dt):
        a = np.ascontiguousarray(a, dtype=dt)
        keep[name] = a
        return a.ctypes.data
    cm = CModel()
    cm.nl, cm.ncp, cm.nb, cm.nsens = model.nl, len(model.cp_link), model.nb, len(model.sensor_body)
    cm.root_fixed, cm.gravity_on = int(model.root_fixed), int(model.gravity_on)
    for n in ("parent", "jtype", "limited", "drive_mode", "cp_link", "cp_body", "body_link", "sensor_body"):
        setattr(cm, n, arr(n, getattr(model, n), np.int32))
    for n in ("axis", "lpos", "lquat", "mass", "com", "inertia", "armature", "damping", "stiffness", "lower", "upper",
              "kp", "kd", "limit_k", "limit_d", "cp_pos", "cp_radius", "body_pos", "body_quat"):
        setattr(cm, n, arr(n, getattr(model, n), np.float32))
    cm.effort = arr("effort", np.minimum(model.effort, 3e38), np.float32)
    cm.cp_mu = arr("cp_mu", np.asarray(model.cp_mu), np.float32)
    cm.contact_kn, cm.contact_cn, cm.contact_vs = model.contact_kn, model.contact_cn, model.contact_vs
    cm.self_collide = 0
    if getattr(model, "self_collide", False):
        cm.self_collide = 1
        cm.self_pairs = arr("self_pairs", model.self_pairs, np.uint8)
        cm.self_kn, cm.self_cn, cm.self_mu = float(model.self_kn), float(model.self_cn), float(model.self_mu)
    cm.angular_damping = float(getattr(model, "angular_damping", 0.0) or 0.0)
    cm.linear_damping = float(getattr(model, "linear_damping", 0.0) or 0.0)
    cm.max_angular_velocity = float(getattr(model, "max_angular_velocity", 0.0) or 0.0)
    return cm, keep


def plan(model, lanes=0, compact=False):
    """The slot programs the engine builds for `model` (host only, no GPU): -> (info dict, slots int32 [24][8][8])."""
    cm, keep = pack_model(model)
    slots = np.zeros((24, 8, 8), np.int32)
    info = (C.c_int32 * 5)()
    _check(lib().b2g_plan(C.byref(cm), C.c_int32(lanes), C.c_int32(int(compact)), C.c_void_p(slots.ctypes.data), info), "b2g_plan")
    return dict(ns=info[0], lanes=info[1], nacc=info[2], root_acc=info[3], cross_lane=info[4]), slots


class Sim:
    """N identical single-actor environments on one GPU (gym.create_sim .. prepare_sim)."""

    def __init__(self, model, num_envs, dt, substeps, gravity=(0.0, 0.0, -9.81), ground_mu=1.0, device="cuda:0",
                 hfield=None, hf_horizontal_scale=1.0, hf_vertical_scale=1.0, hf_origin=(0.0, 0.0), ext=None):
        self.model = model
        self.actors_per_env = int(ext.actors_per_env) if ext is not None else 1
        self.num_envs = int(num_envs)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise EngineError("the CUDA engine has no CPU path: device must be a CUDA device")
        self.nd, self.nb, self.ns = model.ndof, model.nb, len(model.sensor_body)
        cm, self._keep = pack_model(model, ground_mu)
        sp = CSimParams()
        sp.dt, sp.substeps = dt, int(substeps)
        sp.gravity = (C.c_float * 3)(*gravity)
        sp.ground_friction = float(ground_mu)
        if hfield is not None:
            hf = np.ascontiguousarray(hfield, dtype=np.int16)
            self._keep["hf"] = hf
            sp.hf_samples = hf.ctypes.data
            sp.hf_nx, sp.hf_ny = hf.shape
            sp.hf_horizontal_scale, sp.hf_vertical_scale = hf_horizontal_scale, hf_vertical_scale
            sp.hf_origin_x, sp.hf_origin_y = hf_origin
        self._h = C.c_void_p()
        idx = self.device.index if self.device.index is not None else 0
        if ext is not None:
            _check(lib().b2g_create_ext(C.byref(cm), C.byref(ext), C.byref(sp), C.c_int32(self.num_envs), C.c_int32(idx),
                                        C.byref(self._h)), "b2g_create_ext")
        else:
            _check(lib().b2g_create(C.byref(cm), C.byref(sp), C.c_int32(self.num_envs), C.c_int32(idx), C.byref(self._h)),
                   "b2g_create")
        self.tensors = {}
        self._dev_index = idx
        self._step_fn = lib().b2g_task_step
        self._step_fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        N = self.num_envs
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=self.device)
        self.root_state = self._bind(T_ROOT_STATE, z(N * self.actors_per_env, 13))
        self.root_state[:, 6] = 1.0
        self.dof_state = self._bind(T_DOF_STATE, z(N * max(self.nd, 1), 2))
        self.dof_actuation = self._bind(T_DOF_ACTUATION, z(N, max(self.nd, 1)))
        self.dof_target = self._bind(T_DOF_TARGET, z(N, max(self.nd, 1)))
        self.task = None

    # ---- tensor plumbing
    def _bind(self, slot, t):
        assert t.is_contiguous() and t.device == self.device
        _check(lib().b2g_bind(self._h, C.c_int32(slot), C.c_void_p(t.data_ptr()), C.c_size_t(t.numel() * t.element_size())),
               f"b2g_bind({slot})")
        self.tensors[slot] = t
        return t

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def acquire(self, slot):
        """Lazy `gym.acquire_*_tensor`: allocates and binds the optional output tensors."""
        if slot in self.tensors:
            return self.tensors[slot]
        N = self.num_envs
        if slot in (T_JACOBIAN, T_MASS_MATRIX):
            rows, nc = self.kin_shape()
            shape = (N, rows, 6, nc) if slot == T_JACOBIAN else (N, nc, nc)
            return self._bind(slot, torch.zeros(*shape, dtype=torch.float32, device=self.device))
        shape = {T_RIGID_BODY_STATE: (N * (self.nb + self.actors_per_env - 1), 13), T_FORCE_SENSOR: (N * max(self.ns, 1), 6),
                 T_DOF_FORCE: (N * max(self.nd, 1),), T_NET_CONTACT: (N * self.nb, 3)}[slot]
        return self._bind(slot, torch.zeros(*shape, dtype=torch.float32, device=self.device))

    # ---- gym.* calls
    def simulate(self):
        _check(lib().b2g_simulate(self._h, self._stream()), "b2g_simulate")

    def refresh_rigid_body_state(self):
        self.acquire(T_RIGID_BODY_STATE)
        _check(lib().b2g_refresh_rigid_body_state(self._h, self._stream()), "b2g_refresh_rigid_body_state")
        return self.tensors[T_RIGID_BODY_STATE]

    def kin_shape(self):
        """(rows, columns) of the Jacobian tensor: a fixed base has no row for its base body and no base columns; a floating
        base has six leading columns (world linear, world angular velocity of the root origin)."""
        out = (C.c_int32 * 2)()
        lib().b2g_kin_shape.argtypes = [C.c_void_p, C.c_void_p]
        _check(lib().b2g_kin_shape(self._h, out), "b2g_kin_shape")
        return int(out[0]), int(out[1])

    def refresh_kinematic_tensors(self, jacobian=True, mass_matrix=True):
        """gym.refresh_jacobian_tensors / refresh_mass_matrix_tensors (franka_cube_stack.py:439-440), one launch for both."""
        which = 0
        if jacobian:
            self.acquire(T_JACOBIAN); which |= 1
        if mass_matrix:
            self.acquire(T_MASS_MATRIX); which |= 2
        _check(lib().b2g_refresh_kinematic_tensors(self._h, C.c_int32(which), self._stream()), "b2g_refresh_kinematic_tensors")
        return self.tensors.get(T_JACOBIAN), self.tensors.get(T_MASS_MATRIX)

    # ---- fused task step
    def set_task(self, params: CTaskParams, buffers: dict):
        """buffers: slot -> torch tensor for the task-level slots."""
        for slot, t in buffers.items():
            self._bind(slot, t)
        self.task = params
        if isinstance(params, CAnymalParams):
            _check(lib().b2g_set_anymal_task(self._h, C.byref(params)), "b2g_set_anymal_task")
        elif isinstance(params, CHandParams):
            _check(lib().b2g_set_hand_task(self._h, C.byref(params)), "b2g_set_hand_task")
        else:
            _check(lib().b2g_set_task(self._h, C.byref(params)), "b2g_set_task")

    def task_step(self, actions: torch.Tensor):
        """b2g_task_step on the current torch stream; the hot call of VecTask.step (argument conversion pre-bound, raw
        stream handle: a few microseconds of host time per step matter next to a ~10 us kernel)."""
        if actions.dtype is not torch.float32 or not actions.is_cuda or not actions.is_contiguous():
            raise EngineError("task_step: actions must be a contiguous float32 CUDA tensor")
        rc = self._step_fn(self._h, actions.data_ptr(), _raw_stream(self._dev_index))
        if rc != 0:
            _check(rc, "b2g_task_step")

    def task_step_host(self, h_actions, h_obs=None, h_rew=None, h_reset=None, h_timeout=None):
        """Host-buffer step (CPU torch tensors, ideally pinned); synchronises."""
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _check(lib().b2g_task_step_host(self._h, p(h_actions), p(h_obs), p(h_rew), p(h_reset), p(h_timeout),
                                        self._stream()), "b2g_task_step_host")

    def task_rollout(self, actions, obs_out, rew_out, reset_out, timeout_out=None):
        """K x task_step with all actions given up front (K, N, A); results of every step in the (K, N, .) outputs."""
        for t in (actions, obs_out, rew_out, reset_out):
            if not t.is_cuda or not t.is_contiguous():
                raise EngineError("task_rollout: contiguous CUDA tensors expected")
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _check(lib().b2g_task_rollout(self._h, p(actions), C.c_int32(actions.shape[0]), p(obs_out), p(rew_out), p(reset_out),
                                      p(timeout_out), self._stream()), "b2g_task_rollout")

    def reset_flagged(self):
        """reset_idx of every env whose reset flag is set (VecTask.reset_done)."""
        _check(lib().b2g_reset_flagged(self._h, self._stream()), "b2g_reset_flagged")

    def launch_count(self):
        return int(lib().b2g_launch_count(self._h))

    def quad_ns(self):
        """0: generic stepper; 2 / 3: the specialised four-chain stepper (b2g_quad.cuh) with this chain length."""
        lib().b2g_quad_chain_length.argtypes = [C.c_void_p]
        return int(lib().b2g_quad_chain_length(self._h))

    def close(self):
        if self._h:
            lib().b2g_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

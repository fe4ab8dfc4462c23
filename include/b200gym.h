/*
 * b200gym.h -- C ABI of the CUDA-native (H100) vectorised environment stepper.
 *
 * The reference has no C FFI: its boundary for this path is the Python surface of the closed
 * `isaacgym` module (SURVEY.md 8b).  Each entry point below names the reference call it stands
 * behind (file:line under isaacgymenvs/ of the reference).  Conventions, taken from the call sites:
 *   - single caller thread, one sim per process is the common case (tasks/base/vec_task.py:58-64)
 *     but several handles may coexist;
 *   - all work is STREAM-ORDERED on the cudaStream_t passed in (the reference issues on the
 *     current torch stream);
 *   - state lives in buffers the CALLER owns (torch tensors on the host side) and binds once with
 *     b2g_bind(); layouts are exactly the reference's tensor views (`acquire_*_tensor`,
 *     tasks/ant.py:78-95): env-major, float32, quaternions xyzw;
 *   - every function returns 0 on success, a negative B2G_E_* code otherwise and never throws;
 *     b2g_last_error() gives the message.  There is NO CPU fallback: without a CUDA device
 *     b2g_create fails with B2G_E_CUDA.
 */
#ifndef B200GYM_H
#define B200GYM_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2G_VERSION 4
#define B2G_MAX_LINKS 32
#define B2G_MAX_CONTACT_POINTS 96
#define B2G_MAX_BOXES 4
#define B2G_MAX_TENDONS 4
#define B2G_MAX_SENSORS 8

enum {
    B2G_OK = 0,
    B2G_E_INVALID = -1,     /* bad argument / model too large */
    B2G_E_CUDA = -2,        /* CUDA runtime error (message has the cudaError string) */
    B2G_E_UNBOUND = -3,     /* a tensor the call needs was never bound */
    B2G_E_UNSUPPORTED = -4  /* no compiled kernel for this articulation topology / task */
};

/* Articulation model, host memory, copied by b2g_create.  Produced by the asset importer
 * (replaces gym.load_asset + gym.create_actor, tasks/ant.py:149-190).  Link 0 is the root. */
typedef struct {
    int32_t nl, ncp, nb, nsens;
    int32_t root_fixed, gravity_on;
    const int32_t *parent;       /* nl, -1 for the root; parent[i] < i */
    const int32_t *jtype;        /* nl: -1 root, 0 hinge, 1 slide */
    const int32_t *limited;      /* nl */
    const int32_t *drive_mode;   /* nl: gymapi.DOF_MODE_* (1 = position drive) */
    const int32_t *cp_link;      /* ncp: contact sphere -> link */
    const int32_t *cp_body;      /* ncp: contact sphere -> body (public numbering) */
    const int32_t *body_link;    /* nb */
    const int32_t *sensor_body;  /* nsens */
    const float *axis, *lpos, *lquat;          /* nl x 3, 3, 4(xyzw) */
    const float *mass, *com, *inertia;         /* nl x 1, 3, 6 (xx yy zz xy xz yz about the COM) */
    const float *armature, *damping, *stiffness, *lower, *upper, *effort, *kp, *kd, *limit_k, *limit_d; /* nl */
    const float *cp_pos, *cp_radius, *cp_mu;   /* ncp x 3, 1, 1 (mu = the shape's own friction) */
    const float *body_pos, *body_quat;         /* nb x 3, 4: body frame in its link frame */
    float contact_kn, contact_cn, contact_vs;
    /* gymapi.AssetOptions.angular_damping / linear_damping / max_angular_velocity (humanoid.py:153-154,
     * anymal_terrain.py:225-226): damping acceleration -d v on every link's COM twist; clamp of the base's angular speed
     * (0 = no clamp) */
    float angular_damping, linear_damping, max_angular_velocity;
    /* Self-collision = gym.create_actor(env, asset, pose, name, group, filter = 0) (humanoid.py:194): contact spheres of links
     * that are not joint neighbours collide with each other.  self_pairs: ncp x ncp bytes, 1 = the ordered pair may collide
     * (NULL / self_collide 0 = off).  Same contact law as the ground contact; self_kn, self_cn are DIMENSIONLESS: per pair
     * kn = self_kn m_red / h^2, cn = self_cn m_red / h with the reduced mass of the two links (stability of the half-explicit
     * coupling; 0.5 / 0.5 is what the importer sets); ncp <= 64, no second actor.  A four-chain model with chain length 3
     * (ANYmal) keeps the four-chain kernels, which carry the contact when no candidate pair lies within one leg; every other
     * self-colliding model, the chain-length-2 one (Ant) included, runs on the generic sub-step. */
    int32_t self_collide, pad_self;
    const uint8_t *self_pairs;
    float self_kn, self_cn, self_mu, pad_self2;
} b2g_model;

/* Optional extras of an environment with more than one actor (tasks/shadow_hand.py:338-383: hand, object, goal
 * object).  The articulation stays actor 0; actor `obj_actor` is a free rigid box simulated in contact with the
 * articulation's contact spheres, its box primitives and the ground; further actors (the goal marker, created with
 * gravity disabled in its own collision group, shadow_hand.py:281-282,380) are rows of the root-state tensor the
 * engine never moves.  ROOT_STATE / INITIAL_ROOT then are (N * actors_per_env, 13), env-major like the reference's
 * actor_root_state tensor (shadow_hand.py:183). */
typedef struct {
    int32_t actors_per_env;      /* >= 1 */
    int32_t obj_actor;           /* row of the free object inside an env's actors, or -1: none */
    int32_t obj_gravity_on, pad0;
    float obj_mass, obj_inertia[3], obj_half[3];   /* box, principal inertia about the COM */
    float obj_kn, obj_cn, obj_mu;                  /* penalty contact gains / friction of every object contact */
    int32_t nbox;                                  /* box primitives of the articulation (link frame) */
    int32_t box_link[B2G_MAX_BOXES];
    float box_pos[B2G_MAX_BOXES][3], box_quat[B2G_MAX_BOXES][4], box_half[B2G_MAX_BOXES][3];
    /* fixed two-joint tendons with a length limit (open_ai_assets/hand/shared.xml:54-69; stiffness / damping set at
     * shadow_hand.py:255-266): length = c0 q[d0] + c1 q[d1], spring-damper outside [lo, hi] */
    int32_t nten;
    int32_t ten_dof[B2G_MAX_TENDONS][2];
    float ten_coef[B2G_MAX_TENDONS][2], ten_range[B2G_MAX_TENDONS][2];
    float ten_k, ten_d;
    float obj_angular_damping, obj_linear_damping;   /* the object's own AssetOptions (defaults 0.5 / 0, shadow_hand.py:279-282) */
    /* The object is a ROUNDED box: every point within obj_round of the box obj_half.  0 = the block (cube_multicolor.urdf);
     * obj_half = (0, 0, L), obj_round = r is a capsule along z (objectType pen, open_ai_assets/hand/pen.xml:19);
     * a prolate spheroid (objectType egg, egg.xml:10) is carried as the capsule with the same polar and equatorial extent. */
    float obj_round;
    /* the object's AssetOptions.max_angular_velocity (gymapi default 64 rad/s): its angular speed is clamped after every
     * sub-step, 0 = no clamp.  Not cosmetic: a slender object (the pen: I_axial / I_transverse = 1 / 117) that is flicked into a
     * fast tumble makes the explicitly integrated gyroscopic term diverge; PhysX bounds the same case by this clamp. */
    float obj_max_angular_velocity;
} b2g_model_ext;

/* gymapi.SimParams subset that changes the physics (tasks/base/vec_task.py:514-562) */
typedef struct {
    float dt;
    int32_t substeps;
    float gravity[3];
    /* optional height field replacing the z=0 plane (tasks/anymal_terrain.py:196-209): int16
     * samples * vertical_scale, row-major [nx][ny], cell size horizontal_scale, sample (0,0) at
     * world (origin_x, origin_y).  NULL = plane. */
    const int16_t *hf_samples;
    int32_t hf_nx, hf_ny;
    float hf_horizontal_scale, hf_vertical_scale, hf_origin_x, hf_origin_y;
    float ground_friction;   /* PlaneParams / TriangleMeshParams dynamic_friction (ant.py:128-133); combined with a shape's
                                friction by PhysX's default mode, the average */
    float pad_;
} b2g_sim_params;

/* Tensor slots for b2g_bind().  Shapes in elements; N = num_envs, D = dofs, B = bodies, S = sensors. */
enum {
    B2G_T_ROOT_STATE = 0,      /* f32 (N*actors_per_env,13)   acquire_actor_root_state_tensor, ant.py:78 */
    B2G_T_DOF_STATE = 1,       /* f32 (N,D,2)  acquire_dof_state_tensor, ant.py:79 */
    B2G_T_DOF_ACTUATION = 2,   /* f32 (N,D)    set_dof_actuation_force_tensor, ant.py:285 */
    B2G_T_DOF_TARGET = 3,      /* f32 (N,D)    set_dof_position_target_tensor, shadow_hand.py:698 */
    B2G_T_RIGID_BODY_STATE = 4,/* f32 (N,B,13) acquire_rigid_body_state_tensor, shadow_hand.py:172 */
    B2G_T_FORCE_SENSOR = 5,    /* f32 (N,S,6)  acquire_force_sensor_tensor, ant.py:80 */
    B2G_T_DOF_FORCE = 6,       /* f32 (N,D)    acquire_dof_force_tensor, humanoid.py:85 */
    B2G_T_NET_CONTACT = 7,     /* f32 (N,B,3)  acquire_net_contact_force_tensor, anymal_terrain.py:119 */
    /* task-level buffers (VecTask.allocate_buffers, vec_task.py:301-324, + per-task state) */
    B2G_T_ACTIONS = 8,         /* f32 (N,A)   clamped actions kept for the observation */
    B2G_T_OBS = 9,             /* f32 (N,O) */
    B2G_T_REW = 10,            /* f32 (N) */
    B2G_T_RESET = 11,          /* i64 (N) */
    B2G_T_PROGRESS = 12,       /* i64 (N) */
    B2G_T_TIMEOUT = 13,        /* u8  (N)  bool, vec_task.py:394 */
    B2G_T_POTENTIALS = 14,     /* f32 (N) */
    B2G_T_PREV_POTENTIALS = 15,/* f32 (N) */
    B2G_T_UP_VEC = 16,         /* f32 (N,3) */
    B2G_T_HEADING_VEC = 17,    /* f32 (N,3) */
    B2G_T_INITIAL_ROOT = 18,   /* f32 (N,13) initial_root_states, ant.py:89-90 */
    B2G_T_RESET_COUNT = 19,    /* i32 (N)  per-env reset counter feeding the Philox stream */
    B2G_T_OBS_CLIPPED = 20,    /* f32 (N,O) clamp(obs, +-clip_obs), vec_task.py:402 (may alias OBS) */
    /* AnymalTerrain state (anymal_terrain.py:126-150) */
    B2G_T_COMMANDS = 21,       /* f32 (N,4)  x vel, y vel, yaw vel, heading */
    B2G_T_LAST_ACTIONS = 22,   /* f32 (N,A) */
    B2G_T_LAST_DOF_VEL = 23,   /* f32 (N,D) */
    B2G_T_FEET_AIR_TIME = 24,  /* f32 (N,4) */
    B2G_T_TORQUES = 25,        /* f32 (N,A) */
    B2G_T_EPISODE_SUMS = 26,   /* f32 (13,N) rows in the order of anymal_terrain.py:144-146 */
    B2G_T_TERRAIN_LEVELS = 27, /* i64 (N) */
    B2G_T_TERRAIN_TYPES = 28,  /* i64 (N) */
    B2G_T_ENV_ORIGINS = 29,    /* f32 (N,3) */
    B2G_T_TERRAIN_ORIGINS = 30,/* f32 (rows,cols,3) */
    B2G_T_NOISE_SCALE = 31,    /* f32 (O)   noise_scale_vec, anymal_terrain.py:174-186 */
    B2G_T_BASE_SCRATCH = 32,   /* f32 (N,12) base_lin_vel, base_ang_vel, projected_gravity handed from kernel 1 to 2 */
    B2G_T_REDUCE_SCRATCH = 33, /* f32 (>= 1024 + 48) per-block partials of the reset-set norm (anymal_terrain.py:432); then [0,13) sums of
                                  the reset envs' episode sums, 13 their count, 15 ticket, [16,29) extras['episode'] means, 29 mean terrain level,
                                  32 running sum of TERRAIN_LEVELS (the caller initialises it) */
    B2G_T_ENV_FRICTION = 34,   /* f32 (N)   per-env shape friction (friction buckets, anymal_terrain.py:235-281); NULL = the model's */
    /* ShadowHand state (shadow_hand.py:183-200,398-408) */
    B2G_T_GOAL_STATES = 35,    /* f32 (N,13)  goal_states */
    B2G_T_PREV_TARGETS = 36,   /* f32 (N,D)   prev_targets (cur_targets is the DOF_TARGET tensor itself) */
    B2G_T_SUCCESSES = 37,      /* f32 (N) */
    B2G_T_CONSECUTIVE_SUCCESSES = 38, /* f32 (4): [0] consecutive_successes, [1..3] reduction scratch (sum resets, sum finished, ticket) */
    B2G_T_RESET_GOAL = 39,     /* i64 (N)     reset_goal_buf */
    B2G_T_GOAL_RESET_COUNT = 40,/* i32 (N)    per-env goal-only reset counter feeding the Philox stream */
    B2G_T_STATES = 41,         /* f32 (N,S)  states_buf, vec_task.py:306 (asymmetric observations; unclipped, get_state clamps) */
    /* physical domain randomisation (vec_task.py:720-828 writes these per actor through gym.set_actor_*_properties; here they
     * are per-env parameter arrays the step kernels read).  NULL = the model's own values.  Read by every sub-step (the four-chain
     * kernels and the generic one). */
    B2G_T_ENV_MASS_SCALE = 42, /* f32 (N,L)   factor on every link's mass AND rotational inertia (rigid_body_properties.mass is set with
                                  recomputeInertia = True: utils/dr_utils.py:62); the COM stays */
    B2G_T_ENV_DOF_PROPS = 43,  /* f32 (N,D,4) damping, stiffness, lower, upper of every DOF (dof_properties).  For a position-driven DOF
                                  the columns are what get_actor_dof_properties reports for it: damping is all of its velocity
                                  damping (the model's joint damping plus the drive's kd, applied as joint damping), stiffness the
                                  drive's kp; the model's passive stiffness of that DOF stays */
    /* gym.acquire_jacobian_tensor / acquire_mass_matrix_tensor (tasks/franka_cube_stack.py:388-392); shapes from b2g_kin_shape:
     * nc = D for a fixed base, 6 + D for a floating base (base columns first: world linear, world angular velocity of the
     * root origin); rows = B - 1 for a fixed base (no row for the base body), B otherwise */
    B2G_T_JACOBIAN = 44,       /* f32 (N,rows,6,nc)  rows 0:3 linear, 3:6 angular velocity of the body-frame origin, world frame */
    B2G_T_MASS_MATRIX = 45,    /* f32 (N,nc,nc)      joint-space inertia (composite rigid body) + armature on the diagonal */
    /* gym.apply_rigid_body_force_tensors(sim, forces, None, LOCAL_SPACE) for the free object (shadow_hand.py:700-709,
     * forceScale > 0): a force at the object's COM in the OBJECT's frame, held over the simulate calls of a step.  The fused
     * ShadowHand step owns both tensors (decay, redraw with probability RANDOM_FORCE_PROB, zero + redraw the probability on
     * reset); b2g_simulate only reads OBJ_FORCE.  NULL = no force. */
    B2G_T_OBJ_FORCE = 46,      /* f32 (N,3) */
    B2G_T_RANDOM_FORCE_PROB = 47, /* f32 (N)   random_force_prob, shadow_hand.py:198,642 */
    /* physical domain randomisation of a sim with a free object (ShadowHand's actor_params.object, tendon_properties and
     * sim_params.gravity, vec_task.py:722-828).  NULL = the model's own values; b2g_bind refuses ENV_OBJ_PROPS and
     * ENV_TENDON_DAMPING (B2G_E_UNSUPPORTED) on a sim without a free object.  Any per-env parameter bound on such a sim (these three or ENV_MASS_SCALE / ENV_DOF_PROPS /
     * ENV_FRICTION) selects the randomised instantiation of its simulate and ShadowHand step kernels.  Frictions combine as
     * PhysX's default, the average of the two materials: ENV_FRICTION (the articulation's shapes) with the ground and with the
     * object, the object's with the ground; where only one of ENV_FRICTION / ENV_OBJ_PROPS is bound, obj_mu stands in for the
     * other material. */
    B2G_T_ENV_OBJ_PROPS = 48,  /* f32 (N,4)  the object's size scale s (contact extents obj_half and obj_round x s; mass unchanged,
                                  inertia x s^2), mass factor (mass, inertia and the contact gains obj_kn / obj_cn, which are
                                  proportional to the mass), friction, unused */
    B2G_T_ENV_TENDON_DAMPING = 49, /* f32 (N,nten)  damping of each tendon (ten_d) */
    /* f32 (3)  the sim's gravity (bodies with gravity on), read on the device by every sub-step of the kernels that take it: the
     * randomised simulate and ShadowHand step of a free-object sim, and the Humanoid step at its 4 lanes and 64 threads with
     * device or staged I/O (with or without link-link contact).  Bound on any sim; every other physics launch -- b2g_simulate
     * without a free object, the Ant, Cartpole and AnymalTerrain steps, the four-chain kernels, a Humanoid combination without
     * the instantiation -- fails with B2G_E_UNSUPPORTED while it is bound.  Resets, body state and the kinematic tensors
     * involve no gravity and ignore it. */
    B2G_T_GRAVITY = 50,
    B2G_T_COUNT = 51
};

/* fused per-task control steps */
enum { B2G_TASK_NONE = 0, B2G_TASK_CARTPOLE = 1, B2G_TASK_ANT = 2, B2G_TASK_HUMANOID = 3, B2G_TASK_ANYMAL_TERRAIN = 4,
       B2G_TASK_SHADOW_HAND = 5 };
enum { B2G_HAND_OBS_OPENAI = 0, B2G_HAND_OBS_FULL_NO_VEL = 1, B2G_HAND_OBS_FULL = 2, B2G_HAND_OBS_FULL_STATE = 3 };

/* Scalars of the locomotion tasks (cfg/task/Ant.yaml:13-29, Humanoid.yaml; ant.py:47-68). */
typedef struct {
    int32_t task;                    /* B2G_TASK_* */
    int32_t num_obs, num_actions;
    int32_t control_freq_inv;        /* gym.simulate calls per step, vec_task.py:379-382 */
    float clip_actions, clip_obs;    /* vec_task.py:374,402 */
    float max_episode_length;
    float power_scale;
    float joint_gears[B2G_MAX_LINKS];     /* per-DOF effort = action * gear * power_scale, ant.py:283 */
    float motor_efforts[B2G_MAX_LINKS];   /* humanoid.py:160-171 (actuator order, see SURVEY 3.3) */
    float max_motor_effort;
    float dof_limits_lower[B2G_MAX_LINKS], dof_limits_upper[B2G_MAX_LINKS]; /* sorted, ant.py:199-207 */
    float initial_dof_pos[B2G_MAX_LINKS];                                   /* ant.py:96-99 */
    float dof_vel_scale, contact_force_scale, angular_velocity_scale;
    float heading_weight, up_weight, actions_cost_scale, energy_cost_scale, joints_at_limit_cost_scale;
    float death_cost, termination_height, alive_reward;
    float reset_pos_noise, reset_vel_noise;   /* +-0.2, +-0.1: ant.py:257-258 */
    float dt;                                 /* cfg sim.dt as the task divides by it, ant.py:112 */
    float target[3];                          /* ant.py:110 */
    /* cartpole (cartpole.py:44-47,159-163) */
    float max_push_effort, reset_dist;
    uint64_t seed;
    int32_t env_id_offset;                    /* global id of env 0 on this rank: keys the reset RNG so
                                                 results do not depend on how envs are sharded */
    int32_t pad_;
} b2g_task_params;

/* Scalars of AnymalTerrain (cfg/task/AnymalTerrain.yaml, anymal_terrain.py:43-108). */
typedef struct {
    int32_t num_obs, num_actions;           /* 188, 12 */
    int32_t decimation, control_freq_inv;   /* gym.simulate calls: decimation inside pre_physics_step (:441-451) + control_freq_inv after it */
    float clip_actions, clip_obs;
    int32_t max_episode_length, push_interval;
    int32_t push_robots, add_noise, curriculum, allow_knee_contacts, custom_origins, pad0;
    float kp, kd, action_scale, torque_limit;
    float default_dof_pos[B2G_MAX_LINKS];
    float lin_vel_scale, ang_vel_scale, dof_pos_scale, dof_vel_scale, height_meas_scale;
    float rew_scales[14];   /* termination, lin_vel_xy, lin_vel_z, ang_vel_z, ang_vel_xy, orient, torque, joint_acc, base_height,
                               air_time, collision, stumble, action_rate, hip -- already multiplied by dt (:104-105) */
    float dt, max_episode_length_s;
    float command_x[2], command_y[2], command_yaw[2];
    float base_init_state[13];
    float border_size, terrain_hscale, terrain_vscale, env_length;
    int32_t hs_rows, hs_cols, env_rows, env_cols;
    int32_t base_body, knee_bodies[4], feet_bodies[4], pad1;
    uint64_t seed;
    int32_t env_id_offset, pad2;
} b2g_anymal_params;

/* Scalars of ShadowHand (cfg/task/ShadowHand.yaml, shadow_hand.py:52-130).  The sim must have been created with
 * b2g_create_ext: actors hand (0), object (1), goal marker (2).  INITIAL_ROOT holds, per env, the hand start state,
 * object_init_state and goal_init_state (shadow_hand.py:343-346,398-402). */
typedef struct {
    int32_t num_obs, num_actions;          /* 42 / 77 / 157 / 211 ; 20 */
    int32_t obs_type;                      /* B2G_HAND_OBS_* (shadow_hand.py:101-113) */
    int32_t control_freq_inv;
    float clip_actions, clip_obs;
    float max_episode_length;
    int32_t use_relative_control, max_consecutive_successes;
    float dof_speed_scale, act_moving_average, dt;
    float dist_reward_scale, rot_reward_scale, rot_eps, action_penalty_scale, success_tolerance, reach_goal_bonus,
          fall_dist, fall_penalty, av_factor;
    float vel_obs_scale, force_torque_obs_scale;               /* 0.2, 10.0: shadow_hand.py:62-63 */
    float reset_position_noise, reset_dof_pos_noise, reset_dof_vel_noise;
    float goal_displacement[3];                                /* shadow_hand.py:311 */
    int32_t actuated_dof[B2G_MAX_LINKS];                       /* action k drives DOF actuated_dof[k], shadow_hand.py:268-269 */
    float dof_lower[B2G_MAX_LINKS], dof_upper[B2G_MAX_LINKS], dof_default_pos[B2G_MAX_LINKS], dof_default_vel[B2G_MAX_LINKS];
    int32_t fingertip_body[5];                                 /* shadow_hand.py:120,289 */
    int32_t num_states;                                        /* 0, or the full_state size: states_buf is filled too (asymmetric_obs, :457-458) */
    uint64_t seed;
    int32_t env_id_offset, pad1;
    /* random forces on the object (shadow_hand.py:69-72,196-201,700-709); force_scale 0 = off.  force_decay_factor =
     * forceDecay ^ (dt / forceDecayInterval); a new force N(0,1)^3 * object mass * force_scale is drawn when U < random_force_prob,
     * random_force_prob = exp(force_logp_span * U' + force_logp1) redrawn on reset (force_logp_span = log p0 - log p1) */
    float force_scale, force_decay_factor, force_logp_span, force_logp1;
    /* objectType pen (shadow_hand.py:626-629): reset_idx poses the object with randomize_rotation_pen (:810-813: about x by
     * pi/2 + 0.3 rand0, then about z by pi rand0) instead of randomize_rotation; 0 = block / egg */
    int32_t object_is_pen, pad2;
} b2g_hand_params;

typedef struct b2g_sim b2g_sim;

/* gymapi.acquire_gym() + gym.create_sim() + create_env/create_actor x N + gym.prepare_sim()
 * (vec_task.py:247,262; ant.py:185-190): N identical single-actor environments. */
int b2g_create(const b2g_model *model, const b2g_sim_params *params, int32_t num_envs, int32_t device,
               b2g_sim **out);
/* same with the multi-actor extras (ext may be NULL) */
int b2g_create_ext(const b2g_model *model, const b2g_model_ext *ext, const b2g_sim_params *params, int32_t num_envs,
                   int32_t device, b2g_sim **out);
int b2g_destroy(b2g_sim *sim);

/* gymtorch.wrap_tensor in reverse: hand the engine the device buffer behind a tensor view. */
int b2g_bind(b2g_sim *sim, int32_t slot, void *device_ptr, size_t bytes);

/* gym.simulate(sim): `substeps` sub-steps (vec_task.py:382); reads DOF_ACTUATION / DOF_TARGET,
 * updates ROOT_STATE, DOF_STATE and, if bound, FORCE_SENSOR, DOF_FORCE, NET_CONTACT. */
int b2g_simulate(b2g_sim *sim, void *stream);

/* gym.refresh_rigid_body_state_tensor(sim) (shadow_hand.py:443): forward kinematics into
 * RIGID_BODY_STATE. */
int b2g_refresh_rigid_body_state(b2g_sim *sim, void *stream);

/* gym.refresh_jacobian_tensors(sim) / gym.refresh_mass_matrix_tensors(sim) (tasks/franka_cube_stack.py:439-440): recompute
 * JACOBIAN (which & 1) and / or MASS_MATRIX (which & 2) from ROOT_STATE and DOF_STATE -- one launch, one warp per env
 * (csrc/b2g_kin.cuh).  b2g_kin_shape: shape_out = {rows, nc} of this sim's articulation (host only). */
#define B2G_KIN_JACOBIAN 1
#define B2G_KIN_MASS_MATRIX 2
int b2g_kin_shape(const b2g_sim *sim, int32_t shape_out[2]);
int b2g_refresh_kinematic_tensors(b2g_sim *sim, int32_t which, void *stream);

/* One whole VecTask.step() (vec_task.py:360-408) for a fused task: clamp actions, pre_physics_step,
 * control_freq_inv x simulate, post_physics_step (progress, reset_idx, observations, reward),
 * timeout flags and the clipped observation copy -- one kernel launch.
 * `actions` is a DEVICE pointer (N, num_actions). */
int b2g_set_task(b2g_sim *sim, const b2g_task_params *task);
/* AnymalTerrain (tasks/anymal_terrain.py:441-485): b2g_task_step then launches two kernels, physics +
 * termination + reward, and reset (terrain curriculum) + observations. */
int b2g_set_anymal_task(b2g_sim *sim, const b2g_anymal_params *task);
/* ShadowHand (tasks/shadow_hand.py:661-705 pre_physics_step with reset_idx / reset_target_pose, simulate,
 * :707-712 post_physics_step with compute_observations and compute_hand_reward): one kernel launch. */
int b2g_set_hand_task(b2g_sim *sim, const b2g_hand_params *task);
int b2g_task_step(b2g_sim *sim, const float *actions, void *stream);

/* K consecutive VecTask.step() calls whose actions are all known up front -- the open-loop, random-action rollout the
 * reference's README times (README.md:39-51: `for _ in range(K): envs.step(random_actions)`):
 *     for k in range(K): obs[k], rew[k], reset[k], time_outs[k] = step(actions[k])
 * `actions` (K,N,A), `obs_out` (K,N,O: the observation step() returns, i.e. clipped when a clip is configured), `rew_out`
 * (K,N), `reset_out` (K,N) i64, `timeout_out` (K,N) u8 or NULL: DEVICE pointers.  Afterwards every bound tensor holds
 * what it would hold after the K single steps.  Ant on whole tiles of 16 envs runs as ONE launch (state stays on chip
 * between the steps); anything else as K single steps with device copies. */
int b2g_task_rollout(b2g_sim *sim, const float *actions, int32_t K, float *obs_out, float *rew_out, int64_t *reset_out,
                     uint8_t *timeout_out, void *stream);

/* VecTask.reset_done() (vec_task.py:440-455): run reset_idx (ant.py:252-279, humanoid.py:253-279, cartpole.py:144-157,
 * shadow_hand.py:594-659, anymal_terrain.py:384-425) for every env whose RESET flag is set, now, and clear the flag the
 * way the task's reset_idx does.  Observations are refreshed by the next step, as in the reference. */
int b2g_reset_flagged(b2g_sim *sim, void *stream);

/* Same step with HOST buffers (pinned or pageable): copies actions in, runs the step, copies
 * obs / rew / reset / timeout out and synchronises the stream: the call an rl_device="cpu" user
 * makes through VecTask.step (vec_task.py:402,408 `.to(rl_device)`). Any output may be NULL. */
int b2g_task_step_host(b2g_sim *sim, const float *h_actions, float *h_obs, float *h_rew, int64_t *h_reset,
                       uint8_t *h_timeout, void *stream);

/* Introspection, host only (no device needed): the slot programs b2g_create would build for `model` on `lanes`
 * lanes per env (1, 2, 4 or 8; 0 = the engine's own choice).  `compact` selects the env-wide accumulator numbering of
 * the multi-actor kernels.  slots_out receives B2G_PLAN_MAX_SLOTS x B2G_PLAN_MAX_LANES records of 8 int32:
 * link, parent ((lane << 8) | slot + 1; 0 = root), out (-1 carried, -2 dropped, else accumulator id), flags, child[4].
 * info_out: ns, lanes, nacc, root_acc, cross_lane. */
#define B2G_PLAN_MAX_SLOTS 24
#define B2G_PLAN_MAX_LANES 8
int b2g_plan(const b2g_model *model, int32_t lanes, int32_t compact, int32_t *slots_out, int32_t info_out[5]);

/* Which formulation of the sub-step the sim runs: 0 = the generic slot-program stepper, 2 / 3 = the specialised
 * "four hinge chains of this length on a free base" stepper (Ant / ANYmal class articulations).  Same physics. */
int b2g_quad_chain_length(const b2g_sim *sim);

/* number of kernels this library has launched since creation (bench.py "gpu_launches") */
int64_t b2g_launch_count(const b2g_sim *sim);
const char *b2g_last_error(void);
int b2g_version(void);

#ifdef __cplusplus
}
#endif
#endif

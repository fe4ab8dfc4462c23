// b2g_tasks.cuh -- per-task observation / reward / reset arithmetic, fused behind the physics.
//
// Each function restates (file:line under isaacgymenvs/ of the reference) the @torch.jit.script
// function it replaces and keeps its OPERATION ORDER: tests compare against golden vectors produced
// by the reference's own functions (tests/golden) at 1e-6, and `potentials` bit-exactly, because
// progress_reward = potentials - prev_potentials (tasks/ant.py:359) differences two ~6e4 numbers.
#pragma once
#include "b2g_common.cuh"

namespace b2g {

// ------------------------------------------------------------------ utils/torch_jit_utils.py
// quat_mul, torch_jit_utils.py:41-62 (xyzw)
__device__ __forceinline__ void t_quat_mul(const float a[4], const float b[4], float o[4]) {
    const float x1 = a[0], y1 = a[1], z1 = a[2], w1 = a[3], x2 = b[0], y2 = b[1], z2 = b[2], w2 = b[3];
    const float ww = (z1 + x1) * (x2 + y2);
    const float yy = (w1 - y1) * (w2 + z2);
    const float zz = (w1 + y1) * (w2 - z2);
    const float xx = ww + yy + zz;
    const float qq = 0.5f * (xx + (z1 - x1) * (x2 - y2));
    o[3] = qq - ww + (z1 - y1) * (y2 - z2);
    o[0] = qq - xx + (x1 + w1) * (x2 + w2);
    o[1] = qq - yy + (w1 - x1) * (y2 + z2);
    o[2] = qq - zz + (z1 + y1) * (w2 - x2);
}
// quat_rotate :80-90 (sign=+1) / quat_rotate_inverse :93-103 (sign=-1)
__device__ __forceinline__ void t_quat_rotate(const float q[4], const float v[3], float o[3], float sign) {
    const float qw = q[3];
    const float s = 2.0f * qw * qw - 1.0f;
    float cr[3]; cross(q, v, cr);
    const float d = (q[0] * v[0] + q[1] * v[1]) + q[2] * v[2];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float a = v[c] * s, b = cr[c] * qw * 2.0f, cc = q[c] * d * 2.0f;
        o[c] = (sign > 0.f) ? (a + b + cc) : (a - b + cc);
    }
}
// torch.remainder(a, 2*pi) for a in [-pi, pi]  (get_euler_xyz :195)
__device__ __forceinline__ float t_rem_2pi(float a) {
    const float b = 6.2831855f;          // float32(2*np.pi)
    float r = fmodf(a, b);
    if (r != 0.f && (r < 0.f)) r += b;
    return r;
}
// get_euler_xyz :175-195
__device__ __forceinline__ void t_euler_xyz(const float q[4], float &roll, float &pitch, float &yaw) {
    const float qx = q[0], qy = q[1], qz = q[2], qw = q[3];
    const float sinr_cosp = 2.0f * (qw * qx + qy * qz);
    const float cosr_cosp = qw * qw - qx * qx - qy * qy + qz * qz;
    roll = t_rem_2pi(atan2f(sinr_cosp, cosr_cosp));
    const float sinp = 2.0f * (qw * qy - qz * qx);
    const float pr = (fabsf(sinp) >= 1.f) ? copysignf(1.5707964f, sinp) : asinf(sinp);
    pitch = t_rem_2pi(pr);
    const float siny_cosp = 2.0f * (qw * qz + qx * qy);
    const float cosy_cosp = qw * qw + qx * qx - qy * qy - qz * qz;
    yaw = t_rem_2pi(atan2f(siny_cosp, cosy_cosp));
}
// normalize_angle :126-128
__device__ __forceinline__ float t_normalize_angle(float x) { return atan2f(sinf(x), cosf(x)); }

// -norm(to_target)/dt with torch-CPU rounding (plain squares and sum, sqrt, true division; no FMA
// contraction): ant.py:387-391, humanoid.py:389-393.  Bit-exact against the golden vectors.
__device__ __forceinline__ float t_potential(float tx, float ty, float dt) {
    const float s = __fadd_rn(__fmul_rn(tx, tx), __fmul_rn(ty, ty));
    return -__fdiv_rn(__fsqrt_rn(s), dt);
}

// ------------------------------------------------------------------ Philox4x32-10 reset stream
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// the idx-th uniform in [0,1) of env's reset number `count`
__device__ __forceinline__ float reset_uniform(uint64_t seed, uint32_t env, uint32_t count, int idx) {
    uint32_t r[4];
    philox4x32_10((uint32_t)(idx >> 2), count, env, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    return (float)(r[idx & 3] >> 8) * (1.0f / 16777216.0f);
}

// ------------------------------------------------------------------ locomotion (Ant / Humanoid)
// potentials from a root position (ant.py:273-275, 387-391)
__device__ __forceinline__ float loco_potential(const b2g_task_params &P, const float rp[3]) {
    return t_potential(P.target[0] - rp[0], P.target[1] - rp[1], P.dt);
}

// Root-derived part of compute_ant_observations (ant.py:374-408) /
// compute_humanoid_observations (humanoid.py:378-413): fills o[0..11] and the per-env state.
struct LocoRootObs {
    float o[12];
    float potentials, up_vec[3], heading_vec[3];
};
__device__ __forceinline__ void loco_root_obs(const b2g_task_params &P, const float rp[3], const float rq[4],
                                              const float rv[3], const float rw[3], bool humanoid, LocoRootObs &r) {
    const float to_t[3] = {P.target[0] - rp[0], P.target[1] - rp[1], 0.f};
    r.potentials = loco_potential(P, rp);
    // compute_heading_and_up, torch_jit_utils.py:247-262 (inv_start_rot = identity conj, ant.py:106)
    const float nrm = fmaxf(sqrtf(to_t[0] * to_t[0] + to_t[1] * to_t[1] + 0.f), 1e-9f);
    const float td[3] = {to_t[0] / nrm, to_t[1] / nrm, 0.f / nrm};
    const float isr[4] = {-0.f, -0.f, -0.f, 1.f};
    float tq[4]; t_quat_mul(rq, isr, tq);
    const float b0[3] = {1.f, 0.f, 0.f}, b1[3] = {0.f, 0.f, 1.f};
    t_quat_rotate(tq, b1, r.up_vec, 1.f);
    t_quat_rotate(tq, b0, r.heading_vec, 1.f);
    const float up_proj = r.up_vec[2];
    const float heading_proj = (r.heading_vec[0] * td[0] + r.heading_vec[1] * td[1]) + r.heading_vec[2] * td[2];
    // compute_rot, torch_jit_utils.py:265-276
    float vloc[3], wloc[3];
    t_quat_rotate(tq, rv, vloc, -1.f);
    t_quat_rotate(tq, rw, wloc, -1.f);
    float roll, pitch, yaw; t_euler_xyz(tq, roll, pitch, yaw);
    const float walk = atan2f(P.target[2] - rp[2], P.target[0] - rp[0]);
    float ang = walk - yaw;
    if (humanoid) { roll = t_normalize_angle(roll); yaw = t_normalize_angle(yaw); ang = t_normalize_angle(ang); }
    const float avs = humanoid ? P.angular_velocity_scale : 1.f;
    r.o[0] = rp[2];
    r.o[1] = vloc[0]; r.o[2] = vloc[1]; r.o[3] = vloc[2];
    r.o[4] = wloc[0] * avs; r.o[5] = wloc[1] * avs; r.o[6] = wloc[2] * avs;
    r.o[7] = yaw; r.o[8] = roll; r.o[9] = ang; r.o[10] = up_proj; r.o[11] = heading_proj;
}

// unscale, torch_jit_utils.py:238-239
__device__ __forceinline__ float t_unscale(float x, float lo, float hi) { return (2.0f * x - hi - lo) / (hi - lo); }

// reset_idx (ant.py:252-279, humanoid.py:253-279): DOF d of env `gid`'s reset number `count` -- the initial position plus
// uniform noise, clamped to the limits, and a uniform velocity
__device__ __forceinline__ float2 loco_reset_dof(const b2g_task_params &P, uint32_t gid, uint32_t count, int d, int nd) {
    const float up = reset_uniform(P.seed, gid, count, d);
    const float uv = reset_uniform(P.seed, gid, count, nd + d);
    const float pos = (P.reset_pos_noise - (-P.reset_pos_noise)) * up + (-P.reset_pos_noise);
    return make_float2(fmaxf(fminf(P.initial_dof_pos[d] + pos, P.dof_limits_upper[d]), P.dof_limits_lower[d]),
                       (P.reset_vel_noise - (-P.reset_vel_noise)) * uv + (-P.reset_vel_noise));
}

// reset_idx's root: the initial root state; returns the potential that prev_potentials and potentials are both reset to
__device__ __forceinline__ float loco_reset_root(const b2g_task_params &P, const Buffers &B, int e, RootState &rs) {
    load_root((const float *)B.p[B2G_T_INITIAL_ROOT] + 13 * (size_t)e, rs);
    return loco_potential(P, rs.rp);
}

// the per-DOF sums of compute_ant_reward (ant.py:353-355) / compute_humanoid_reward (humanoid.py:352-359), from the clamped
// action a and the observed ps (unscaled position) and vs (scaled velocity)
struct LocoCosts {
    float actions = 0.f, electricity = 0.f, at_limit = 0.f;
    __device__ __forceinline__ void add(const b2g_task_params &P, int d, float a, float ps, float vs, bool humanoid) {
        actions += a * a;
        if (humanoid) {
            const float ratio = P.motor_efforts[d] / P.max_motor_effort;
            const float scaled = P.joints_at_limit_cost_scale * (fabsf(ps) - 0.98f) / 0.02f;
            at_limit += (fabsf(ps) > 0.98f) ? scaled * ratio : 0.f;
            electricity += fabsf(a * vs) * ratio;
        } else {
            at_limit += (ps > 0.99f) ? 1.f : 0.f;
            electricity += fabsf(a * vs);
        }
    }
    template <int L> __device__ __forceinline__ void sum_lanes() {
        actions = lane_sum<L>(actions);
        electricity = lane_sum<L>(electricity);
        at_limit = lane_sum<L>(at_limit);
    }
};

// the rest of compute_ant_reward (ant.py:326-371) / compute_humanoid_reward (humanoid.py:324-375): the reward and the two
// reasons to reset -- the torso fell below termination_height (the reward is then death_cost) or the episode ran out.
// reset_buf was cleared by reset_idx or was already 0, so reset = died || timed, and time_out = timed (vec_task.py:394).
struct LocoReward {
    float rew;
    bool died, timed;
};
__device__ __forceinline__ LocoReward loco_reward(const b2g_task_params &P, float up_proj, float heading_proj, float potentials,
                                                  float prev_potentials, const LocoCosts &c, float height, long long progress,
                                                  bool humanoid) {
    const float heading_reward = (heading_proj > 0.8f) ? P.heading_weight : P.heading_weight * heading_proj / 0.8f;
    const float up_reward = (up_proj > 0.93f) ? P.up_weight : 0.f;
    const float progress_reward = potentials - prev_potentials;
    LocoReward r;
    r.rew = progress_reward + P.alive_reward + up_reward + heading_reward - P.actions_cost_scale * c.actions -
            P.energy_cost_scale * c.electricity - (humanoid ? c.at_limit : c.at_limit * P.joints_at_limit_cost_scale);
    r.died = height < P.termination_height;
    if (r.died) r.rew = P.death_cost;
    r.timed = (float)progress >= P.max_episode_length - 1.f;
    return r;
}

// compute_cartpole_reward, cartpole.py:180-196
__device__ __forceinline__ void cartpole_reward(float pole_angle, float pole_vel, float cart_vel, float cart_pos,
                                                float reset_dist, long long progress, float max_len,
                                                float &rew, long long &reset) {
    float reward = 1.0f - pole_angle * pole_angle - 0.01f * fabsf(cart_vel) - 0.005f * fabsf(pole_vel);
    if (fabsf(cart_pos) > reset_dist) reward = -2.0f;
    if (fabsf(pole_angle) > 1.5707964f) reward = -2.0f;
    if (fabsf(cart_pos) > reset_dist) reset = 1;
    if (fabsf(pole_angle) > 1.5707964f) reset = 1;
    if ((float)progress >= max_len - 1.f) reset = 1;
    rew = reward;
}
// reset_idx, cartpole.py:144-157: DOF s (0 cart, 1 pole) of env `gid`'s reset number `count` -- (position, velocity)
__device__ __forceinline__ float2 cartpole_reset_dof(const b2g_task_params &P, uint32_t gid, uint32_t count, int s) {
    return make_float2(0.2f * (reset_uniform(P.seed, gid, count, s) - 0.5f), 0.5f * (reset_uniform(P.seed, gid, count, 2 + s) - 0.5f));
}

// ------------------------------------------------------------------ AnymalTerrain helpers (tasks/anymal_terrain.py)
// uniform in [0,1) number `idx` of stream (env, step, tag)
__device__ __forceinline__ float anymal_uniform(uint64_t seed, uint32_t env, uint32_t step, uint32_t tag, int idx) {
    uint32_t r[4];
    philox4x32_10((uint32_t)(idx >> 2), step, env, tag, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    return (float)(r[idx & 3] >> 8) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float t_rand_float(float lo, float hi, float u) { return (hi - lo) * u + lo; }   // torch_rand_float, torch_jit_utils.py:215-218

// wrap_to_pi, anymal_terrain.py:683-687: the in-place `%=` is aten::fmod_ (keeps the dividend's sign)
__device__ __forceinline__ float t_wrap_to_pi(float a) {
    a = fmodf(a, 6.2831855f);
    return a - 6.2831855f * ((a > 3.1415927f) ? 1.f : 0.f);
}
// quat_apply, torch_jit_utils.py:70-77
__device__ __forceinline__ void t_quat_apply(const float q[4], const float b[3], float o[3]) {
    float t[3], u[3];
    cross(q, b, t);
    t[0] *= 2.f; t[1] *= 2.f; t[2] *= 2.f;
    cross(q, t, u);
#pragma unroll
    for (int c = 0; c < 3; c++) o[c] = b[c] + q[3] * t[c] + u[c];
}

enum { TAG_PUSH = 1, TAG_RESET = 2, TAG_NOISE = 3 };
constexpr int REDUCE_PARTIALS = 1024;      // REDUCE_SCRATCH: [0,1024) block partials, then 16 floats of extras sums

// pre_physics_step's PD torque of DOF d from the clamped action a (:443-444)
__device__ __forceinline__ float anymal_pd_torque(const b2g_anymal_params &P, int d, float a, float q, float qd) {
    const float t = P.kp * (P.action_scale * a + P.default_dof_pos[d] - q) - P.kd * qd;
    return fminf(fmaxf(t, -P.torque_limit), P.torque_limit);
}

// push_robots (:437-439)
__device__ __forceinline__ void anymal_push(const b2g_anymal_params &P, uint32_t gid, unsigned step_counter, RootState &rs) {
    if (P.push_robots && P.push_interval > 0 && (step_counter % (unsigned)P.push_interval) == 0) {
        rs.rv[0] = t_rand_float(-1.f, 1.f, anymal_uniform(P.seed, gid, step_counter, TAG_PUSH, 0));
        rs.rv[1] = t_rand_float(-1.f, 1.f, anymal_uniform(P.seed, gid, step_counter, TAG_PUSH, 1));
    }
}

// the per-DOF reward sums of compute_reward (:339,342,355,361), from DOF d's last PD torque t, clamped action a and state
struct AnymalCosts {
    float torque = 0.f, jacc = 0.f, arate = 0.f, hip = 0.f;
    __device__ __forceinline__ void add(const b2g_anymal_params &P, int d, float t, float a, float q, float qd,
                                        const float *last_a, const float *last_v) {
        torque += t * t;
        const float dv = last_v[d] - qd; jacc += dv * dv;
        const float da = last_a[d] - a; arate += da * da;
        if (d % 3 == 0) hip += fabsf(q - P.default_dof_pos[d]);          // dof_pos[:, [0,3,6,9]]
    }
    template <int L> __device__ __forceinline__ void sum_lanes() {
        torque = lane_sum<L>(torque); jacc = lane_sum<L>(jacc); arate = lane_sum<L>(arate); hip = lane_sum<L>(hip);
    }
};

// post_physics_step (:453-475) of AnymalTerrain's first launch, four lanes per env (lane k owns leg k): progress, push,
// the DOF and root write-back, the contact-force terms, the base quantities, check_termination, compute_reward and its
// stores, and this block's partial of the norm over the reset set that reset_idx's curriculum needs (:432).
// write_back(c) is the kernel's own part: it stores the env's DOF states (and, on lane 0, the root) and adds this lane's
// DOFs to the costs c.  cf: the env's NET_CONTACT rows; s_part: BLOCK / 32 floats of shared memory.
template <int BLOCK, class WRITE_BACK>
__device__ __forceinline__ void anymal_post_physics(const b2g_anymal_params &P, const Buffers &B, int N, int e, int lane, bool valid,
                                                    unsigned step_counter, RootState &rs, const float *cf, float *s_part,
                                                    WRITE_BACK write_back) {
    long long *progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *reset_b = (long long *)B.p[B2G_T_RESET];
    const long long progress = progress_b[e] + 1;
    const uint32_t gid = (uint32_t)(e + P.env_id_offset);
    anymal_push(P, gid, step_counter, rs);
    AnymalCosts c;
    write_back(c);
    c.sum_lanes<4>();

    // contact-force terms: every lane looks at bodies base / knee[lane] / foot[lane]
    float *fat_b = (float *)B.p[B2G_T_FEET_AIR_TIME] + (size_t)e * 4;
    float n_knee = 0.f, n_stumble = 0.f, air = 0.f;
    __syncwarp();
    const float *fk = cf + 3 * P.knee_bodies[lane], *ff = cf + 3 * P.feet_bodies[lane];
    const bool knee_hit = sqrtf(fk[0] * fk[0] + fk[1] * fk[1] + fk[2] * fk[2]) > 1.f;
    n_knee += knee_hit ? 1.f : 0.f;
    n_stumble += ((sqrtf(ff[0] * ff[0] + ff[1] * ff[1]) > 5.f) && (fabsf(ff[2]) < 1.f)) ? 1.f : 0.f;
    const bool contact = ff[2] > 1.f;
    float fat = fat_b[lane];
    const bool first = (fat > 0.f) && contact;
    fat += P.dt;
    air += (fat - 0.5f) * (first ? 1.f : 0.f);
    fat = contact ? 0.f : fat;
    if (valid) fat_b[lane] = fat;
    n_knee = lane_sum<4>(n_knee); n_stumble = lane_sum<4>(n_stumble); air = lane_sum<4>(air);
    const float any_knee = lane_sum<4>(knee_hit ? 1.f : 0.f);

    // prepare quantities (:464-471)
    float *cmd = (float *)B.p[B2G_T_COMMANDS] + (size_t)e * 4;
    const float gvec[3] = {0.f, 0.f, -1.f}, fvec[3] = {1.f, 0.f, 0.f};
    float blv[3], bav[3], pg[3], fwd[3];
    t_quat_rotate(rs.rq, rs.rv, blv, -1.f);
    t_quat_rotate(rs.rq, rs.rw, bav, -1.f);
    t_quat_rotate(rs.rq, gvec, pg, -1.f);
    t_quat_apply(rs.rq, fvec, fwd);
    const float heading = atan2f(fwd[1], fwd[0]);
    const float c0 = cmd[0], c1 = cmd[1], c3 = cmd[3];
    const float c2 = fminf(fmaxf(0.5f * t_wrap_to_pi(c3 - heading), -1.f), 1.f);

    // check_termination (:294-300)
    const float *fb = cf + 3 * P.base_body;
    bool reset = sqrtf(fb[0] * fb[0] + fb[1] * fb[1] + fb[2] * fb[2]) > 1.f;
    if (!P.allow_knee_contacts) reset = reset || (any_knee > 0.f);
    if (progress >= (long long)P.max_episode_length - 1) reset = true;

    float part = 0.f;
    if (lane == 0 && valid) {
        // compute_reward (:315-382)
        const float *R = P.rew_scales;
        const float ex = c0 - blv[0], ey = c1 - blv[1];
        const float lin_err = ex * ex + ey * ey;
        const float ang_err = (c2 - bav[2]) * (c2 - bav[2]);
        float t[13];
        t[0] = expf(-lin_err / 0.25f) * R[1];                    // lin_vel_xy
        t[1] = blv[2] * blv[2] * R[2];                           // lin_vel_z
        t[2] = expf(-ang_err / 0.25f) * R[3];                    // ang_vel_z
        t[3] = (bav[0] * bav[0] + bav[1] * bav[1]) * R[4];       // ang_vel_xy
        t[4] = (pg[0] * pg[0] + pg[1] * pg[1]) * R[5];           // orient
        t[5] = c.torque * R[6];                                  // torques
        t[6] = c.jacc * R[7];                                    // joint_acc
        t[7] = (rs.rp[2] - 0.52f) * (rs.rp[2] - 0.52f) * R[8];   // base_height
        t[8] = air * R[9] * ((sqrtf(c0 * c0 + c1 * c1) > 0.1f) ? 1.f : 0.f);   // air_time
        t[9] = n_knee * R[10];                                   // collision
        t[10] = n_stumble * R[11];                               // stumble
        t[11] = c.arate * R[12];                                 // action_rate
        t[12] = c.hip * R[13];                                   // hip
        float rew = t[0] + t[2] + t[1] + t[3] + t[4] + t[7] + t[5] + t[6] + t[9] + t[11] + t[8] + t[12] + t[10];
        rew = fmaxf(rew, 0.f);
        const uint8_t *to = (const uint8_t *)B.p[B2G_T_TIMEOUT];
        rew += R[0] * (reset ? 1.f : 0.f) * ((to && to[e]) ? 0.f : 1.f);
        ((float *)B.p[B2G_T_REW])[e] = rew;
        float *es = (float *)B.p[B2G_T_EPISODE_SUMS];
#pragma unroll
        for (int k = 0; k < 13; k++) es[(size_t)k * N + e] += t[k];
        reset_b[e] = reset ? 1 : 0;
        progress_b[e] = progress;
        cmd[2] = c2;
        float *bs = (float *)B.p[B2G_T_BASE_SCRATCH] + (size_t)e * 12;
        bs[0] = blv[0]; bs[1] = blv[1]; bs[2] = blv[2]; bs[3] = bav[0]; bs[4] = bav[1]; bs[5] = bav[2];
        bs[6] = pg[0]; bs[7] = pg[1]; bs[8] = pg[2];
        if (reset) part = c0 * c0 + c1 * c1;
    }
    // deterministic per-block partial of sum over the reset set of |commands_xy|^2
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int w = 0; w < BLOCK / 32; w++) tot += s_part[w];
        float *red = (float *)B.p[B2G_T_REDUCE_SCRATCH];
        red[blockIdx.x] = tot;
        if (blockIdx.x == 0) for (int k = 0; k < 16; k++) red[REDUCE_PARTIALS + k] = 0.f;
    }
}

}  // namespace b2g

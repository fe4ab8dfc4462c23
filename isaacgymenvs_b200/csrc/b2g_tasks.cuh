// b2g_tasks.cuh -- per-task observation / reward / reset arithmetic, fused behind the physics.
//
// Each function restates (file:line under isaacgymenvs/ of the reference) the @torch.jit.script
// function it replaces and keeps its OPERATION ORDER: tests compare against golden vectors produced
// by the reference's own functions (tests/golden) at 1e-6, and `potentials` bit-exactly, because
// progress_reward = potentials - prev_potentials (tasks/ant.py:359) differences two ~6e4 numbers.
#pragma once
#include "b2g_device.cuh"
#include "../../include/b200gym.h"

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
// Root-derived part of compute_ant_observations (ant.py:374-408) /
// compute_humanoid_observations (humanoid.py:378-413): fills o[0..11] and the per-env state.
struct LocoRootObs {
    float o[12];
    float potentials, up_vec[3], heading_vec[3];
};
__device__ __forceinline__ void loco_root_obs(const b2g_task_params &P, const float rp[3], const float rq[4],
                                              const float rv[3], const float rw[3], bool humanoid, LocoRootObs &r) {
    const float to_t[3] = {P.target[0] - rp[0], P.target[1] - rp[1], 0.f};
    r.potentials = t_potential(to_t[0], to_t[1], P.dt);
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

}  // namespace b2g

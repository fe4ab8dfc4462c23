// b2g_hand.cuh -- one whole VecTask.step() of ShadowHand (tasks/shadow_hand.py) in one kernel:
//   vec_task.py:374 clamp -> pre_physics_step (:661-705: reset_target_pose :594-610, reset_idx :612-659, position
//   targets) -> control_freq_inv x gym.simulate (hand + free cube, Stepper<.., OBJ=true>) -> post_physics_step
//   (:707-712: progress, compute_observations :436-458 in the four layouts :460-592, compute_hand_reward :749-804).
// An env is owned by L lanes (the fingers run in parallel); per-env scalars are computed on every lane and written by
// lane 0, per-DOF quantities by the lane whose slot program holds the DOF.
#pragma once
#include "b2g_device.cuh"
#include "b2g_tasks.cuh"

namespace b2g {

struct HandDev {                      // host-derived tables (b2g_set_hand_task)
    int ft_ref[5];                    // ((lane << 8) | slot) of each fingertip's link
    float ft_bpos[5][3], ft_bR[5][9]; // fingertip body frame in its link frame
    int dof_action[MAX_LINKS];        // action index driving a DOF, -1: not actuated
    // offsets of the pieces inside an observation vector (-1: absent); [0] = obs_buf in the configured layout,
    // [1] = states_buf, always the full_state layout (asymmetric observations, shadow_hand.py:457-458,529-556)
    struct Layout { int o_dofpos, o_dofvel, o_dofforce, o_objpose, n_objpose, o_objvel, o_goalpose, o_qdiff, o_ft, ft_stride, o_sens, o_act; } lay[2];
    int num_states;                   // 0: no states_buf
};

// quat_from_angle_axis (torch_jit_utils.py:118-123) about a unit coordinate axis, then quat_unit
__device__ __forceinline__ void t_quat_axis(float angle, int axis, float q[4]) {
    const float th = angle / 2.f;
    const float sn = sinf(th), cs = cosf(th);
    float v[4] = {0.f, 0.f, 0.f, cs};
    v[axis] = 1.f * sn;
    const float nrm = fmaxf(sqrtf((v[0] * v[0] + v[1] * v[1]) + (v[2] * v[2] + v[3] * v[3])), 1e-9f);
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = v[c] / nrm;
}
// randomize_rotation, shadow_hand.py:807-810
__device__ __forceinline__ void t_randomize_rotation(float rand0, float rand1, float q[4]) {
    float qx[4], qy[4];
    t_quat_axis(rand0 * 3.1415927f, 0, qx);
    t_quat_axis(rand1 * 3.1415927f, 1, qy);
    t_quat_mul(qx, qy, q);
}
// randomize_rotation_pen, shadow_hand.py:810-813 (called with max_angle = tensor(0.3), :627): quat_from_angle_axis(0.5 pi + rand0 *
// max_angle, x) * quat_from_angle_axis(rand0 pi, z); 0.5 * np.pi enters the float32 tensor arithmetic as 1.5707964
__device__ __forceinline__ void t_randomize_rotation_pen(float rand0, float q[4]) {
    float qx[4], qz[4];
    t_quat_axis(1.5707964f + rand0 * 0.3f, 0, qx);
    t_quat_axis(rand0 * 3.1415927f, 2, qz);
    t_quat_mul(qx, qz, q);
}
// torch_rand_float(-1, 1): (upper - lower) * rand + lower
__device__ __forceinline__ float hand_rand(uint64_t seed, uint32_t gid, uint32_t count, int idx) {
    return 2.0f * reset_uniform(seed, gid, count, idx) + (-1.0f);
}

// ---- reset_idx (:612-659), reset_target_pose (:594-610): shared by the fused step and reset_done (b2g_reset.cuh).  Reset
// stream of reset number `count`, by index: object position 0-2, rotation 3-4 (:625-629); DOF d's position 5 + d (also its
// target), velocity 5 + nd + d; goal rotation 2 nd + 5, 2 nd + 6; random_force_prob 2 nd + 7.  A goal-only reset
// draws 0, 1 of stream *goal_count | 2^31.  write: store goal_states, the goal's root row (rows + 26), the new goal_count.
__device__ __forceinline__ void hand_reset_goal(const b2g_hand_params &P, uint32_t gid, uint32_t count, int nd, bool goal_only,
                                                int *goal_count, const float *init_rows, float *goal_row, float *rows,
                                                bool write, float goal_pos[3], float goal_rot[4]) {
    float r0, r1;
    if (!goal_only) { r0 = hand_rand(P.seed, gid, count, 2 * nd + 5); r1 = hand_rand(P.seed, gid, count, 2 * nd + 6); }
    else {
        const uint32_t gc = (uint32_t)*goal_count | 0x80000000u;
        r0 = hand_rand(P.seed, gid, gc, 0); r1 = hand_rand(P.seed, gid, gc, 1);
        if (write) *goal_count = (int)(((uint32_t)*goal_count + 1u) & 0x7fffffffu);
    }
    t_randomize_rotation(r0, r1, goal_rot);
#pragma unroll
    for (int c = 0; c < 3; c++) goal_pos[c] = init_rows[26 + c];
    if (write) {
#pragma unroll
        for (int c = 0; c < 3; c++) { goal_row[c] = goal_pos[c]; rows[26 + c] = goal_pos[c] + P.goal_displacement[c]; }
#pragma unroll
        for (int c = 0; c < 4; c++) { goal_row[3 + c] = goal_rot[c]; rows[29 + c] = goal_rot[c]; }
#pragma unroll
        for (int c = 7; c < 13; c++) rows[26 + c] = 0.f;
    }
}
__device__ __forceinline__ void hand_reset_obj(const b2g_hand_params &P, uint32_t gid, uint32_t count, const float *init_rows, ObjState &ob) {
#pragma unroll
    for (int c = 0; c < 3; c++) ob.p[c] = init_rows[13 + c] + P.reset_position_noise * hand_rand(P.seed, gid, count, c);
    const float r3 = hand_rand(P.seed, gid, count, 3), r4 = hand_rand(P.seed, gid, count, 4);
    if (P.object_is_pen) t_randomize_rotation_pen(r3, ob.q);
    else t_randomize_rotation(r3, r4, ob.q);
#pragma unroll
    for (int c = 0; c < 3; c++) { ob.v[c] = 0.f; ob.w[c] = 0.f; }
}
__device__ __forceinline__ float2 hand_reset_dof(const b2g_hand_params &P, uint32_t gid, uint32_t count, int d, int nd) {
    const float delta_max = P.dof_upper[d] - P.dof_default_pos[d], delta_min = P.dof_lower[d] - P.dof_default_pos[d];
    const float rand_delta = delta_min + (delta_max - delta_min) * 0.5f * (hand_rand(P.seed, gid, count, 5 + d) + 1.0f);
    return make_float2(P.dof_default_pos[d] + P.reset_dof_pos_noise * rand_delta,
                       P.dof_default_vel[d] + P.reset_dof_vel_noise * hand_rand(P.seed, gid, count, 5 + nd + d));
}

// ---- random forces on the object (shadow_hand.py:700-709, forceScale > 0).  The reference draws from torch's global generator;
// here, like the reset stream, the draws are counter-based: Philox counter (step within the episode, reset count, global
// env id, 1 | 2), so the result does not depend on the sharding.  f: the force carried over from the previous step.
__device__ __forceinline__ float hand_force_prob(const b2g_hand_params &P, uint32_t gid, uint32_t count, int nd) {
    // random_force_prob = exp((log p0 - log p1) * rand + log p1), :198,642; index 2 nd + 7 of the env's reset stream
    return expf(P.force_logp_span * reset_uniform(P.seed, gid, count, 2 * nd + 7) + P.force_logp1);
}
__device__ __forceinline__ void hand_force_update(const b2g_hand_params &P, uint32_t gid, uint32_t rcount, uint32_t step, float mass,
                                                  float prob, float f[3]) {
#pragma unroll
    for (int c = 0; c < 3; c++) f[c] *= P.force_decay_factor;                     // rb_forces *= decay ^ (dt / interval), :701
    uint32_t r[4];
    philox4x32_10(step, rcount, gid, 1u, (uint32_t)P.seed, (uint32_t)(P.seed >> 32), r);
    const float k24 = 1.0f / 16777216.0f;
    if ((float)(r[0] >> 8) * k24 < prob) {                                        // torch.rand(num_envs) < random_force_prob, :704
        uint32_t r2[4];
        philox4x32_10(step, rcount, gid, 2u, (uint32_t)P.seed, (uint32_t)(P.seed >> 32), r2);
        // Box-Muller: two pairs of uniforms -> three standard normals (torch.randn, :705)
        const float ra = sqrtf(-2.0f * logf((float)((r[1] >> 8) + 1u) * k24)), ta = 6.2831855f * ((float)(r[2] >> 8) * k24);
        const float rb = sqrtf(-2.0f * logf((float)((r[3] >> 8) + 1u) * k24)), tb = 6.2831855f * ((float)(r2[0] >> 8) * k24);
        const float n[3] = {ra * cosf(ta), ra * sinf(ta), rb * cosf(tb)};
#pragma unroll
        for (int c = 0; c < 3; c++) f[c] = n[c] * mass * P.force_scale;
    }
}

// DR: the instantiation that reads the per-env object, tendon and gravity parameters (b200gym.cu attach_object_params)
template <int L, int BLOCK, bool DR = false>
__global__ void __launch_bounds__(BLOCK) hand_step_kernel(const DevModel *__restrict__ gm, Buffers B,
                                                          const __grid_constant__ b2g_hand_params P,
                                                          const __grid_constant__ HandDev H,
                                                          const float *__restrict__ actions_in, int N) {
    __shared__ DevModel sm;
    __shared__ alignas(8) uint64_t mbar;
    load_model_hot(&sm, &mbar, gm);
    using ST = Stepper<L, false, BLOCK, true, false, DR>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const bool w0 = valid && lane == 0;
    const int nd = sm.nl - 1, NS = sm.ns, NA = P.num_actions, O = P.num_obs;
    ST st = make_stepper<L, false, BLOCK, true, false, DR>(&sm, nullptr, lane);
    attach_env_params_generic(st, sm, B, e);                 // per-env link masses / joint properties / friction, when bound
    if (DR) attach_object_params(st, sm, B, e);             // object size / mass / friction, tendon damping, gravity

    float *const rows = (float *)B.p[B2G_T_ROOT_STATE] + (size_t)e * 39;          // hand | object | goal marker
    const float *const init_rows = (const float *)B.p[B2G_T_INITIAL_ROOT] + (size_t)e * 39;
    float *const goal_row = (float *)B.p[B2G_T_GOAL_STATES] + (size_t)e * 13;
    float2 *const row_dof = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    float *const cur_t = (float *)B.p[B2G_T_DOF_TARGET] + (size_t)e * nd;
    float *const prev_t = (float *)B.p[B2G_T_PREV_TARGETS] + (size_t)e * nd;
    float *const act_out = B.p[B2G_T_ACTIONS] ? (float *)B.p[B2G_T_ACTIONS] + (size_t)e * NA : nullptr;
    long long *const reset_b = (long long *)B.p[B2G_T_RESET], *const goal_reset_b = (long long *)B.p[B2G_T_RESET_GOAL];
    long long *const progress_b = (long long *)B.p[B2G_T_PROGRESS];
    float *const succ_b = (float *)B.p[B2G_T_SUCCESSES];
    int *const rc = (int *)B.p[B2G_T_RESET_COUNT], *const grc = (int *)B.p[B2G_T_GOAL_RESET_COUNT];

    RootState rs; load_root(rows, rs);
    ObjState ob; load_obj(rows + 13, ob);
    const bool do_reset = reset_b[e] != 0;
    const bool do_goal = do_reset || goal_reset_b[e] != 0;
    long long progress = progress_b[e];
    float successes = succ_b[e];
    const uint32_t gid = (uint32_t)(e + P.env_id_offset);
    const uint32_t count = do_reset ? (uint32_t)rc[e] : 0u;

    // ---- pre_physics_step: reset_target_pose.  An env that resets draws its goal inside reset_idx, which overrides :667-670
    float goal_pos[3], goal_rot[4];
    if (do_goal) {
        hand_reset_goal(P, gid, count, nd, !do_reset, grc + e, init_rows, goal_row, rows, w0, goal_pos, goal_rot);
    } else {
#pragma unroll
        for (int c = 0; c < 3; c++) goal_pos[c] = goal_row[c];
#pragma unroll
        for (int c = 0; c < 4; c++) goal_rot[c] = goal_row[3 + c];
    }
    // ---- reset_idx (:612-659): object pose, then the hand's joints and targets
    if (do_reset) {
        hand_reset_obj(P, gid, count, init_rows, ob);
        progress = 0; successes = 0.f;
        if (w0) rc[e] = (int)(count + 1u);
    }
    // ---- joints: reset state, position targets (:672-698), clamp of VecTask.step (:374)
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int link = st.link_of(s), d = link - 1;
        if (link < 0) continue;
        float2 qv = row_dof[d];
        float cur = cur_t[d], prev = prev_t[d];
        const float lo = P.dof_lower[d], hi = P.dof_upper[d];
        if (do_reset) {
            qv = hand_reset_dof(P, gid, count, d, nd);
            cur = qv.x; prev = qv.x;
        }
        const int k = H.dof_action[d];
        if (k >= 0) {
            const float a = fminf(fmaxf(actions_in[(size_t)e * NA + k], -P.clip_actions), P.clip_actions);
            if (P.use_relative_control) {
                const float tg = prev + P.dof_speed_scale * P.dt * a;
                cur = fmaxf(fminf(tg, hi), lo);                                   // tensor_clamp: max(min(t, hi), lo)
            } else {
                cur = 0.5f * (a + 1.0f) * (hi - lo) + lo;                         // scale, torch_jit_utils.py:234
                cur = P.act_moving_average * cur + (1.0f - P.act_moving_average) * prev;
                cur = fmaxf(fminf(cur, hi), lo);
            }
            prev = cur;
            if (valid && act_out) act_out[k] = a;
        }
        if (valid) { cur_t[d] = cur; prev_t[d] = prev; }
        st.set_joint(s, qv.x, qv.y, (st.links[link].flags & LF_POSDRIVE) ? cur : 0.f);
    }

    // ---- random forces on the object (:700-709): every lane of the env computes them, lane 0 stores
    if (P.force_scale > 0.f) {
        float *const of = (float *)B.p[B2G_T_OBJ_FORCE] + 3 * (size_t)e, *const pb = (float *)B.p[B2G_T_RANDOM_FORCE_PROB] + e;
        float f[3] = {of[0], of[1], of[2]}, prob = *pb;
        if (do_reset) { f[0] = f[1] = f[2] = 0.f; prob = hand_force_prob(P, gid, count, nd); }      // reset_idx, :616,642
        hand_force_update(P, gid, do_reset ? count + 1u : (uint32_t)rc[e], (uint32_t)progress, sm.obj_mass, prob, f);
        __syncwarp();                                   // every lane has read the old values
        if (w0) { of[0] = f[0]; of[1] = f[1]; of[2] = f[2]; *pb = prob; }
        st.set_obj_force(f[0], f[1], f[2]);
    } else st.set_obj_force(0.f, 0.f, 0.f);

    // ---- control_freq_inv x gym.simulate.  control_freq_inv == 0: no simulate (the observation then reads the
    // sensor / joint-force tensors as they stand); pins the task arithmetic against the reference's golden vectors
    typename ST::Outputs o;
    o.write = valid;
    o.net_contact = B.p[B2G_T_NET_CONTACT] ? (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * sm.nb * 3 : nullptr;
    o.sensor = B.p[B2G_T_FORCE_SENSOR] ? (float *)B.p[B2G_T_FORCE_SENSOR] + (size_t)e * sm.nsens * 6 : nullptr;
    o.dof_force = B.p[B2G_T_DOF_FORCE] ? (float *)B.p[B2G_T_DOF_FORCE] + (size_t)e * nd : nullptr;
    const int total = P.control_freq_inv * sm.substeps;
    for (int k = 0; k < total; k++) st.substep(rs, k == total - 1, o, &ob);
    st.pass1(rs);                                   // link poses of the new state (fingertips)

    // ---- post_physics_step
    progress += 1;
    if (w0) store_obj(rows + 13, ob);
    float *const obs = (float *)B.p[B2G_T_OBS] + (size_t)e * O;
    float *obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    obsc = (obsc && obsc != (float *)B.p[B2G_T_OBS]) ? obsc + (size_t)e * O : nullptr;
    const float clipo = P.clip_obs;
    float *const states = (H.num_states > 0 && B.p[B2G_T_STATES]) ? (float *)B.p[B2G_T_STATES] + (size_t)e * H.num_states : nullptr;
    // put(piece, i, v): element i of an observation piece, into obs_buf (+ its clipped copy) and, if present, states_buf
    auto put = [&](int HandDev::Layout::*piece, int i, float v) {
        if (!valid) return;
        const int io = H.lay[0].*piece;
        if (io >= 0) {
            obs[io + i] = v;
            if (obsc) obsc[io + i] = fminf(fmaxf(v, -clipo), clipo);
        }
        if (states) { const int is = H.lay[1].*piece; if (is >= 0) states[is + i] = v; }
    };
    using LY = HandDev::Layout;
    float action_penalty = 0.f;
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int link = st.link_of(s), d = link - 1;
        if (link < 0) continue;
        const float2 qv = st.get_q(s);
        if (valid) row_dof[d] = qv;
        put(&LY::o_dofpos, d, t_unscale(qv.x, P.dof_lower[d], P.dof_upper[d]));
        put(&LY::o_dofvel, d, P.vel_obs_scale * qv.y);
        put(&LY::o_dofforce, d, P.force_torque_obs_scale * (o.dof_force ? o.dof_force[d] : 0.f));
        const int k = H.dof_action[d];
        if (k >= 0) {
            const float a = fminf(fmaxf(actions_in[(size_t)e * NA + k], -P.clip_actions), P.clip_actions);
            put(&LY::o_act, k, a);
            action_penalty += a * a;
        }
    }
    // fingertips (:456-457): rigid-body state of the five distal links, force sensors
#pragma unroll 1
    for (int f = 0; f < 5; f++) {
        const int ref = H.ft_ref[f];
        if ((ref >> 8) != lane) continue;
        float R[9], x[3], vw[3], vl[3];
        st.load_pose(ref & 255, R, x, vw, vl);
        const float bp[3] = {H.ft_bpos[f][0], H.ft_bpos[f][1], H.ft_bpos[f][2]};
        float wb[3]; matvec(R, bp, wb);
        const float xb[3] = {x[0] + wb[0], x[1] + wb[1], x[2] + wb[2]};
        // fingertip block: 3 (position only) or 13 floats per fingertip, per destination layout
        float Rwb[9], q[4], wxr[3];
        matmul(R, H.ft_bR[f], Rwb); mat_to_quat(Rwb, q);
        cross(vw, xb, wxr);
        auto put_ft = [&](float *dst, float *dstc, const HandDev::Layout &ly) {
            if (!valid || !dst || ly.o_ft < 0) return;
            const int o0 = ly.o_ft + ly.ft_stride * f;
            float v[13] = {rs.rp[0] + xb[0], rs.rp[1] + xb[1], rs.rp[2] + xb[2], q[0], q[1], q[2], q[3],
                           vl[0] + wxr[0], vl[1] + wxr[1], vl[2] + wxr[2], vw[0], vw[1], vw[2]};
#pragma unroll
            for (int c = 0; c < 13; c++) {
                if (c < ly.ft_stride) {
                    dst[o0 + c] = v[c];
                    if (dstc) dstc[o0 + c] = fminf(fmaxf(v[c], -clipo), clipo);
                }
            }
        };
        put_ft(obs, obsc, H.lay[0]);
        put_ft(states, nullptr, H.lay[1]);
#pragma unroll
        for (int c = 0; c < 6; c++) put(&LY::o_sens, 6 * f + c, P.force_torque_obs_scale * (o.sensor ? o.sensor[6 * f + c] : 0.f));
    }
    action_penalty = lane_sum<L>(action_penalty);

    // object / goal part of the observation and compute_hand_reward (:749-804), replicated; lane 0 writes
    const float gconj[4] = {-goal_rot[0], -goal_rot[1], -goal_rot[2], goal_rot[3]};
    float qdiff[4]; t_quat_mul(ob.q, gconj, qdiff);
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 3; c++) put(&LY::o_objpose, c, ob.p[c]);
        if (valid) {       // orientation only where the layout carries the full pose
            if (H.lay[0].o_objpose >= 0 && H.lay[0].n_objpose == 7) {
#pragma unroll
                for (int c = 0; c < 4; c++) { obs[H.lay[0].o_objpose + 3 + c] = ob.q[c]; if (obsc) obsc[H.lay[0].o_objpose + 3 + c] = fminf(fmaxf(ob.q[c], -clipo), clipo); }
            }
            if (states) {
#pragma unroll
                for (int c = 0; c < 4; c++) states[H.lay[1].o_objpose + 3 + c] = ob.q[c];
            }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) { put(&LY::o_objvel, c, ob.v[c]); put(&LY::o_objvel, 3 + c, P.vel_obs_scale * ob.w[c]); }
#pragma unroll
        for (int c = 0; c < 3; c++) put(&LY::o_goalpose, c, goal_pos[c]);
#pragma unroll
        for (int c = 0; c < 4; c++) put(&LY::o_goalpose, 3 + c, goal_rot[c]);
#pragma unroll
        for (int c = 0; c < 4; c++) put(&LY::o_qdiff, c, qdiff[c]);
    }
    {
        const float dx = ob.p[0] - goal_pos[0], dy = ob.p[1] - goal_pos[1], dz = ob.p[2] - goal_pos[2];
        const float goal_dist = sqrtf(dx * dx + dy * dy + dz * dz);
        const float vn = sqrtf(qdiff[0] * qdiff[0] + qdiff[1] * qdiff[1] + qdiff[2] * qdiff[2]);
        const float rot_dist = 2.0f * asinf(fminf(vn, 1.0f));
        const float dist_rew = goal_dist * P.dist_reward_scale;
        const float rot_rew = 1.0f / (fabsf(rot_dist) + P.rot_eps) * P.rot_reward_scale;
        float reward = dist_rew + rot_rew + action_penalty * P.action_penalty_scale;
        const bool hit = fabsf(rot_dist) <= P.success_tolerance;
        const long long goal_resets = hit ? 1 : 0;                 // reset_goal_buf is 0 here: cleared by reset_target_pose
        successes = successes + (float)goal_resets;
        if (goal_resets == 1) reward = reward + P.reach_goal_bonus;
        if (goal_dist >= P.fall_dist) reward = reward + P.fall_penalty;
        long long resets = (goal_dist >= P.fall_dist) ? 1 : 0;     // reset_buf is 0 here: cleared by reset_idx
        if (P.max_consecutive_successes > 0) {
            if (hit) progress = 0;
            if (successes >= (float)P.max_consecutive_successes) resets = 1;
        }
        if ((float)progress >= P.max_episode_length - 1.f) resets = 1;
        if (P.max_consecutive_successes > 0 && (float)progress >= P.max_episode_length - 1.f) reward = reward + 0.5f * P.fall_penalty;
        float *const cs = (float *)B.p[B2G_T_CONSECUTIVE_SUCCESSES];
        if (w0) {
            ((float *)B.p[B2G_T_REW])[e] = reward;
            reset_b[e] = resets; goal_reset_b[e] = goal_resets; progress_b[e] = progress; succ_b[e] = successes;
            uint8_t *to = (uint8_t *)B.p[B2G_T_TIMEOUT];
            if (to) to[e] = (uint8_t)(((float)progress >= P.max_episode_length - 1.f) && resets != 0);   // vec_task.py:394
            if (resets != 0) { atomicAdd(cs + 1, 1.0f); atomicAdd(cs + 2, successes); }               // integer-valued: order-free
        }
        // consecutive_successes (:797-801): the last block to finish folds the two sums in
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            unsigned *ticket = reinterpret_cast<unsigned *>(cs + 3);
            if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
                __threadfence();
                const float num_resets = atomicAdd(cs + 1, 0.f), finished = atomicAdd(cs + 2, 0.f);
                if (num_resets > 0.f) cs[0] = P.av_factor * finished / num_resets + (1.0f - P.av_factor) * cs[0];
                cs[1] = 0.f; cs[2] = 0.f; *ticket = 0u;
            }
        }
    }
}

}  // namespace b2g

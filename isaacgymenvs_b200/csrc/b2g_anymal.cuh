// b2g_anymal.cuh -- fused AnymalTerrain control step (reference: tasks/anymal_terrain.py).
//
// Two launches per VecTask.step(), because reset_idx's terrain curriculum compares each env with a
// norm taken over ALL envs being reset this step (`torch.norm(self.commands[env_ids,:2])` without
// dim, anymal_terrain.py:432 -- SURVEY.md 3.3), i.e. a grid-wide reduction between termination
// and reset:
//   kernel 1  pre_physics_step (PD torque + gym.simulate x decimation, :441-451) + the extra
//             control_freq_inv simulate of VecTask.step (vec_task.py:379-382) + post_physics_step
//             up to compute_reward (:453-475): push, base quantities, termination, 13 reward terms;
//   kernel 2  reset_idx (:384-425) incl. update_terrain_level (:427-435), compute_observations
//             (:302-313) with get_heights (:515-538), observation noise (:481-482), last_* (:484-485).
#pragma once
#include "b2g_device.cuh"
#include "b2g_tasks.cuh"

namespace b2g {

// four lanes per env on the generic Stepper (lane k owns leg k), 128 threads
template <bool HF>
__global__ void __launch_bounds__(128) anymal_physics_kernel(const DevModel *__restrict__ gm, const int16_t *__restrict__ hf,
                                                              Buffers B, const __grid_constant__ b2g_anymal_params P,
                                                              const float *__restrict__ actions_in, int N, unsigned step_counter) {
    constexpr int L = 4, BLOCK = 128;
    __shared__ DevModel sm;
    __shared__ alignas(8) uint64_t mbar;
    __shared__ float s_part[BLOCK / 32];
    load_model_hot(&sm, &mbar, gm);
    using ST = Stepper<L, HF, BLOCK>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const int nd = sm.nl - 1, NS = sm.ns;
    ST st = make_stepper<L, HF, BLOCK>(&sm, hf, lane);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
    RootState rs; load_root((const float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
    const float2 *dofs = (const float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    float *act_out = (float *)B.p[B2G_T_ACTIONS];
    float *torq = (float *)B.p[B2G_T_TORQUES] + (size_t)e * nd;
    const float *last_a = (const float *)B.p[B2G_T_LAST_ACTIONS] + (size_t)e * nd;
    const float *last_v = (const float *)B.p[B2G_T_LAST_DOF_VEL] + (size_t)e * nd;
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int d = st.link_of(s) - 1;
        if (d < 0) continue;
        const float2 v = dofs[d];
        const float a = fminf(fmaxf(actions_in[(size_t)e * nd + d], -P.clip_actions), P.clip_actions);
        if (valid) act_out[(size_t)e * nd + d] = a;
        st.set_joint(s, v.x, v.y, 0.f);
    }
    typename ST::Outputs o;
    o.write = valid; o.sensor = nullptr; o.dof_force = nullptr;
    o.net_contact = (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * sm.nb * 3;
    // ---- pre_physics_step (:441-451): decimation x {PD torque from the refreshed dof state, simulate},
    //      then VecTask.step's own control_freq_inv x simulate with the last torques (vec_task.py:379-382)
    const int total = (P.decimation + P.control_freq_inv) * sm.substeps;
    for (int k = 0; k < total; k++) {
        if (k < P.decimation * sm.substeps && (k % sm.substeps) == 0) {
#pragma unroll 1
            for (int s = 0; s < NS; s++) {
                const int d = st.link_of(s) - 1;
                if (d < 0) continue;
                const float2 qv = st.get_q(s);
                const float t = anymal_pd_torque(P, d, act_out[(size_t)e * nd + d], qv.x, qv.y);
                st.set_act(s, t);
                if (valid) torq[d] = t;
            }
        }
        st.substep(rs, k == total - 1, o);
    }

    // ---- post_physics_step (:453-475)
    anymal_post_physics<BLOCK>(P, B, N, e, lane, valid, step_counter, rs, o.net_contact, s_part, [&](AnymalCosts &c) {
        float2 *dw = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
#pragma unroll 1
        for (int s = 0; s < NS; s++) {
            const int d = st.link_of(s) - 1;
            if (d < 0) continue;
            const float2 qv = st.get_q(s);
            if (valid) dw[d] = qv;
            c.add(P, d, torq[d], act_out[(size_t)e * nd + d], qv.x, qv.y, last_a, last_v);
        }
        if (valid && lane == 0 && !sm.root_fixed) store_root((float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
    });
}

// one warp per env, 128 threads
__global__ void __launch_bounds__(128) anymal_reset_obs_kernel(Buffers B, const __grid_constant__ b2g_anymal_params P,
                                                                const int16_t *__restrict__ hs, int N, int nd,
                                                                int nblocks1, unsigned step_counter, int reset_only) {
    constexpr int L = 32, BLOCK = 128;
    // reset_only (VecTask.reset_done, vec_task.py:440-455 -> reset_idx :384-425 of the flagged envs, no step): the norm
    // over the reset set is summed here from the flags themselves; observations and last_* are left to the next step
    __shared__ float s_norm;
    __shared__ int s_done;
    if (threadIdx.x == 0) s_done = 0;
    if (threadIdx.x < 32) {
        const float *red = (const float *)B.p[B2G_T_REDUCE_SCRATCH];
        float t = 0.f;
        if (reset_only) {
            const long long *rb = (const long long *)B.p[B2G_T_RESET];
            const float *cm = (const float *)B.p[B2G_T_COMMANDS];
            for (int i = threadIdx.x; i < N; i += 32) t += (rb[i] != 0) ? cm[4 * i] * cm[4 * i] + cm[4 * i + 1] * cm[4 * i + 1] : 0.f;
        } else
        for (int i = threadIdx.x; i < nblocks1; i += 32) t += red[i];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
        if (threadIdx.x == 0) s_norm = sqrtf(t);
    }
    __syncthreads();
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    if (env >= N) return;
    const int e = env;
    const uint32_t gid = (uint32_t)(e + P.env_id_offset);
    float *root = (float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e;
    float2 *dofs = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    float *cmd = (float *)B.p[B2G_T_COMMANDS] + (size_t)e * 4;
    long long *reset_b = (long long *)B.p[B2G_T_RESET], *progress_b = (long long *)B.p[B2G_T_PROGRESS];
    const float *acts = (const float *)B.p[B2G_T_ACTIONS] + (size_t)e * nd;
    float *last_a = (float *)B.p[B2G_T_LAST_ACTIONS] + (size_t)e * nd, *last_v = (float *)B.p[B2G_T_LAST_DOF_VEL] + (size_t)e * nd;
    const bool do_reset = reset_b[e] != 0;
    int *rcnt = (int *)B.p[B2G_T_RESET_COUNT];
    const uint32_t count = (uint32_t)rcnt[e];
    __syncwarp();
    if (do_reset) {
        // reset_idx (:384-425).  uniform indices: [0,nd) position offsets, [nd,2nd) velocities, 2nd..2nd+1 xy, then x, y, heading
        auto U = [&](int i) { return anymal_uniform(P.seed, gid, count, TAG_RESET, i); };
        for (int d = lane; d < nd; d += L)
            dofs[d] = make_float2(P.default_dof_pos[d] * t_rand_float(0.5f, 1.5f, U(d)), t_rand_float(-0.1f, 0.1f, U(nd + d)));
        if (lane == 0) {
            float org[3] = {0.f, 0.f, 0.f};
            if (P.custom_origins) {
                float *eo = (float *)B.p[B2G_T_ENV_ORIGINS] + 3 * (size_t)e;
                if (P.curriculum) {                                   // update_terrain_level (:427-435)
                    long long *lv = (long long *)B.p[B2G_T_TERRAIN_LEVELS];
                    const long long ty = ((const long long *)B.p[B2G_T_TERRAIN_TYPES])[e];
                    const float dx = root[0] - eo[0], dy = root[1] - eo[1];
                    const float dist = sqrtf(dx * dx + dy * dy);
                    long long level = lv[e];
                    level -= (dist < s_norm * P.max_episode_length_s * 0.25f) ? 1 : 0;
                    level += (dist > P.env_length / 2.f) ? 1 : 0;
                    level = (level < 0 ? 0 : level) % P.env_rows;
                    atomicAdd((float *)B.p[B2G_T_REDUCE_SCRATCH] + REDUCE_PARTIALS + 32, (float)(level - lv[e]));   // running sum of terrain_levels (integer-valued)
                    lv[e] = level;
                    const float *to = (const float *)B.p[B2G_T_TERRAIN_ORIGINS] + 3 * ((size_t)level * P.env_cols + ty);
                    eo[0] = to[0]; eo[1] = to[1]; eo[2] = to[2];
                }
                org[0] = eo[0]; org[1] = eo[1]; org[2] = eo[2];
            }
#pragma unroll
            for (int c = 0; c < 13; c++) root[c] = P.base_init_state[c];
            root[0] += org[0]; root[1] += org[1]; root[2] += org[2];
            if (P.custom_origins) { root[0] += t_rand_float(-0.5f, 0.5f, U(2 * nd)); root[1] += t_rand_float(-0.5f, 0.5f, U(2 * nd + 1)); }
            float c0 = t_rand_float(P.command_x[0], P.command_x[1], U(2 * nd + 2));
            float c1 = t_rand_float(P.command_y[0], P.command_y[1], U(2 * nd + 3));
            float c3 = t_rand_float(P.command_yaw[0], P.command_yaw[1], U(2 * nd + 4));
            const float keep = (sqrtf(c0 * c0 + c1 * c1) > 0.25f) ? 1.f : 0.f;    // set small commands to zero
            cmd[0] = c0 * keep; cmd[1] = c1 * keep; cmd[2] = cmd[2] * keep; cmd[3] = c3 * keep;
            float *fat = (float *)B.p[B2G_T_FEET_AIR_TIME] + 4 * (size_t)e;
            fat[0] = fat[1] = fat[2] = fat[3] = 0.f;
            progress_b[e] = 0;
            reset_b[e] = 1;
            rcnt[e] = (int)(count + 1);
            float *es = (float *)B.p[B2G_T_EPISODE_SUMS];
            float *red = (float *)B.p[B2G_T_REDUCE_SCRATCH] + REDUCE_PARTIALS;          // extras["episode"] sums (logging)
            for (int k = 0; k < 13; k++) { atomicAdd(red + k, es[(size_t)k * N + e]); es[(size_t)k * N + e] = 0.f; }
            atomicAdd(red + 13, 1.f);
            __threadfence();                  // these sums are read by the grid's last warp (ticket below): order them before this warp's arrival
        }
    }
    __syncwarp();
    if (reset_only) return;
    // ---- compute_observations (:302-313) + noise (:481-482)
    float *obs = (float *)B.p[B2G_T_OBS] + (size_t)e * P.num_obs;
    float *obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    obsc = (obsc && obsc != (float *)B.p[B2G_T_OBS]) ? obsc + (size_t)e * P.num_obs : nullptr;
    const float *nsv = (const float *)B.p[B2G_T_NOISE_SCALE];
    // observation noise (:481-482): uniform number idx of stream (env, step); one Philox block serves 4 neighbours.
    // The env's 47 Philox blocks are generated ONCE, spread over the 32 lanes (<= 2 each), and the noise terms parked in
    // shared memory -- with each lane generating the blocks of the indices it happens to write, the Philox rounds were
    // most of this kernel's instructions.
    __shared__ float s_noise[BLOCK / 32][192];
    float *const my_noise = s_noise[threadIdx.x >> 5];
    if (P.add_noise) {
        for (int blk = lane; 4 * blk < P.num_obs && blk < 48; blk += 32) {
            uint32_t r4[4];
            philox4x32_10((uint32_t)blk, step_counter, gid, TAG_NOISE, (uint32_t)P.seed, (uint32_t)(P.seed >> 32), r4);
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int idx = 4 * blk + c;
                if (idx < P.num_obs) my_noise[idx] = (2.f * ((float)(r4[c] >> 8) * (1.0f / 16777216.0f)) - 1.f) * nsv[idx];
            }
        }
        __syncwarp();
    }
    auto put = [&](int idx, float v) {
        if (P.add_noise) v += my_noise[idx];
        obs[idx] = v;
        if (obsc) obsc[idx] = fminf(fmaxf(v, -P.clip_obs), P.clip_obs);
    };
    const float *bs = (const float *)B.p[B2G_T_BASE_SCRATCH] + (size_t)e * 12;
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            put(c, bs[c] * P.lin_vel_scale);
            put(3 + c, bs[3 + c] * P.ang_vel_scale);
            put(6 + c, bs[6 + c]);
        }
        put(9, cmd[0] * P.lin_vel_scale); put(10, cmd[1] * P.lin_vel_scale); put(11, cmd[2] * P.ang_vel_scale);
    }
    for (int d = lane; d < nd; d += L) {
        const float2 qv = dofs[d];
        const float a = acts[d];
        put(12 + d, qv.x * P.dof_pos_scale);
        put(12 + nd + d, qv.y * P.dof_vel_scale);
        put(12 + 2 * nd + 140 + d, a);
        last_a[d] = a; last_v[d] = qv.y;                                           // :484-485
    }
    // get_heights (:515-538): yaw-rotate the 14 x 10 grid, index the int16 samples, min of two neighbours
    {
        float qy[4] = {0.f, 0.f, root[5], root[6]};
        const float nq = fmaxf(sqrtf(qy[2] * qy[2] + qy[3] * qy[3]), 1e-9f);
        qy[2] /= nq; qy[3] /= nq;
        const float bz = root[2];
        constexpr int PER = (140 + L - 1) / L;
        const float rx = root[0], ry = root[1];
        // the two height samples of a point are independent global loads: fetch a chunk of points' samples together
        // (their latencies overlap), then emit the chunk's observations
        constexpr int CH = PER < 7 ? PER : 7;
        const int p_end = min(140, (lane + 1) * PER);
#pragma unroll 1
        for (int p0 = lane * PER; p0 < p_end; p0 += CH) {
            int hmin[CH];
#pragma unroll
            for (int j = 0; j < CH; j++) {
                const int p = min(p0 + j, 139);
                const int ix = p / 10, iy = p % 10;
                const int xi = (ix < 7) ? ix - 8 : ix - 5;            // -8..-2, 2..8
                const int yi = (iy < 5) ? iy - 5 : iy - 4;            // -5..-1, 1..5
                const float pt[3] = {0.1f * (float)xi, 0.1f * (float)yi, 0.f};
                float w[3]; t_quat_apply(qy, pt, w);
                hmin[j] = 0;
                if (hs) {
                    const float fx = (w[0] + rx + P.border_size) / P.terrain_hscale;
                    const float fy = (w[1] + ry + P.border_size) / P.terrain_hscale;
                    int px = (int)fx, py = (int)fy;                   // .long(): truncation toward zero
                    px = max(0, min(px, P.hs_rows - 2)); py = max(0, min(py, P.hs_cols - 2));
                    const int h1 = __ldg(hs + (size_t)px * P.hs_cols + py), h2 = __ldg(hs + (size_t)(px + 1) * P.hs_cols + py + 1);
                    hmin[j] = min(h1, h2);
                }
            }
#pragma unroll
            for (int j = 0; j < CH; j++) {
                if (p0 + j < p_end) put(12 + 2 * nd + p0 + j, fminf(fmaxf(bz - 0.5f - (float)hmin[j] * P.terrain_vscale, -1.f), 1.f) * P.height_meas_scale);
            }
        }
    }
    if (lane == 0) {
        uint8_t *to = (uint8_t *)B.p[B2G_T_TIMEOUT];                                // vec_task.py:394
        if (to) to[e] = (uint8_t)((progress_b[e] >= (long long)P.max_episode_length - 1) && reset_b[e] != 0);
    }
    // extras["episode"] (reset_idx :420-425): the last warp of the grid to get here turns this step's sums over the reset
    // envs into the per-second means the task publishes (kept as they are when no env was reset), so that the host side
    // of VecTask.step issues no torch kernels for them.  Layout after the 1024 partials: [0,13) sums, 13 count,
    // 15 ticket, [16,29) means, 29 mean terrain level, 32 running sum of terrain_levels.
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        const int nwarps = min(BLOCK / 32, N - (int)blockIdx.x * (BLOCK / 32));    // warps of this block that own an env
        // (no grid-scope fence here: only the few warps that reset an env touched the sums, and they fenced there; a
        // __threadfence by every warp invalidates L1 4096 times per launch -- measured +13 us)
        if (atomicAdd(&s_done, 1) == nwarps - 1) {
            float *red = (float *)B.p[B2G_T_REDUCE_SCRATCH] + REDUCE_PARTIALS;
            unsigned *ticket = reinterpret_cast<unsigned *>(red + 15);
            if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
                __threadfence();
                const float cnt = atomicAdd(red + 13, 0.f);
                if (cnt > 0.f) {
                    for (int k = 0; k < 13; k++) red[16 + k] = atomicAdd(red + k, 0.f) / cnt / P.max_episode_length_s;
                    red[29] = atomicAdd(red + 32, 0.f) / (float)N;
                }
                *ticket = 0u;
            }
        }
    }
}

}  // namespace b2g

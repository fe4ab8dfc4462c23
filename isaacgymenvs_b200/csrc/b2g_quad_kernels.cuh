// b2g_quad_kernels.cuh -- kernels on the quad sub-step (b2g_quad.cuh).  Included by b200gym.cu after Buffers /
// TileArgs / the task helpers.
//
//   quad_simulate_kernel   gym.simulate() (vec_task.py:379-382) for "4 chains on a free base" articulations
//   quad_loco_kernel       one whole VecTask.step() of Ant (vec_task.py:360-408 + ant.py:281-297), tiles by bulk copy
#pragma once
#include "b2g_quad.cuh"
#include "b2g_tasks.cuh"

namespace b2g {

// dynamic shared memory of the quad kernels: [park: quad_park_f4(NS) x BLOCK float4][tiles ...][quad model]
template <int NS, bool HF, int SP, bool SELF = false>
__device__ __forceinline__ QLane<NS, HF, SP, SELF> make_qlane(const float4 *qm, const int16_t *hf, float4 *park_base, int block, int lane) {
    QLane<NS, HF, SP, SELF> L;
    L.qm = qm; L.hf = hf; L.park = park_base + threadIdx.x; L.pstride = block; L.lane = lane; L.env_mu = -1.f;
    L.dr_mass = nullptr; L.dr_dof = nullptr;
    return L;
}

// per-env physical parameters (domain randomisation tensors; null = the model's own)
template <class QL>
__device__ __forceinline__ void attach_env_params(QL &L, const Buffers &B, int e, int nd, bool arrays = true) {
    const float *ms = arrays ? (const float *)B.p[B2G_T_ENV_MASS_SCALE] : nullptr;
    const float4 *dp = arrays ? (const float4 *)B.p[B2G_T_ENV_DOF_PROPS] : nullptr;
    const float *envmu = (const float *)B.p[B2G_T_ENV_FRICTION];
    if (ms) L.dr_mass = ms + (size_t)e * (nd + 1);
    if (dp) L.dr_dof = dp + (size_t)e * nd;
    if (envmu) L.env_mu = 0.5f * (envmu[e] + L.qm[18].x);             // PhysX default combine mode: the average of the two materials
}

// SELF: link-link contact (a self-colliding model; its blob and park area are larger, see b2g_quad.cuh)
template <int NS, bool HF, int SP, int BLOCK, bool SELF = false>
__global__ void __launch_bounds__(BLOCK) quad_simulate_kernel(const float4 *__restrict__ gqm, const int16_t *__restrict__ hf, Buffers B, int N, int substeps) {
    float4 *const park = b2g_dyn_smem;
    float4 *const qm = b2g_dyn_smem + quad_park_f4(NS, SELF) * BLOCK;
    for (int i = threadIdx.x; i < quad_model_f4(NS, SELF); i += BLOCK) qm[i] = gqm[i];
    __syncthreads();
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt >> 2, lane = gt & 3;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    constexpr int nd = 4 * NS;
    QLane<NS, HF, SP, SELF> L = make_qlane<NS, HF, SP, SELF>(qm, hf, park, BLOCK, lane);
    attach_env_params(L, B, e, nd);
    float *const root_row = (float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e;
    RootState rs; load_root(root_row, rs);
    float2 *const d = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    const float *act = (const float *)B.p[B2G_T_DOF_ACTUATION];
    int dofi[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) {
        dofi[s] = q_f2i(L.LK(s, 16).w);
        const float2 v = d[dofi[s]];
        L.q[s] = v.x; L.qd[s] = v.y; L.act[s] = act ? act[(size_t)e * nd + dofi[s]] : 0.f;
    }
    const int cnt = q_f2i(qm[7].w), n_sens = cnt & 255, n_body = cnt >> 8;
    float *fs = (float *)B.p[B2G_T_FORCE_SENSOR], *df = (float *)B.p[B2G_T_DOF_FORCE], *nc = (float *)B.p[B2G_T_NET_CONTACT];
    QOutputs o;
    o.sensor = fs ? fs + (size_t)e * n_sens * 6 : nullptr;
    o.dof_force = df ? df + (size_t)e * nd : nullptr;
    o.net_contact = nc ? nc + (size_t)e * n_body * 3 : nullptr;
    o.write = valid;
    // `substeps` is a kernel parameter (warp-uniform by construction): the shuffles inside need no re-convergence code
#pragma unroll 1
    for (int k = 0; k < substeps; k++) L.substep(rs, k == substeps - 1, o);
    if (!valid) return;
#pragma unroll
    for (int s = 0; s < NS; s++) d[dofi[s]] = make_float2(L.q[s], L.qd[s]);
    if (lane == 0) store_root(root_row, rs);
}

// -------------------------------------------------------------------------------------------
// compute_observations of Ant (ant.py:374-408) on the four lanes of env e, with the per-DOF sums of its reward (summed on
// this lane only).  put(idx, v) stores element idx of the observation; lane 0 also returns the up / heading vectors and
// projections.  The sensor rows come from the staged tile row s_row after a simulate (stage_out), else from the tensor.
struct AntRootObs {
    float up_proj = 0.f, heading_proj = 0.f;
    float up_vec[3], heading_vec[3];
};
template <int NS, class PUT>
__device__ __forceinline__ LocoCosts ant_obs(const b2g_task_params &P, const RootState &rs, const float (&q)[NS], const float (&qd)[NS],
                                             const int (&dofi)[NS], const int (&sens)[NS], const float (&a_cl)[NS], const float4 *qm, int lane,
                                             const float *s_sens, const float *g_sens, int e, int el, int nsens6, bool stage_out, AntRootObs &ro, PUT put) {
    constexpr int nd = 4 * NS;
    // The three Euler / heading angles are three atan2f calls on different arguments: the lanes of the env take one each
    // (same instruction stream, different data) and hand it to lane 0.
    const float to_t[3] = {P.target[0] - rs.rp[0], P.target[1] - rs.rp[1], 0.f};
    const float isr[4] = {-0.f, -0.f, -0.f, 1.f};
    float tq[4]; t_quat_mul(rs.rq, isr, tq);                   // compute_heading_and_up, torch_jit_utils.py:247-262
    float ang_mine;
    {
        const float qx = tq[0], qy = tq[1], qz = tq[2], qw = tq[3];
        // get_euler_xyz :175-195 (roll, yaw) and compute_rot :265-276 (walk_target_angle); lane 3 duplicates lane 0
        const float ay = (lane == 1) ? 2.0f * (qw * qx + qy * qz) : (lane == 2) ? P.target[2] - rs.rp[2] : 2.0f * (qw * qz + qx * qy);
        const float ax = (lane == 1) ? qw * qw - qx * qx - qy * qy + qz * qz : (lane == 2) ? P.target[0] - rs.rp[0] : qw * qw + qx * qx - qy * qy - qz * qz;
        const float a = atan2f(ay, ax);
        // torch.remainder(a, 2 pi) for a in [-pi, pi] (fmod leaves such an `a` unchanged); the walk angle is not wrapped
        ang_mine = (lane != 2 && a < 0.f) ? a + 6.2831855f : a;
    }
    const float roll = __shfl_sync(0xffffffffu, ang_mine, (threadIdx.x & 28) | 1);
    const float walk = __shfl_sync(0xffffffffu, ang_mine, (threadIdx.x & 28) | 2);
    const float yaw = __shfl_sync(0xffffffffu, ang_mine, (threadIdx.x & 28));
    if (lane == 0) {
        const float nrm = fmaxf(sqrtf(to_t[0] * to_t[0] + to_t[1] * to_t[1] + 0.f), 1e-9f);
        const float td[3] = {to_t[0] / nrm, to_t[1] / nrm, 0.f / nrm};
        const float b0[3] = {1.f, 0.f, 0.f}, b1[3] = {0.f, 0.f, 1.f};
        t_quat_rotate(tq, b1, ro.up_vec, 1.f);
        t_quat_rotate(tq, b0, ro.heading_vec, 1.f);
        ro.up_proj = ro.up_vec[2];
        ro.heading_proj = (ro.heading_vec[0] * td[0] + ro.heading_vec[1] * td[1]) + ro.heading_vec[2] * td[2];
        float vloc[3], wloc[3];
        t_quat_rotate(tq, rs.rv, vloc, -1.f);
        t_quat_rotate(tq, rs.rw, wloc, -1.f);
        put(0, rs.rp[2]);
        put(1, vloc[0]); put(2, vloc[1]); put(3, vloc[2]);
        put(4, wloc[0]); put(5, wloc[1]); put(6, wloc[2]);
        put(7, yaw); put(8, roll); put(9, walk - yaw); put(10, ro.up_proj); put(11, ro.heading_proj);
    }
    // layout: ant.py:401-406  [12 | nd pos | nd vel | 6*nsens sensors | nd actions]
    const int o_pos = 12, o_vel = 12 + nd, o_sens = 12 + 2 * nd, o_act = o_sens + nsens6;
    LocoCosts cost;
#pragma unroll
    for (int s = 0; s < NS; s++) {
        const int d = dofi[s];
        const float a = a_cl[s];
        const float ps = t_unscale(q[s], P.dof_limits_lower[d], P.dof_limits_upper[d]);
        const float vs = qd[s] * P.dof_vel_scale;
        put(o_pos + d, ps); put(o_vel + d, vs); put(o_act + d, a);
        if (sens[s] >= 0) {                                    // typed pointers: shared-memory loads of the staged tile, not generic ones
            float sv[6];
            if (stage_out) {
                const float *sp_ = s_sens + nsens6 * el + 6 * sens[s];
#pragma unroll
                for (int c = 0; c < 6; c++) sv[c] = sp_[c];
            } else {                                           // no simulate: the tensor as it stands (golden-vector mode)
#pragma unroll
                for (int c = 0; c < 6; c++) sv[c] = g_sens ? g_sens[(size_t)e * nsens6 + 6 * sens[s] + c] : 0.f;
            }
            if (stage_out || g_sens) {
#pragma unroll
                for (int c = 0; c < 6; c++) put(o_sens + 6 * sens[s] + c, sv[c] * P.contact_force_scale);
            }
        }
        cost.add(P, d, a, ps, vs, false);
    }
    {
        const int rsens = q_f2i(qm[3].w);                      // a sensor on the base itself (not Ant): through the tensor
        const float *sp_ = stage_out ? s_sens + nsens6 * el : (g_sens ? g_sens + (size_t)e * nsens6 : nullptr);
        if (lane == 0 && rsens >= 0 && sp_) {
#pragma unroll
            for (int c = 0; c < 6; c++) put(o_sens + 6 * rsens + c, sp_[6 * rsens + c] * P.contact_force_scale);
        }
    }
    return cost;
}

// -------------------------------------------------------------------------------------------
// One whole VecTask.step() of Ant on the quad sub-step.  Same data movement as loco_step_kernel: every tensor of
// the step is ONE bulk-async (TMA) copy per block in and out; whole tiles only (the host falls back to
// loco_step_kernel otherwise).
#ifndef B2G_QUAD_MINBLOCKS
#define B2G_QUAD_MINBLOCKS(BLOCK) ((BLOCK) == 128 ? 4 : ((BLOCK) == 64 ? 7 : 14))
#endif
// LEAN: no per-env physical parameters, no dof-force / net-contact outputs bound (the plain Ant task): those pointers
// become compile-time nulls -- their branches and the registers they occupy across the sub-step loop disappear
template <int NS, int SP, int BLOCK, bool HOSTIO, bool LEAN = false>
__global__ void __launch_bounds__(BLOCK, B2G_QUAD_MINBLOCKS(BLOCK)) quad_loco_kernel(
    const float4 *__restrict__ gqm, Buffers B, const __grid_constant__ b2g_task_params P, const float *__restrict__ actions_in, int N, int substeps, TileArgs ta) {
    __shared__ alignas(8) uint64_t mbar, mbar2;
    constexpr int EPB = BLOCK / 4;
    constexpr int nd = 4 * NS;
    float4 *const park = b2g_dyn_smem;
    float4 *const qm = b2g_dyn_smem + ta.model_f4;
    float *const io = reinterpret_cast<float *>(b2g_dyn_smem + ta.io_f4);
    const int O = P.num_obs;
    const int nsens6 = O - 12 - 3 * nd;                      // 6 * nsens, from the obs layout (checked by b2g_set_task)
    const int env0 = blockIdx.x * EPB;
    const TileLayout tl = tile_layout(EPB, nd, nsens6, false);
    float *const s_root = io, *const s_dof = io + tl.dof, *const s_act = io + tl.act, *const s_sens = io + tl.sens;
    long long *const progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    float *const pot_b = (float *)B.p[B2G_T_POTENTIALS];
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int e = gt >> 2, lane = gt & 3;                    // whole tiles: every env of the block exists
    const int el = e - env0;
    // ---- prologue: the model before griddepcontrol.wait, the state tiles after it
    if (threadIdx.x == 0) { mbar_init(&mbar, 1); mbar_init(&mbar2, 1); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&mbar, quad_model_f4(NS) * 16);
        bulk_g2s(qm, gqm, quad_model_f4(NS) * 16, &mbar);
    }
    load_state_tiles<EPB, BLOCK, true, HOSTIO>(&mbar2, io, tl, B, nd, actions_in, env0, ta);
    const long long progress_in = progress_b[e];
    const long long reset_in = reset_b[e];
    const float potentials_in = pot_b[e];
    int *const rc = (int *)B.p[B2G_T_RESET_COUNT];
    // read here (unconditionally: a load that depended on reset_in would stall the prologue on it), written after the
    // physics by lane 0: no intra-warp race
    const uint32_t count = (uint32_t)rc[e];
    mbar_wait(&mbar, 0);
    mbar_wait(&mbar2, 0);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    QLane<NS, false, SP> L = make_qlane<NS, false, SP>(qm, nullptr, park, BLOCK, lane);
    if (!LEAN) attach_env_params(L, B, e, nd);
    float *const row_root = s_root + 13 * el;
    float2 *const row_dof = reinterpret_cast<float2 *>(s_dof + 2 * nd * el);
    float *const row_act = s_act + nd * el;
    RootState rs; load_root(row_root, rs);

    // ---- VecTask.step :374 clamp ; pre_physics_step (ant.py:281-285)
    int dofi[NS], sens[NS];
    float a_cl[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) {
        const float4 k16 = L.LK(s, 16);
        dofi[s] = q_f2i(k16.w); sens[s] = q_f2i(k16.y);
        const float2 v = row_dof[dofi[s]];
        const float a = fminf(fmaxf(row_act[dofi[s]], -P.clip_actions), P.clip_actions);
        row_act[dofi[s]] = a;                                 // the tile becomes the clamped-action output
        a_cl[s] = a;
        L.q[s] = v.x; L.qd[s] = v.y; L.act[s] = a * P.joint_gears[dofi[s]] * P.power_scale;
    }

    // ---- control_freq_inv x gym.simulate (vec_task.py:379-382); 0: the observation reads the tensors as they stand
    const int total = P.control_freq_inv * substeps;          // kernel parameters: warp-uniform trip count
    float *const g_sens = (float *)B.p[B2G_T_FORCE_SENSOR], *const g_dfrc = (float *)B.p[B2G_T_DOF_FORCE];
    QOutputs o;
    o.write = true;
    o.net_contact = (!LEAN && B.p[B2G_T_NET_CONTACT]) ? (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * (q_f2i(qm[7].w) >> 8) * 3 : nullptr;
    const bool stage_out = total > 0;
    o.sensor = stage_out ? s_sens + nsens6 * el : (g_sens ? g_sens + (size_t)e * nsens6 : nullptr);
    o.dof_force = (!LEAN && g_dfrc) ? g_dfrc + (size_t)e * nd : nullptr;
#pragma unroll 1
    for (int k = 0; k < total; k++) L.substep(rs, k == total - 1, o);

    // ---- post_physics_step (ant.py:287-297): progress, reset_idx, observations, reward
    long long progress = progress_in + 1;
    float potentials = potentials_in;
    const bool do_reset = reset_in != 0;
    if (do_reset) {                                           // reset_idx, ant.py:252-279
        const uint32_t gid = (uint32_t)(e + P.env_id_offset);
#pragma unroll
        for (int s = 0; s < NS; s++) {
            const float2 qv = loco_reset_dof(P, gid, count, dofi[s], nd);
            L.q[s] = qv.x; L.qd[s] = qv.y;
        }
        potentials = loco_reset_root(P, B, e, rs);
        progress = 0;
        if (lane == 0) rc[e] = (int)(count + 1);
    }
#pragma unroll
    for (int s = 0; s < NS; s++) row_dof[dofi[s]] = make_float2(L.q[s], L.qd[s]);
    if (lane == 0) store_root(row_root, rs);

    // the parking area is dead from here on: it becomes the output staging area
    __syncthreads();
    float *const g_obs = (float *)B.p[B2G_T_OBS];
    float *g_obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    if (g_obsc == g_obs) g_obsc = nullptr;
    const LocoStage t = loco_stage(reinterpret_cast<float *>(b2g_dyn_smem), EPB, O, g_obsc != nullptr);
    float *const obs = t.obs + (size_t)el * O;
    float *const obsc = g_obsc ? t.obsc + (size_t)el * O : nullptr;

    // compute_observations (ant.py:374-408)
    const float prev_potentials = potentials;                  // prev_potentials_new = potentials.clone(), ant.py:390
    potentials = loco_potential(P, rs.rp);
    const float clipo = P.clip_obs;
    AntRootObs ro;
    LocoCosts cost = ant_obs<NS>(P, rs, L.q, L.qd, dofi, sens, a_cl, qm, lane, s_sens, g_sens, e, el, nsens6, stage_out, ro,
                                 [&](int idx, float v) {
                                     obs[idx] = v;
                                     if (obsc) obsc[idx] = fminf(fmaxf(v, -clipo), clipo);
                                 });
    cost.sum_lanes<4>();
    if (lane == 0) {
        const LocoReward r = loco_reward(P, ro.up_proj, ro.heading_proj, potentials, prev_potentials, cost, rs.rp[2], progress, false);
        stage_row(t, el, r.rew, r.died || r.timed, progress, potentials, prev_potentials, ro.up_vec, ro.heading_vec, r.timed);
    }
    fence_async_smem();
    __syncthreads();
    static_assert(EPB % 16 == 0, "bulk copies move multiples of 16 bytes: the timeout tile is EPB bytes");
    drain_tiles<EPB, BLOCK / 32, false>(B, t, io, tl, s_act, nd, O, nsens6, env0, true, stage_out, true);
    if (HOSTIO) loco_copy_to_host<BLOCK>(ta, t, (size_t)env0, EPB, O, g_obsc != nullptr);
}


// -------------------------------------------------------------------------------------------
// AnymalTerrain kernel 1 on the quad sub-step (same contract as anymal_physics_kernel, b2g_anymal.cuh): pre_physics_step
// (PD torque + gym.simulate x decimation, anymal_terrain.py:441-451) + the control_freq_inv simulates of VecTask.step
// (vec_task.py:379-382) + post_physics_step up to compute_reward (:453-475).  The joint state stays in registers across
// the 5 sub-steps; the PD law reads it there.
// DR = false: no per-env link-mass / joint-property arrays bound -- their pointers are compile-time nulls (smaller code: this kernel runs one
// warp per scheduler, so instruction fetch is exposed: 27 % of its stall cycles are "no instruction")
// SELF: link-link contact (env.selfCollision; the model's self-collision table follows the link table)
template <bool HF, int BLOCK, bool DR = true, bool SELF = false>
__global__ void __launch_bounds__(BLOCK) quad_anymal_physics_kernel(const float4 *__restrict__ gqm, const int16_t *__restrict__ hf,
                                                                    Buffers B, const __grid_constant__ b2g_anymal_params P,
                                                                    const float *__restrict__ actions_in, int N, int substeps, unsigned step_counter) {
    constexpr int NS = 3, nd = 12;
    __shared__ float s_part[BLOCK / 32];
    float4 *const park = b2g_dyn_smem;
    float4 *const qm = b2g_dyn_smem + quad_park_f4(NS, SELF) * BLOCK;
    for (int i = threadIdx.x; i < quad_model_f4(NS, SELF); i += BLOCK) qm[i] = gqm[i];
    __syncthreads();
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt >> 2, lane = gt & 3;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    QLane<NS, HF, 0, SELF> L = make_qlane<NS, HF, 0, SELF>(qm, hf, park, BLOCK, lane);
    attach_env_params(L, B, e, nd, DR);                      // the per-env friction (terrain buckets, anymal_terrain.py:238-247) is always honoured
    RootState rs; load_root((const float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
    const float2 *dofs = (const float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    float *act_out = (float *)B.p[B2G_T_ACTIONS] + (size_t)e * nd;
    float *torq = (float *)B.p[B2G_T_TORQUES] + (size_t)e * nd;
    const float *last_a = (const float *)B.p[B2G_T_LAST_ACTIONS] + (size_t)e * nd;
    const float *last_v = (const float *)B.p[B2G_T_LAST_DOF_VEL] + (size_t)e * nd;
    int dofi[NS];
    float a_cl[NS], tq[NS] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int s = 0; s < NS; s++) {
        dofi[s] = q_f2i(L.LK(s, 16).w);
        const float2 v = dofs[dofi[s]];
        a_cl[s] = fminf(fmaxf(actions_in[(size_t)e * nd + dofi[s]], -P.clip_actions), P.clip_actions);
        if (valid) act_out[dofi[s]] = a_cl[s];
        L.q[s] = v.x; L.qd[s] = v.y; L.act[s] = 0.f;
    }
    QOutputs o;
    o.write = valid; o.sensor = nullptr; o.dof_force = nullptr;
    o.net_contact = (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * (q_f2i(qm[7].w) >> 8) * 3;
    const int total = (P.decimation + P.control_freq_inv) * substeps;
    const int pd_until = P.decimation * substeps;
#pragma unroll 1
    for (int k = 0; k < total; k++) {
        if (k < pd_until && (k % substeps) == 0) {
#pragma unroll
            for (int s = 0; s < NS; s++) {
                const float t = anymal_pd_torque(P, dofi[s], a_cl[s], L.q[s], L.qd[s]);
                L.act[s] = t; tq[s] = t;
            }
        }
        L.substep(rs, k == total - 1, o);
    }

    // ---- post_physics_step (:453-475)
    anymal_post_physics<BLOCK>(P, B, N, e, lane, valid, step_counter, rs, o.net_contact, s_part, [&](AnymalCosts &c) {
        float2 *dw = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
#pragma unroll
        for (int s = 0; s < NS; s++) {
            const int d = dofi[s];
            if (valid) { dw[d] = make_float2(L.q[s], L.qd[s]); if (total > 0 && pd_until > 0) torq[d] = tq[s]; }
            c.add(P, d, (total > 0 && pd_until > 0) ? tq[s] : torq[d], a_cl[s], L.q[s], L.qd[s], last_a, last_v);
        }
        if (valid && lane == 0) store_root((float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
    });
}

}  // namespace b2g

// b2g_quad_rollout.cuh -- K control steps of Ant in ONE launch (b2g_task_rollout): the open-loop rollout the benchmark's
// metric is defined on ("env-steps/s on random-action rollouts", README.md:39-51 of the reference; SURVEY.md 7 hard part 1).
//
// It is K x VecTask.step() (vec_task.py:360-408 + ant.py:281-297) with the actions of all K steps given up front:
//   for k in range(K): obs[k], rew[k], reset[k], time_outs[k] = env.step(actions[k])
// Same device functions, same order of operations as quad_loco_kernel, so the results are the ones K single steps produce;
// what disappears is everything a step pays for being its own launch: the launch itself, the model / state tile loads (the
// joint and base state stay in registers from one step to the next), the drain of the output stores (they overlap the next
// step's physics: the staging area does not alias the sweep scratch here) -- ncu on the single-step kernel attributes
// ~40 % of its time to that once-per-step code.  Actions arrive as double-buffered bulk-async tiles, one step ahead.
//
// Whole tiles of 16 envs (64 threads per CTA); the host falls back to K single steps otherwise.
#pragma once
#include "b2g_quad_kernels.cuh"

namespace b2g {

struct RollArgs {
    const float *actions;      // (K, N, A) device
    float *obs_out;            // (K, N, O): what step() returns -- the clipped observation when a clip is configured
    float *rew_out;            // (K, N)
    long long *reset_out;      // (K, N)
    uint8_t *timeout_out;      // (K, N) or null
    int K;
    int io_f4, model_f4, stage_f4;     // float4 offsets inside dynamic shared memory
};

// output staging of the rollout, epb envs per block.  Per step (never aliases the sweep scratch):
// obs | rew | reset(i64) | timeout(u8).  Last step only, the remaining state tensors in the (then dead) sweep scratch:
// obs (unclipped, when a separate clipped tensor exists) | pot | ppot | up(3) | head(3) | progress(i64)
struct RollStage {
    float *obs, *rew;
    long long *reset;
    uint8_t *to;
};
__device__ __forceinline__ RollStage roll_stage(float *base, int epb, int O) {
    RollStage t;
    t.obs = base;
    t.rew = t.obs + epb * O;
    t.reset = reinterpret_cast<long long *>(t.rew + epb);
    t.to = reinterpret_cast<uint8_t *>(t.reset + epb);
    return t;
}
// the last step's results as drain_tiles stores them: the per-step tiles of t, the rest in base (obs: the unclipped copy,
// written only when a separate clipped tensor exists)
__device__ __forceinline__ LocoStage roll_last(float *base, const RollStage &t, int epb, int O) {
    LocoStage l;
    l.obs = base; l.obsc = t.obs; l.rew = t.rew; l.reset = t.reset; l.to = t.to;
    l.pot = base + epb * O; l.ppot = l.pot + epb; l.up = l.ppot + epb; l.head = l.up + 3 * epb;
    l.prog = reinterpret_cast<long long *>(l.head + 3 * epb);
    return l;
}
__host__ __device__ inline size_t roll_stage_bytes(int epb, int O) { return (size_t)epb * (O * 4 + 4 + 8 + 1); }
__host__ __device__ inline size_t roll_last_bytes(int epb, int O) { return (size_t)epb * (O * 4 + 4 * 2 + 12 * 2 + 8); }

template <int NS, int SP>
__global__ void __launch_bounds__(64, 7) quad_rollout_kernel(const float4 *__restrict__ gqm, Buffers B, const __grid_constant__ b2g_task_params P,
                                                              int N, int substeps, const __grid_constant__ RollArgs ra) {
    constexpr int BLOCK = 64, EPB = 16, nd = 4 * NS;
    __shared__ alignas(8) uint64_t mbar, mbar2, mbarA[2];
    float4 *const park = b2g_dyn_smem;
    float4 *const qm = b2g_dyn_smem + ra.model_f4;
    float *const io = reinterpret_cast<float *>(b2g_dyn_smem + ra.io_f4);
    float *const stage = reinterpret_cast<float *>(b2g_dyn_smem + ra.stage_f4);
    const int O = P.num_obs, K = ra.K;
    const int nsens6 = O - 12 - 3 * nd;
    const int env0 = blockIdx.x * EPB;
    const TileLayout tl = tile_layout(EPB, nd, nsens6, false, 2);
    float *const s_root = io, *const s_dof = io + tl.dof, *const s_sens = io + tl.sens;
    float *const s_actb[2] = {io + tl.act, io + tl.act + EPB * nd};
    long long *const progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    float *const pot_b = (float *)B.p[B2G_T_POTENTIALS];
    float *const g_obs = (float *)B.p[B2G_T_OBS];
    float *g_obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    if (g_obsc == g_obs) g_obsc = nullptr;
    const bool clip_sep = g_obsc != nullptr;
    const RollStage t = roll_stage(stage, EPB, O);
    const LocoStage l = roll_last(reinterpret_cast<float *>(park), t, EPB, O);
    float *const g_sens = (float *)B.p[B2G_T_FORCE_SENSOR], *const g_dfrc = (float *)B.p[B2G_T_DOF_FORCE];
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int e = gt >> 2, lane = gt & 3;
    const int el = e - env0;
    if (threadIdx.x == 0) { mbar_init(&mbar, 1); mbar_init(&mbar2, 1); mbar_init(&mbarA[0], 1); mbar_init(&mbarA[1], 1); }
    __syncthreads();
    constexpr uint32_t ab = EPB * nd * 4;
    if (threadIdx.x == 0) {
        mbar_expect_tx(&mbar, quad_model_f4(NS) * 16);
        bulk_g2s(qm, gqm, quad_model_f4(NS) * 16, &mbar);
    }
    load_state_tiles<EPB, BLOCK, true, false, false>(&mbar2, io, tl, B, nd, nullptr, env0, TileArgs{});
    if (threadIdx.x == 0) {
        mbar_expect_tx(&mbarA[0], ab);
        bulk_g2s(s_actb[0], ra.actions + (size_t)env0 * nd, ab, &mbarA[0]);
    }
    long long progress = progress_b[e];
    bool do_reset = reset_b[e] != 0;
    float potentials = pot_b[e];
    int *const rc = (int *)B.p[B2G_T_RESET_COUNT];
    uint32_t count = (uint32_t)rc[e];
    const uint32_t count0 = count;
    mbar_wait(&mbar, 0);
    mbar_wait(&mbar2, 0);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    QLane<NS, false, SP> L = make_qlane<NS, false, SP>(qm, nullptr, park, BLOCK, lane);
    attach_env_params(L, B, e, nd);
    float *const row_root = s_root + 13 * el;
    float2 *const row_dof = reinterpret_cast<float2 *>(s_dof + 2 * nd * el);
    RootState rs; load_root(row_root, rs);
    int dofi[NS], sens[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) {
        const float4 k16 = L.LK(s, 16);
        dofi[s] = q_f2i(k16.w); sens[s] = q_f2i(k16.y);
        const float2 v = row_dof[dofi[s]];
        L.q[s] = v.x; L.qd[s] = v.y;
    }
    const int total = P.control_freq_inv * substeps;
    QOutputs o;
    o.write = true;
    o.net_contact = B.p[B2G_T_NET_CONTACT] ? (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * (q_f2i(qm[7].w) >> 8) * 3 : nullptr;
    const bool stage_out = total > 0;
    o.sensor = stage_out ? s_sens + nsens6 * el : (g_sens ? g_sens + (size_t)e * nsens6 : nullptr);
    o.dof_force = g_dfrc ? g_dfrc + (size_t)e * nd : nullptr;
    const float clipo = P.clip_obs;
    const uint32_t gid = (uint32_t)(e + P.env_id_offset);

#pragma unroll 1
    for (int kk = 0; kk < K; kk++) {
        const bool last = kk == K - 1;
        float *const s_act = s_actb[kk & 1];
        if (threadIdx.x == 0 && !last) {                      // next step's actions, one step ahead
            mbar_expect_tx(&mbarA[(kk + 1) & 1], ab);
            bulk_g2s(s_actb[(kk + 1) & 1], ra.actions + ((size_t)(kk + 1) * N + env0) * nd, ab, &mbarA[(kk + 1) & 1]);
        }
        mbar_wait(&mbarA[kk & 1], (uint32_t)((kk >> 1) & 1));
        float *const row_act = s_act + nd * el;
        // ---- VecTask.step :374 clamp ; pre_physics_step (ant.py:281-285)
        float a_cl[NS];
#pragma unroll
        for (int s = 0; s < NS; s++) {
            const float a = fminf(fmaxf(row_act[dofi[s]], -P.clip_actions), P.clip_actions);
            row_act[dofi[s]] = a;
            a_cl[s] = a;
            L.act[s] = a * P.joint_gears[dofi[s]] * P.power_scale;
        }
        // ---- control_freq_inv x gym.simulate
#pragma unroll 1
        for (int k = 0; k < total; k++) L.substep(rs, k == total - 1, o);
        // ---- post_physics_step (ant.py:287-297)
        progress += 1;
        if (do_reset) {                                       // reset_idx, ant.py:252-279
#pragma unroll
            for (int s = 0; s < NS; s++) {
                const float2 qv = loco_reset_dof(P, gid, count, dofi[s], nd);
                L.q[s] = qv.x; L.qd[s] = qv.y;
            }
            potentials = loco_reset_root(P, B, e, rs);
            progress = 0;
            count += 1;
        }
        // the previous step's output stores must have read their staging tiles before these are rewritten
        if ((threadIdx.x & 31) == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncthreads();
        float *const obs = t.obs + (size_t)el * O;            // per-step output tile: the observation step() returns
        float *const obs_raw = l.obs + (size_t)el * O;        // last step only, when a separate unclipped tensor exists
        const float prev_potentials = potentials;
        potentials = loco_potential(P, rs.rp);
        AntRootObs ro;
        LocoCosts cost = ant_obs<NS>(P, rs, L.q, L.qd, dofi, sens, a_cl, qm, lane, s_sens, g_sens, e, el, nsens6, stage_out, ro,
                                     [&](int idx, float v) {
                                         obs[idx] = clip_sep ? fminf(fmaxf(v, -clipo), clipo) : v;
                                         if (last && clip_sep) obs_raw[idx] = v;
                                     });
        cost.sum_lanes<4>();
        // reset / time-out depend on the height and the step count only: every lane of the env knows them (the flag drives
        // the NEXT step's reset_idx on all four lanes)
        const LocoReward r = loco_reward(P, ro.up_proj, ro.heading_proj, potentials, prev_potentials, cost, rs.rp[2], progress, false);
        do_reset = r.died || r.timed;
        if (lane == 0) {
            t.rew[el] = r.rew; t.reset[el] = do_reset ? 1 : 0;
            t.to[el] = r.timed;                                                                             // vec_task.py:394
            if (last) {
                l.pot[el] = potentials; l.ppot[el] = prev_potentials; l.prog[el] = progress;
                l.up[3 * el] = ro.up_vec[0]; l.up[3 * el + 1] = ro.up_vec[1]; l.up[3 * el + 2] = ro.up_vec[2];
                l.head[3 * el] = ro.heading_vec[0]; l.head[3 * el + 1] = ro.heading_vec[1]; l.head[3 * el + 2] = ro.heading_vec[2];
                if (count != count0) rc[e] = (int)count;
            }
        }
        if (last) {
#pragma unroll
            for (int s = 0; s < NS; s++) row_dof[dofi[s]] = make_float2(L.q[s], L.qd[s]);
            if (lane == 0) store_root(row_root, rs);
        }
        fence_async_smem();
        __syncthreads();
        if (last) {
            LocoStage v = l;                                  // without a separate clipped tensor, obs is the per-step tile
            if (!clip_sep) v.obs = t.obs;
            drain_tiles<EPB, BLOCK / 32, false>(B, v, io, tl, s_act, nd, O, nsens6, env0, true, stage_out, false);
        }
        {
            const size_t kN = (size_t)kk * N + env0;
            if (threadIdx.x == 0) {
                bulk_s2g(ra.obs_out + kN * O, t.obs, (uint32_t)(EPB * O * 4));
                bulk_s2g(ra.rew_out + kN, t.rew, EPB * 4);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            } else if (threadIdx.x == 32) {
                bulk_s2g(ra.reset_out + kN, t.reset, EPB * 8);
                if (ra.timeout_out) bulk_s2g(ra.timeout_out + kN, t.to, EPB);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if ((threadIdx.x & 31) == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

}  // namespace b2g

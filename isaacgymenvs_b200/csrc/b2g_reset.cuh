// b2g_reset.cuh -- VecTask.reset_done() (tasks/base/vec_task.py:440-455): `reset_idx(nonzero(reset_buf))` right at
// the call, for callers that reset outside step() (rl_games' env wrapper calls it once before the first rollout).
// The fused step kernels perform the same reset_idx for flagged envs inside the step; these small kernels call the
// step kernels' reset helpers (same Philox stream: seed, global env id, reset count) on their own, one thread per env,
// and clear reset_buf, so the next step finds nothing to reset -- exactly the reference's order of events.
// Observations are NOT recomputed (the reference's reset_idx does not either: obs_buf is refreshed by the next step).
#pragma once
#include "b2g_common.cuh"
#include "b2g_tasks.cuh"
#include "b2g_hand.cuh"

namespace b2g {

// Ant / Humanoid reset_idx (ant.py:252-279, humanoid.py:253-279) and Cartpole reset_idx (cartpole.py:144-157)
__global__ void __launch_bounds__(128) loco_reset_kernel(Buffers B, const __grid_constant__ b2g_task_params P, int N, int nd) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    if (reset_b[e] == 0) return;
    int *const rc = (int *)B.p[B2G_T_RESET_COUNT];
    const uint32_t count = (uint32_t)rc[e], gid = (uint32_t)(e + P.env_id_offset);
    float2 *const dof = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    if (P.task == B2G_TASK_CARTPOLE) {
        for (int s = 0; s < 2; s++) dof[s] = cartpole_reset_dof(P, gid, count, s);
    } else {
        for (int d = 0; d < nd; d++) dof[d] = loco_reset_dof(P, gid, count, d, nd);
        RootState rs;
        const float pot = loco_reset_root(P, B, e, rs);
        store_root((float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
        ((float *)B.p[B2G_T_POTENTIALS])[e] = pot;                       // prev_potentials = potentials = -|to_target| / dt (:273-276)
        ((float *)B.p[B2G_T_PREV_POTENTIALS])[e] = pot;
    }
    ((long long *)B.p[B2G_T_PROGRESS])[e] = 0;
    reset_b[e] = 0;
    rc[e] = (int)(count + 1);
}

// ShadowHand reset_idx incl. its reset_target_pose (shadow_hand.py:594-659) for envs with reset_buf set; goal-only resets
// (reset_goal_buf) stay with the next step's pre_physics_step, as in the reference
__global__ void __launch_bounds__(128) hand_reset_kernel(Buffers B, const __grid_constant__ b2g_hand_params P, int N, int nd) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    if (reset_b[e] == 0) return;
    int *const rc = (int *)B.p[B2G_T_RESET_COUNT];
    const uint32_t count = (uint32_t)rc[e], gid = (uint32_t)(e + P.env_id_offset);
    float *const rows = (float *)B.p[B2G_T_ROOT_STATE] + (size_t)e * 39;
    const float *const init_rows = (const float *)B.p[B2G_T_INITIAL_ROOT] + (size_t)e * 39;
    float *const goal_row = (float *)B.p[B2G_T_GOAL_STATES] + (size_t)e * 13;
    float goal_pos[3], goal_rot[4];
    hand_reset_goal(P, gid, count, nd, false, nullptr, init_rows, goal_row, rows, true, goal_pos, goal_rot);
    ObjState ob;
    hand_reset_obj(P, gid, count, init_rows, ob);
    store_obj(rows + 13, ob);
    float2 *const dof = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    float *const cur_t = (float *)B.p[B2G_T_DOF_TARGET] + (size_t)e * nd, *const prev_t = (float *)B.p[B2G_T_PREV_TARGETS] + (size_t)e * nd;
    for (int d = 0; d < nd; d++) {
        const float2 qv = hand_reset_dof(P, gid, count, d, nd);
        dof[d] = qv; cur_t[d] = qv.x; prev_t[d] = qv.x;
    }
    if (P.force_scale > 0.f) {                                           // rb_forces[env_ids] = 0, new random_force_prob (:616,642)
        float *const of = (float *)B.p[B2G_T_OBJ_FORCE] + 3 * (size_t)e;
        of[0] = of[1] = of[2] = 0.f;
        ((float *)B.p[B2G_T_RANDOM_FORCE_PROB])[e] = hand_force_prob(P, gid, count, nd);
    }
    ((long long *)B.p[B2G_T_PROGRESS])[e] = 0;
    ((float *)B.p[B2G_T_SUCCESSES])[e] = 0.f;
    reset_b[e] = 0;
    ((long long *)B.p[B2G_T_RESET_GOAL])[e] = 0;                         // reset_target_pose clears it (:610)
    rc[e] = (int)(count + 1);
}

}  // namespace b2g

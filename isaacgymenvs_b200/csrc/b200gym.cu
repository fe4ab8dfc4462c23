// b200gym.cu -- kernels + C ABI (include/b200gym.h) of the CUDA-native (H100) environment stepper.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include <memory>

#include "../../include/b200gym.h"
#include "b2g_device.cuh"
#include "b2g_tasks.cuh"
#include "b2g_common.cuh"
#include "b2g_kin_host.h"

using namespace b2g;

// ============================================================================================
// kernels
// ============================================================================================

// whole-struct copy (forward-kinematics kernel, which also reads the cold tables)
__device__ __forceinline__ void load_model_full(DevModel *sm, const DevModel *__restrict__ gm) {
    const uint4 *src = reinterpret_cast<const uint4 *>(gm);
    uint4 *dst = reinterpret_cast<uint4 *>(sm);
    for (int i = threadIdx.x; i < (int)(sizeof(DevModel) / 16); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

template <int L, bool HF, int BLOCK, bool OBJ = false, bool SELF = false, bool DR = false>
__device__ __forceinline__ Stepper<L, HF, BLOCK, OBJ, SELF, DR> make_stepper(const DevModel *sm, const int16_t *hf, int lane) {
    Stepper<L, HF, BLOCK, OBJ, SELF, DR> st;
    st.m = sm; st.gr = Ground{sm, hf, sm->cps, -1.f};
    st.slots = &sm->slots[0][0]; st.links = sm->links;
    if (OBJ) {      // [link][k][env] layout: the env's column
        st.ss = b2g_dyn_smem + threadIdx.x / L;
        st.acc = b2g_dyn_smem + (sm->nl - 1) * SLOT_F4 * Stepper<L, HF, BLOCK, OBJ>::KS + threadIdx.x / L;
    } else {
        st.ss = b2g_dyn_smem + threadIdx.x;
        st.acc = b2g_dyn_smem + sm->ns * SLOT_F4 * BLOCK + threadIdx.x;
    }
    st.lane = lane;
    st.gmodel = nullptr;
    st.dr_mass = nullptr; st.dr_dof = nullptr; st.dr_ten = nullptr; st.dr_grav = nullptr;
    st.scen = nullptr; st.scs = 1;
    if (SELF) {
        if (sm->self_f4) st.scen = b2g_dyn_smem + (sm->ns * SLOT_F4 + sm->nacc * ACC_F4) * BLOCK + (threadIdx.x / L) * sm->self_f4;
        else { st.scen = b2g_dyn_smem + (sm->self_cell & 255) * SLOT_F4 * BLOCK + (threadIdx.x - lane + (sm->self_cell >> 8)); st.scs = BLOCK; }
    }
    return st;
}

// per-env physical parameters (domain randomisation arrays; null = the model's own), any sub-step
template <class ST>
__device__ __forceinline__ void attach_env_params_generic(ST &st, const DevModel &sm, const Buffers &B, int e) {
    const float *ms = (const float *)B.p[B2G_T_ENV_MASS_SCALE];
    const float4 *dp = (const float4 *)B.p[B2G_T_ENV_DOF_PROPS];
    const float *envmu = (const float *)B.p[B2G_T_ENV_FRICTION];
    if (ms) st.dr_mass = ms + (size_t)e * sm.nl;
    if (dp) st.dr_dof = dp + (size_t)e * (sm.nl - 1);
    if (envmu) st.gr.env_mu = 0.5f * (envmu[e] + sm.ground_mu);      // PhysX default combine mode: the average of the two materials
}

// the free object's per-env parameters, the tendon damping and the gravity (the DR instantiations of the free-object kernels;
// null = the model's own).  Frictions combine as PhysX does by default, the average of the two materials: hand (ENV_FRICTION)
// with object (ENV_OBJ_PROPS.z) for their contacts, object with ground for the object's ground contacts.  Where only one of the
// two tensors is bound, the model's object friction obj_mu stands in for the missing material.
template <class ST>
__device__ __forceinline__ void attach_object_params(ST &st, const DevModel &sm, const Buffers &B, int e) {
    const float4 *op = (const float4 *)B.p[B2G_T_ENV_OBJ_PROPS];
    const float *hand_mu = (const float *)B.p[B2G_T_ENV_FRICTION];
    const float *td = (const float *)B.p[B2G_T_ENV_TENDON_DAMPING];
    const float4 v = op ? op[e] : make_float4(1.f, 1.f, sm.obj_mu, 0.f);
    const float mu_h = hand_mu ? hand_mu[e] : sm.obj_mu;
    st.set_obj_params(v.x, v.y, (op || hand_mu) ? 0.5f * (mu_h + v.z) : sm.obj_mu, op ? 0.5f * (v.z + sm.ground_mu) : sm.obj_mu);
    if (td) st.dr_ten = td + (size_t)e * sm.nten;
    st.dr_grav = (const float *)B.p[B2G_T_GRAVITY];
}

template <class ST>
__device__ __forceinline__ typename ST::Outputs make_outputs(const DevModel &sm, const Buffers &B, int e, bool valid) {
    typename ST::Outputs o;
    const int nd = sm.nl - 1;
    float *fs = (float *)B.p[B2G_T_FORCE_SENSOR], *df = (float *)B.p[B2G_T_DOF_FORCE], *nc = (float *)B.p[B2G_T_NET_CONTACT];
    o.sensor = fs ? fs + (size_t)e * sm.nsens * 6 : nullptr;
    o.dof_force = df ? df + (size_t)e * nd : nullptr;
    o.net_contact = nc ? nc + (size_t)e * sm.nb * 3 : nullptr;
    o.write = valid;
    return o;
}

// -------------------------------------------------------------------------------------------
// gym.simulate(): physics only
template <int L, bool HF, int BLOCK, bool OBJ = false, bool SELF = false, bool DR = false>
__global__ void __launch_bounds__(BLOCK) simulate_kernel(const DevModel *__restrict__ gm, const int16_t *__restrict__ hf,
                                                         Buffers B, int N) {
    __shared__ DevModel sm;
    __shared__ alignas(8) uint64_t mbar;
    load_model_hot(&sm, &mbar, gm);
    using ST = Stepper<L, HF, BLOCK, OBJ, SELF, DR>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const int nd = sm.nl - 1, NS = sm.ns;
    ST st = make_stepper<L, HF, BLOCK, OBJ, SELF, DR>(&sm, hf, lane);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
    if (DR) attach_object_params(st, sm, B, e);
    float *const root_row = (float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e * sm.root_stride;
    RootState rs; load_root(root_row, rs);
    ObjState ob;
    if (OBJ) {
        load_obj(root_row + 13 * sm.obj_row, ob);
        const float *of = (const float *)B.p[B2G_T_OBJ_FORCE];
        if (of) st.set_obj_force(of[3 * (size_t)e], of[3 * (size_t)e + 1], of[3 * (size_t)e + 2]);
        else st.set_obj_force(0.f, 0.f, 0.f);
    }
    const float2 *d = (const float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    const float *act = (const float *)B.p[B2G_T_DOF_ACTUATION];
    const float *tgt = (const float *)B.p[B2G_T_DOF_TARGET];
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int link = st.link_of(s);
        if (link < 0) continue;
        const float2 v = d[link - 1];
        const float *src = (sm.links[link].flags & LF_POSDRIVE) ? tgt : act;
        st.set_joint(s, v.x, v.y, src ? src[(size_t)e * nd + link - 1] : 0.f);
    }
    const typename ST::Outputs o = make_outputs<ST>(sm, B, e, valid);
    for (int k = 0; k < sm.substeps; k++) st.substep(rs, k == sm.substeps - 1, o, &ob);
    if (!valid) return;
    float2 *dw = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
#pragma unroll 1
    for (int s = 0; s < NS; s++) { const int link = st.link_of(s); if (link >= 0) dw[link - 1] = st.get_q(s); }
    if (lane == 0 && !sm.root_fixed) store_root(root_row, rs);
    if (OBJ && lane == 0) store_obj(root_row + 13 * sm.obj_row, ob);
}

// -------------------------------------------------------------------------------------------
// One whole VecTask.step() of Ant / Humanoid (vec_task.py:360-408 + ant.py:281-297 / humanoid.py)
//
// Data movement: with whole 16-byte-aligned tiles per block (TILES) every tensor of the step moves as ONE bulk-async
// copy per block (the tile helpers of b2g_common.cuh); the output tiles are staged in the shared memory that held the
// slot state during the physics.  Without tiles the kernel reads and writes the tensors directly.
#ifndef B2G_MINBLOCKS
#define B2G_MINBLOCKS 4
#endif

// DR: the sub-steps read a bound gravity vector (B2G_T_GRAVITY; the Humanoid's sim_params.gravity randomisation), a separate
// instantiation chosen at run time when the tensor is bound
template <int L, bool HF, bool HUM, int BLOCK, bool TILES, bool HOSTIO = false, bool SELF = false, bool DR = false>
__global__ void __launch_bounds__(BLOCK, (BLOCK == 128 ? B2G_MINBLOCKS : (BLOCK == 64 && !HUM ? 2 * B2G_MINBLOCKS : 1))) loco_step_kernel(
    const DevModel *__restrict__ gm, const int16_t *__restrict__ hf, Buffers B, const __grid_constant__ b2g_task_params P,
    const float *__restrict__ actions_in, int N, TileArgs ta) {
    __shared__ alignas(8) uint64_t mbar;
    // the model's hot part, packed: header | links[0..nl) | cps[0..ncp)
    DevModel &sm = *reinterpret_cast<DevModel *>(b2g_dyn_smem + ta.model_f4);
    constexpr int EPB = BLOCK / L;
    const int nd = P.num_actions;                       // == dofs for the locomotion tasks (checked by b2g_set_task)
    const int O = P.num_obs;
    const int env0 = blockIdx.x * EPB;
    constexpr bool tiles = TILES;
    float *const io = reinterpret_cast<float *>(b2g_dyn_smem + ta.io_f4);
    const int nsens6 = 6 * ((P.num_obs - 12 - (HUM ? 4 : 3) * nd) / 6);          // 6 * nsens, from the obs layout
    const TileLayout tl = tile_layout(EPB, nd, nsens6, HUM);
    float *const s_root = io, *const s_dof = io + tl.dof, *const s_act = io + tl.act, *const s_sens = io + tl.sens, *const s_dfrc = io + tl.dfrc;
    // ---- prologue: barrier set-up and the bulk copy of the (constant) model before griddepcontrol.wait, the state tiles
    // and per-env scalars after it
    __shared__ alignas(8) uint64_t mbar2;
    long long *const progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    float *const pot_b = (float *)B.p[B2G_T_POTENTIALS], *const ppot_b = (float *)B.p[B2G_T_PREV_POTENTIALS];
    const int e_pre = min((int)((blockIdx.x * BLOCK + threadIdx.x) / L), N - 1);
    if (threadIdx.x == 0) { mbar_init(&mbar, 1); mbar_init(&mbar2, 1); }
    __syncthreads();
    if (threadIdx.x == 0) {
        const ModelHot h = model_hot_bytes(gm->ns, gm->nl, gm->ncp);   // three scalar loads; everything else arrives by bulk copy
        mbar_expect_tx(&mbar, h.total());
        bulk_g2s(&sm, gm, h.head, &mbar);                                  // header | slots[0..ns)
        char *const pk = reinterpret_cast<char *>(&sm) + h.head;           // links and cps packed right behind
        bulk_g2s(pk, gm->links, h.links, &mbar);
        if (h.cps) bulk_g2s(pk + h.links, gm->cps, h.cps, &mbar);
    }
    load_state_tiles<EPB, BLOCK, TILES, HOSTIO>(&mbar2, io, tl, B, nd, actions_in, env0, ta);
    // per-env scalars of post_physics_step: issued now, consumed after the physics
    const long long progress_in = progress_b[e_pre];
    const long long reset_in = reset_b[e_pre];
    const float potentials_in = pot_b[e_pre];
    mbar_wait(&mbar, 0);
    if (tiles) mbar_wait(&mbar2, 0);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");       // the next step's grid may begin its own prologue
    using ST = Stepper<L, HF, BLOCK, false, SELF, DR>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const int el = e - env0;                             // env index inside this block's tiles
    const int NS = sm.ns;
    ST st = make_stepper<L, HF, BLOCK, false, SELF, DR>(&sm, hf, lane);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
    if (DR) st.dr_grav = (const float *)B.p[B2G_T_GRAVITY];
    {
        // model_hot_bytes's layout with 64-bit offset arithmetic: its 32-bit form costs the Humanoid DR instantiations registers
        const char *pk = reinterpret_cast<const char *>(&sm) + offsetof(DevModel, slots) + (size_t)sm.ns * MAX_LANES * sizeof(SlotRec);
        st.links = reinterpret_cast<const LinkC *>(pk);
        st.gr.cps = reinterpret_cast<const CpC *>(pk + round16((uint32_t)sm.nl * (uint32_t)sizeof(LinkC)));
    }

    // this env's rows: shared-memory tiles, or the tensors themselves
    float *const row_root = tiles ? s_root + 13 * el : (float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e;
    float2 *const row_dof = reinterpret_cast<float2 *>(tiles ? s_dof + 2 * nd * el : (float *)B.p[B2G_T_DOF_STATE] + 2 * (size_t)nd * e);
    const float *const row_act_in = tiles ? s_act + nd * el : actions_in + (size_t)nd * e;
    float *const g_act_out = (float *)B.p[B2G_T_ACTIONS];
    float *const row_act_out = tiles ? s_act + nd * el : (g_act_out ? g_act_out + (size_t)nd * e : nullptr);
    float *const g_sens = (float *)B.p[B2G_T_FORCE_SENSOR], *const g_dfrc = (float *)B.p[B2G_T_DOF_FORCE];

    RootState rs; load_root(row_root, rs);

    // ---- VecTask.step :374 clamp ; pre_physics_step (ant.py:281-285 / humanoid.py:281-285)
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int d = st.link_of(s) - 1;
        if (d < 0) continue;
        const float2 v = row_dof[d];
        const float a = fminf(fmaxf(row_act_in[d], -P.clip_actions), P.clip_actions);
        if (valid && row_act_out) row_act_out[d] = a;   // in tile mode this overwrites the raw action in place
        st.set_joint(s, v.x, v.y, a * (HUM ? P.motor_efforts[d] : P.joint_gears[d]) * P.power_scale);
    }

    // ---- control_freq_inv x gym.simulate (vec_task.py:379-382).  control_freq_inv == 0: no simulate --
    // the observation then reads the sensor / joint-force tensors as they stand (what refresh_*_tensor
    // would return); used to pin the observation/reward arithmetic against the reference's golden vectors
    const int total = P.control_freq_inv * sm.substeps;
    typename ST::Outputs o;
    o.write = valid;
    o.net_contact = B.p[B2G_T_NET_CONTACT] ? (float *)B.p[B2G_T_NET_CONTACT] + (size_t)e * sm.nb * 3 : nullptr;
    const bool stage_out = tiles && total > 0;           // sensor / dof-force tiles are produced by the physics
    o.sensor = stage_out ? s_sens + nsens6 * el : (g_sens ? g_sens + (size_t)e * nsens6 : nullptr);
    o.dof_force = (stage_out && HUM) ? s_dfrc + nd * el : (g_dfrc ? g_dfrc + (size_t)e * nd : nullptr);
    for (int k = 0; k < total; k++) st.substep(rs, k == total - 1, o);

    // ---- post_physics_step (ant.py:287-297): progress, reset_idx, observations, reward
    long long progress = progress_in + 1;
    float potentials = potentials_in;
    const bool do_reset = reset_in != 0;
    // final joint state -> dof rows (reset_idx, ant.py:252-279 / humanoid.py:253-279, overrides it)
    uint32_t count = 0;
    int *rc = (int *)B.p[B2G_T_RESET_COUNT];
    if (do_reset) count = (uint32_t)rc[e];
    const uint32_t gid = (uint32_t)(e + P.env_id_offset);
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int d = st.link_of(s) - 1;
        if (d < 0) continue;
        float2 qv = st.get_q(s);
        if (do_reset) qv = loco_reset_dof(P, gid, count, d, nd);
        if (valid) row_dof[d] = qv;
    }
    if (do_reset) {
        potentials = loco_reset_root(P, B, e, rs);
        progress = 0;
        if (valid && lane == 0) rc[e] = (int)(count + 1);
    }
    if (valid && lane == 0 && !sm.root_fixed) store_root(row_root, rs);

    // the slot state is dead from here on: its shared memory becomes the output staging area
    __syncthreads();
    float *const g_obs = (float *)B.p[B2G_T_OBS];
    float *g_obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    if (g_obsc == g_obs) g_obsc = nullptr;
    const LocoStage t = loco_stage(reinterpret_cast<float *>(b2g_dyn_smem), EPB, O, g_obsc != nullptr);
    float *const obs = tiles ? t.obs + (size_t)el * O : g_obs + (size_t)e * O;
    float *const obsc = g_obsc ? (tiles ? t.obsc + (size_t)el * O : g_obsc + (size_t)e * O) : nullptr;

    // compute_observations
    LocoRootObs ro;
    loco_root_obs(P, rs.rp, rs.rq, rs.rv, rs.rw, HUM, ro);
    const float prev_potentials = potentials;     // prev_potentials_new = potentials.clone(), ant.py:390
    potentials = ro.potentials;
    const float clipo = P.clip_obs;
    auto put = [&](int idx, float v) {
        if (!valid) return;
        obs[idx] = v;
        if (obsc) obsc[idx] = fminf(fmaxf(v, -clipo), clipo);
    };
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 12; c++) put(c, ro.o[c]);
    }
    // layout: ant.py:401-406  [12 | nd pos | nd vel | 24 sensors | nd actions]
    //    humanoid.py:407-411  [12 | nd pos | nd vel | nd dof_force | 12 sensors | nd actions]
    const int o_pos = 12, o_vel = 12 + nd, o_frc = 12 + 2 * nd;
    const int o_sens = HUM ? 12 + 3 * nd : 12 + 2 * nd;
    const int o_act = o_sens + nsens6;
    LocoCosts cost;
#pragma unroll 1
    for (int s = 0; s < NS; s++) {
        const int link = st.link_of(s), d = link - 1;
        if (link < 0) continue;
        const float2 qv = row_dof[d];
        const float a = tiles ? row_act_out[d] : fminf(fmaxf(row_act_in[d], -P.clip_actions), P.clip_actions);
        const float ps = t_unscale(qv.x, P.dof_limits_lower[d], P.dof_limits_upper[d]);
        const float vs = qv.y * P.dof_vel_scale;
        put(o_pos + d, ps); put(o_vel + d, vs); put(o_act + d, a);
        if (HUM) put(o_frc + d, (o.dof_force ? o.dof_force[d] : 0.f) * P.contact_force_scale);
        const int sk = st.links[link].sensor;
        if (sk >= 0 && o.sensor) {
#pragma unroll
            for (int c = 0; c < 6; c++) put(o_sens + 6 * sk + c, o.sensor[6 * sk + c] * P.contact_force_scale);
        }
        cost.add(P, d, a, ps, vs, HUM);
    }
    if (lane == 0 && st.links[0].sensor >= 0 && o.sensor) {
        const int sk = st.links[0].sensor;
#pragma unroll
        for (int c = 0; c < 6; c++) put(o_sens + 6 * sk + c, o.sensor[6 * sk + c] * P.contact_force_scale);
    }
    cost.sum_lanes<L>();

    if (valid && lane == 0) {
        const LocoReward r = loco_reward(P, ro.o[10], ro.o[11], potentials, prev_potentials, cost, ro.o[0], progress, HUM);
        const float total_r = r.rew;
        const long long reset = (r.died || r.timed) ? 1 : 0;
        const uint8_t tout = r.timed;
        float *uv = (float *)B.p[B2G_T_UP_VEC], *hv = (float *)B.p[B2G_T_HEADING_VEC];
        uint8_t *to = (uint8_t *)B.p[B2G_T_TIMEOUT];
        if (tiles) {
            stage_row(t, el, total_r, r.died || r.timed, progress, potentials, prev_potentials, ro.up_vec, ro.heading_vec, r.timed);
        } else {
            ((float *)B.p[B2G_T_REW])[e] = total_r;
            reset_b[e] = reset; progress_b[e] = progress;
            pot_b[e] = potentials; ppot_b[e] = prev_potentials;
            if (uv) { uv[3 * e] = ro.up_vec[0]; uv[3 * e + 1] = ro.up_vec[1]; uv[3 * e + 2] = ro.up_vec[2]; }
            if (hv) { hv[3 * e] = ro.heading_vec[0]; hv[3 * e + 1] = ro.heading_vec[1]; hv[3 * e + 2] = ro.heading_vec[2]; }
            if (to) to[e] = tout;
        }
    }
    if (tiles) {
        fence_async_smem();
        __syncthreads();
        // one issuing thread, as before: dealt across the warps, the Humanoid step measured no faster (H100, 700 W)
        drain_tiles<EPB, 1, HUM>(B, t, io, tl, s_act, nd, O, nsens6, env0, !sm.root_fixed, stage_out, true);
        if (HOSTIO) loco_copy_to_host<BLOCK>(ta, t, (size_t)env0, EPB, O, g_obsc != nullptr);
    }
}

// -------------------------------------------------------------------------------------------
// One whole VecTask.step() of Cartpole (cartpole.py:131-163)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) cartpole_step_kernel(const DevModel *__restrict__ gm, Buffers B,
                                                              const __grid_constant__ b2g_task_params P,
                                                              const float *__restrict__ actions_in, int N) {
    __shared__ DevModel sm;
    __shared__ alignas(8) uint64_t mbar;
    load_model_hot(&sm, &mbar, gm);
    using ST = Stepper<1, false, BLOCK>;
    const int env = blockIdx.x * BLOCK + threadIdx.x;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    ST st = make_stepper<1, false, BLOCK>(&sm, nullptr, 0);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
    RootState rs; load_root((const float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e, rs);
    const float2 *dofs = (const float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * 2;
    const float a = fminf(fmaxf(actions_in[e], -P.clip_actions), P.clip_actions);
    st.set_joint(0, dofs[0].x, dofs[0].y, a * P.max_push_effort);   // cartpole.py:159-163: effort on DOF 0 only
    st.set_joint(1, dofs[1].x, dofs[1].y, 0.f);
    typename ST::Outputs o; o.sensor = nullptr; o.dof_force = nullptr; o.net_contact = nullptr; o.write = false;
    const int total = P.control_freq_inv * sm.substeps;
    for (int k = 0; k < total; k++) st.substep(rs, false, o);
    long long *progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *reset_b = (long long *)B.p[B2G_T_RESET];
    long long progress = progress_b[e] + 1;
    if (reset_b[e] != 0) {   // reset_idx, cartpole.py:144-157
        int *rc = (int *)B.p[B2G_T_RESET_COUNT];
        const uint32_t count = (uint32_t)rc[e], gid = (uint32_t)(e + P.env_id_offset);
#pragma unroll
        for (int s = 0; s < 2; s++) { const float2 qv = cartpole_reset_dof(P, gid, count, s); st.set_q(s, qv.x, qv.y); }
        progress = 0;
        if (valid) rc[e] = (int)(count + 1);
    }
    if (!valid) return;
    const float2 q0 = st.get_q(0), q1 = st.get_q(1);
    float2 *dw = (float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * 2;
    dw[0] = q0; dw[1] = q1;
    float *act_out = (float *)B.p[B2G_T_ACTIONS];
    if (act_out) act_out[e] = a;
    // compute_observations, cartpole.py:131-142
    const float ob[4] = {q0.x, q0.y, q1.x, q1.y};
    float *obs = (float *)B.p[B2G_T_OBS] + 4 * (size_t)e;
    float *obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    obsc = (obsc && obsc != (float *)B.p[B2G_T_OBS]) ? obsc + 4 * (size_t)e : nullptr;
#pragma unroll
    for (int c = 0; c < 4; c++) { obs[c] = ob[c]; if (obsc) obsc[c] = fminf(fmaxf(ob[c], -P.clip_obs), P.clip_obs); }
    float rew; long long reset = 0;
    cartpole_reward(q1.x, q1.y, q0.y, q0.x, P.reset_dist, progress, P.max_episode_length, rew, reset);
    ((float *)B.p[B2G_T_REW])[e] = rew;
    reset_b[e] = reset; progress_b[e] = progress;
    uint8_t *to = (uint8_t *)B.p[B2G_T_TIMEOUT];
    if (to) to[e] = (uint8_t)(((float)progress >= P.max_episode_length - 1.f) && reset != 0);
}

#include "b2g_anymal.cuh"
#include "b2g_hand.cuh"
#include "b2g_quad_kernels.cuh"
#include "b2g_model_host.h"
#include "b2g_reset.cuh"
#include "b2g_quad_rollout.cuh"

// -------------------------------------------------------------------------------------------
// gym.refresh_rigid_body_state_tensor(): forward kinematics, one thread per env, any topology
__global__ void __launch_bounds__(128) body_state_kernel(const DevModel *__restrict__ gm, Buffers B, int N) {
    __shared__ DevModel sm;
    load_model_full(&sm, gm);
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    const int nl = sm.nl, nd = nl - 1;
    float R[MAX_LINKS][9], x[MAX_LINKS][3], wv[MAX_LINKS][3], lv[MAX_LINKS][3];
    const float *r = (const float *)B.p[B2G_T_ROOT_STATE] + 13 * (size_t)e * sm.root_stride;
    const float q0[4] = {r[3], r[4], r[5], r[6]};
    quat_to_mat(q0, R[0]);
    for (int c = 0; c < 3; c++) { x[0][c] = r[c]; lv[0][c] = sm.root_fixed ? 0.f : r[7 + c]; wv[0][c] = sm.root_fixed ? 0.f : r[10 + c]; }
    const float2 *d = (const float2 *)B.p[B2G_T_DOF_STATE] + (size_t)e * nd;
    for (int i = 1; i < nl; i++) {
        const LinkC &lk = sm.links[i];
        const int p = sm.link_parent[i];
        const float2 qv = d[i - 1];
        float Rt[9], ax[3] = {lk.axis[0], lk.axis[1], lk.axis[2]}, w[3], lp[3] = {lk.lpos[0], lk.lpos[1], lk.lpos[2]}, dd[3], wxd[3];
        matmul(R[p], lk.R0, Rt); matvec(Rt, ax, w);
        if (!(lk.flags & LF_SLIDE)) {
            float sn, cs; sincosf(qv.x, &sn, &cs);
            const float oc = 1.f - cs;
            for (int j = 0; j < 3; j++) {
                float col[3] = {Rt[j], Rt[3 + j], Rt[6 + j]}, wxc[3];
                cross(w, col, wxc);
                const float wd = dot3(w, col) * oc;
                R[i][j] = col[0] * cs + wxc[0] * sn + w[0] * wd;
                R[i][3 + j] = col[1] * cs + wxc[1] * sn + w[1] * wd;
                R[i][6 + j] = col[2] * cs + wxc[2] * sn + w[2] * wd;
            }
            matvec(R[p], lp, dd);
        } else {
            for (int c = 0; c < 9; c++) R[i][c] = Rt[c];
            matvec(R[p], lp, dd);
            for (int c = 0; c < 3; c++) dd[c] += w[c] * qv.x;
        }
        cross(wv[p], dd, wxd);
        for (int c = 0; c < 3; c++) {
            x[i][c] = x[p][c] + dd[c];
            lv[i][c] = lv[p][c] + wxd[c] + ((lk.flags & LF_SLIDE) ? w[c] * qv.y : 0.f);
            wv[i][c] = wv[p][c] + ((lk.flags & LF_SLIDE) ? 0.f : w[c] * qv.y);
        }
    }
    // bodies of an env: the articulation's, then one per further actor (single rigid bodies: their root rows)
    const int nb_env = sm.nb + sm.root_stride - 1;
    float *bs = (float *)B.p[B2G_T_RIGID_BODY_STATE] + 13 * (size_t)e * nb_env;
    for (int a = 1; a < sm.root_stride; a++)
        for (int c = 0; c < 13; c++) bs[13 * (sm.nb + a - 1) + c] = r[13 * a + c];
    for (int b = 0; b < sm.nb; b++) {
        const int i = sm.body_link[b];
        float bp[3] = {sm.body_pos[b][0], sm.body_pos[b][1], sm.body_pos[b][2]}, wb[3], wxb[3], Rb[9], Rwb[9], q[4];
        matvec(R[i], bp, wb); cross(wv[i], wb, wxb);
        quat_to_mat(sm.body_quat[b], Rb); matmul(R[i], Rb, Rwb); mat_to_quat(Rwb, q);
        float *o = bs + 13 * b;
        for (int c = 0; c < 3; c++) { o[c] = x[i][c] + wb[c]; o[7 + c] = lv[i][c] + wxb[c]; o[10 + c] = wv[i][c]; }
        o[3] = q[0]; o[4] = q[1]; o[5] = q[2]; o[6] = q[3];
    }
}

// ============================================================================================
// host side
// ============================================================================================
struct b2g_sim : SimModel {
    int device = 0;
    int num_envs = 0;
    DevModel *dm = nullptr;      // device copy of hm
    int16_t *d_hf = nullptr;
    float4 *d_qm = nullptr;      // device copy of qm
    KinModel *d_kin = nullptr;   // device copy of hk
    Buffers buf = {};
    size_t buf_bytes[B2G_T_COUNT] = {};
    b2g_task_params task;
    b2g_anymal_params anymal;
    b2g_hand_params hand;
    HandDev hand_dev;
    bool has_task = false, has_anymal = false, has_hand = false;
    unsigned step_counter = 0;   // common_step_counter, anymal_terrain.py:459
    float *d_actions_stage = nullptr;    // device staging for b2g_task_step_host
    int64_t launches = 0;
    std::vector<const void *> smem_set;      // kernels whose dynamic shared-memory limit has been raised (once per sim)

    b2g_sim() = default;
    b2g_sim(const b2g_sim &) = delete;
    b2g_sim &operator=(const b2g_sim &) = delete;
    ~b2g_sim() {
        cudaSetDevice(device);
        for (void *p : {(void *)dm, (void *)d_hf, (void *)d_qm, (void *)d_kin, (void *)d_actions_stage}) if (p) cudaFree(p);
    }
};

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }
#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(B2G_E_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

extern "C" const char *b2g_last_error(void) { return g_err.c_str(); }
extern "C" int b2g_version(void) { return B2G_VERSION; }
extern "C" int64_t b2g_launch_count(const b2g_sim *sim) { return sim ? sim->launches : 0; }
extern "C" int b2g_quad_chain_length(const b2g_sim *sim) { return sim ? sim->quad_ns : 0; }

static_assert(B2G_PLAN_MAX_SLOTS == MAX_SLOTS && B2G_PLAN_MAX_LANES == MAX_LANES, "plan table size");
extern "C" int b2g_plan(const b2g_model *m, int32_t lanes, int32_t compact, int32_t *slots_out, int32_t info_out[5]) {
    if (!m || !slots_out || !info_out) return fail(B2G_E_INVALID, "b2g_plan: null argument");
    if (m->nl < 1 || m->nl > MAX_LINKS || m->nl - 1 > MAX_SLOTS) return fail(B2G_E_INVALID, "b2g_plan: model exceeds compiled limits");
    if (lanes != 0 && lanes != 1 && lanes != 2 && lanes != 4 && lanes != 8) return fail(B2G_E_INVALID, "b2g_plan: lanes must be 0, 1, 2, 4 or 8");
    DevModel *h = new DevModel();
    memset(h, 0, sizeof(*h));
    const int L = lanes ? lanes : pick_lanes(m, false);
    const int rc = schedule(m, L, *h, compact != 0);
    if (rc != 0) { delete h; return fail(B2G_E_INVALID, "b2g_plan: the articulation does not fit the slot program limits"); }
    for (int sl = 0; sl < MAX_SLOTS; sl++) for (int l = 0; l < MAX_LANES; l++) {
        const SlotRec &r = h->slots[sl][l];
        int32_t *o = slots_out + 8 * (sl * MAX_LANES + l);
        o[0] = r.link; o[1] = r.parent; o[2] = r.out; o[3] = r.flags;
        for (int c = 0; c < MAX_CHILD_REFS; c++) o[4 + c] = r.child[c];
    }
    info_out[0] = h->ns; info_out[1] = h->lanes; info_out[2] = h->nacc; info_out[3] = h->root_acc; info_out[4] = h->cross_lane;
    delete h;
    return B2G_OK;
}

extern "C" int b2g_create(const b2g_model *m, const b2g_sim_params *sp, int32_t num_envs, int32_t device, b2g_sim **out) {
    return b2g_create_ext(m, nullptr, sp, num_envs, device, out);
}

extern "C" int b2g_create_ext(const b2g_model *m, const b2g_model_ext *ext, const b2g_sim_params *sp, int32_t num_envs, int32_t device,
                              b2g_sim **out) {
    if (!m || !sp || !out || num_envs <= 0) return fail(B2G_E_INVALID, "b2g_create: null argument or num_envs <= 0");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
        return fail(B2G_E_CUDA, std::string("b2g_create: no CUDA device (there is no CPU fallback): ") + cudaGetErrorString(ce));
    CUDA_TRY(cudaSetDevice(device));
    std::unique_ptr<b2g_sim> s(new b2g_sim());
    s->device = device; s->num_envs = num_envs;
    // the reference paths the tests compare with: B2G_SINGLE_LANE=1 one thread per env, B2G_NO_QUAD=1 the generic Stepper
    const char *single = getenv("B2G_SINGLE_LANE"), *no_quad = getenv("B2G_NO_QUAD");
    const char *err = "";
    const int rc = build_sim_model(m, ext, sp, single && single[0] == '1', no_quad && no_quad[0] == '1', *s, &err);
    if (rc != B2G_OK) return fail(rc, err);
    if (sp->hf_samples) {
        const size_t bytes = (size_t)sp->hf_nx * sp->hf_ny * sizeof(int16_t);
        CUDA_TRY(cudaMalloc(&s->d_hf, bytes));
        CUDA_TRY(cudaMemcpy(s->d_hf, sp->hf_samples, bytes, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMalloc(&s->dm, sizeof(DevModel)));
    CUDA_TRY(cudaMemcpy(s->dm, &s->hm, sizeof(DevModel), cudaMemcpyHostToDevice));
    if (s->kin_ok) {
        CUDA_TRY(cudaMalloc(&s->d_kin, sizeof(KinModel)));
        CUDA_TRY(cudaMemcpy(s->d_kin, &s->hk, sizeof(KinModel), cudaMemcpyHostToDevice));
    }
    if (s->quad_ns) {
        CUDA_TRY(cudaMalloc(&s->d_qm, s->qm.size() * sizeof(float)));
        CUDA_TRY(cudaMemcpy(s->d_qm, s->qm.data(), s->qm.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    *out = s.release();
    return B2G_OK;
}

extern "C" int b2g_destroy(b2g_sim *s) {
    delete s;
    return B2G_OK;
}

extern "C" int b2g_bind(b2g_sim *s, int32_t slot, void *ptr, size_t bytes) {
    if (!s || slot < 0 || slot >= B2G_T_COUNT) return fail(B2G_E_INVALID, "b2g_bind: bad slot");
    const int N = s->num_envs, nd = s->hm.nl - 1, nb = s->hm.nb, ns = s->hm.nsens;
    size_t need = 0;
    switch (slot) {
        case B2G_T_ROOT_STATE: case B2G_T_INITIAL_ROOT: need = (size_t)N * s->hm.root_stride * 13 * 4; break;
        case B2G_T_DOF_STATE: need = (size_t)N * nd * 8; break;
        case B2G_T_DOF_ACTUATION: case B2G_T_DOF_TARGET: case B2G_T_DOF_FORCE: need = (size_t)N * nd * 4; break;
        case B2G_T_RIGID_BODY_STATE: need = (size_t)N * (nb + s->hm.root_stride - 1) * 13 * 4; break;
        case B2G_T_FORCE_SENSOR: need = (size_t)N * ns * 6 * 4; break;
        case B2G_T_NET_CONTACT: need = (size_t)N * nb * 3 * 4; break;
        case B2G_T_GOAL_STATES: need = (size_t)N * 13 * 4; break;
        case B2G_T_PREV_TARGETS: need = (size_t)N * nd * 4; break;
        case B2G_T_SUCCESSES: case B2G_T_GOAL_RESET_COUNT: need = (size_t)N * 4; break;
        case B2G_T_CONSECUTIVE_SUCCESSES: need = 16; break;
        case B2G_T_RESET_GOAL: need = (size_t)N * 8; break;
        case B2G_T_REW: case B2G_T_POTENTIALS: case B2G_T_PREV_POTENTIALS: case B2G_T_RESET_COUNT: need = (size_t)N * 4; break;
        case B2G_T_RESET: case B2G_T_PROGRESS: need = (size_t)N * 8; break;
        case B2G_T_TIMEOUT: need = (size_t)N; break;
        case B2G_T_UP_VEC: case B2G_T_HEADING_VEC: need = (size_t)N * 12; break;
        case B2G_T_ENV_MASS_SCALE: need = (size_t)N * (nd + 1) * 4; break;
        case B2G_T_ENV_DOF_PROPS: need = (size_t)N * nd * 16; break;
        case B2G_T_ENV_FRICTION: need = (size_t)N * 4; break;
        case B2G_T_OBJ_FORCE: need = (size_t)N * 12; break;
        case B2G_T_RANDOM_FORCE_PROB: need = (size_t)N * 4; break;
        case B2G_T_ENV_OBJ_PROPS: need = (size_t)N * 16; break;
        case B2G_T_ENV_TENDON_DAMPING: need = (size_t)N * s->hm.nten * 4; break;
        case B2G_T_GRAVITY: need = 12; break;
        case B2G_T_JACOBIAN: need = (size_t)N * s->hk.rows * 6 * s->hk.nc * 4; break;
        case B2G_T_MASS_MATRIX: need = (size_t)N * s->hk.nc * s->hk.nc * 4; break;
        default: need = 0; break;   // ACTIONS / OBS / OBS_CLIPPED are checked against the task in b2g_set_task
    }
    if (ptr && bytes < need) return fail(B2G_E_INVALID, "b2g_bind: buffer smaller than the tensor's layout requires");
    if ((slot == B2G_T_ENV_OBJ_PROPS || slot == B2G_T_ENV_TENDON_DAMPING) && !s->hm.obj_on)
        return fail(B2G_E_UNSUPPORTED, "b2g_bind: object and tendon parameters need a sim with a free object");
    s->buf.p[slot] = ptr; s->buf_bytes[slot] = bytes;
    return B2G_OK;
}

static int require(const b2g_sim *s, std::initializer_list<int> slots, const char *who) {
    for (int k : slots) if (!s->buf.p[k]) return fail(B2G_E_UNBOUND, std::string(who) + ": tensor slot " + std::to_string(k) + " is not bound");
    return B2G_OK;
}

// A bound gravity vector (B2G_T_GRAVITY) is read by the free-object DR kernels and the Humanoid's gravity instantiations
// only: every other physics launch refuses it rather than step under the model's gravity
static int refuse_gravity(const b2g_sim *s, const std::string &who) {
    if (!s->buf.p[B2G_T_GRAVITY]) return B2G_OK;
    return fail(B2G_E_UNSUPPORTED, who + ": no kernel of this combination reads a bound GRAVITY vector; unbind it or use a sim whose "
                                         "kernels read it (a free object, or the Humanoid task)");
}

// the action and observation counts of the task set on the sim
static void task_sizes(const b2g_sim *s, int *n_act, int *n_obs) {
    if (s->has_anymal) { *n_act = s->anymal.num_actions; *n_obs = s->anymal.num_obs; }
    else if (s->has_hand) { *n_act = s->hand.num_actions; *n_obs = s->hand.num_obs; }
    else { *n_act = s->task.num_actions; *n_obs = s->task.num_obs; }
}

// Whole tiles for the bulk-copy step kernels: the envs fill whole CTAs of `epb`, and every per-env tile of a CTA, down to
// the one-byte time-out flags, is a whole number of 16-byte units (epb % 16 == 0 covers every wider row as well)
static bool whole_tiles(size_t N, int epb) { return N % epb == 0 && epb % 16 == 0; }

// ---------------------------------------------------------------------------------------------------------------------
// launches

// raise a kernel's dynamic shared-memory limit, once per (sim, kernel): the attribute call costs microseconds of host
// time, comparable to a whole step when issued before every launch
template <typename K>
static int set_smem(b2g_sim *s, K kernel, size_t bytes) {
    const void *key = reinterpret_cast<const void *>(kernel);
    for (const void *k : s->smem_set) if (k == key) return B2G_OK;
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024 > (int)bytes ? 200 * 1024 : (int)bytes));
    s->smem_set.push_back(key);
    return B2G_OK;
}

// PLAIN: as is.  SMEM: raise the kernel's dynamic shared-memory limit first (set_smem; the attribute can also change the
// shared-memory carveout, so only the kernels that size their shared memory at run time ask for it).  SMEM_PDL: and let the
// grid start while the previous kernel in the stream drains (programmatic dependent launch: the kernel's griddepcontrol.wait).
enum LaunchMode { PLAIN, SMEM, SMEM_PDL };

template <typename... P, typename... A>
static int launch(b2g_sim *s, void (*kernel)(P...), int grid, int block, size_t dyn, cudaStream_t st, LaunchMode mode, A... args) {
    if (mode != PLAIN) { const int rc = set_smem(s, kernel, dyn); if (rc) return rc; }
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(grid); lc.blockDim = dim3(block); lc.dynamicSmemBytes = dyn; lc.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    if (mode == SMEM_PDL) { lc.attrs = at; lc.numAttrs = 1; }
    CUDA_TRY(cudaLaunchKernelEx(&lc, kernel, args...));
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Instantiation lists: one function per kernel family maps the runtime key to the compiled instantiation, null when there
// is none; every instantiation the library contains is listed once.  The kernels are compiled in the order they are first
// named, so the lists keep the order the entry points have always named them in: quad simulate, simulate, (Jacobian),
// ShadowHand, AnymalTerrain, (Cartpole), quad locomotion, locomotion, (rollout).
static constexpr int key(int lanes, int block) { return (lanes << 8) | block; }

// gym.simulate() on the quad sub-step: (chain length, height field, specialisation, link-link contact); 128 threads, one
// env per 4.  A self-colliding model is packed for chain length 3 in the general layout (quad_build)
constexpr int QUAD_SIM_BLOCK = 128;
using QuadSimKernel = void (*)(const float4 *, const int16_t *, Buffers, int, int);
static QuadSimKernel quad_simulate_kernel_for(int ns, bool hf, int spec, bool self) {
    constexpr int B = QUAD_SIM_BLOCK;
    const bool sp3 = spec == 3;
    if (!self) {
        if (ns == 2 && !hf) return sp3 ? quad_simulate_kernel<2, false, 3, B> : quad_simulate_kernel<2, false, 0, B>;
        if (ns == 2) return sp3 ? quad_simulate_kernel<2, true, 3, B> : quad_simulate_kernel<2, true, 0, B>;
        if (ns == 3 && !hf) return sp3 ? quad_simulate_kernel<3, false, 3, B> : quad_simulate_kernel<3, false, 0, B>;
        if (ns == 3) return sp3 ? quad_simulate_kernel<3, true, 3, B> : quad_simulate_kernel<3, true, 0, B>;
        return nullptr;
    }
    if (ns != 3 || spec != 0) return nullptr;
    return hf ? quad_simulate_kernel<3, true, 0, B, true> : quad_simulate_kernel<3, false, 0, B, true>;
}

// gym.simulate() on the generic Stepper: (lanes, CTA size, height field, free object, self-collision, per-env physical
// parameters of the free-object sim bound)
using SimulateKernel = void (*)(const DevModel *, const int16_t *, Buffers, int);
static SimulateKernel simulate_kernel_for(int lanes, int block, bool hf, bool obj, bool self, bool dr) {
    if (obj && !dr) {            // the free object (b2g_create_ext keeps it on the ground plane)
        switch (key(lanes, block)) {
            case key(8, 128): return simulate_kernel<8, false, 128, true>;
            case key(8, 64): return simulate_kernel<8, false, 64, true>;
            case key(4, 128): return simulate_kernel<4, false, 128, true>;
            case key(4, 64): return simulate_kernel<4, false, 64, true>;
            case key(4, 32): return simulate_kernel<4, false, 32, true>;
            case key(1, 32): return simulate_kernel<1, false, 32, true>;
        }
        return nullptr;
    }
    if (self) {                  // link-link contact, on the ground plane
        if (hf) return nullptr;
        switch (key(lanes, block)) {
            case key(4, 128): return simulate_kernel<4, false, 128, false, true>;
            case key(4, 64): return simulate_kernel<4, false, 64, false, true>;
            case key(4, 32): return simulate_kernel<4, false, 32, false, true>;
            case key(1, 64): return simulate_kernel<1, false, 64, false, true>;
            case key(1, 32): return simulate_kernel<1, false, 32, false, true>;
        }
        return nullptr;
    }
    if (!obj) {
        if (hf && key(lanes, block) != key(4, 128)) return nullptr;      // the height field: 4 lanes, 128 threads
        switch (key(lanes, block)) {
            case key(4, 128): return !hf ? simulate_kernel<4, false, 128> : simulate_kernel<4, true, 128>;
            case key(4, 64): return simulate_kernel<4, false, 64>;
            case key(4, 32): return simulate_kernel<4, false, 32>;
            case key(2, 128): return simulate_kernel<2, false, 128>;
            case key(2, 64): return simulate_kernel<2, false, 64>;
            case key(2, 32): return simulate_kernel<2, false, 32>;
            case key(1, 128): return simulate_kernel<1, false, 128>;
            case key(1, 64): return simulate_kernel<1, false, 64>;
            case key(1, 32): return simulate_kernel<1, false, 32>;
        }
        return nullptr;
    }
    // the free object with per-env physical parameters: the hand's 4 lanes, 128 threads
    return key(lanes, block) == key(4, 128) ? simulate_kernel<4, false, 128, true, false, true> : nullptr;
}

// a free-object sim with any per-env physical parameter bound runs the DR instantiation of its kernels
static bool object_dr_bound(const b2g_sim *s) {
    if (!s->hm.obj_on) return false;
    for (int k : {B2G_T_ENV_MASS_SCALE, B2G_T_ENV_DOF_PROPS, B2G_T_ENV_FRICTION, B2G_T_ENV_OBJ_PROPS, B2G_T_ENV_TENDON_DAMPING, B2G_T_GRAVITY})
        if (s->buf.p[k]) return true;
    return false;
}

// ---------------------------------------------------------------------------------------------------------------------

extern "C" int b2g_simulate(b2g_sim *s, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "b2g_simulate: null sim");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE}, "b2g_simulate"); if (rc) return rc;
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int N = s->num_envs;
    if (!s->hm.obj_on) { rc = refuse_gravity(s, "b2g_simulate(sim without a free object)"); if (rc) return rc; }
    if (s->quad_ns) {
        const bool self = s->hm.self_on != 0;
        const size_t dyn = ((size_t)quad_park_f4(s->quad_ns, self) * QUAD_SIM_BLOCK + quad_model_f4(s->quad_ns, self)) * sizeof(float4);
        return launch(s, quad_simulate_kernel_for(s->quad_ns, s->d_hf != nullptr, s->quad_spec, self), (N * 4 + QUAD_SIM_BLOCK - 1) / QUAD_SIM_BLOCK,
                      QUAD_SIM_BLOCK, dyn, st, SMEM, s->d_qm, s->d_hf, s->buf, N, s->hm.substeps);
    }
    const int blk = s->block, grid = (N * s->lanes + blk - 1) / blk;
    const SimulateKernel k = simulate_kernel_for(s->lanes, blk, s->d_hf != nullptr, s->hm.obj_on, s->hm.self_on, object_dr_bound(s));
    if (!k) return fail(B2G_E_UNSUPPORTED, "no simulate kernel instantiated for this (lanes, CTA size, terrain, free object, self-collision, randomised) combination");
    return launch(s, k, grid, blk, s->dyn_smem, st, SMEM, s->dm, s->d_hf, s->buf, N);
}

extern "C" int b2g_refresh_rigid_body_state(b2g_sim *s, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "null sim");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_RIGID_BODY_STATE}, "b2g_refresh_rigid_body_state"); if (rc) return rc;
    CUDA_TRY(cudaSetDevice(s->device));
    const int N = s->num_envs;
    return launch(s, body_state_kernel, (N + 127) / 128, 128, 0, (cudaStream_t)stream, PLAIN, s->dm, s->buf, N);
}

extern "C" int b2g_kin_shape(const b2g_sim *s, int32_t shape_out[2]) {
    if (!s || !shape_out) return fail(B2G_E_INVALID, "b2g_kin_shape: null argument");
    if (!s->kin_ok) return fail(B2G_E_UNSUPPORTED, "b2g_kin_shape: articulation exceeds the kernel's limits");
    shape_out[0] = s->hk.rows; shape_out[1] = s->hk.nc;
    return B2G_OK;
}

extern "C" int b2g_refresh_kinematic_tensors(b2g_sim *s, int32_t which, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "null sim");
    if (!s->kin_ok) return fail(B2G_E_UNSUPPORTED, "b2g_refresh_kinematic_tensors: articulation exceeds the kernel's limits");
    if (!(which & (B2G_KIN_JACOBIAN | B2G_KIN_MASS_MATRIX))) return fail(B2G_E_INVALID, "b2g_refresh_kinematic_tensors: nothing selected");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE}, "b2g_refresh_kinematic_tensors"); if (rc) return rc;
    if (which & B2G_KIN_JACOBIAN) { rc = require(s, {B2G_T_JACOBIAN}, "b2g_refresh_kinematic_tensors"); if (rc) return rc; }
    if (which & B2G_KIN_MASS_MATRIX) { rc = require(s, {B2G_T_MASS_MATRIX}, "b2g_refresh_kinematic_tensors"); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(s->device));
    const int N = s->num_envs;
    constexpr int WARPS = 4;
    const float *root = (const float *)s->buf.p[B2G_T_ROOT_STATE], *dof = (const float *)s->buf.p[B2G_T_DOF_STATE];
    float *J = (which & B2G_KIN_JACOBIAN) ? (float *)s->buf.p[B2G_T_JACOBIAN] : nullptr;
    float *M = (which & B2G_KIN_MASS_MATRIX) ? (float *)s->buf.p[B2G_T_MASS_MATRIX] : nullptr;
    // one warp per env -- or per two envs when links and bodies fit 16 lanes (arms, quadrupeds); at most a few resident waves of
    // CTAs, the warps stride over the envs
    int sms = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (s->hk.nl <= 16 && s->hk.nb <= 16)
        return launch(s, kin_tensors_kernel<WARPS, 16>, std::min((N + 2 * WARPS - 1) / (2 * WARPS), sms * 8), WARPS * 32, 0, st, PLAIN,
                      s->d_kin, root, dof, J, M, N);
    return launch(s, kin_tensors_kernel<WARPS, 32>, std::min((N + WARPS - 1) / WARPS, sms * 8), WARPS * 32, 0, st, PLAIN,
                  s->d_kin, root, dof, J, M, N);
}

extern "C" int b2g_set_task(b2g_sim *s, const b2g_task_params *t) {
    if (!s || !t) return fail(B2G_E_INVALID, "b2g_set_task: null argument");
    const int nd = s->hm.nl - 1;
    if (t->task == B2G_TASK_CARTPOLE) {
        if (s->hm.nl != 3 || !s->hm.root_fixed || t->num_obs != 4 || t->num_actions != 1) return fail(B2G_E_UNSUPPORTED, "cartpole task needs the 2-DOF fixed-base chain, 4 obs, 1 action");
    } else if (t->task == B2G_TASK_ANT) {
        if (t->num_actions != nd || t->num_obs != 12 + 3 * nd + 6 * s->hm.nsens) return fail(B2G_E_UNSUPPORTED, "ant task: observation size does not match the articulation");
    } else if (t->task == B2G_TASK_HUMANOID) {
        if (t->num_actions != nd || t->num_obs != 12 + 4 * nd + 6 * s->hm.nsens) return fail(B2G_E_UNSUPPORTED, "humanoid task: observation size does not match the articulation");
    } else return fail(B2G_E_UNSUPPORTED, "b2g_set_task: unknown task id");
    if (t->control_freq_inv < 0) return fail(B2G_E_INVALID, "control_freq_inv < 0");
    if (s->hm.root_stride != 1) return fail(B2G_E_UNSUPPORTED, "b2g_set_task: single-actor environments only");
    s->task = *t; s->has_task = true; s->has_anymal = false; s->has_hand = false;
    return B2G_OK;
}

extern "C" int b2g_set_anymal_task(b2g_sim *s, const b2g_anymal_params *t) {
    if (!s || !t) return fail(B2G_E_INVALID, "b2g_set_anymal_task: null argument");
    const int nd = s->hm.nl - 1;
    if (s->lanes != 4 || s->hm.ns != 3 || nd != 12 || t->num_actions != 12 || t->num_obs != 12 + 3 * nd + 140)
        return fail(B2G_E_UNSUPPORTED, "AnymalTerrain needs the 4-leg x 3-DOF articulation, 12 actions, 188 observations");
    if (t->decimation < 0 || t->control_freq_inv < 0) return fail(B2G_E_INVALID, "negative simulate count");
    if (s->hm.root_stride != 1) return fail(B2G_E_UNSUPPORTED, "b2g_set_anymal_task: single-actor environments only");
    s->anymal = *t; s->has_anymal = true; s->has_task = false; s->has_hand = false; s->step_counter = 0;
    return B2G_OK;
}

extern "C" int b2g_set_hand_task(b2g_sim *s, const b2g_hand_params *t) {
    if (!s || !t) return fail(B2G_E_INVALID, "b2g_set_hand_task: null argument");
    const DevModel &h = s->hm;
    const int nd = h.nl - 1;
    if (!h.obj_on || h.root_stride != 3 || h.obj_row != 1 || !h.root_fixed)
        return fail(B2G_E_UNSUPPORTED, "ShadowHand needs a fixed-base articulation created with b2g_create_ext: actors hand, object, goal");
    if (t->num_actions < 1 || t->num_actions > nd || h.nsens != 5) return fail(B2G_E_UNSUPPORTED, "ShadowHand: 1..dofs actions and 5 fingertip force sensors expected");
    if (t->control_freq_inv < 0) return fail(B2G_E_INVALID, "control_freq_inv < 0");
    HandDev H; memset(&H, 0, sizeof(H));
    for (int d = 0; d < MAX_LINKS; d++) H.dof_action[d] = -1;
    for (int k = 0; k < t->num_actions; k++) {
        const int d = t->actuated_dof[k];
        if (d < 0 || d >= nd || H.dof_action[d] >= 0) return fail(B2G_E_INVALID, "ShadowHand: bad actuated_dof table");
        H.dof_action[d] = k;
    }
    for (int f = 0; f < 5; f++) {
        const int b = t->fingertip_body[f];
        if (b < 0 || b >= h.nb || h.sensor_body[f] != b) return fail(B2G_E_INVALID, "ShadowHand: fingertip bodies must be the five force-sensor bodies, in order");
        const int ref = slot_of_link(h, h.body_link[b]);
        if (ref < 0) return fail(B2G_E_UNSUPPORTED, "ShadowHand: a fingertip rides on the root link");
        H.ft_ref[f] = ref;
        for (int c = 0; c < 3; c++) H.ft_bpos[f][c] = h.body_pos[b][c];
        host_quat_to_mat(h.body_quat[b], H.ft_bR[f]);
    }
    // observation layouts, shadow_hand.py:460-592
    const int A = t->num_actions;
    auto layout = [&](int type, HandDev::Layout &Y) -> int {
        Y.o_dofpos = Y.o_dofvel = Y.o_dofforce = Y.o_objpose = Y.o_objvel = Y.o_goalpose = Y.o_sens = -1; Y.n_objpose = 0;
        switch (type) {
            case B2G_HAND_OBS_OPENAI:      Y.o_ft = 0; Y.ft_stride = 3; Y.o_objpose = 15; Y.n_objpose = 3; Y.o_qdiff = 18; Y.o_act = 22; return 22 + A;
            case B2G_HAND_OBS_FULL_NO_VEL: Y.o_dofpos = 0; Y.o_objpose = nd; Y.n_objpose = 7; Y.o_goalpose = nd + 7; Y.o_qdiff = nd + 14; Y.o_ft = nd + 18; Y.ft_stride = 3;
                                           Y.o_act = nd + 33; return nd + 33 + A;
            case B2G_HAND_OBS_FULL:        Y.o_dofpos = 0; Y.o_dofvel = nd; Y.o_objpose = 2 * nd; Y.n_objpose = 7; Y.o_objvel = 2 * nd + 7; Y.o_goalpose = 2 * nd + 13;
                                           Y.o_qdiff = 2 * nd + 20; Y.o_ft = 2 * nd + 24; Y.ft_stride = 13; Y.o_act = 2 * nd + 89; return 2 * nd + 89 + A;
            case B2G_HAND_OBS_FULL_STATE:  Y.o_dofpos = 0; Y.o_dofvel = nd; Y.o_dofforce = 2 * nd; Y.o_objpose = 3 * nd; Y.n_objpose = 7; Y.o_objvel = 3 * nd + 7;
                                           Y.o_goalpose = 3 * nd + 13; Y.o_qdiff = 3 * nd + 20; Y.o_ft = 3 * nd + 24; Y.ft_stride = 13; Y.o_sens = 3 * nd + 89;
                                           Y.o_act = 3 * nd + 119; return 3 * nd + 119 + A;
            default: return -1;
        }
    };
    const int expect = layout(t->obs_type, H.lay[0]);
    if (expect < 0) return fail(B2G_E_INVALID, "ShadowHand: unknown observation type");
    const int expect_states = layout(B2G_HAND_OBS_FULL_STATE, H.lay[1]);
    if (t->num_states != 0 && t->num_states != expect_states) return fail(B2G_E_UNSUPPORTED, "ShadowHand: num_states must be 0 or the full_state size");
    H.num_states = t->num_states;
    if (t->num_obs != expect) return fail(B2G_E_UNSUPPORTED, "ShadowHand: observation size does not match the layout of this observation type");
    s->hand = *t; s->hand_dev = H; s->has_hand = true; s->has_task = false; s->has_anymal = false;
    return B2G_OK;
}

// the fused ShadowHand step: (lanes, CTA size, per-env physical parameters bound)
using HandKernel = void (*)(const DevModel *, Buffers, b2g_hand_params, HandDev, const float *, int);
static HandKernel hand_kernel_for(int lanes, int block, bool dr) {
    if (!dr) {
        switch (key(lanes, block)) {
            case key(8, 128): return hand_step_kernel<8, 128>;
            case key(8, 64): return hand_step_kernel<8, 64>;
            case key(4, 128): return hand_step_kernel<4, 128>;
            case key(4, 64): return hand_step_kernel<4, 64>;
            case key(4, 32): return hand_step_kernel<4, 32>;
            case key(1, 32): return hand_step_kernel<1, 32>;
        }
        return nullptr;
    }
    return key(lanes, block) == key(4, 128) ? hand_step_kernel<4, 128, true> : nullptr;     // the hand's 4 lanes, 128 threads
}

static int hand_step(b2g_sim *s, const float *actions, void *stream) {
    const b2g_hand_params &P = s->hand;
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_DOF_TARGET, B2G_T_OBS, B2G_T_REW, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT,
                         B2G_T_INITIAL_ROOT, B2G_T_GOAL_STATES, B2G_T_PREV_TARGETS, B2G_T_SUCCESSES, B2G_T_CONSECUTIVE_SUCCESSES,
                         B2G_T_RESET_GOAL, B2G_T_GOAL_RESET_COUNT}, "b2g_task_step(ShadowHand)");
    if (rc) return rc;
    if (s->hand_dev.lay[0].o_sens >= 0 || s->hand_dev.num_states > 0) { rc = require(s, {B2G_T_FORCE_SENSOR, B2G_T_DOF_FORCE}, "b2g_task_step(ShadowHand, full_state)"); if (rc) return rc; }
    if (s->hand_dev.num_states > 0) {
        rc = require(s, {B2G_T_STATES}, "b2g_task_step(ShadowHand, asymmetric observations)"); if (rc) return rc;
        if (s->buf_bytes[B2G_T_STATES] < (size_t)s->num_envs * s->hand_dev.num_states * 4) return fail(B2G_E_INVALID, "STATES buffer too small");
    }
    if (P.force_scale > 0.f) { rc = require(s, {B2G_T_OBJ_FORCE, B2G_T_RANDOM_FORCE_PROB}, "b2g_task_step(ShadowHand, forceScale > 0)"); if (rc) return rc; }
    const size_t N = s->num_envs;
    if (s->buf_bytes[B2G_T_OBS] < N * P.num_obs * 4) return fail(B2G_E_INVALID, "OBS buffer too small");
    CUDA_TRY(cudaSetDevice(s->device));
    const int blk = s->block, grid = ((int)N * s->lanes + blk - 1) / blk;
    const HandKernel k = hand_kernel_for(s->lanes, blk, object_dr_bound(s));
    if (!k) return fail(B2G_E_UNSUPPORTED, "no ShadowHand kernel instantiated for this (lanes, CTA size, randomised) combination");
    return launch(s, k, grid, blk, s->dyn_smem, (cudaStream_t)stream, SMEM, s->dm, s->buf, P, s->hand_dev, actions, (int)N);
}

// AnymalTerrain physics (the first of its two kernels): the quad sub-step when the model is on the quad path (on a height
// field with or without per-env physical parameters; with link-link contact when the model self-collides), else the
// generic Stepper; plane or height field.  128 threads.
static int launch_anymal_physics(b2g_sim *s, const b2g_anymal_params &P, const float *actions, int N, int grid, cudaStream_t st) {
    const bool hf = s->d_hf != nullptr, self = s->hm.self_on != 0;
    if (s->quad_ns == 3) {
        const bool dr = s->buf.p[B2G_T_ENV_MASS_SCALE] || s->buf.p[B2G_T_ENV_DOF_PROPS];
        auto k = hf ? (dr ? quad_anymal_physics_kernel<true, 128, true> : quad_anymal_physics_kernel<true, 128, false>) : quad_anymal_physics_kernel<false, 128>;
        if (self) k = hf ? quad_anymal_physics_kernel<true, 128, true, true> : quad_anymal_physics_kernel<false, 128, true, true>;
        const size_t dyn = ((size_t)quad_park_f4(3, self) * 128 + quad_model_f4(3, self)) * sizeof(float4);
        return launch(s, k, grid, 128, dyn, st, SMEM, s->d_qm, s->d_hf, s->buf, P, actions, N, s->hm.substeps, s->step_counter);
    }
    // the generic AnymalTerrain kernel has no link-link contact: never drop it silently
    if (self) return fail(B2G_E_UNSUPPORTED, "b2g_task_step(AnymalTerrain): link-link contact needs the four-chain kernels (unset B2G_NO_QUAD)");
    const auto k = hf ? anymal_physics_kernel<true> : anymal_physics_kernel<false>;
    return launch(s, k, grid, 128, s->dyn_smem, st, SMEM, s->dm, s->d_hf, s->buf, P, actions, N, s->step_counter);
}

static int anymal_step(b2g_sim *s, const float *actions, void *stream) {
    const b2g_anymal_params &P = s->anymal;
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_OBS, B2G_T_REW, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT,
                         B2G_T_ACTIONS, B2G_T_NET_CONTACT, B2G_T_COMMANDS, B2G_T_LAST_ACTIONS, B2G_T_LAST_DOF_VEL, B2G_T_FEET_AIR_TIME,
                         B2G_T_TORQUES, B2G_T_EPISODE_SUMS, B2G_T_BASE_SCRATCH, B2G_T_REDUCE_SCRATCH, B2G_T_NOISE_SCALE},
                     "b2g_task_step(AnymalTerrain)");
    if (rc) return rc;
    if (P.custom_origins) { rc = require(s, {B2G_T_ENV_ORIGINS, B2G_T_TERRAIN_LEVELS, B2G_T_TERRAIN_TYPES, B2G_T_TERRAIN_ORIGINS}, "b2g_task_step(AnymalTerrain)"); if (rc) return rc; }
    rc = refuse_gravity(s, "b2g_task_step(AnymalTerrain)"); if (rc) return rc;
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int N = s->num_envs, grid = (N * 4 + 127) / 128;
    if (s->block != 128) return fail(B2G_E_UNSUPPORTED, "AnymalTerrain: unexpected CTA size");
    if (grid > REDUCE_PARTIALS) return fail(B2G_E_INVALID, "AnymalTerrain: too many blocks for the reduction scratch (num_envs <= 32768)");
    if (s->buf_bytes[B2G_T_REDUCE_SCRATCH] < (REDUCE_PARTIALS + 48) * 4) return fail(B2G_E_INVALID, "REDUCE_SCRATCH too small");
    s->step_counter++;                                   // common_step_counter += 1 (:459) before the push test
    rc = launch_anymal_physics(s, P, actions, N, grid, st); if (rc) return rc;
    // kernel 2: one WARP per env -- the 140-point height gather (anymal_terrain.py:515-538) and the 188 observation
    // stores dominate it; with 4 lanes per env the 4096-env workload was 512 warps on 592 schedulers
    return launch(s, anymal_reset_obs_kernel, (N * 32 + 127) / 128, 128, 0, st, PLAIN,
                  s->buf, P, s->d_hf, N, s->hm.nl - 1, grid, s->step_counter, 0);
}

// b2g_task_step_host with pinned host buffers: the step kernel reads its actions from host memory and writes what
// VecTask.step returns straight to these buffers
struct HostOut {
    float *obs, *rew;
    long long *reset;
    uint8_t *timeout;
};

static TileArgs tile_args(size_t io_bytes_at, size_t model_bytes_at, const float *actions, const HostOut *io) {
    TileArgs ta;
    ta.io_f4 = (int)(io_bytes_at / 16); ta.model_f4 = (int)(model_bytes_at / 16);
    ta.h_act = io ? actions : nullptr;
    ta.h_obs = io ? io->obs : nullptr; ta.h_rew = io ? io->rew : nullptr; ta.h_reset = io ? io->reset : nullptr; ta.h_timeout = io ? io->timeout : nullptr;
    return ta;
}

// the locomotion step lists, defined behind task_step (see "Instantiation lists")
constexpr int QUAD_LOCO_BLOCK = 64;
using QuadLocoKernel = void (*)(const float4 *, Buffers, b2g_task_params, const float *, int, int, TileArgs);
using LocoKernel = void (*)(const DevModel *, const int16_t *, Buffers, b2g_task_params, const float *, int, TileArgs);
static QuadLocoKernel quad_loco_kernel_for(int spec, bool hostio, bool lean);
static LocoKernel loco_kernel_for(int lanes, int block, bool hum, bool tiles, bool hostio, bool self, bool grav);
static LocoKernel loco_gravity_kernel_for(int lanes, int block, bool hum, bool tiles, bool hostio, bool self);

// One VecTask.step(); io: the pinned host buffers the Ant / Humanoid step kernel writes to itself (null: device I/O)
static int task_step(b2g_sim *s, const float *actions, void *stream, const HostOut *io) {
    if (!s || !actions) return fail(B2G_E_INVALID, "b2g_task_step: null argument");
    if (s->has_anymal) return anymal_step(s, actions, stream);
    if (s->has_hand) return hand_step(s, actions, stream);
    if (!s->has_task) return fail(B2G_E_INVALID, "b2g_task_step: call b2g_set_task first");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_OBS, B2G_T_REW, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT}, "b2g_task_step");
    if (rc) return rc;
    const b2g_task_params &P = s->task;
    const size_t N = s->num_envs;
    if (s->buf_bytes[B2G_T_OBS] < N * P.num_obs * 4) return fail(B2G_E_INVALID, "OBS buffer too small");
    if (s->buf.p[B2G_T_ACTIONS] && s->buf_bytes[B2G_T_ACTIONS] < N * P.num_actions * 4) return fail(B2G_E_INVALID, "ACTIONS buffer too small");
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int blk = s->block, grid = ((int)N * s->lanes + blk - 1) / blk;
    if (P.task == B2G_TASK_CARTPOLE) {
        rc = refuse_gravity(s, "b2g_task_step(Cartpole)"); if (rc) return rc;
        if (blk != 128) return fail(B2G_E_UNSUPPORTED, "cartpole: unexpected CTA size");
        return launch(s, cartpole_step_kernel<128>, grid, blk, s->dyn_smem, st, SMEM, s->dm, s->buf, P, actions, (int)N);
    }
    rc = require(s, {B2G_T_POTENTIALS, B2G_T_PREV_POTENTIALS, B2G_T_INITIAL_ROOT}, "b2g_task_step"); if (rc) return rc;
    const bool hum = P.task == B2G_TASK_HUMANOID, grav = s->buf.p[B2G_T_GRAVITY] != nullptr;
    if (!hum) { rc = refuse_gravity(s, "b2g_task_step(Ant)"); if (rc) return rc; }
    const int O = P.num_obs, ns6 = 6 * s->hm.nsens;
    const bool clip_sep = s->buf.p[B2G_T_OBS_CLIPPED] && s->buf.p[B2G_T_OBS_CLIPPED] != s->buf.p[B2G_T_OBS];
    if (!hum && s->quad_ns == 2 && !s->d_hf) {           // Ant on the quad sub-step (whole tiles only)
        constexpr int EPB = QUAD_LOCO_BLOCK / 4, ND = 8;
        const size_t park_bytes = (size_t)quad_park_f4(2) * QUAD_LOCO_BLOCK * sizeof(float4);
        const size_t io_bytes = tile_layout(EPB, ND, ns6, false).bytes;
        if (whole_tiles(N, EPB) && loco_stage_bytes(EPB, O, clip_sep) <= park_bytes) {
            const size_t dyn = park_bytes + io_bytes + (size_t)quad_model_f4(2) * sizeof(float4);
            const bool lean = !s->buf.p[B2G_T_ENV_MASS_SCALE] && !s->buf.p[B2G_T_ENV_DOF_PROPS] && !s->buf.p[B2G_T_ENV_FRICTION] &&
                              !s->buf.p[B2G_T_NET_CONTACT] && !s->buf.p[B2G_T_DOF_FORCE];
            return launch(s, quad_loco_kernel_for(s->quad_spec, io != nullptr, lean), (int)N / EPB, QUAD_LOCO_BLOCK, dyn, st, SMEM_PDL,
                          (const float4 *)s->d_qm, s->buf, P, actions, (int)N, (int)s->hm.substeps,
                          tile_args(park_bytes, park_bytes + io_bytes, actions, io));
        }
    }
    if (s->d_hf) return fail(B2G_E_UNSUPPORTED, "locomotion tasks run on the ground plane");
    // tiles by bulk copy: whole blocks only, every tile a multiple of 16 bytes at a 16-byte-aligned address
    const int epb = blk / s->lanes, ndof = s->hm.nl - 1;
    const size_t state_bytes = s->dyn_smem;                                   // slot state + accumulators
    const size_t io_bytes = tile_layout(epb, ndof, ns6, hum).bytes;
    const bool tiles = whole_tiles(N, epb) && loco_stage_bytes(epb, O, clip_sep) <= state_bytes && s->buf.p[B2G_T_ACTIONS];
    const size_t model_bytes = model_hot_bytes(s->hm.ns, s->hm.nl, s->hm.ncp).total();
    const size_t io_used = tiles ? io_bytes : 16;
    const size_t dyn = state_bytes + io_used + model_bytes;
    const LocoKernel k = loco_kernel_for(s->lanes, blk, hum, tiles, io != nullptr, s->hm.self_on, grav);
    if (!k) {
        char what[160];
        snprintf(what, sizeof(what), "(lanes %d, CTA size %d, %s, tiles %d, host I/O %d, self-collision %d, gravity bound %d)", s->lanes, blk,
                 hum ? "Humanoid" : "Ant", (int)tiles, (int)(io != nullptr), (int)(s->hm.self_on != 0), (int)grav);
        return fail(B2G_E_UNSUPPORTED, std::string("no locomotion step kernel instantiated for this combination ") + what);
    }
    return launch(s, k, grid, blk, dyn, st, SMEM_PDL, (const DevModel *)s->dm, (const int16_t *)s->d_hf, s->buf, P, actions, (int)N,
                  tile_args(state_bytes, state_bytes + io_used, actions, io));
}

// the fused Ant step on the quad sub-step: (specialisation, host I/O, lean); 64 threads, 16 envs per CTA.  Lean: the plain
// task (no per-env physical parameters, no dof-force / net-contact tensors acquired), device or staged I/O
static QuadLocoKernel quad_loco_kernel_for(int spec, bool hostio, bool lean) {
    constexpr int B = QUAD_LOCO_BLOCK;
    const bool sp3 = spec == 3;
    if (hostio) return sp3 ? quad_loco_kernel<2, 3, B, true> : quad_loco_kernel<2, 0, B, true>;
    if (lean) return sp3 ? quad_loco_kernel<2, 3, B, false, true> : quad_loco_kernel<2, 0, B, false, true>;
    return sp3 ? quad_loco_kernel<2, 3, B, false> : quad_loco_kernel<2, 0, B, false>;
}

// the fused Ant / Humanoid step on the generic Stepper (ground plane): (lanes, CTA size, Humanoid, tiles, host I/O,
// self-collision, gravity bound).  Host I/O needs the tiles; self-collision runs 4-lane Humanoid-type tasks with device or
// staged I/O.
static LocoKernel loco_kernel_for(int lanes, int block, bool hum, bool tiles, bool hostio, bool self, bool grav) {
    if (hostio && !tiles) return nullptr;
    if (grav) return loco_gravity_kernel_for(lanes, block, hum, tiles, hostio, self);
    if (self) {
        if (!hum || lanes != 4 || hostio) return nullptr;
        if (block == 64) return tiles ? loco_step_kernel<4, false, true, 64, true, false, true> : loco_step_kernel<4, false, true, 64, false, false, true>;
        if (block == 32) return tiles ? loco_step_kernel<4, false, true, 32, true, false, true> : loco_step_kernel<4, false, true, 32, false, false, true>;
        return nullptr;
    }
#define LOCO_IO(L, HUM, B) (tiles ? (hostio ? loco_step_kernel<L, false, HUM, B, true, true> : loco_step_kernel<L, false, HUM, B, true, false>) \
                                  : loco_step_kernel<L, false, HUM, B, false, false>)
    if (!hum) {
        switch (key(lanes, block)) {
            case key(4, 128): return LOCO_IO(4, false, 128);
            case key(4, 64): return LOCO_IO(4, false, 64);
            case key(1, 128): return LOCO_IO(1, false, 128);
        }
        return nullptr;
    }
    switch (key(lanes, block)) {
        case key(4, 128): return LOCO_IO(4, true, 128);
        case key(4, 64): return LOCO_IO(4, true, 64);
        case key(4, 32): return LOCO_IO(4, true, 32);
        case key(2, 64): return LOCO_IO(2, true, 64);
        case key(2, 32): return LOCO_IO(2, true, 32);
        case key(1, 64): return LOCO_IO(1, true, 64);
        case key(1, 32): return LOCO_IO(1, true, 32);
    }
#undef LOCO_IO
    return nullptr;
}

// the Humanoid step reading a bound gravity vector: the Humanoid's own 4 lanes and 64 threads, with and without link-link
// contact (the reference's collision filter 0), device or staged I/O
static LocoKernel loco_gravity_kernel_for(int lanes, int block, bool hum, bool tiles, bool hostio, bool self) {
    if (!hum || hostio || key(lanes, block) != key(4, 64)) return nullptr;
    if (self) return tiles ? loco_step_kernel<4, false, true, 64, true, false, true, true> : loco_step_kernel<4, false, true, 64, false, false, true, true>;
    return tiles ? loco_step_kernel<4, false, true, 64, true, false, false, true> : loco_step_kernel<4, false, true, 64, false, false, false, true>;
}

extern "C" int b2g_task_step(b2g_sim *s, const float *actions, void *stream) { return task_step(s, actions, stream, nullptr); }

// K x VecTask.step() with the actions of all K steps given up front (open-loop / random-action rollouts)
extern "C" int b2g_task_rollout(b2g_sim *s, const float *actions, int32_t K, float *obs_out, float *rew_out, int64_t *reset_out,
                                uint8_t *timeout_out, void *stream) {
    if (!s || !actions || !obs_out || !rew_out || !reset_out || K < 1) return fail(B2G_E_INVALID, "b2g_task_rollout: null argument or K < 1");
    if (!s->has_task && !s->has_anymal && !s->has_hand) return fail(B2G_E_INVALID, "b2g_task_rollout: call b2g_set_task first");
    const size_t N = s->num_envs;
    constexpr int QB = 64, EPB = 16;
    // (a bound gravity vector takes the single-step path, whose Ant step refuses it)
    const bool fused = s->has_task && s->task.task == B2G_TASK_ANT && s->quad_ns == 2 && !s->d_hf && whole_tiles(N, EPB) && !s->buf.p[B2G_T_GRAVITY];
    cudaStream_t st = (cudaStream_t)stream;
    if (!fused) {
        // every other task / shape: K single steps, their results copied into the (K, N, .) outputs (same semantics, no fusion)
        int A, O;
        task_sizes(s, &A, &O);
        const void *obs_src = s->buf.p[B2G_T_OBS_CLIPPED] ? s->buf.p[B2G_T_OBS_CLIPPED] : s->buf.p[B2G_T_OBS];
        for (int k = 0; k < K; k++) {
            int rc = b2g_task_step(s, actions + (size_t)k * N * A, stream); if (rc) return rc;
            CUDA_TRY(cudaMemcpyAsync(obs_out + (size_t)k * N * O, obs_src, N * O * 4, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(rew_out + (size_t)k * N, s->buf.p[B2G_T_REW], N * 4, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(reset_out + (size_t)k * N, s->buf.p[B2G_T_RESET], N * 8, cudaMemcpyDeviceToDevice, st));
            if (timeout_out && s->buf.p[B2G_T_TIMEOUT]) CUDA_TRY(cudaMemcpyAsync(timeout_out + (size_t)k * N, s->buf.p[B2G_T_TIMEOUT], N, cudaMemcpyDeviceToDevice, st));
        }
        return B2G_OK;
    }
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_OBS, B2G_T_REW, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT,
                         B2G_T_POTENTIALS, B2G_T_PREV_POTENTIALS, B2G_T_INITIAL_ROOT}, "b2g_task_rollout"); if (rc) return rc;
    const b2g_task_params &P = s->task;
    if (s->buf_bytes[B2G_T_OBS] < N * P.num_obs * 4) return fail(B2G_E_INVALID, "OBS buffer too small");
    CUDA_TRY(cudaSetDevice(s->device));
    const int nd_ = 8, O = P.num_obs, ns6 = 6 * s->hm.nsens;
    const size_t park_f4 = (size_t)quad_park_f4(2) * QB;
    const size_t io_f4 = tile_layout(EPB, nd_, ns6, false, 2).bytes / 16;
    const size_t model_f4 = quad_model_f4(2);
    const size_t stage_f4 = (roll_stage_bytes(EPB, O) + 15) / 16;
    if (roll_last_bytes(EPB, O) > park_f4 * 16) return fail(B2G_E_UNSUPPORTED, "b2g_task_rollout: observation too large for the last-step staging");
    RollArgs ra;
    ra.actions = actions; ra.obs_out = obs_out; ra.rew_out = rew_out; ra.reset_out = (long long *)reset_out; ra.timeout_out = timeout_out;
    ra.K = K; ra.io_f4 = (int)park_f4; ra.model_f4 = (int)(park_f4 + io_f4); ra.stage_f4 = (int)(park_f4 + io_f4 + model_f4);
    const size_t dyn = (park_f4 + io_f4 + model_f4 + stage_f4) * 16;
    return launch(s, s->quad_spec == 3 ? quad_rollout_kernel<2, 3> : quad_rollout_kernel<2, 0>, (int)N / EPB, QB, dyn, st, SMEM_PDL,
                  (const float4 *)s->d_qm, s->buf, P, (int)N, (int)s->hm.substeps, ra);
}

// VecTask.reset_done() (vec_task.py:440-455): reset_idx of every env whose reset_buf is set, right now (stream-ordered)
extern "C" int b2g_reset_flagged(b2g_sim *s, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "b2g_reset_flagged: null sim");
    if (!s->has_task && !s->has_anymal && !s->has_hand) return fail(B2G_E_INVALID, "b2g_reset_flagged: call b2g_set_task first");
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int N = s->num_envs, nd = s->hm.nl - 1;
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT}, "b2g_reset_flagged"); if (rc) return rc;
    if (s->has_anymal) {
        rc = require(s, {B2G_T_COMMANDS, B2G_T_FEET_AIR_TIME, B2G_T_EPISODE_SUMS, B2G_T_REDUCE_SCRATCH}, "b2g_reset_flagged(AnymalTerrain)"); if (rc) return rc;
        if (s->anymal.custom_origins) { rc = require(s, {B2G_T_ENV_ORIGINS, B2G_T_TERRAIN_LEVELS, B2G_T_TERRAIN_TYPES, B2G_T_TERRAIN_ORIGINS}, "b2g_reset_flagged(AnymalTerrain)"); if (rc) return rc; }
        CUDA_TRY(cudaMemsetAsync((float *)s->buf.p[B2G_T_REDUCE_SCRATCH] + REDUCE_PARTIALS, 0, 16 * sizeof(float), st));
        return launch(s, anymal_reset_obs_kernel, (N * 32 + 127) / 128, 128, 0, st, PLAIN, s->buf, s->anymal, s->d_hf, N, nd, 0, s->step_counter, 1);
    }
    if (s->has_hand) {
        rc = require(s, {B2G_T_INITIAL_ROOT, B2G_T_GOAL_STATES, B2G_T_DOF_TARGET, B2G_T_PREV_TARGETS, B2G_T_SUCCESSES, B2G_T_RESET_GOAL}, "b2g_reset_flagged(ShadowHand)"); if (rc) return rc;
        if (s->hand.force_scale > 0.f) { rc = require(s, {B2G_T_OBJ_FORCE, B2G_T_RANDOM_FORCE_PROB}, "b2g_reset_flagged(ShadowHand, forceScale > 0)"); if (rc) return rc; }
        return launch(s, hand_reset_kernel, (N + 127) / 128, 128, 0, st, PLAIN, s->buf, s->hand, N, nd);
    }
    if (s->task.task != B2G_TASK_CARTPOLE) { rc = require(s, {B2G_T_POTENTIALS, B2G_T_PREV_POTENTIALS, B2G_T_INITIAL_ROOT}, "b2g_reset_flagged"); if (rc) return rc; }
    return launch(s, loco_reset_kernel, (N + 127) / 128, 128, 0, st, PLAIN, s->buf, s->task, N, nd);
}

extern "C" int b2g_task_step_host(b2g_sim *s, const float *h_actions, float *h_obs, float *h_rew, int64_t *h_reset,
                                  uint8_t *h_timeout, void *stream) {
    if (!s || !h_actions) return fail(B2G_E_INVALID, "b2g_task_step_host: null argument");
    if (!s->has_task && !s->has_anymal && !s->has_hand) return fail(B2G_E_INVALID, "b2g_task_step_host: call b2g_set_task first");
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    int n_act, n_obs;
    task_sizes(s, &n_act, &n_obs);
    const size_t N = s->num_envs, abytes = N * n_act * 4;
    // fast path (Ant / Humanoid tiled kernel, every host buffer pinned): no copy launches at all.  This pre-check counts the
    // generic step's envs per CTA even when Ant runs the quad kernel (16 per CTA), so some env counts the quad kernel could
    // tile take the staged path; a step that turns out untiled returns B2G_E_UNSUPPORTED and takes it as well.
    if (s->has_task && s->task.task != B2G_TASK_CARTPOLE) {
        auto pinned = [](const void *p) {
            if (!p) return true;
            cudaPointerAttributes a;
            if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
            return a.type == cudaMemoryTypeHost;
        };
        if (whole_tiles(N, s->block / s->lanes) && s->buf.p[B2G_T_ACTIONS] && !s->d_hf &&
            pinned(h_actions) && pinned(h_obs) && pinned(h_rew) && pinned(h_reset) && pinned(h_timeout)) {
            const HostOut io = {h_obs, h_rew, (long long *)h_reset, h_timeout};
            const int rc = task_step(s, h_actions, stream, &io);
            if (rc == B2G_OK) { CUDA_TRY(cudaStreamSynchronize(st)); return B2G_OK; }
            if (rc != B2G_E_UNSUPPORTED) return rc;       // else: the staged path below
        }
    }
    if (!s->d_actions_stage) CUDA_TRY(cudaMalloc(&s->d_actions_stage, abytes));
    CUDA_TRY(cudaMemcpyAsync(s->d_actions_stage, h_actions, abytes, cudaMemcpyHostToDevice, st));
    int rc = task_step(s, s->d_actions_stage, stream, nullptr); if (rc) return rc;
    const void *obs_src = s->buf.p[B2G_T_OBS_CLIPPED] ? s->buf.p[B2G_T_OBS_CLIPPED] : s->buf.p[B2G_T_OBS];
    if (h_obs) CUDA_TRY(cudaMemcpyAsync(h_obs, obs_src, N * n_obs * 4, cudaMemcpyDeviceToHost, st));
    if (h_rew) CUDA_TRY(cudaMemcpyAsync(h_rew, s->buf.p[B2G_T_REW], N * 4, cudaMemcpyDeviceToHost, st));
    if (h_reset) CUDA_TRY(cudaMemcpyAsync(h_reset, s->buf.p[B2G_T_RESET], N * 8, cudaMemcpyDeviceToHost, st));
    if (h_timeout && s->buf.p[B2G_T_TIMEOUT]) CUDA_TRY(cudaMemcpyAsync(h_timeout, s->buf.p[B2G_T_TIMEOUT], N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return B2G_OK;
}

// b200gym.cu -- kernels + C ABI (include/b200gym.h) of the CUDA-native (H100) environment stepper.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>

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

// Step-kernel prologue: ONE mbarrier transaction brings the hot part of the model (header, links,
// contact spheres) and, when the block owns whole 16-byte-aligned tiles, this block's slice of
// root_state / dof_state / actions into shared memory with bulk-async (TMA) copies.
struct Tiles {
    const float *root;     // [envs_per_block][13]   (shared memory, or global when !on)
    const float2 *dof;     // [envs_per_block][nd]
    const float *act;      // [envs_per_block][na]
    bool on;
};
__device__ __forceinline__ uint32_t round16(uint32_t b) { return (b + 15u) & ~15u; }

__device__ __forceinline__ Tiles prologue(DevModel *sm, uint64_t *mbar, const DevModel *__restrict__ gm, float4 *tile_smem,
                                          bool tiles_on, int env0, int epb, const float *g_root, const float *g_dof,
                                          const float *g_act, int nd_hint, int na_hint) {
    Tiles t;
    if (threadIdx.x == 0) mbar_init(mbar, 1);
    __syncthreads();
    const uint32_t rb = (uint32_t)epb * 13u * 4u, db = (uint32_t)epb * (uint32_t)nd_hint * 8u, ab = (uint32_t)epb * (uint32_t)na_hint * 4u;
    float *s_root = reinterpret_cast<float *>(tile_smem);
    float *s_dof = s_root + rb / 4;
    float *s_act = s_dof + db / 4;
    if (threadIdx.x == 0) {
        const int nl = gm->nl, ncp = gm->ncp, ns = gm->ns;   // three scalar loads; everything else arrives by bulk copy
        const uint32_t hb = (uint32_t)offsetof(DevModel, slots) + (uint32_t)ns * MAX_LANES * (uint32_t)sizeof(SlotRec);
        const uint32_t lb = round16((uint32_t)nl * (uint32_t)sizeof(LinkC)), cb = round16((uint32_t)ncp * (uint32_t)sizeof(CpC));
        uint32_t total = hb + lb + cb;
        if (tiles_on) total += rb + db + (g_act ? ab : 0u);
        mbar_expect_tx(mbar, total);
        bulk_g2s(sm, gm, hb, mbar);
        bulk_g2s(sm->links, gm->links, lb, mbar);
        if (cb) bulk_g2s(sm->cps, gm->cps, cb, mbar);
        if (tiles_on) {
            bulk_g2s(s_root, g_root + (size_t)env0 * 13, rb, mbar);
            bulk_g2s(s_dof, g_dof + (size_t)env0 * nd_hint * 2, db, mbar);
            if (g_act) bulk_g2s(s_act, g_act + (size_t)env0 * na_hint, ab, mbar);
        }
    }
    mbar_wait(mbar, 0);
    t.on = tiles_on;
    t.root = tiles_on ? s_root : g_root + (size_t)env0 * 13;
    t.dof = reinterpret_cast<const float2 *>(tiles_on ? s_dof : g_dof + (size_t)env0 * nd_hint * 2);
    t.act = g_act ? (tiles_on ? s_act : g_act + (size_t)env0 * na_hint) : nullptr;
    return t;
}


template <int L, bool HF, int BLOCK, bool OBJ = false, bool SELF = false>
__device__ __forceinline__ Stepper<L, HF, BLOCK, OBJ, SELF> make_stepper(const DevModel *sm, const int16_t *hf, int lane) {
    Stepper<L, HF, BLOCK, OBJ, SELF> st;
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
    st.dr_mass = nullptr; st.dr_dof = nullptr;
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
template <int L, bool HF, int BLOCK, bool OBJ = false, bool SELF = false>
__global__ void __launch_bounds__(BLOCK) simulate_kernel(const DevModel *__restrict__ gm, const int16_t *__restrict__ hf,
                                                         Buffers B, int N) {
    __shared__ DevModel sm;
    __shared__ alignas(8) uint64_t mbar;
    prologue(&sm, &mbar, gm, nullptr, false, 0, 0, nullptr, nullptr, nullptr, 0, 0);
    using ST = Stepper<L, HF, BLOCK, OBJ, SELF>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const int nd = sm.nl - 1, NS = sm.ns;
    ST st = make_stepper<L, HF, BLOCK, OBJ, SELF>(&sm, hf, lane);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
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
// Data movement: with whole 16-byte-aligned tiles per block (tiles_on) every tensor of the step
// moves as ONE bulk-async copy per block: in  -- model, root_state, dof_state, actions;
// out -- root_state, dof_state, clamped actions, force sensors, dof forces, obs (+ clipped obs),
// rew, reset, progress, potentials, prev_potentials, up_vec, heading_vec, time-outs.  The output
// tiles are staged in the shared memory that held the slot state during the physics.
#ifndef B2G_MINBLOCKS
#define B2G_MINBLOCKS 4
#endif

template <int L, bool HF, bool HUM, int BLOCK, bool TILES, bool HOSTIO = false, bool SELF = false>
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
    // ---- in/out tile region: root | dof | act | sensors | dof_force
    const int nsens6 = 6 * ((P.num_obs - 12 - (HUM ? 4 : 3) * nd) / 6);          // 6 * nsens, from the obs layout
    float *const s_root = io;
    float *const s_dof = s_root + EPB * 13;
    float *const s_act = s_dof + EPB * nd * 2;
    float *const s_sens = s_act + EPB * nd;
    float *const s_dfrc = s_sens + EPB * nsens6;
    // ---- prologue.  Programmatic dependent launch: this grid may start while the previous kernel in the
    // stream (the previous control step) is still draining.  Everything that does not depend on it --
    // barrier set-up and the bulk copy of the (constant) model -- happens before griddepcontrol.wait;
    // the state tiles and per-env scalars are fetched after it.
    __shared__ alignas(8) uint64_t mbar2;
    long long *const progress_b = (long long *)B.p[B2G_T_PROGRESS];
    long long *const reset_b = (long long *)B.p[B2G_T_RESET];
    float *const pot_b = (float *)B.p[B2G_T_POTENTIALS], *const ppot_b = (float *)B.p[B2G_T_PREV_POTENTIALS];
    const int e_pre = min((int)((blockIdx.x * BLOCK + threadIdx.x) / L), N - 1);
    if (threadIdx.x == 0) { mbar_init(&mbar, 1); mbar_init(&mbar2, 1); }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nl = gm->nl, ncp = gm->ncp, ns = gm->ns;   // three scalar loads; everything else arrives by bulk copy
        const uint32_t hb = (uint32_t)offsetof(DevModel, slots) + (uint32_t)ns * MAX_LANES * (uint32_t)sizeof(SlotRec);
        const uint32_t lb = round16((uint32_t)nl * (uint32_t)sizeof(LinkC)), cb = round16((uint32_t)ncp * (uint32_t)sizeof(CpC));
        mbar_expect_tx(&mbar, hb + lb + cb);
        bulk_g2s(&sm, gm, hb, &mbar);                                      // header | slots[0..ns)
        char *const pk = reinterpret_cast<char *>(&sm) + hb;               // links and cps packed right behind
        bulk_g2s(pk, gm->links, lb, &mbar);
        if (cb) bulk_g2s(pk + lb, gm->cps, cb, &mbar);
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");                     // previous step's writes are now visible
    if (tiles && threadIdx.x == 0) {
        const uint32_t rb = EPB * 13 * 4, db = (uint32_t)(EPB * nd * 8), ab = (uint32_t)(EPB * nd * 4);
        mbar_expect_tx(&mbar2, rb + db + (HOSTIO ? 0u : ab));
        bulk_g2s(s_root, (const float *)B.p[B2G_T_ROOT_STATE] + (size_t)env0 * 13, rb, &mbar2);
        bulk_g2s(s_dof, (const float *)B.p[B2G_T_DOF_STATE] + (size_t)env0 * nd * 2, db, &mbar2);
        if (!HOSTIO) bulk_g2s(s_act, actions_in + (size_t)env0 * nd, ab, &mbar2);
    }
    if (tiles && HOSTIO) {         // actions straight from pinned host memory
        const float4 *src = reinterpret_cast<const float4 *>(ta.h_act + (size_t)env0 * nd);
        float4 *dst = reinterpret_cast<float4 *>(s_act);
        for (int i = threadIdx.x; i < EPB * nd / 4; i += BLOCK) dst[i] = src[i];
        __syncthreads();
    }
    // per-env scalars of post_physics_step: issued now, consumed after the physics
    const long long progress_in = progress_b[e_pre];
    const long long reset_in = reset_b[e_pre];
    const float potentials_in = pot_b[e_pre];
    mbar_wait(&mbar, 0);
    if (tiles) mbar_wait(&mbar2, 0);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");       // the next step's grid may begin its own prologue
    using ST = Stepper<L, HF, BLOCK, false, SELF>;
    const int gt = blockIdx.x * BLOCK + threadIdx.x;
    const int env = gt / L, lane = gt % L;
    const bool valid = env < N;
    const int e = valid ? env : N - 1;
    const int el = e - env0;                             // env index inside this block's tiles
    const int NS = sm.ns;
    ST st = make_stepper<L, HF, BLOCK, false, SELF>(&sm, hf, lane);
    st.gmodel = gm;
    attach_env_params_generic(st, sm, B, e);
    {
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
        if (do_reset) {
            const float up = reset_uniform(P.seed, gid, count, d);
            const float uv = reset_uniform(P.seed, gid, count, nd + d);
            const float pos = (P.reset_pos_noise - (-P.reset_pos_noise)) * up + (-P.reset_pos_noise);
            qv.x = fmaxf(fminf(P.initial_dof_pos[d] + pos, P.dof_limits_upper[d]), P.dof_limits_lower[d]);
            qv.y = (P.reset_vel_noise - (-P.reset_vel_noise)) * uv + (-P.reset_vel_noise);
        }
        if (valid) row_dof[d] = qv;
    }
    if (do_reset) {
        const float *ir = (const float *)B.p[B2G_T_INITIAL_ROOT] + 13 * (size_t)e;
        rs.rp[0] = ir[0]; rs.rp[1] = ir[1]; rs.rp[2] = ir[2];
        rs.rq[0] = ir[3]; rs.rq[1] = ir[4]; rs.rq[2] = ir[5]; rs.rq[3] = ir[6];
        rs.rv[0] = ir[7]; rs.rv[1] = ir[8]; rs.rv[2] = ir[9];
        rs.rw[0] = ir[10]; rs.rw[1] = ir[11]; rs.rw[2] = ir[12];
        potentials = t_potential(P.target[0] - rs.rp[0], P.target[1] - rs.rp[1], P.dt);
        progress = 0;
        if (valid && lane == 0) rc[e] = (int)(count + 1);
    }
    if (valid && lane == 0 && !sm.root_fixed) store_root(row_root, rs);

    // the slot state is dead from here on: its shared memory becomes the output staging area
    // layout (floats unless noted): obs | obs_clipped? | rew | pot | ppot | up(3) | head(3) | reset(i64) | progress(i64) | timeout(u8)
    __syncthreads();
    float *const g_obs = (float *)B.p[B2G_T_OBS];
    float *g_obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    if (g_obsc == g_obs) g_obsc = nullptr;
    float *const so = reinterpret_cast<float *>(b2g_dyn_smem);
    float *const t_obs = so;
    float *const t_obsc = t_obs + EPB * O;
    float *const t_rew = t_obsc + (g_obsc ? EPB * O : 0);
    float *const t_pot = t_rew + EPB, *const t_ppot = t_pot + EPB, *const t_up = t_ppot + EPB, *const t_head = t_up + 3 * EPB;
    long long *const t_reset = reinterpret_cast<long long *>(t_head + 3 * EPB), *const t_prog = t_reset + EPB;
    uint8_t *const t_to = reinterpret_cast<uint8_t *>(t_prog + EPB);
    float *const obs = tiles ? t_obs + (size_t)el * O : g_obs + (size_t)e * O;
    float *const obsc = g_obsc ? (tiles ? t_obsc + (size_t)el * O : g_obsc + (size_t)e * O) : nullptr;

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
    float actions_cost = 0.f, electricity = 0.f, at_limit = 0.f;
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
        // compute_ant_reward (ant.py:353-355) / compute_humanoid_reward (humanoid.py:352-359)
        actions_cost += a * a;
        if (HUM) {
            const float ratio = P.motor_efforts[d] / P.max_motor_effort;
            const float scaled = P.joints_at_limit_cost_scale * (fabsf(ps) - 0.98f) / 0.02f;
            at_limit += (fabsf(ps) > 0.98f) ? scaled * ratio : 0.f;
            electricity += fabsf(a * vs) * ratio;
        } else {
            at_limit += (ps > 0.99f) ? 1.f : 0.f;
            electricity += fabsf(a * vs);
        }
    }
    if (lane == 0 && st.links[0].sensor >= 0 && o.sensor) {
        const int sk = st.links[0].sensor;
#pragma unroll
        for (int c = 0; c < 6; c++) put(o_sens + 6 * sk + c, o.sensor[6 * sk + c] * P.contact_force_scale);
    }
    actions_cost = lane_sum<L>(actions_cost);
    electricity = lane_sum<L>(electricity);
    at_limit = lane_sum<L>(at_limit);

    if (valid && lane == 0) {
        const float heading_proj = ro.o[11], up_proj = ro.o[10], height = ro.o[0];
        const float heading_reward = (heading_proj > 0.8f) ? P.heading_weight : P.heading_weight * heading_proj / 0.8f;
        const float up_reward = (up_proj > 0.93f) ? P.up_weight : 0.f;
        const float progress_reward = potentials - prev_potentials;
        float total_r = progress_reward + P.alive_reward + up_reward + heading_reward - P.actions_cost_scale * actions_cost -
                        P.energy_cost_scale * electricity - (HUM ? at_limit : at_limit * P.joints_at_limit_cost_scale);
        long long reset = 0;                       // reset_buf was cleared by reset_idx or was already 0
        if (height < P.termination_height) { total_r = P.death_cost; reset = 1; }
        if ((float)progress >= P.max_episode_length - 1.f) reset = 1;
        const uint8_t tout = (uint8_t)(((float)progress >= P.max_episode_length - 1.f) && reset != 0);   // vec_task.py:394
        float *uv = (float *)B.p[B2G_T_UP_VEC], *hv = (float *)B.p[B2G_T_HEADING_VEC];
        uint8_t *to = (uint8_t *)B.p[B2G_T_TIMEOUT];
        if (tiles) {
            t_rew[el] = total_r; t_reset[el] = reset; t_prog[el] = progress; t_pot[el] = potentials; t_ppot[el] = prev_potentials;
            t_up[3 * el] = ro.up_vec[0]; t_up[3 * el + 1] = ro.up_vec[1]; t_up[3 * el + 2] = ro.up_vec[2];
            t_head[3 * el] = ro.heading_vec[0]; t_head[3 * el + 1] = ro.heading_vec[1]; t_head[3 * el + 2] = ro.heading_vec[2];
            t_to[el] = tout;
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
        if (threadIdx.x == 0) {
            const size_t e0 = (size_t)env0;
            if (!sm.root_fixed) bulk_s2g((float *)B.p[B2G_T_ROOT_STATE] + e0 * 13, s_root, EPB * 13 * 4);
            bulk_s2g((float *)B.p[B2G_T_DOF_STATE] + e0 * nd * 2, s_dof, (uint32_t)(EPB * nd * 8));
            if (g_act_out) bulk_s2g(g_act_out + e0 * nd, s_act, (uint32_t)(EPB * nd * 4));
            if (stage_out && g_sens && nsens6) bulk_s2g(g_sens + e0 * nsens6, s_sens, (uint32_t)(EPB * nsens6 * 4));
            if (stage_out && HUM && g_dfrc) bulk_s2g(g_dfrc + e0 * nd, s_dfrc, (uint32_t)(EPB * nd * 4));
            bulk_s2g(g_obs + e0 * O, t_obs, (uint32_t)(EPB * O * 4));
            if (g_obsc) bulk_s2g(g_obsc + e0 * O, t_obsc, (uint32_t)(EPB * O * 4));
            bulk_s2g((float *)B.p[B2G_T_REW] + e0, t_rew, EPB * 4);
            bulk_s2g(pot_b + e0, t_pot, EPB * 4);
            bulk_s2g(ppot_b + e0, t_ppot, EPB * 4);
            if (B.p[B2G_T_UP_VEC]) bulk_s2g((float *)B.p[B2G_T_UP_VEC] + 3 * e0, t_up, EPB * 12);
            if (B.p[B2G_T_HEADING_VEC]) bulk_s2g((float *)B.p[B2G_T_HEADING_VEC] + 3 * e0, t_head, EPB * 12);
            bulk_s2g(reset_b + e0, t_reset, EPB * 8);
            bulk_s2g(progress_b + e0, t_prog, EPB * 8);
            if (B.p[B2G_T_TIMEOUT]) bulk_s2g((uint8_t *)B.p[B2G_T_TIMEOUT] + e0, t_to, EPB);

            bulk_commit_wait();
        }
        // host copies of what VecTask.step returns (vec_task.py:402-408), straight over PCIe: coalesced 16-byte stores
        if (HOSTIO) {
            const size_t e0 = (size_t)env0;
            auto copy16 = [&](void *dst, const void *src, int bytes) {
                float4 *d = reinterpret_cast<float4 *>(dst); const float4 *sp = reinterpret_cast<const float4 *>(src);
                for (int i = threadIdx.x; i < bytes / 16; i += BLOCK) d[i] = sp[i];
            };
            if (ta.h_obs) copy16(ta.h_obs + e0 * O, g_obsc ? t_obsc : t_obs, EPB * O * 4);
            if (ta.h_rew) copy16(ta.h_rew + e0, t_rew, EPB * 4);
            if (ta.h_reset) copy16(ta.h_reset + e0, t_reset, EPB * 8);
            if (ta.h_timeout) copy16(ta.h_timeout + e0, t_to, EPB);
        }
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
    prologue(&sm, &mbar, gm, nullptr, false, 0, 0, nullptr, nullptr, nullptr, 0, 0);
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
        for (int s = 0; s < 2; s++)
            st.set_q(s, 0.2f * (reset_uniform(P.seed, gid, count, s) - 0.5f), 0.5f * (reset_uniform(P.seed, gid, count, 2 + s) - 0.5f));
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
#include "b2g_quad_host.h"
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
struct b2g_sim {
    int device = 0;
    int num_envs = 0;
    int lanes = 1;
    int block = 128;             // threads per CTA, chosen so the slot state fits in shared memory
    size_t dyn_smem = 0;
    DevModel hm;                 // host copy
    DevModel *dm = nullptr;      // device copy
    int16_t *d_hf = nullptr;
    Buffers buf;
    size_t buf_bytes[B2G_T_COUNT];
    b2g_task_params task;
    b2g_anymal_params anymal;
    b2g_hand_params hand;
    HandDev hand_dev;
    bool has_task = false, has_anymal = false, has_hand = false;
    unsigned step_counter = 0;   // common_step_counter, anymal_terrain.py:459
    float *d_actions_stage = nullptr;    // device staging for b2g_task_step_host
    struct { bool on = false; float *obs = nullptr, *rew = nullptr; long long *reset = nullptr; uint8_t *timeout = nullptr; } zero_copy;
    int64_t launches = 0;
    // quad path (b2g_quad.cuh): chain length (2 Ant-like, 3 ANYmal-like) or 0 = generic Stepper; the packed constants
    int quad_ns = 0;
    int quad_spec = 0;                        // QLane specialisation flags the constants are packed for (b2g_quad.cuh)
    int quad_block = 64;                      // threads per CTA of the quad step kernels (B2G_QUAD_BLOCK: 32 / 64 / 128)
    float4 *d_qm = nullptr;
    KinModel hk;                              // constant tables of the Jacobian / mass-matrix kernel (b2g_kin.cuh)
    KinModel *d_kin = nullptr;
    bool kin_ok = false;
    std::vector<const void *> smem_set;      // kernels whose dynamic shared-memory limit has been raised (once per sim)
    bool no_zero_copy = false;
    size_t hostio_pad = 0;                    // extra dynamic shared memory of the host-I/O Ant launch (see b2g_task_step_host)
};

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }
#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(B2G_E_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

extern "C" const char *b2g_last_error(void) { return g_err.c_str(); }
extern "C" int b2g_version(void) { return B2G_VERSION; }
extern "C" int64_t b2g_launch_count(const b2g_sim *sim) { return sim ? sim->launches : 0; }
extern "C" int b2g_quad_chain_length(const b2g_sim *sim) { return sim ? sim->quad_ns : 0; }

// Build the lanes' slot programs: list-schedule the links over `L` lanes, critical path first; a lane
// keeps following a chain (parent at step s-1 in the same lane -> state travels in registers), any
// other parent/child relation goes through shared memory (parked inertia / pose / acceleration).
static int schedule(const b2g_model *m, int L, DevModel &h, bool compact = false) {
    const int nl = m->nl;
    std::vector<int> height(nl, 1);
    for (int i = nl - 1; i >= 1; i--) height[m->parent[i]] = std::max(height[m->parent[i]], height[i] + 1);
    std::vector<int> t_of(nl, -1), lane_of(nl, -1);
    t_of[0] = -1;
    std::vector<int> lane_last(L, -1);
    int remaining = nl - 1, t = 0;
    for (int s = 0; s < MAX_SLOTS; s++) for (int l = 0; l < MAX_LANES; l++) {
        SlotRec &r = h.slots[s][l]; r.link = -1; r.parent = 0; r.out = -1; r.flags = 0;
        for (int c = 0; c < MAX_CHILD_REFS; c++) r.child[c] = -1;
    }
    while (remaining > 0) {
        if (t >= MAX_SLOTS) return -1;
        std::vector<int> ready;
        for (int i = 1; i < nl; i++) if (t_of[i] < 0 && (m->parent[i] == 0 || (t_of[m->parent[i]] >= 0 && t_of[m->parent[i]] < t))) ready.push_back(i);
        std::stable_sort(ready.begin(), ready.end(), [&](int a, int b) { return height[a] > height[b]; });
        std::vector<int> pick(L, -1);
        std::vector<char> used(nl, 0);
        for (int l = 0; l < L; l++) {                                   // continue chains first
            if (lane_last[l] < 0) continue;
            for (int i : ready) if (!used[i] && m->parent[i] == lane_last[l]) { pick[l] = i; used[i] = 1; break; }
        }
        for (int i : ready) {                                            // then the most critical remaining links
            if (used[i]) continue;
            int l = 0; while (l < L && pick[l] >= 0) l++;
            if (l == L) break;
            pick[l] = i; used[i] = 1;
        }
        for (int l = 0; l < L; l++) {
            lane_last[l] = pick[l];
            if (pick[l] >= 0) { t_of[pick[l]] = t; lane_of[pick[l]] = l; h.slots[t][l].link = pick[l]; remaining--; }
        }
        t++;
    }
    h.ns = t; h.lanes = L; h.cross_lane = 0; h.root_acc = -1;
    std::vector<int> nacc(L, 0);
    bool need_root_acc = false;
    for (int i = 1; i < nl; i++) if (m->parent[i] == 0 && t_of[i] > 0) need_root_acc = true;
    // compact (env-wide) accumulator ids: per-lane ones take L consecutive ids, parked inertias one each
    int gacc = 0;
    if (compact && m->root_fixed) need_root_acc = false;                 // nothing collects a fixed root's children
    if (need_root_acc) { h.root_acc = 0; for (int l = 0; l < L; l++) nacc[l] = 1; gacc = L; }
    for (int i = 1; i < nl; i++) {
        const int l = lane_of[i], s = t_of[i], p = m->parent[i];
        SlotRec &r = h.slots[s][l];
        if (p == 0) {
            r.parent = 0;
            r.out = (s == 0) ? -1 : h.root_acc;
            if (compact && m->root_fixed) r.out = (s == 0) ? -1 : -2;
        } else {
            const int lp = lane_of[p], sp = t_of[p];
            r.parent = (lp << 8) | (sp + 1);
            if (lp != l) h.cross_lane = 1;
            if (lp == l && sp == s - 1) r.out = -1;
            else {
                r.out = compact ? gacc++ : nacc[l]++;
                SlotRec &pr = h.slots[sp][lp];
                int c = 0; while (c < MAX_CHILD_REFS && pr.child[c] >= 0) c++;
                if (c == MAX_CHILD_REFS) return -2;
                pr.child[c] = (l << 8) | r.out;
                pr.flags |= 1;
            }
        }
    }
    h.nacc = 0;
    for (int l = 0; l < L; l++) h.nacc = std::max(h.nacc, nacc[l]);
    if (compact) h.nacc = gacc;
    return 0;
}
static int pick_lanes(const b2g_model *m, bool single) {
    if (single) return 1;
    int root_children = 0;
    for (int i = 1; i < m->nl; i++) if (m->parent[i] == 0) root_children++;
    const char *env = getenv("B2G_LANES");
    if (env && (env[0] == '1' || env[0] == '2' || env[0] == '4' || env[0] == '8') && env[1] == 0) return env[0] - '0';
    if (m->nl - 1 >= 16) return 4;                 // long trees (Humanoid, hands): chains run in parallel lanes
    if (root_children >= 4) return 4;              // quadrupeds
    if (root_children >= 2) return 2;
    return 1;
}

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
    if (ext && (ext->actors_per_env < 1 || ext->obj_actor >= ext->actors_per_env || ext->obj_actor == 0 || ext->nbox < 0 ||
                ext->nbox > MAX_BOX || ext->nten < 0 || ext->nten > MAX_TEN))
        return fail(B2G_E_INVALID, "b2g_create_ext: bad actor / box / tendon counts");
    if (ext && ext->obj_actor > 0 && sp->hf_samples) return fail(B2G_E_UNSUPPORTED, "b2g_create_ext: the free object needs the ground plane");
    if (m->nl < 1 || m->nl > MAX_LINKS || m->nl - 1 > MAX_SLOTS || m->ncp > MAX_CP || m->nsens > MAX_SENS || m->nb > MAX_LINKS)
        return fail(B2G_E_INVALID, "b2g_create: model exceeds compiled limits (links/contact points/sensors)");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
        return fail(B2G_E_CUDA, std::string("b2g_create: no CUDA device (there is no CPU fallback): ") + cudaGetErrorString(ce));
    CUDA_TRY(cudaSetDevice(device));
    b2g_sim *s = new b2g_sim();
    s->device = device; s->num_envs = num_envs;
    memset(&s->buf, 0, sizeof(s->buf)); memset(s->buf_bytes, 0, sizeof(s->buf_bytes));
    DevModel &h = s->hm;
    memset(&h, 0, sizeof(h));
    h.nl = m->nl; h.ncp = m->ncp; h.nb = m->nb; h.nsens = m->nsens;
    h.root_fixed = m->root_fixed; h.gravity_on = m->gravity_on; h.substeps = sp->substeps;
    h.h = sp->dt / (float)sp->substeps;
    for (int c = 0; c < 3; c++) h.g[c] = m->gravity_on ? sp->gravity[c] : 0.f;
    h.kn = m->contact_kn; h.cn = m->contact_cn; h.vs2 = m->contact_vs * m->contact_vs;
    h.ground_mu = sp->ground_friction;
    h.ang_damp = m->angular_damping; h.lin_damp = m->linear_damping; h.max_angvel = m->max_angular_velocity;
    h.obj_ang_damp = ext ? ext->obj_angular_damping : 0.f; h.obj_lin_damp = ext ? ext->obj_linear_damping : 0.f;
    // topology
    const char *force1 = getenv("B2G_SINGLE_LANE");
    const bool compact = ext && ext->obj_actor > 0;                     // [link][k][env] state layout (Stepper<.., OBJ>)
    if (schedule(m, pick_lanes(m, force1 && force1[0] == '1'), h, compact) != 0) { delete s; return fail(B2G_E_INVALID, "b2g_create: the articulation does not fit the slot program limits"); }
    s->lanes = h.lanes;
    h.root_stride = ext ? ext->actors_per_env : 1;
    h.obj_on = 0; h.obj_acc = h.obj_pose_acc = -1;
    if (ext) {
        if (ext->obj_actor > 0) {
            h.obj_on = 1; h.obj_row = ext->obj_actor; h.obj_gravity_on = ext->obj_gravity_on;
            h.obj_mass = ext->obj_mass; h.obj_kn = ext->obj_kn; h.obj_cn = ext->obj_cn; h.obj_mu = ext->obj_mu;
            for (int c = 0; c < 3; c++) { h.obj_I[c] = ext->obj_inertia[c]; h.obj_half[c] = ext->obj_half[c]; }
            h.obj_round = ext->obj_round; h.obj_max_angvel = ext->obj_max_angular_velocity;
            if (ext->obj_round < 0.f || (ext->obj_round == 0.f && (ext->obj_half[0] <= 0.f || ext->obj_half[1] <= 0.f || ext->obj_half[2] <= 0.f))) {
                delete s; return fail(B2G_E_INVALID, "b2g_create_ext: the object needs positive half extents, or a rounding radius");
            }
            h.obj_acc = h.nacc; h.obj_pose_acc = h.nacc + h.lanes; h.nacc += h.lanes + 1;   // env-wide ids: one sum per lane, one pose
            // the object's gravity does not follow the articulation's disable_gravity flag (shadow_hand.py:239,279-282)
            for (int c = 0; c < 3; c++) h.obj_g[c] = ext->obj_gravity_on ? sp->gravity[c] : 0.f;
        }
        h.nbox = ext->nbox;
        for (int b = 0; b < ext->nbox; b++) {
            h.box_link[b] = ext->box_link[b];
            if (ext->box_link[b] < 0 || ext->box_link[b] >= m->nl) { delete s; return fail(B2G_E_INVALID, "b2g_create_ext: box link out of range"); }
            const float *q = ext->box_quat[b];
            float x = q[0], y = q[1], z = q[2], w = q[3], n = sqrtf(x * x + y * y + z * z + w * w);
            x /= n; y /= n; z /= n; w /= n;
            const float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                                2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                                2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
            memcpy(h.box_R[b], R, sizeof(R));
            for (int c = 0; c < 3; c++) { h.box_pos[b][c] = ext->box_pos[b][c]; h.box_half[b][c] = ext->box_half[b][c]; }
        }
        h.nten = ext->nten; h.ten_k = ext->ten_k; h.ten_d = ext->ten_d;
        for (int t = 0; t < ext->nten; t++) for (int k = 0; k < 2; k++) {
            const int link = ext->ten_dof[t][k] + 1;
            int ref = -1;
            for (int sl = 0; sl < h.ns && ref < 0; sl++) for (int l = 0; l < h.lanes; l++) if (h.slots[sl][l].link == link) { ref = (l << 8) | sl; break; }
            if (ref < 0) { delete s; return fail(B2G_E_INVALID, "b2g_create_ext: tendon joint index out of range"); }
            h.ten_ref[t][k] = ref; h.ten_coef[t][k] = ext->ten_coef[t][k]; h.ten_range[t][k] = ext->ten_range[t][k];
        }
        if (h.nten > 0 && !h.obj_on) { delete s; return fail(B2G_E_UNSUPPORTED, "b2g_create_ext: tendons are only compiled into the object-enabled kernels"); }
    }
    if (compact) {
        // per-env rows; one CTA = `blk / lanes` envs (+1 column of padding when that is even).  Prefer the CTA size that
        // puts the most envs on an SM (registers: ~248 per thread in these kernels -> at most 256 threads per SM)
        const size_t rows = (size_t)(h.nl - 1) * SLOT_F4 + (size_t)h.nacc * ACC_F4;
        const size_t static_smem = sizeof(DevModel) + 64;
        int best = 0; size_t best_envs = 0;
        for (int blk : {128, 64, 32}) {
            const int epb = blk / h.lanes;
            if (epb < 1) continue;
            const size_t bytes = rows * (size_t)(epb | 1) * sizeof(float4);
            if (bytes + static_smem > 200 * 1024) continue;
            const size_t ctas = std::min<size_t>((227 * 1024) / (bytes + static_smem + 1024), 256 / blk);
            if (ctas * epb > best_envs) { best_envs = ctas * epb; best = blk; }
        }
        if (!best) { delete s; return fail(B2G_E_INVALID, "b2g_create: articulation too large for shared-memory slot state"); }
        s->block = best; s->dyn_smem = rows * (size_t)((best / h.lanes) | 1) * sizeof(float4);
    } else {   // CTA size: the per-thread slot state must fit in shared memory, preferably several CTAs per SM
        const size_t per_thread = ((size_t)h.ns * SLOT_F4 + (size_t)h.nacc * ACC_F4) * sizeof(float4);
        // self-collision scratch per ENV behind the accumulator pool: sphere centres, hit count, hit list (odd float4 count: banks)
        h.self_on = (m->self_collide && m->self_pairs) ? 1 : 0;
        h.self_f4 = 0;
        if (h.self_on) {
            // preferably in a run of consecutive slot cells of one lane that no link occupies (10 float4 each): no extra shared
            // memory, the CTA size is unchanged
            const int need = (m->ncp + 1 + SELF_HITS * 2 / 16 + SLOT_F4 - 1) / SLOT_F4;
            int found = -1;
            for (int l = 0; l < h.lanes && found < 0; l++) for (int s0 = 0; s0 + need <= h.ns && found < 0; s0++) {
                bool idle = true;
                for (int k = 0; k < need; k++) idle = idle && h.slots[s0 + k][l].link < 0;
                if (idle) found = (l << 8) | s0;
            }
            h.self_cell = found;
            if (found < 0 || getenv("B2G_SELF_APPENDED")) h.self_f4 = (m->ncp + 1 + SELF_HITS * 2 / 16) | 1;
        }
        auto bytes_of = [&](int b) { return per_thread * b + (size_t)(b / h.lanes) * h.self_f4 * sizeof(float4); };
        int blk = 128;
        const char *fb = getenv("B2G_BLOCK");                       // experiment hook: force a smaller CTA
        if (fb && (atoi(fb) == 64 || atoi(fb) == 32)) blk = atoi(fb);
        while (blk > 32 && bytes_of(blk) > 104 * 1024) blk >>= 1;
        if (bytes_of(blk) > 200 * 1024) { delete s; return fail(B2G_E_INVALID, "b2g_create: articulation too large for shared-memory slot state"); }
        s->block = blk; s->dyn_smem = bytes_of(blk);
    }
    // links
    std::vector<int> order(m->ncp);
    for (int i = 0; i < m->ncp; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return m->cp_link[a] < m->cp_link[b]; });
    for (int i = 0; i < MAX_LINKS; i++) h.link_body[i] = -1;
    for (int b = m->nb - 1; b >= 0; b--) { h.body_link[b] = m->body_link[b]; h.link_body[m->body_link[b]] = b; }
    for (int b = 0; b < m->nb; b++) {
        for (int c = 0; c < 3; c++) h.body_pos[b][c] = m->body_pos[3 * b + c];
        for (int c = 0; c < 4; c++) h.body_quat[b][c] = m->body_quat[4 * b + c];
    }
    for (int i = 0; i < m->nl; i++) h.link_parent[i] = m->parent[i];
    for (int k = 0; k < m->nsens; k++) {
        h.sensor_body[k] = m->sensor_body[k];
        for (int c = 0; c < 3; c++) h.sensor_bpos[k][c] = m->body_pos[3 * m->sensor_body[k] + c];
    }
    for (int i = 0; i < m->nl; i++) {
        LinkC &l = h.links[i];
        const float *q = m->lquat + 4 * i;
        float x = q[0], y = q[1], z = q[2], w = q[3], n = sqrtf(x * x + y * y + z * z + w * w);
        x /= n; y /= n; z /= n; w /= n;
        float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        memcpy(l.R0, R, sizeof(R));
        for (int c = 0; c < 3; c++) { l.lpos[c] = m->lpos[3 * i + c]; l.axis[c] = m->axis[3 * i + c]; l.com[c] = m->com[3 * i + c]; }
        for (int c = 0; c < 6; c++) l.Ic[c] = m->inertia[6 * i + c];
        l.mass = m->mass[i];
        l.armature = m->armature[i]; l.damping = m->damping[i]; l.stiffness = m->stiffness[i];
        l.lower = m->lower[i]; l.upper = m->upper[i]; l.effort = m->effort[i];
        l.kp = m->kp[i]; l.kd = m->kd[i]; l.limit_k = m->limit_k[i]; l.limit_d = m->limit_d[i];
        {
            const bool ident = fabsf(R[0] - 1.f) < 1e-7f && fabsf(R[4] - 1.f) < 1e-7f && fabsf(R[8] - 1.f) < 1e-7f;
            l.flags = (m->jtype[i] == 1 ? LF_SLIDE : 0) | (m->limited[i] ? LF_LIMITED : 0) | (m->drive_mode[i] == 1 ? LF_POSDRIVE : 0) | (ident ? LF_R0_IDENTITY : 0);
        }
        l.sensor = -1;
        l.cp_begin = l.cp_end = 0;
    }
    for (int k = 0; k < m->nsens; k++) h.links[m->body_link[m->sensor_body[k]]].sensor = k;
    for (int k = 0; k < m->ncp; k++) {
        int src = order[k];
        CpC &c = h.cps[k];
        for (int j = 0; j < 3; j++) c.pos[j] = m->cp_pos[3 * src + j];
        c.radius = m->cp_radius[src]; c.mu = 0.5f * (m->cp_mu[src] + sp->ground_friction); c.body = m->cp_body[src]; c.pad = m->cp_link[src];
        LinkC &l = h.links[m->cp_link[src]];
        if (l.cp_end == 0 && l.cp_begin == 0) l.cp_begin = k;
        l.cp_end = k + 1;
    }
    if (ext) for (int b = 0; b < ext->nbox; b++) h.links[ext->box_link[b]].flags |= LF_HAS_BOX;
    {   // reach: bound on the distance of any contact sphere's far side from the root origin, over all joint positions
        std::vector<float> dist(m->nl, 0.f);
        for (int i = 1; i < m->nl; i++) {
            const float *lp = m->lpos + 3 * i;
            float d = sqrtf(lp[0] * lp[0] + lp[1] * lp[1] + lp[2] * lp[2]);
            if (m->jtype[i] == 1) d += m->limited[i] ? std::max(fabsf(m->lower[i]), fabsf(m->upper[i])) : 1e30f;
            dist[i] = dist[m->parent[i]] + d;
        }
        h.reach = 0.f;
        for (int k = 0; k < m->ncp; k++) {
            const float *cp = m->cp_pos + 3 * k;
            h.reach = std::max(h.reach, dist[m->cp_link[k]] + sqrtf(cp[0] * cp[0] + cp[1] * cp[1] + cp[2] * cp[2]) + m->cp_radius[k]);
        }
    }
    // self-collision tables (create_actor collision filter 0)
    if (m->self_collide && m->self_pairs) {
        if (compact || (ext && ext->obj_actor >= 0)) { delete s; return fail(B2G_E_UNSUPPORTED, "b2g_create_ext: self-collision is not compiled into the object-enabled kernels"); }
        if (m->ncp > 64 || m->nl > MAX_LINKS) { delete s; return fail(B2G_E_UNSUPPORTED, "b2g_create: self-collision supports at most 64 contact spheres / 32 links"); }
        h.self_kn = m->self_kn; h.self_cn = m->self_cn; h.self_mu = m->self_mu;
        std::vector<int> inv(m->ncp);
        for (int k = 0; k < m->ncp; k++) inv[order[k]] = k;
        for (int i = 0; i < MAX_LINKS; i++) h.link_slot[i] = -1;
        h.npairs = 0;
        for (int a = 0; a < m->ncp; a++) for (int b = a + 1; b < m->ncp; b++) {
            if (!m->self_pairs[(size_t)a * m->ncp + b] && !m->self_pairs[(size_t)b * m->ncp + a]) continue;
            if (h.npairs >= MAX_PAIRS) { delete s; return fail(B2G_E_UNSUPPORTED, "b2g_create: too many self-collision pairs"); }
            const int ia = std::min(inv[a], inv[b]), ib = std::max(inv[a], inv[b]);
            h.pair_list[h.npairs++] = (unsigned short)(ia | (ib << 8));
        }
        while (h.npairs % (4 * h.lanes)) { if (h.npairs >= MAX_PAIRS) { delete s; return fail(B2G_E_UNSUPPORTED, "b2g_create: too many self-collision pairs"); } h.pair_list[h.npairs++] = 0; }
        h.npairs /= 4;                                              // quads from here on
        for (int sl = 0; sl < h.ns; sl++) for (int l = 0; l < h.lanes; l++) if (h.slots[sl][l].link > 0) h.link_slot[h.slots[sl][l].link] = (l << 8) | sl;
    }
    // height field
    if (sp->hf_samples) {
        h.has_hf = 1; h.hf_nx = sp->hf_nx; h.hf_ny = sp->hf_ny;
        h.hf_scale = sp->hf_horizontal_scale; h.hf_inv_scale = 1.f / sp->hf_horizontal_scale; h.hf_vscale = sp->hf_vertical_scale;
        h.hf_ox = sp->hf_origin_x; h.hf_oy = sp->hf_origin_y;
        size_t bytes = (size_t)sp->hf_nx * sp->hf_ny * sizeof(int16_t);
        CUDA_TRY(cudaMalloc(&s->d_hf, bytes));
        CUDA_TRY(cudaMemcpy(s->d_hf, sp->hf_samples, bytes, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMalloc(&s->dm, sizeof(DevModel)));
    CUDA_TRY(cudaMemcpy(s->dm, &h, sizeof(DevModel), cudaMemcpyHostToDevice));
    s->kin_ok = kin_build(m, h.root_stride, s->hk) == 0;
    if (s->kin_ok) {
        CUDA_TRY(cudaMalloc(&s->d_kin, sizeof(KinModel)));
        CUDA_TRY(cudaMemcpy(s->d_kin, &s->hk, sizeof(KinModel), cudaMemcpyHostToDevice));
    }
    {   // the specialised path of "four hinge chains on a free base" (Ant, ANYmal): b2g_quad.cuh
        const char *nq = getenv("B2G_NO_QUAD"), *qb = getenv("B2G_QUAD_BLOCK"), *nz = getenv("B2G_NO_ZERO_COPY");
        s->no_zero_copy = nz != nullptr;
        if (const char *hc = getenv("B2G_HOSTIO_CTAS")) {      // experiment hook: resident CTAs per SM of the host-I/O Ant step (2..6)
            const int c = atoi(hc);
            if (c >= 2 && c <= 6) s->hostio_pad = (size_t)(227 * 1024 / c - 1024 - 32 * 1024) & ~(size_t)15;
        }
        if (qb && (atoi(qb) == 32 || atoi(qb) == 64 || atoi(qb) == 128)) s->quad_block = atoi(qb);
        if (!(nq && nq[0] == '1') && !ext && !h.self_on && !(force1 && force1[0] == '1') && !getenv("B2G_LANES") && !getenv("B2G_BLOCK")) {
            std::vector<float> qm; int leg_link[12], spec = 0;
            const char *nsp = getenv("B2G_QUAD_NO_SPEC");
            const int ns = quad_build(m, sp, qm, leg_link, &spec, (nsp && nsp[0] == '1') ? 0 : 3);
            s->quad_spec = spec;
            if (ns) {
                CUDA_TRY(cudaMalloc(&s->d_qm, qm.size() * sizeof(float)));
                CUDA_TRY(cudaMemcpy(s->d_qm, qm.data(), qm.size() * sizeof(float), cudaMemcpyHostToDevice));
                s->quad_ns = ns;
            }
        }
    }
    *out = s;
    return B2G_OK;
}

extern "C" int b2g_destroy(b2g_sim *s) {
    if (!s) return B2G_OK;
    cudaSetDevice(s->device);
    if (s->dm) cudaFree(s->dm);
    if (s->d_hf) cudaFree(s->d_hf);
    if (s->d_actions_stage) cudaFree(s->d_actions_stage);
    if (s->d_qm) cudaFree(s->d_qm);
    if (s->d_kin) cudaFree(s->d_kin);
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
        case B2G_T_JACOBIAN: need = (size_t)N * s->hk.rows * 6 * s->hk.nc * 4; break;
        case B2G_T_MASS_MATRIX: need = (size_t)N * s->hk.nc * s->hk.nc * 4; break;
        default: need = 0; break;   // ACTIONS / OBS / OBS_CLIPPED are checked against the task in b2g_set_task
    }
    if (ptr && bytes < need) return fail(B2G_E_INVALID, "b2g_bind: buffer smaller than the tensor's layout requires");
    s->buf.p[slot] = ptr; s->buf_bytes[slot] = bytes;
    return B2G_OK;
}

// developer switches read once per process (never on the step path)
static bool getenv_once(const char *name) {
    static std::vector<std::pair<std::string, bool>> cache;
    for (auto &kv : cache) if (kv.first == name) return kv.second;
    const char *v = getenv(name);
    cache.emplace_back(name, v && v[0] == '1');
    return cache.back().second;
}

static int require(const b2g_sim *s, std::initializer_list<int> slots, const char *who) {
    for (int k : slots) if (!s->buf.p[k]) return fail(B2G_E_UNBOUND, std::string(who) + ": tensor slot " + std::to_string(k) + " is not bound");
    return B2G_OK;
}

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
#define B2G_LAUNCH(KERNEL, ...)                                                                  \
    do {                                                                                          \
        int rc_ = set_smem(s, KERNEL, s->dyn_smem); if (rc_) return rc_;                          \
        KERNEL<<<grid, blk, s->dyn_smem, st>>>(__VA_ARGS__);                                      \
    } while (0)
// dispatch on (lanes, height field, CTA size)
#define B2G_DISPATCH_LHB(NAME, ...)                                                                                   \
    do {                                                                                                               \
        const bool hf_ = s->d_hf != nullptr;                                                                           \
        if (s->lanes == 4 && !hf_ && blk == 128) B2G_LAUNCH((NAME<4, false, 128>), __VA_ARGS__);                       \
        else if (s->lanes == 4 && hf_ && blk == 128) B2G_LAUNCH((NAME<4, true, 128>), __VA_ARGS__);                    \
        else if (s->lanes == 4 && !hf_ && blk == 64) B2G_LAUNCH((NAME<4, false, 64>), __VA_ARGS__);                    \
        else if (s->lanes == 4 && !hf_ && blk == 32) B2G_LAUNCH((NAME<4, false, 32>), __VA_ARGS__);                    \
        else if (s->lanes == 2 && !hf_ && blk == 128) B2G_LAUNCH((NAME<2, false, 128>), __VA_ARGS__);                  \
        else if (s->lanes == 2 && !hf_ && blk == 64) B2G_LAUNCH((NAME<2, false, 64>), __VA_ARGS__);                    \
        else if (s->lanes == 2 && !hf_ && blk == 32) B2G_LAUNCH((NAME<2, false, 32>), __VA_ARGS__);                    \
        else if (s->lanes == 1 && !hf_ && blk == 128) B2G_LAUNCH((NAME<1, false, 128>), __VA_ARGS__);                  \
        else if (s->lanes == 1 && !hf_ && blk == 64) B2G_LAUNCH((NAME<1, false, 64>), __VA_ARGS__);                    \
        else if (s->lanes == 1 && !hf_ && blk == 32) B2G_LAUNCH((NAME<1, false, 32>), __VA_ARGS__);                    \
        else return fail(B2G_E_UNSUPPORTED, "no kernel instantiated for this (lanes, terrain, CTA size) combination"); \
    } while (0)

extern "C" int b2g_simulate(b2g_sim *s, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "b2g_simulate: null sim");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE}, "b2g_simulate"); if (rc) return rc;
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (s->quad_ns) {
        constexpr int QB = 128;
        const int N = s->num_envs, grid = (N * 4 + QB - 1) / QB;
        const size_t dyn = ((size_t)quad_park_f4(s->quad_ns) * QB + quad_model_f4(s->quad_ns)) * sizeof(float4);
#define QSIM(NS_, HF_, SP_)                                                                                         \
        do {                                                                                                        \
            int rc_ = set_smem(s, quad_simulate_kernel<NS_, HF_, SP_, QB>, dyn); if (rc_) return rc_;               \
            quad_simulate_kernel<NS_, HF_, SP_, QB><<<grid, QB, dyn, st>>>(s->d_qm, s->d_hf, s->buf, N, s->hm.substeps); \
        } while (0)
        const bool sp3 = s->quad_spec == 3;
        if (s->quad_ns == 2 && !s->d_hf) { if (sp3) QSIM(2, false, 3); else QSIM(2, false, 0); }
        else if (s->quad_ns == 2) { if (sp3) QSIM(2, true, 3); else QSIM(2, true, 0); }
        else if (s->quad_ns == 3 && !s->d_hf) { if (sp3) QSIM(3, false, 3); else QSIM(3, false, 0); }
        else { if (sp3) QSIM(3, true, 3); else QSIM(3, true, 0); }
#undef QSIM
        s->launches++;
        CUDA_TRY(cudaGetLastError());
        return B2G_OK;
    }
    const int N = s->num_envs, blk = s->block, grid = (N * s->lanes + blk - 1) / blk;
    if (s->hm.obj_on) {
        if (s->lanes == 8 && blk == 128) B2G_LAUNCH((simulate_kernel<8, false, 128, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 8 && blk == 64) B2G_LAUNCH((simulate_kernel<8, false, 64, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 4 && blk == 128) B2G_LAUNCH((simulate_kernel<4, false, 128, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 4 && blk == 64) B2G_LAUNCH((simulate_kernel<4, false, 64, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 4 && blk == 32) B2G_LAUNCH((simulate_kernel<4, false, 32, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 1 && blk == 32) B2G_LAUNCH((simulate_kernel<1, false, 32, true>), s->dm, s->d_hf, s->buf, N);
        else return fail(B2G_E_UNSUPPORTED, "no object-enabled kernel instantiated for this (lanes, CTA size) combination");
    } else if (s->hm.self_on) {      // link-link contact: its own instantiations
        if (s->d_hf) return fail(B2G_E_UNSUPPORTED, "self-collision kernels are instantiated for the ground plane");
        if (s->lanes == 4 && blk == 128) B2G_LAUNCH((simulate_kernel<4, false, 128, false, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 4 && blk == 64) B2G_LAUNCH((simulate_kernel<4, false, 64, false, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 4 && blk == 32) B2G_LAUNCH((simulate_kernel<4, false, 32, false, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 1 && blk == 64) B2G_LAUNCH((simulate_kernel<1, false, 64, false, true>), s->dm, s->d_hf, s->buf, N);
        else if (s->lanes == 1 && blk == 32) B2G_LAUNCH((simulate_kernel<1, false, 32, false, true>), s->dm, s->d_hf, s->buf, N);
        else return fail(B2G_E_UNSUPPORTED, "no self-collision kernel instantiated for this (lanes, CTA size) combination");
    } else
        B2G_DISPATCH_LHB(simulate_kernel, s->dm, s->d_hf, s->buf, N);
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

extern "C" int b2g_refresh_rigid_body_state(b2g_sim *s, void *stream) {
    if (!s) return fail(B2G_E_INVALID, "null sim");
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_RIGID_BODY_STATE}, "b2g_refresh_rigid_body_state"); if (rc) return rc;
    CUDA_TRY(cudaSetDevice(s->device));
    const int N = s->num_envs;
    body_state_kernel<<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(s->dm, s->buf, N);
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
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
    if (s->hk.nl <= 16 && s->hk.nb <= 16) {
        const int grid = std::min((N + 2 * WARPS - 1) / (2 * WARPS), sms * 8);
        kin_tensors_kernel<WARPS, 16><<<grid, WARPS * 32, 0, (cudaStream_t)stream>>>(s->d_kin, root, dof, J, M, N);
    } else {
        const int grid = std::min((N + WARPS - 1) / WARPS, sms * 8);
        kin_tensors_kernel<WARPS, 32><<<grid, WARPS * 32, 0, (cudaStream_t)stream>>>(s->d_kin, root, dof, J, M, N);
    }
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
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
        const int link = h.body_link[b];
        int ref = -1;
        for (int sl = 0; sl < h.ns && ref < 0; sl++) for (int l = 0; l < h.lanes; l++) if (h.slots[sl][l].link == link) { ref = (l << 8) | sl; break; }
        if (ref < 0) return fail(B2G_E_UNSUPPORTED, "ShadowHand: a fingertip rides on the root link");
        H.ft_ref[f] = ref;
        for (int c = 0; c < 3; c++) H.ft_bpos[f][c] = h.body_pos[b][c];
        const float *q = h.body_quat[b];
        float x = q[0], y = q[1], z = q[2], w = q[3], n = sqrtf(x * x + y * y + z * z + w * w);
        x /= n; y /= n; z /= n; w /= n;
        const float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        memcpy(H.ft_bR[f], R, sizeof(R));
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
    cudaStream_t st = (cudaStream_t)stream;
    const int blk = s->block, grid = ((int)N * s->lanes + blk - 1) / blk;
    if (s->lanes == 8 && blk == 128) B2G_LAUNCH((hand_step_kernel<8, 128>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else if (s->lanes == 8 && blk == 64) B2G_LAUNCH((hand_step_kernel<8, 64>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else if (s->lanes == 4 && blk == 128) B2G_LAUNCH((hand_step_kernel<4, 128>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else if (s->lanes == 4 && blk == 64) B2G_LAUNCH((hand_step_kernel<4, 64>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else if (s->lanes == 4 && blk == 32) B2G_LAUNCH((hand_step_kernel<4, 32>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else if (s->lanes == 1 && blk == 32) B2G_LAUNCH((hand_step_kernel<1, 32>), s->dm, s->buf, P, s->hand_dev, actions, (int)N);
    else return fail(B2G_E_UNSUPPORTED, "no ShadowHand kernel instantiated for this (lanes, CTA size) combination");
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

static int anymal_step(b2g_sim *s, const float *actions, void *stream) {
    const b2g_anymal_params &P = s->anymal;
    int rc = require(s, {B2G_T_ROOT_STATE, B2G_T_DOF_STATE, B2G_T_OBS, B2G_T_REW, B2G_T_RESET, B2G_T_PROGRESS, B2G_T_RESET_COUNT,
                         B2G_T_ACTIONS, B2G_T_NET_CONTACT, B2G_T_COMMANDS, B2G_T_LAST_ACTIONS, B2G_T_LAST_DOF_VEL, B2G_T_FEET_AIR_TIME,
                         B2G_T_TORQUES, B2G_T_EPISODE_SUMS, B2G_T_BASE_SCRATCH, B2G_T_REDUCE_SCRATCH, B2G_T_NOISE_SCALE},
                     "b2g_task_step(AnymalTerrain)");
    if (rc) return rc;
    if (P.custom_origins) { rc = require(s, {B2G_T_ENV_ORIGINS, B2G_T_TERRAIN_LEVELS, B2G_T_TERRAIN_TYPES, B2G_T_TERRAIN_ORIGINS}, "b2g_task_step(AnymalTerrain)"); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int N = s->num_envs, blk = 128, grid = (N * 4 + blk - 1) / blk;
    if (s->block != 128) return fail(B2G_E_UNSUPPORTED, "AnymalTerrain: unexpected CTA size");
    if (grid > REDUCE_PARTIALS) return fail(B2G_E_INVALID, "AnymalTerrain: too many blocks for the reduction scratch (num_envs <= 32768)");
    if (s->buf_bytes[B2G_T_REDUCE_SCRATCH] < (REDUCE_PARTIALS + 48) * 4) return fail(B2G_E_INVALID, "REDUCE_SCRATCH too small");
    s->step_counter++;                                   // common_step_counter += 1 (:459) before the push test
    if (s->quad_ns == 3) {                               // the specialised sub-step (b2g_quad.cuh), joint state in registers
        const size_t dyn = ((size_t)quad_park_f4(3) * 128 + quad_model_f4(3)) * sizeof(float4);
        if (s->d_hf) {
            const bool dr = s->buf.p[B2G_T_ENV_MASS_SCALE] || s->buf.p[B2G_T_ENV_DOF_PROPS];
            if (dr) {
                rc = set_smem(s, quad_anymal_physics_kernel<true, 128, true>, dyn); if (rc) return rc;
                quad_anymal_physics_kernel<true, 128, true><<<grid, blk, dyn, st>>>(s->d_qm, s->d_hf, s->buf, P, actions, N, s->hm.substeps, s->step_counter);
            } else {
                rc = set_smem(s, quad_anymal_physics_kernel<true, 128, false>, dyn); if (rc) return rc;
                quad_anymal_physics_kernel<true, 128, false><<<grid, blk, dyn, st>>>(s->d_qm, s->d_hf, s->buf, P, actions, N, s->hm.substeps, s->step_counter);
            }
        } else {
            rc = set_smem(s, quad_anymal_physics_kernel<false, 128>, dyn); if (rc) return rc;
            quad_anymal_physics_kernel<false, 128><<<grid, blk, dyn, st>>>(s->d_qm, s->d_hf, s->buf, P, actions, N, s->hm.substeps, s->step_counter);
        }
    } else if (s->d_hf) {
        rc = set_smem(s, anymal_physics_kernel<4, true, 128>, s->dyn_smem); if (rc) return rc;
        anymal_physics_kernel<4, true, 128><<<grid, blk, s->dyn_smem, st>>>(s->dm, s->d_hf, s->buf, P, actions, N, s->step_counter);
    } else {
        rc = set_smem(s, anymal_physics_kernel<4, false, 128>, s->dyn_smem); if (rc) return rc;
        anymal_physics_kernel<4, false, 128><<<grid, blk, s->dyn_smem, st>>>(s->dm, s->d_hf, s->buf, P, actions, N, s->step_counter);
    }
    // kernel 2: one WARP per env -- the 140-point height gather (anymal_terrain.py:515-538) and the 188 observation
    // stores dominate it; with 4 lanes per env the 4096-env workload was 512 warps on 592 schedulers
    anymal_reset_obs_kernel<32, 128><<<(N * 32 + 127) / 128, 128, 0, st>>>(s->buf, P, s->d_hf, N, s->hm.nl - 1, grid, s->step_counter, 0);
    s->launches += 2;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

extern "C" int b2g_task_step(b2g_sim *s, const float *actions, void *stream) {
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
        if (blk != 128) return fail(B2G_E_UNSUPPORTED, "cartpole: unexpected CTA size");
        B2G_LAUNCH((cartpole_step_kernel<128>), s->dm, s->buf, P, actions, (int)N);
    } else {
        rc = require(s, {B2G_T_POTENTIALS, B2G_T_PREV_POTENTIALS, B2G_T_INITIAL_ROOT}, "b2g_task_step"); if (rc) return rc;
        const bool hum = P.task == B2G_TASK_HUMANOID;
        if (!hum && s->quad_ns == 2 && !s->d_hf) {           // Ant on the quad sub-step (whole tiles only)
            const int qb = s->quad_block, epb = qb / 4, nd_ = 8, O = P.num_obs, ns6 = 6 * s->hm.nsens;
            const bool clip_sep = s->buf.p[B2G_T_OBS_CLIPPED] && s->buf.p[B2G_T_OBS_CLIPPED] != s->buf.p[B2G_T_OBS];
            const size_t park_bytes = (size_t)quad_park_f4(2) * qb * sizeof(float4);
            const size_t io_bytes = ((size_t)epb * (13 + 3 * nd_ + ns6) * 4 + 15) & ~(size_t)15;
            const size_t out_bytes = (size_t)epb * ((clip_sep ? 2 : 1) * O * 4 + 4 * 3 + 12 * 2 + 8 * 2 + 1);
            const bool ok = (N % epb == 0) && ((epb * ns6 * 4) % 16 == 0) && ((epb * O * 4) % 16 == 0) && out_bytes <= park_bytes;
            if (ok) {
                // Host-I/O launches ask for more shared memory than they use: fewer CTAs are resident, the grid runs in several waves,
                // and a later wave computes while the PCIe writes of an earlier one drain (all CTAs of a single wave reach their
                // store phase together and the link idles while they compute).
                const size_t dyn = park_bytes + io_bytes + (size_t)quad_model_f4(2) * sizeof(float4) + (s->zero_copy.on ? s->hostio_pad : 0);
                TileArgs ta; ta.on = 1; ta.io_f4 = (int)(park_bytes / 16); ta.model_f4 = (int)((park_bytes + io_bytes) / 16);
                ta.h_act = nullptr; ta.h_obs = ta.h_rew = nullptr; ta.h_reset = nullptr; ta.h_timeout = nullptr;
                if (s->zero_copy.on) { ta.h_act = actions; ta.h_obs = s->zero_copy.obs; ta.h_rew = s->zero_copy.rew; ta.h_reset = s->zero_copy.reset; ta.h_timeout = s->zero_copy.timeout; }
                const int qgrid = (int)N / epb;
#define COMMA ,
#define QLOCO(SP_, BK, HIO)                                                                                               \
    do {                                                                                                                   \
        int rc_ = set_smem(s, quad_loco_kernel<2, SP_, BK, HIO>, dyn); if (rc_) return rc_;                                \
        cudaLaunchConfig_t lc = {};                                                                                        \
        lc.gridDim = dim3(qgrid); lc.blockDim = dim3(BK); lc.dynamicSmemBytes = dyn; lc.stream = st;                       \
        cudaLaunchAttribute at[1];                                                                                         \
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                                     \
        at[0].val.programmaticStreamSerializationAllowed = 1;                                                              \
        lc.attrs = at; lc.numAttrs = 1;                                                                                    \
        CUDA_TRY(cudaLaunchKernelEx(&lc, quad_loco_kernel<2, SP_, BK, HIO>, (const float4 *)s->d_qm, s->buf, P, actions, (int)N, (int)s->hm.substeps, ta)); \
    } while (0)
#define QLOCO_S(BK, HIO) do { if (s->quad_spec == 3) QLOCO(3, BK, HIO); else QLOCO(0, BK, HIO); } while (0)
                // the plain task (no per-env physical parameters, no dof-force / net-contact tensors acquired): the lean instantiation
                const bool lean = !s->buf.p[B2G_T_ENV_MASS_SCALE] && !s->buf.p[B2G_T_ENV_DOF_PROPS] && !s->buf.p[B2G_T_ENV_FRICTION] &&
                                  !s->buf.p[B2G_T_NET_CONTACT] && !s->buf.p[B2G_T_DOF_FORCE] && !getenv_once("B2G_NO_LEAN");
                if (qb == 128) { if (s->zero_copy.on) QLOCO_S(128, true); else QLOCO_S(128, false); }
                else if (qb == 32) { if (s->zero_copy.on) QLOCO_S(32, true); else QLOCO_S(32, false); }
                else if (s->zero_copy.on) QLOCO_S(64, true);
                else if (lean) { if (s->quad_spec == 3) QLOCO(3, 64, false COMMA true); else QLOCO(0, 64, false COMMA true); }
                else QLOCO_S(64, false);
#undef QLOCO_S
#undef QLOCO
#undef COMMA
                s->launches++;
                CUDA_TRY(cudaGetLastError());
                return B2G_OK;
            }
        }
        // tiles by bulk copy: whole blocks only, every tile a multiple of 16 bytes at a 16-byte-aligned address
        const int epb = blk / s->lanes, ndof = s->hm.nl - 1, O = P.num_obs, ns6 = 6 * s->hm.nsens;
        const bool clip_sep = s->buf.p[B2G_T_OBS_CLIPPED] && s->buf.p[B2G_T_OBS_CLIPPED] != s->buf.p[B2G_T_OBS];
        const size_t state_bytes = s->dyn_smem;                                   // slot state + accumulators
        const size_t io_bytes = ((size_t)epb * (13 + 3 * ndof + ns6 + (hum ? ndof : 0)) * 4 + 15) & ~(size_t)15;
        const size_t out_bytes = (size_t)epb * ((clip_sep ? 2 : 1) * O * 4 + 4 * 3 + 12 * 2 + 8 * 2 + 1);
        const bool tiles = (N % epb == 0) && (epb % 16 == 0) && ((epb * ndof * 4) % 16 == 0) && ((epb * ns6 * 4) % 16 == 0) &&
                           ((epb * O * 4) % 16 == 0) && out_bytes <= state_bytes && s->buf.p[B2G_T_ACTIONS];
        const size_t model_bytes = offsetof(DevModel, slots) + (size_t)s->hm.ns * MAX_LANES * sizeof(SlotRec) + (((size_t)s->hm.nl * sizeof(LinkC) + 15) & ~(size_t)15) +
                                   (((size_t)s->hm.ncp * sizeof(CpC) + 15) & ~(size_t)15);
        const size_t io_used = tiles ? io_bytes : 16;
        const size_t dyn = state_bytes + io_used + model_bytes;
        TileArgs ta; ta.on = tiles ? 1 : 0; ta.io_f4 = (int)(state_bytes / 16); ta.model_f4 = (int)((state_bytes + io_used) / 16);
        ta.h_act = nullptr; ta.h_obs = ta.h_rew = nullptr; ta.h_reset = nullptr; ta.h_timeout = nullptr;
        if (s->zero_copy.on) {
            if (!tiles) return fail(B2G_E_UNSUPPORTED, "zero-copy host step needs the tiled kernel");
            ta.h_act = actions; ta.h_obs = s->zero_copy.obs; ta.h_rew = s->zero_copy.rew; ta.h_reset = s->zero_copy.reset; ta.h_timeout = s->zero_copy.timeout;
        }
#define LOCO_T(LN, HM, BK, TL) do { if (TL && s->zero_copy.on) LOCO_K(LN, HM, BK, TL, TL); else LOCO_K(LN, HM, BK, TL, false); } while (0)
#define LOCO_K(LN, HM, BK, TL, HIO)                                                                                       \
    do {                                                                                                                   \
        int rc_ = set_smem(s, loco_step_kernel<LN, false, HM, BK, TL, HIO>, dyn); if (rc_) return rc_;                       \
        cudaLaunchConfig_t lc = {};                                                                                        \
        lc.gridDim = dim3(grid); lc.blockDim = dim3(blk); lc.dynamicSmemBytes = dyn; lc.stream = st;                       \
        cudaLaunchAttribute at[1];                                                                                         \
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                                     \
        at[0].val.programmaticStreamSerializationAllowed = 1;                                                              \
        lc.attrs = at; lc.numAttrs = 1;                                                                                    \
        CUDA_TRY(cudaLaunchKernelEx(&lc, loco_step_kernel<LN, false, HM, BK, TL, HIO>, (const DevModel *)s->dm,            \
                                    (const int16_t *)s->d_hf, s->buf, P, actions, (int)N, ta));                            \
    } while (0)
#define LOCO(LN, HM, BK) do { if (tiles) LOCO_T(LN, HM, BK, true); else LOCO_T(LN, HM, BK, false); } while (0)
        if (s->d_hf) return fail(B2G_E_UNSUPPORTED, "locomotion tasks run on the ground plane");
        if (s->hm.self_on) {             // link-link contact: separate instantiations (Humanoid-type tasks, device or staged I/O)
#define LOCO_S(BK, TL)                                                                                                     \
    do {                                                                                                                   \
        int rc_ = set_smem(s, loco_step_kernel<4, false, true, BK, TL, false, true>, dyn); if (rc_) return rc_;            \
        cudaLaunchConfig_t lc = {};                                                                                        \
        lc.gridDim = dim3(grid); lc.blockDim = dim3(blk); lc.dynamicSmemBytes = dyn; lc.stream = st;                       \
        cudaLaunchAttribute at[1];                                                                                         \
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                                     \
        at[0].val.programmaticStreamSerializationAllowed = 1;                                                              \
        lc.attrs = at; lc.numAttrs = 1;                                                                                    \
        CUDA_TRY(cudaLaunchKernelEx(&lc, loco_step_kernel<4, false, true, BK, TL, false, true>, (const DevModel *)s->dm,   \
                                    (const int16_t *)s->d_hf, s->buf, P, actions, (int)N, ta));                            \
    } while (0)
            if (!hum || s->lanes != 4 || s->zero_copy.on) return fail(B2G_E_UNSUPPORTED, "self-collision: fused step instantiated for 4-lane Humanoid-type tasks with device or staged I/O");
            if (blk == 64) { if (tiles) LOCO_S(64, true); else LOCO_S(64, false); }
            else if (blk == 32) { if (tiles) LOCO_S(32, true); else LOCO_S(32, false); }
            else return fail(B2G_E_UNSUPPORTED, "self-collision: no fused step instantiated for this CTA size");
#undef LOCO_S
        }
        else if (!hum && s->lanes == 4 && blk == 128) LOCO(4, false, 128);
        else if (!hum && s->lanes == 4 && blk == 64) LOCO(4, false, 64);
        else if (!hum && s->lanes == 1 && blk == 128) LOCO(1, false, 128);
        else if (hum && s->lanes == 4 && blk == 128) LOCO(4, true, 128);
        else if (hum && s->lanes == 4 && blk == 64) LOCO(4, true, 64);
        else if (hum && s->lanes == 4 && blk == 32) LOCO(4, true, 32);
        else if (hum && s->lanes == 2 && blk == 64) LOCO(2, true, 64);
        else if (hum && s->lanes == 2 && blk == 32) LOCO(2, true, 32);
        else if (hum && s->lanes == 1 && blk == 64) LOCO(1, true, 64);
        else if (hum && s->lanes == 1 && blk == 32) LOCO(1, true, 32);
        else return fail(B2G_E_UNSUPPORTED, "no locomotion kernel instantiated for this (lanes, CTA size) combination");
#undef LOCO
#undef LOCO_T
#undef LOCO_K
    }
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

// K x VecTask.step() with the actions of all K steps given up front (open-loop / random-action rollouts)
extern "C" int b2g_task_rollout(b2g_sim *s, const float *actions, int32_t K, float *obs_out, float *rew_out, int64_t *reset_out,
                                uint8_t *timeout_out, void *stream) {
    if (!s || !actions || !obs_out || !rew_out || !reset_out || K < 1) return fail(B2G_E_INVALID, "b2g_task_rollout: null argument or K < 1");
    if (!s->has_task && !s->has_anymal && !s->has_hand) return fail(B2G_E_INVALID, "b2g_task_rollout: call b2g_set_task first");
    const size_t N = s->num_envs;
    const bool fused = s->has_task && s->task.task == B2G_TASK_ANT && s->quad_ns == 2 && !s->d_hf && (N % 16 == 0) &&
                       ((16 * 6 * s->hm.nsens * 4) % 16 == 0);
    cudaStream_t st = (cudaStream_t)stream;
    if (!fused) {
        // every other task / shape: K single steps, their results copied into the (K, N, .) outputs (same semantics, no fusion)
        const int A = s->has_anymal ? s->anymal.num_actions : (s->has_hand ? s->hand.num_actions : s->task.num_actions);
        const int O = s->has_anymal ? s->anymal.num_obs : (s->has_hand ? s->hand.num_obs : s->task.num_obs);
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
    constexpr int QB = 64, EPB = 16;
    const int nd_ = 8, O = P.num_obs, ns6 = 6 * s->hm.nsens;
    const size_t park_f4 = (size_t)quad_park_f4(2) * QB;
    const size_t io_f4 = ((size_t)EPB * (13 + 2 * nd_ + 2 * nd_ + ns6) * 4 + 15) / 16;
    const size_t model_f4 = quad_model_f4(2);
    const size_t stage_f4 = ((size_t)EPB * (O * 4 + 4 + 8 + 1) + 15) / 16;
    if ((size_t)EPB * (O * 4 + 4 * 2 + 12 * 2 + 8) > park_f4 * 16) return fail(B2G_E_UNSUPPORTED, "b2g_task_rollout: observation too large for the last-step staging");
    RollArgs ra;
    ra.actions = actions; ra.obs_out = obs_out; ra.rew_out = rew_out; ra.reset_out = (long long *)reset_out; ra.timeout_out = timeout_out;
    ra.K = K; ra.io_f4 = (int)park_f4; ra.model_f4 = (int)(park_f4 + io_f4); ra.stage_f4 = (int)(park_f4 + io_f4 + model_f4);
    const size_t dyn = (park_f4 + io_f4 + model_f4 + stage_f4) * 16;
    const int grid = (int)N / EPB;
#define QROLL(SP_)                                                                                                         \
    do {                                                                                                                   \
        int rc_ = set_smem(s, quad_rollout_kernel<2, SP_>, dyn); if (rc_) return rc_;                                      \
        cudaLaunchConfig_t lc = {};                                                                                        \
        lc.gridDim = dim3(grid); lc.blockDim = dim3(QB); lc.dynamicSmemBytes = dyn; lc.stream = st;                        \
        cudaLaunchAttribute at[1];                                                                                         \
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                                     \
        at[0].val.programmaticStreamSerializationAllowed = 1;                                                              \
        lc.attrs = at; lc.numAttrs = 1;                                                                                    \
        CUDA_TRY(cudaLaunchKernelEx(&lc, quad_rollout_kernel<2, SP_>, (const float4 *)s->d_qm, s->buf, P, (int)N, (int)s->hm.substeps, ra)); \
    } while (0)
    if (s->quad_spec == 3) QROLL(3); else QROLL(0);
#undef QROLL
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
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
        anymal_reset_obs_kernel<32, 128><<<(N * 32 + 127) / 128, 128, 0, st>>>(s->buf, s->anymal, s->d_hf, N, nd, 0, s->step_counter, 1);
    } else if (s->has_hand) {
        rc = require(s, {B2G_T_INITIAL_ROOT, B2G_T_GOAL_STATES, B2G_T_DOF_TARGET, B2G_T_PREV_TARGETS, B2G_T_SUCCESSES, B2G_T_RESET_GOAL}, "b2g_reset_flagged(ShadowHand)"); if (rc) return rc;
        if (s->hand.force_scale > 0.f) { rc = require(s, {B2G_T_OBJ_FORCE, B2G_T_RANDOM_FORCE_PROB}, "b2g_reset_flagged(ShadowHand, forceScale > 0)"); if (rc) return rc; }
        hand_reset_kernel<<<(N + 127) / 128, 128, 0, st>>>(s->buf, s->hand, N, nd);
    } else {
        if (s->task.task != B2G_TASK_CARTPOLE) { rc = require(s, {B2G_T_POTENTIALS, B2G_T_PREV_POTENTIALS, B2G_T_INITIAL_ROOT}, "b2g_reset_flagged"); if (rc) return rc; }
        loco_reset_kernel<<<(N + 127) / 128, 128, 0, st>>>(s->buf, s->task, N, nd);
    }
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2G_OK;
}

extern "C" int b2g_task_step_host(b2g_sim *s, const float *h_actions, float *h_obs, float *h_rew, int64_t *h_reset,
                                  uint8_t *h_timeout, void *stream) {
    if (!s || !h_actions) return fail(B2G_E_INVALID, "b2g_task_step_host: null argument");
    if (!s->has_task && !s->has_anymal && !s->has_hand) return fail(B2G_E_INVALID, "b2g_task_step_host: call b2g_set_task first");
    CUDA_TRY(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int n_act = s->has_anymal ? s->anymal.num_actions : (s->has_hand ? s->hand.num_actions : s->task.num_actions);
    const int n_obs = s->has_anymal ? s->anymal.num_obs : (s->has_hand ? s->hand.num_obs : s->task.num_obs);
    const size_t N = s->num_envs, abytes = N * n_act * 4;
    // fast path (Ant / Humanoid tiled kernel, every host buffer pinned): no copy launches at all
    if (s->has_task && s->task.task != B2G_TASK_CARTPOLE && !s->no_zero_copy) {
        auto pinned = [](const void *p) {
            if (!p) return true;
            cudaPointerAttributes a;
            if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
            return a.type == cudaMemoryTypeHost;
        };
        const int epb = s->block / s->lanes, ndof = s->hm.nl - 1;
        const bool tiles_ok = (N % epb == 0) && (epb % 16 == 0) && ((epb * ndof * 4) % 16 == 0) && ((epb * 6 * s->hm.nsens * 4) % 16 == 0) &&
                              ((epb * n_obs * 4) % 16 == 0) && s->buf.p[B2G_T_ACTIONS] && !s->d_hf;
        if (tiles_ok && pinned(h_actions) && pinned(h_obs) && pinned(h_rew) && pinned(h_reset) && pinned(h_timeout)) {
            s->zero_copy.on = true; s->zero_copy.obs = h_obs; s->zero_copy.rew = h_rew;
            s->zero_copy.reset = (long long *)h_reset; s->zero_copy.timeout = h_timeout;
            int rc = b2g_task_step(s, h_actions, stream);
            s->zero_copy.on = false;
            if (rc == B2G_OK) { CUDA_TRY(cudaStreamSynchronize(st)); return B2G_OK; }
            if (rc != B2G_E_UNSUPPORTED) return rc;       // else: the generic path below
        }
    }
    if (!s->d_actions_stage) CUDA_TRY(cudaMalloc(&s->d_actions_stage, abytes));
    CUDA_TRY(cudaMemcpyAsync(s->d_actions_stage, h_actions, abytes, cudaMemcpyHostToDevice, st));
    int rc = b2g_task_step(s, s->d_actions_stage, stream); if (rc) return rc;
    const void *obs_src = s->buf.p[B2G_T_OBS_CLIPPED] ? s->buf.p[B2G_T_OBS_CLIPPED] : s->buf.p[B2G_T_OBS];
    if (h_obs) CUDA_TRY(cudaMemcpyAsync(h_obs, obs_src, N * n_obs * 4, cudaMemcpyDeviceToHost, st));
    if (h_rew) CUDA_TRY(cudaMemcpyAsync(h_rew, s->buf.p[B2G_T_REW], N * 4, cudaMemcpyDeviceToHost, st));
    if (h_reset) CUDA_TRY(cudaMemcpyAsync(h_reset, s->buf.p[B2G_T_RESET], N * 8, cudaMemcpyDeviceToHost, st));
    if (h_timeout && s->buf.p[B2G_T_TIMEOUT]) CUDA_TRY(cudaMemcpyAsync(h_timeout, s->buf.p[B2G_T_TIMEOUT], N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return B2G_OK;
}

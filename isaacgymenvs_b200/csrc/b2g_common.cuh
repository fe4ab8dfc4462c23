// b2g_common.cuh -- definitions shared by the kernel headers: the bound-tensor table, the tile descriptor of the
// bulk-copy step kernels, root-state row helpers.
#pragma once
#include "b2g_device.cuh"
#include "../../include/b200gym.h"

using namespace b2g;

struct Buffers {
    void *p[B2G_T_COUNT];
};

extern __shared__ float4 b2g_dyn_smem[];

struct TileArgs {
    int io_f4;       // float4 offset (per block) of the in/out tile region inside dynamic smem
    int model_f4;    // float4 offset of the packed model
    // b2g_task_step_host with PINNED host buffers: the kernel reads its action tile from, and writes its result tiles
    // to, host memory directly (unified addressing, plain coalesced 16-byte loads / stores -- not TMA), so the step
    // needs no separate copy launches.  Null = off.
    const float *h_act;
    float *h_obs, *h_rew;
    long long *h_reset;
    uint8_t *h_timeout;
};

__host__ __device__ constexpr uint32_t round16(uint32_t b) { return (b + 15u) & ~15u; }

// The hot part of the model a step kernel copies into shared memory, in bytes: the header with slots[0..ns), the links
// [0..nl) and the contact spheres [0..ncp), each rounded to 16 bytes (bulk copies move multiples of 16 bytes).
struct ModelHot {
    uint32_t head, links, cps;
    __host__ __device__ uint32_t total() const { return head + links + cps; }
};
__host__ __device__ inline ModelHot model_hot_bytes(int ns, int nl, int ncp) {
    return {(uint32_t)offsetof(DevModel, slots) + (uint32_t)ns * MAX_LANES * (uint32_t)sizeof(SlotRec),
            round16((uint32_t)nl * (uint32_t)sizeof(LinkC)), round16((uint32_t)ncp * (uint32_t)sizeof(CpC))};
}

// The model-only prologue of the kernels without tiles: ONE mbarrier transaction brings the hot part of the model into
// the shared DevModel (three scalar loads; everything else arrives by bulk copy).
__device__ __forceinline__ void load_model_hot(DevModel *sm, uint64_t *mbar, const DevModel *__restrict__ gm) {
    if (threadIdx.x == 0) mbar_init(mbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        const ModelHot h = model_hot_bytes(gm->ns, gm->nl, gm->ncp);
        mbar_expect_tx(mbar, h.total());
        bulk_g2s(sm, gm, h.head, mbar);
        bulk_g2s(sm->links, gm->links, h.links, mbar);
        if (h.cps) bulk_g2s(sm->cps, gm->cps, h.cps, mbar);
    }
    mbar_wait(mbar, 0);
}

// ---------------------------------------------------------------------------------------------------------------------
// The tiles of the fused Ant / Humanoid step kernels (loco_step_kernel, quad_loco_kernel, quad_rollout_kernel): every tensor
// of the step moves as ONE bulk-async (TMA) copy per block, epb envs per block, whole 16-byte-aligned tiles only.
//
// The input region, in floats: root(13) | dof(2 nd) | act(nd) x n_act | sensors(nsens6) | dof_force(nd, Humanoid only).
// n_act = 2: the rollout's double-buffered action stream.  Offsets count from the region's start (the root tile).
struct TileLayout {
    int dof, act, sens, dfrc;
    uint32_t bytes;            // the whole region, rounded to 16 bytes
};
__host__ __device__ constexpr TileLayout tile_layout(int epb, int nd, int nsens6, bool dof_force, int n_act = 1) {
    const int dof = epb * 13, act = dof + epb * 2 * nd, sens = act + epb * n_act * nd, dfrc = sens + epb * nsens6;
    return {dof, act, sens, dfrc, round16((uint32_t)(dfrc + (dof_force ? epb * nd : 0)) * 4u)};
}

// The state half of a step kernel's prologue.  griddepcontrol.wait (programmatic dependent launch: everything before it --
// barrier set-up, the model copy -- overlaps the previous step's drain; the previous step's writes are visible after it),
// then this block's root / dof tiles and, with ACT, its action tile on `mbar`.  HOSTIO: the actions come straight from
// pinned host memory instead (plain coalesced 16-byte loads).  !TILES: the wait alone.
template <int EPB, int BLOCK, bool TILES, bool HOSTIO, bool ACT = true>
__device__ __forceinline__ void load_state_tiles(uint64_t *mbar, float *io, const TileLayout &tl, const Buffers &B, int nd,
                                                 const float *actions_in, int env0, const TileArgs &ta) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (!TILES) return;
    constexpr bool dev_act = ACT && !HOSTIO;
    if (threadIdx.x == 0) {
        const uint32_t rb = EPB * 13 * 4, db = (uint32_t)(EPB * nd * 8), ab = (uint32_t)(EPB * nd * 4);
        mbar_expect_tx(mbar, rb + db + (dev_act ? ab : 0u));
        bulk_g2s(io, (const float *)B.p[B2G_T_ROOT_STATE] + (size_t)env0 * 13, rb, mbar);
        bulk_g2s(io + tl.dof, (const float *)B.p[B2G_T_DOF_STATE] + (size_t)env0 * nd * 2, db, mbar);
        if (dev_act) bulk_g2s(io + tl.act, actions_in + (size_t)env0 * nd, ab, mbar);
    }
    if (ACT && HOSTIO) {
        const float4 *src = reinterpret_cast<const float4 *>(ta.h_act + (size_t)env0 * nd);
        float4 *dst = reinterpret_cast<float4 *>(io + tl.act);
        for (int i = threadIdx.x; i < EPB * nd / 4; i += BLOCK) dst[i] = src[i];
        __syncthreads();
    }
}

// output staging of the fused Ant / Humanoid steps, epb envs per block (floats unless noted):
// obs | obs_clipped (only when it is a separate tensor) | rew | pot | ppot | up(3) | head(3) | reset(i64) | progress(i64) | timeout(u8)
struct LocoStage {
    float *obs, *obsc, *rew, *pot, *ppot, *up, *head;
    long long *reset, *prog;
    uint8_t *to;
};
__device__ __forceinline__ LocoStage loco_stage(float *base, int epb, int O, bool clip_sep) {
    LocoStage t;
    t.obs = base;
    t.obsc = t.obs + epb * O;
    t.rew = t.obsc + (clip_sep ? epb * O : 0);
    t.pot = t.rew + epb; t.ppot = t.pot + epb; t.up = t.ppot + epb; t.head = t.up + 3 * epb;
    t.reset = reinterpret_cast<long long *>(t.head + 3 * epb); t.prog = t.reset + epb;
    t.to = reinterpret_cast<uint8_t *>(t.prog + epb);
    return t;
}
__host__ __device__ inline size_t loco_stage_bytes(int epb, int O, bool clip_sep) {
    return (size_t)epb * ((clip_sep ? 2 : 1) * O * 4 + 4 * 3 + 12 * 2 + 8 * 2 + 1);
}

// lane 0's row el of the staged per-env results
__device__ __forceinline__ void stage_row(const LocoStage &t, int el, float rew, bool reset, long long progress, float pot, float ppot,
                                          const float (&up)[3], const float (&head)[3], bool timed) {
    t.rew[el] = rew; t.reset[el] = reset ? 1 : 0; t.prog[el] = progress; t.pot[el] = pot; t.ppot[el] = ppot;
    t.up[3 * el] = up[0]; t.up[3 * el + 1] = up[1]; t.up[3 * el + 2] = up[2];
    t.head[3 * el] = head[0]; t.head[3 * el + 1] = head[1]; t.head[3 * el + 2] = head[2];
    t.to[el] = timed;
}

// The drain: one bulk-async store per output tensor of this block's tiles -- the state tiles of `io` (s_act: the action
// tile, which the rollout double-buffers) and the staged results of `t`.  The stores are dealt to the FIRST THREAD of each
// of the first NW warps at compile time (`threadIdx.x == 32 w` branches, each a single-thread region the compiler keeps on
// the uniform datapath): their issue -- address arithmetic + UBLKCP each -- runs in parallel instead of as one thread's
// serial tail.
// Optional tensors are stored only when bound; the root tile only with `root` (not a fixed base), the sensor tile only
// with `stage_out` (the physics produced it), the dof-force tile only with DFRC (Humanoid) and `stage_out`.
// The host launches the tiled kernels only with EPB % 16 == 0 (the timeout tile is EPB bytes).
// commit_wait: each issuing thread commits its stores and waits until they have read shared memory; otherwise the caller
// commits (and waits before the tiles are rewritten).
template <int EPB, int NW, bool DFRC>
__device__ __forceinline__ void drain_tiles(const Buffers &B, const LocoStage &t, const float *io, const TileLayout &tl, const float *s_act,
                                            int nd, int O, int nsens6, int env0, bool root, bool stage_out, bool commit_wait) {
    static_assert(NW >= 1 && NW <= 4, "the stores are dealt to one to four warps");
    const size_t e0 = (size_t)env0;
    float *const g_obs = (float *)B.p[B2G_T_OBS];
    float *g_obsc = (float *)B.p[B2G_T_OBS_CLIPPED];
    if (g_obsc == g_obs) g_obsc = nullptr;
    float *const g_act = (float *)B.p[B2G_T_ACTIONS], *const g_sens = (float *)B.p[B2G_T_FORCE_SENSOR];
    float *const g_dfrc = (float *)B.p[B2G_T_DOF_FORCE];
    auto issue = [&](int w) {
        int k = 0;
        auto st = [&](bool cond, void *dst, const void *src, uint32_t bytes) {
            if ((k++ % NW) == w && cond) bulk_s2g(dst, src, bytes);
        };
        st(true, g_obs + e0 * O, t.obs, (uint32_t)(EPB * O * 4));
        st(g_obsc != nullptr, g_obsc + e0 * O, t.obsc, (uint32_t)(EPB * O * 4));
        st(root, (float *)B.p[B2G_T_ROOT_STATE] + e0 * 13, io, EPB * 13 * 4);
        st(true, (float *)B.p[B2G_T_DOF_STATE] + e0 * nd * 2, io + tl.dof, (uint32_t)(EPB * nd * 8));
        st(g_act != nullptr, g_act + e0 * nd, s_act, (uint32_t)(EPB * nd * 4));
        st(stage_out && g_sens && nsens6, g_sens + e0 * nsens6, io + tl.sens, (uint32_t)(EPB * nsens6 * 4));
        st(true, (float *)B.p[B2G_T_REW] + e0, t.rew, EPB * 4);
        st(true, (float *)B.p[B2G_T_POTENTIALS] + e0, t.pot, EPB * 4);
        st(true, (float *)B.p[B2G_T_PREV_POTENTIALS] + e0, t.ppot, EPB * 4);
        st(B.p[B2G_T_UP_VEC] != nullptr, (float *)B.p[B2G_T_UP_VEC] + 3 * e0, t.up, EPB * 12);
        st(B.p[B2G_T_HEADING_VEC] != nullptr, (float *)B.p[B2G_T_HEADING_VEC] + 3 * e0, t.head, EPB * 12);
        st(true, (long long *)B.p[B2G_T_RESET] + e0, t.reset, EPB * 8);
        st(true, (long long *)B.p[B2G_T_PROGRESS] + e0, t.prog, EPB * 8);
        st(B.p[B2G_T_TIMEOUT] != nullptr, (uint8_t *)B.p[B2G_T_TIMEOUT] + e0, t.to, EPB);
        if (DFRC) st(stage_out && g_dfrc, g_dfrc + e0 * nd, io + tl.dfrc, (uint32_t)(EPB * nd * 4));
        if (commit_wait) bulk_commit_wait();
    };
    if (threadIdx.x == 0) issue(0);
    else if (NW > 1 && threadIdx.x == 32) issue(1);
    else if (NW > 2 && threadIdx.x == 64) issue(2);
    else if (NW > 3 && threadIdx.x == 96) issue(3);
}

// b2g_task_step_host: what VecTask.step returns (vec_task.py:402-408), from the staging tiles straight to the pinned host
// buffers over PCIe as coalesced 16-byte stores.  Whole tiles only (epb % 16 == 0): every copy is a multiple of 16 bytes.
template <int BLOCK>
__device__ __forceinline__ void loco_copy_to_host(const TileArgs &ta, const LocoStage &t, size_t e0, int epb, int O, bool clip_sep) {
    auto copy16 = [&](void *dst, const void *src, int bytes) {
        float4 *d = reinterpret_cast<float4 *>(dst); const float4 *sp = reinterpret_cast<const float4 *>(src);
        for (int i = threadIdx.x; i < bytes / 16; i += BLOCK) d[i] = sp[i];
    };
    if (ta.h_obs) copy16(ta.h_obs + e0 * O, clip_sep ? t.obsc : t.obs, epb * O * 4);
    if (ta.h_rew) copy16(ta.h_rew + e0, t.rew, epb * 4);
    if (ta.h_reset) copy16(ta.h_reset + e0, t.reset, epb * 8);
    if (ta.h_timeout) copy16(ta.h_timeout + e0, t.to, epb);
}

__device__ __forceinline__ void load_root(const float *r, RootState &rs) {
    rs.rp[0] = r[0]; rs.rp[1] = r[1]; rs.rp[2] = r[2];
    rs.rq[0] = r[3]; rs.rq[1] = r[4]; rs.rq[2] = r[5]; rs.rq[3] = r[6];
    rs.rv[0] = r[7]; rs.rv[1] = r[8]; rs.rv[2] = r[9];
    rs.rw[0] = r[10]; rs.rw[1] = r[11]; rs.rw[2] = r[12];
}
__device__ __forceinline__ void load_obj(const float *r, ObjState &ob) {
    ob.p[0] = r[0]; ob.p[1] = r[1]; ob.p[2] = r[2];
    ob.q[0] = r[3]; ob.q[1] = r[4]; ob.q[2] = r[5]; ob.q[3] = r[6];
    ob.v[0] = r[7]; ob.v[1] = r[8]; ob.v[2] = r[9];
    ob.w[0] = r[10]; ob.w[1] = r[11]; ob.w[2] = r[12];
}
__device__ __forceinline__ void store_obj(float *r, const ObjState &ob) {
    r[0] = ob.p[0]; r[1] = ob.p[1]; r[2] = ob.p[2];
    r[3] = ob.q[0]; r[4] = ob.q[1]; r[5] = ob.q[2]; r[6] = ob.q[3];
    r[7] = ob.v[0]; r[8] = ob.v[1]; r[9] = ob.v[2];
    r[10] = ob.w[0]; r[11] = ob.w[1]; r[12] = ob.w[2];
}
__device__ __forceinline__ void store_root(float *r, const RootState &rs) {
    r[0] = rs.rp[0]; r[1] = rs.rp[1]; r[2] = rs.rp[2];
    r[3] = rs.rq[0]; r[4] = rs.rq[1]; r[5] = rs.rq[2]; r[6] = rs.rq[3];
    r[7] = rs.rv[0]; r[8] = rs.rv[1]; r[9] = rs.rv[2];
    r[10] = rs.rw[0]; r[11] = rs.rw[1]; r[12] = rs.rw[2];
}


// b2g_device.cuh -- device-side articulated-body sub-step (sm_90a).
//
// Replaces the closed `gym.simulate(sim)` (call sites tasks/base/vec_task.py:379-382,
// tasks/anymal_terrain.py:448 in the reference) with the algorithm BASELINE.json's north_star names:
// reduced-coordinate Featherstone ABA + PD/effort actuators + semi-implicit Euler + penalty contact.
//
// Formulation (differs on purpose from oracle/aba_oracle.c, which is body-coordinate ABA):
//   * all spatial quantities are expressed in WORLD-ALIGNED axes about the root link's origin O,
//     so child->parent accumulation of articulated inertias is a plain sum (no 6x6 congruence
//     transforms) and contact normals need no rotation;
//   * articulated inertia = packed symmetric 6x6: A (ang-ang, 6) | B (ang-lin, 9) | C (lin-lin, 6);
//   * every DOF is a 1-DOF link; joint damping / stiffness / PD gains / limit springs and the
//     contact spring-damper-friction are integrated implicitly by augmenting the joint-space
//     diagonal and the link inertia (DESIGN.md "time stepping").
//
// Work decomposition: an environment is owned by L lanes of a warp (L = 1, 2, 4 or 8).  Each lane runs a
// "slot program" (one 1-DOF link per step, parents before children; the host list-schedules the links
// over the lanes, b200gym.cu schedule()); the root is replicated on the L lanes and the lanes'
// contributions meet in an xor-butterfly (warp shuffles).  The three ABA sweeps are ROLLED loops over
// the slots: per-slot state (10 float4) lives in shared memory -- [slot][k][thread] (conflict-free
// 128-bit accesses) or, for the multi-actor kernels, [link][k][env] (no storage for idle slots) --
// and the articulated inertia being swept travels in registers along chains, through parked
// accumulators otherwise.  This keeps the kernel ~1/5 the code size and ~1/2 the registers of the
// fully unrolled first version.
//
// OBJ = true adds a second, free rigid body per env (a box: ShadowHand's cube) in contact with the
// articulation's spheres and box primitives and with the ground, plus fixed two-joint tendons.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#ifndef B2G_FAST_TRIG
#define B2G_FAST_TRIG 1
#endif

#define B2G_HD __host__ __device__ __forceinline__
// arithmetic-form switches (see "fused forms" below; measured in DESIGN.md section 6)
#ifndef B2G_FUSE_ADD
#define B2G_FUSE_ADD 1
#endif
#ifndef B2G_FUSE_ACC
#define B2G_FUSE_ACC 1
#endif
#ifndef B2G_RAW_RSQRT
#define B2G_RAW_RSQRT 1
#endif


namespace b2g {

constexpr int MAX_LINKS = 32;
constexpr int MAX_CP = 96;
constexpr int MAX_PAIRS = 1024; // self-collision: candidate sphere pairs
constexpr int SELF_HITS = 32;   // self-collision: overlapping pairs kept per env and sub-step (64 bytes = 4 float4)
constexpr int MAX_BOX = 4;      // box primitives of the articulation the free object's corners are tested against
constexpr int MAX_TEN = 4;      // fixed two-joint tendons
constexpr int MAX_SENS = 8;
constexpr int MAX_SLOTS = 24;
constexpr int MAX_LANES = 8;

// ---------------------------------------------------------------------------------------------
// model constants (global memory -> shared memory at kernel start; strides are odd so that the
// L lanes of an env, which read different links at the same time, hit different banks)
enum : int { LF_SLIDE = 1, LF_LIMITED = 2, LF_POSDRIVE = 4, LF_R0_IDENTITY = 8, LF_HAS_BOX = 16 };
struct LinkC {
    float R0[9];          // link frame in the parent link frame at q = 0, row-major
    float lpos[3];
    float axis[3];        // joint axis, link frame
    float com[3];
    float Ic[6];          // xx yy zz xy xz yz about the COM, link axes
    float mass;
    float armature, damping, stiffness, lower, upper, effort, kp, kd, limit_k, limit_d;
    int flags;            // LF_*
    int cp_begin, cp_end; // contact spheres of this link: [begin, end) in the link-sorted cp array
    int sensor;           // force sensor attached to this link's body (-1 none)
};                        // 39 words (odd: the L lanes of an env read different links -> different banks)
static_assert(sizeof(LinkC) == 39 * 4, "LinkC stride");

struct CpC {
    float pos[3];
    float radius, mu;
    int body;
    int pad;
};                        // 7 words
static_assert(sizeof(CpC) == 7 * 4, "CpC stride");

// One entry of a lane's slot program: which link the lane processes at sweep step s, where its
// parent lives, where its projected articulated inertia goes and which parked contributions it
// collects.  A lane may idle at a step (link < 0) while it waits for another lane's chain.
constexpr int MAX_CHILD_REFS = 4;
struct SlotRec {
    int link;                       // link index, -1 = idle
    int parent;                     // 0 = root, else ((lane << 8) | (slot + 1)) of the parent's slot
    int out;                        // -1: carried in registers to the next-lower slot of this lane (or to the root after slot 0);
                                    // else index of the accumulator (own thread column) the projected inertia is parked in
    int flags;                      // bit 0: park the acceleration after pass 3 (a child is not the next slot of this lane)
    int child[MAX_CHILD_REFS];      // parked contributions to add: ((lane << 8) | accumulator), -1 = none
};
static_assert(sizeof(SlotRec) == 32, "SlotRec");

// Hot part first (what the step kernels read) in 16-byte-aligned regions, so the model reaches shared
// memory as bulk-async copies of exactly the used bytes: header | slots[0..ns) | links[0..nl) |
// cps[0..ncp).  The cold tail is only read by the forward-kinematics kernel.
struct alignas(16) DevModel {
    int nl, ncp, nb, nsens;
    int root_fixed, gravity_on, substeps, has_hf;
    float h;              // sub-step length dt / substeps
    float g[3];
    float kn, cn, vs2;    // contact stiffness, damping, (slip regularisation speed)^2
    int hf_nx, hf_ny;
    float hf_inv_scale, hf_scale, hf_vscale, hf_ox, hf_oy;
    int ns, lanes, nacc;  // sweep steps per lane, lanes per env, accumulators per thread
    int root_acc;         // accumulator index collecting this lane's root children other than slot 0's (-1: none)
    int cross_lane;       // some slot's parent lives in another lane (needs the shared-memory handoff + __syncwarp)
    int self_on;          // link-link contacts within the articulation (tables in the cold tail below)
    int self_f4;          // float4 per env of the self-collision scratch behind the accumulator pool (0: off, or it lives in idle cells)
    int self_cell;        // self_f4 == 0: ((lane << 8) | first slot) of a run of consecutive slot cells no link occupies, the scratch's home
    float ground_mu;      // friction of the ground material (combined per contact as the average, PhysX default)
    float ang_damp, lin_damp, max_angvel;   // AssetOptions.angular_damping / linear_damping / max_angular_velocity (0: no clamp)
    float obj_ang_damp, obj_lin_damp;       // the free object's own
    // ---- optional second actor per env: a free box (ShadowHand's cube, shadow_hand.py:372-378) + fixed tendons
    int obj_on, obj_gravity_on, nbox, nten;
    float reach;          // no contact sphere can be farther than this from the root origin (ground test short-cut)
    int root_stride;      // actors per env in the root-state tensor (row of the articulation = env * root_stride)
    int obj_row;          // the object's row inside an env's actors
    int obj_acc, obj_pose_acc;             // accumulator indices: object inertia/bias sum, object pose of the sub-step
    float obj_mass, obj_I[3], obj_half[3], obj_kn, obj_cn, obj_mu, obj_g[3];
    float obj_max_angvel; // the object's AssetOptions.max_angular_velocity (0: no clamp)
    float obj_round;      // the object is the box obj_half inflated by this radius (0: block; capsule = segment + radius)
    float ten_k, ten_d;
    int box_link[MAX_BOX];
    float box_pos[MAX_BOX][3], box_R[MAX_BOX][9], box_half[MAX_BOX][3];   // link frame
    int ten_ref[MAX_TEN][2];               // ((lane << 8) | slot) of the tendon's two joints
    float ten_coef[MAX_TEN][2], ten_range[MAX_TEN][2];
    int sensor_body[MAX_SENS];
    float sensor_bpos[MAX_SENS][3];        // body-frame origin of the sensor's body in its link frame
    int link_body[MAX_LINKS];              // first body riding on the link (-1: massless virtual link)
    alignas(16) SlotRec slots[MAX_SLOTS][MAX_LANES];
    alignas(16) LinkC links[MAX_LINKS];
    alignas(16) CpC cps[MAX_CP];
    // ---- cold
    alignas(16) int body_link[MAX_LINKS];
    int link_parent[MAX_LINKS];
    float body_pos[MAX_LINKS][3];
    float body_quat[MAX_LINKS][4];
    // ---- self-collision (create_actor collision filter 0): read through the GLOBAL copy of the model (Stepper::gmodel)
    float self_kn, self_cn, self_mu;
    int npairs;                            // QUADS of candidate pairs (the list is padded to a multiple of 4 x lanes)
    int link_slot[MAX_LINKS];              // ((lane << 8) | slot) of the link's slot, -1 for the root
    alignas(8) unsigned short pair_list[MAX_PAIRS];   // (a | b << 8), link-sorted sphere indices, a < b; padding (0, 0)
};
static_assert(offsetof(DevModel, slots) % 16 == 0 && offsetof(DevModel, links) % 16 == 0 && offsetof(DevModel, cps) % 16 == 0, "bulk-copy alignment");

// ---------------------------------------------------------------------------------------------
// bulk-async (TMA) copies + mbarrier, sm_90+ PTX
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// small vector helpers (all fully inlined, arrays are register-resident after unrolling)
B2G_HD void cross(const float a[3], const float b[3], float o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
B2G_HD float dot3(const float a[3], const float b[3]) {
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}
B2G_HD void matvec(const float R[9], const float v[3], float o[3]) {
    o[0] = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
    o[1] = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
    o[2] = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
}
B2G_HD void matTvec(const float R[9], const float v[3], float o[3]) {
    o[0] = R[0] * v[0] + R[3] * v[1] + R[6] * v[2];
    o[1] = R[1] * v[0] + R[4] * v[1] + R[7] * v[2];
    o[2] = R[2] * v[0] + R[5] * v[1] + R[8] * v[2];
}
B2G_HD void matmul(const float A[9], const float B[9], float C[9]) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
            C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// 1/sqrt(x) for x that is never denormal (sums of squares with a positive floor, SPD pivots): one MUFU, no range fix-up
B2G_HD float b2g_rsqrt(float x) {
#if defined(__CUDA_ARCH__) && B2G_RAW_RSQRT
    float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
#elif defined(__CUDA_ARCH__)
    return rsqrtf(x);
#else
    return 1.0f / sqrtf(x);
#endif
}
B2G_HD void quat_to_mat(const float q[4], float R[9]) {
    float x = q[0], y = q[1], z = q[2], w = q[3];
    float inv = b2g_rsqrt(x * x + y * y + z * z + w * w);
    x *= inv; y *= inv; z *= inv; w *= inv;
    R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - z * w); R[2] = 2.f * (x * z + y * w);
    R[3] = 2.f * (x * y + z * w); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - x * w);
    R[6] = 2.f * (x * z - y * w); R[7] = 2.f * (y * z + x * w); R[8] = 1.f - 2.f * (x * x + y * y);
}
B2G_HD void mat_to_quat(const float R[9], float q[4]) {
    float t = R[0] + R[4] + R[8], s;
    if (t > 0.f) { s = sqrtf(t + 1.f) * 2.f; q[3] = 0.25f * s; q[0] = (R[7] - R[5]) / s; q[1] = (R[2] - R[6]) / s; q[2] = (R[3] - R[1]) / s; }
    else if (R[0] > R[4] && R[0] > R[8]) { s = sqrtf(1.f + R[0] - R[4] - R[8]) * 2.f; q[3] = (R[7] - R[5]) / s; q[0] = 0.25f * s; q[1] = (R[1] + R[3]) / s; q[2] = (R[2] + R[6]) / s; }
    else if (R[4] > R[8]) { s = sqrtf(1.f + R[4] - R[0] - R[8]) * 2.f; q[3] = (R[2] - R[6]) / s; q[0] = (R[1] + R[3]) / s; q[1] = 0.25f * s; q[2] = (R[5] + R[7]) / s; }
    else { s = sqrtf(1.f + R[8] - R[0] - R[4]) * 2.f; q[3] = (R[3] - R[1]) / s; q[0] = (R[2] + R[6]) / s; q[1] = (R[5] + R[7]) / s; q[2] = 0.25f * s; }
    if (q[3] < 0.f) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
}
B2G_HD void b2g_sincos(float a, float *s, float *c) {
#if B2G_FAST_TRIG && defined(__CUDA_ARCH__)
    __sincosf(a, s, c);
#else
    sincosf(a, s, c);
#endif
}

// packed symmetric 6x6:  IA[0..5] = A (xx yy zz xy xz yz), IA[6..14] = B row-major (ang x lin),
// IA[15..20] = C (xx yy zz xy xz yz).   y = IA * (a ; l)
// fused forms (one FMA per product: no separate add of a finished cross product / matrix-vector product).
// B2G_FUSE_ADD: "out = c + product" forms (shorten the dependency chain); B2G_FUSE_ACC / the FUSE template argument:
// "acc += product" forms -- fewer instructions, but the accumulator joins the dependency chain and the live range grows:
// measured +0.6 us on the register-capped Ant kernel (128 registers, 44 instead of 32 spilled floats), -2 us on ANYmal
// (196 registers, no spills), so the quad sub-step turns it on per chain length (QLane::FACC)
// out = c + a x b
B2G_HD void cross_add(const float a[3], const float b[3], const float c[3], float out[3]) {
#if B2G_FUSE_ADD
    out[0] = fmaf(a[1], b[2], fmaf(-a[2], b[1], c[0]));
    out[1] = fmaf(a[2], b[0], fmaf(-a[0], b[2], c[1]));
    out[2] = fmaf(a[0], b[1], fmaf(-a[1], b[0], c[2]));
#else
    float t[3]; cross(a, b, t);
    out[0] = c[0] + t[0]; out[1] = c[1] + t[1]; out[2] = c[2] + t[2];
#endif
}
// acc += a x b
template <bool FUSE = (B2G_FUSE_ACC != 0)>
B2G_HD void cross_acc(const float a[3], const float b[3], float acc[3]) {
    if (FUSE) {
        acc[0] = fmaf(a[1], b[2], fmaf(-a[2], b[1], acc[0]));
        acc[1] = fmaf(a[2], b[0], fmaf(-a[0], b[2], acc[1]));
        acc[2] = fmaf(a[0], b[1], fmaf(-a[1], b[0], acc[2]));
    } else {
        float t[3]; cross(a, b, t);
        acc[0] += t[0]; acc[1] += t[1]; acc[2] += t[2];
    }
}
// acc -= a x b
template <bool FUSE = (B2G_FUSE_ACC != 0)>
B2G_HD void cross_sub(const float a[3], const float b[3], float acc[3]) {
    if (FUSE) {
        acc[0] = fmaf(-a[1], b[2], fmaf(a[2], b[1], acc[0]));
        acc[1] = fmaf(-a[2], b[0], fmaf(a[0], b[2], acc[1]));
        acc[2] = fmaf(-a[0], b[1], fmaf(a[1], b[0], acc[2]));
    } else {
        float t[3]; cross(a, b, t);
        acc[0] -= t[0]; acc[1] -= t[1]; acc[2] -= t[2];
    }
}
// out = c + R v   (R row-major 3x3)
B2G_HD void matvec_add(const float R[9], const float v[3], const float c[3], float out[3]) {
#if B2G_FUSE_ADD
    out[0] = fmaf(R[0], v[0], fmaf(R[1], v[1], fmaf(R[2], v[2], c[0])));
    out[1] = fmaf(R[3], v[0], fmaf(R[4], v[1], fmaf(R[5], v[2], c[1])));
    out[2] = fmaf(R[6], v[0], fmaf(R[7], v[1], fmaf(R[8], v[2], c[2])));
#else
    float t[3]; matvec(R, v, t);
    out[0] = c[0] + t[0]; out[1] = c[1] + t[1]; out[2] = c[2] + t[2];
#endif
}
B2G_HD void sym6_mul(const float IA[21], const float a[3], const float l[3], float ya[3], float yl[3]) {
    const float *A = IA, *B = IA + 6, *C = IA + 15;
    ya[0] = A[0] * a[0] + A[3] * a[1] + A[4] * a[2] + B[0] * l[0] + B[1] * l[1] + B[2] * l[2];
    ya[1] = A[3] * a[0] + A[1] * a[1] + A[5] * a[2] + B[3] * l[0] + B[4] * l[1] + B[5] * l[2];
    ya[2] = A[4] * a[0] + A[5] * a[1] + A[2] * a[2] + B[6] * l[0] + B[7] * l[1] + B[8] * l[2];
    yl[0] = B[0] * a[0] + B[3] * a[1] + B[6] * a[2] + C[0] * l[0] + C[3] * l[1] + C[4] * l[2];
    yl[1] = B[1] * a[0] + B[4] * a[1] + B[7] * a[2] + C[3] * l[0] + C[1] * l[1] + C[5] * l[2];
    yl[2] = B[2] * a[0] + B[5] * a[1] + B[8] * a[2] + C[4] * l[0] + C[5] * l[1] + C[2] * l[2];
}
// (ya; yl) += IA (a; l)
template <bool FUSE = (B2G_FUSE_ACC != 0)>
B2G_HD void sym6_mul_acc(const float IA[21], const float a[3], const float l[3], float ya[3], float yl[3]) {
    if (FUSE) {
    const float *A = IA, *B = IA + 6, *C = IA + 15;
    ya[0] = fmaf(A[0], a[0], fmaf(A[3], a[1], fmaf(A[4], a[2], fmaf(B[0], l[0], fmaf(B[1], l[1], fmaf(B[2], l[2], ya[0]))))));
    ya[1] = fmaf(A[3], a[0], fmaf(A[1], a[1], fmaf(A[5], a[2], fmaf(B[3], l[0], fmaf(B[4], l[1], fmaf(B[5], l[2], ya[1]))))));
    ya[2] = fmaf(A[4], a[0], fmaf(A[5], a[1], fmaf(A[2], a[2], fmaf(B[6], l[0], fmaf(B[7], l[1], fmaf(B[8], l[2], ya[2]))))));
    yl[0] = fmaf(B[0], a[0], fmaf(B[3], a[1], fmaf(B[6], a[2], fmaf(C[0], l[0], fmaf(C[3], l[1], fmaf(C[4], l[2], yl[0]))))));
    yl[1] = fmaf(B[1], a[0], fmaf(B[4], a[1], fmaf(B[7], a[2], fmaf(C[3], l[0], fmaf(C[1], l[1], fmaf(C[5], l[2], yl[1]))))));
    yl[2] = fmaf(B[2], a[0], fmaf(B[5], a[1], fmaf(B[8], a[2], fmaf(C[4], l[0], fmaf(C[5], l[1], fmaf(C[2], l[2], yl[2]))))));
    } else {
    float ta[3], tl[3]; sym6_mul(IA, a, l, ta, tl);
    ya[0] += ta[0]; ya[1] += ta[1]; ya[2] += ta[2]; yl[0] += tl[0]; yl[1] += tl[1]; yl[2] += tl[2];
    }
}
// IA += s * (ja; jl)(ja; jl)^T
B2G_HD void sym6_rank1(float IA[21], float s, const float ja[3], const float jl[3]) {
    float sa0 = s * ja[0], sa1 = s * ja[1], sa2 = s * ja[2];
    float sl0 = s * jl[0], sl1 = s * jl[1], sl2 = s * jl[2];
    IA[0] += sa0 * ja[0]; IA[1] += sa1 * ja[1]; IA[2] += sa2 * ja[2];
    IA[3] += sa0 * ja[1]; IA[4] += sa0 * ja[2]; IA[5] += sa1 * ja[2];
    IA[6] += sa0 * jl[0]; IA[7] += sa0 * jl[1]; IA[8] += sa0 * jl[2];
    IA[9] += sa1 * jl[0]; IA[10] += sa1 * jl[1]; IA[11] += sa1 * jl[2];
    IA[12] += sa2 * jl[0]; IA[13] += sa2 * jl[1]; IA[14] += sa2 * jl[2];
    IA[15] += sl0 * jl[0]; IA[16] += sl1 * jl[1]; IA[17] += sl2 * jl[2];
    IA[18] += sl0 * jl[1]; IA[19] += sl0 * jl[2]; IA[20] += sl1 * jl[2];
}

// solve the SPD system  IA * (xa; xl) = (ba; bl)  (root of a floating base) by Cholesky
B2G_HD void sym6_solve(const float IA[21], const float ba[3], const float bl[3], float xa[3], float xl[3]) {
    float M[6][6];
    const float *A = IA, *B = IA + 6, *C = IA + 15;
    M[0][0] = A[0]; M[1][1] = A[1]; M[2][2] = A[2]; M[1][0] = A[3]; M[2][0] = A[4]; M[2][1] = A[5];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[3 + j][i] = B[3 * i + j];   // lower-left block = B^T
    M[3][3] = C[0]; M[4][4] = C[1]; M[5][5] = C[2]; M[4][3] = C[3]; M[5][3] = C[4]; M[5][4] = C[5];
    float Lm[6][6], dinv[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
#pragma unroll
        for (int j = 0; j <= i; j++) {
            float s = M[i][j];
#pragma unroll
            for (int k = 0; k < j; k++) s -= Lm[i][k] * Lm[j][k];
            if (i == j) { dinv[i] = b2g_rsqrt(s); Lm[i][i] = s * dinv[i]; }
            else Lm[i][j] = s * dinv[j];
        }
    }
    float b[6] = {ba[0], ba[1], ba[2], bl[0], bl[1], bl[2]}, y[6], x[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        float s = b[i];
#pragma unroll
        for (int k = 0; k < i; k++) s -= Lm[i][k] * y[k];
        y[i] = s * dinv[i];
    }
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        float s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; k++) s -= Lm[k][i] * x[k];
        x[i] = s * dinv[i];
    }
    xa[0] = x[0]; xa[1] = x[1]; xa[2] = x[2]; xl[0] = x[3]; xl[1] = x[4]; xl[2] = x[5];
}

// sphere (centre cen, radius rad) against a box (centre xb, axes Rb, half sizes hb), all in one frame:
// penetration and the unit normal from the box towards the sphere.  rad = 0 tests a point (a box corner).
__device__ __forceinline__ bool sphere_box(const float cen[3], float rad, const float xb[3], const float Rb[9], const float hb[3],
                                           float &pen, float n[3]) {
    const float d[3] = {cen[0] - xb[0], cen[1] - xb[1], cen[2] - xb[2]};
    float p[3]; matTvec(Rb, d, p);
    if (fabsf(p[0]) > hb[0] + rad || fabsf(p[1]) > hb[1] + rad || fabsf(p[2]) > hb[2] + rad) return false;
    float e[3], nl[3] = {0.f, 0.f, 0.f};
    bool inside = true;
#pragma unroll
    for (int k = 0; k < 3; k++) { const float q = fminf(fmaxf(p[k], -hb[k]), hb[k]); inside = inside && (q == p[k]); e[k] = p[k] - q; }
    if (!inside) {
        const float d2 = dot3(e, e);
        if (d2 >= rad * rad) return false;
        const float inv = rsqrtf(d2);
        pen = rad - d2 * inv; nl[0] = e[0] * inv; nl[1] = e[1] * inv; nl[2] = e[2] * inv;
    } else {
        int ax = 0; float best = hb[0] - fabsf(p[0]);
#pragma unroll
        for (int k = 1; k < 3; k++) { const float m_ = hb[k] - fabsf(p[k]); if (m_ < best) { best = m_; ax = k; } }
        pen = rad + best;
        const float sg = p[ax] >= 0.f ? 1.f : -1.f;
        nl[0] = ax == 0 ? sg : 0.f; nl[1] = ax == 1 ? sg : 0.f; nl[2] = ax == 2 ? sg : 0.f;
    }
    matvec(Rb, nl, n);
    return true;
}
// h * J^T G J of a point contact at r (about O) with G = gam*1 + (gn-gam) n n^T, added to a packed 6x6
__device__ __forceinline__ void contact_inertia(float IA[21], float h, float gam, float gn, const float r[3], const float n[3]) {
    const float hgam = h * gam;
    const float jx[3] = {0.f, r[2], -r[1]}, jy[3] = {-r[2], 0.f, r[0]}, jz[3] = {r[1], -r[0], 0.f};
    const float ex[3] = {1.f, 0.f, 0.f}, ey[3] = {0.f, 1.f, 0.f}, ez[3] = {0.f, 0.f, 1.f};
    sym6_rank1(IA, hgam, jx, ex); sym6_rank1(IA, hgam, jy, ey); sym6_rank1(IA, hgam, jz, ez);
    float rxn[3]; cross(r, n, rxn);
    sym6_rank1(IA, h * (gn - gam), rxn, n);
}

struct Ground {
    const DevModel *m;
    const int16_t *hf;
    const CpC *cps;       // contact spheres (shared memory; packed right behind the used links)
    float env_mu;         // >= 0: this env's combined friction (per-env friction buckets), else use the sphere's
    // height and unit normal at world (x, y)
    __device__ __forceinline__ void sample(float x, float y, float &h, float n[3]) const {
        if (!m->has_hf) { h = 0.f; n[0] = 0.f; n[1] = 0.f; n[2] = 1.f; return; }
        float fx = (x - m->hf_ox) * m->hf_inv_scale, fy = (y - m->hf_oy) * m->hf_inv_scale;
        int ix = (int)floorf(fx), iy = (int)floorf(fy);
        ix = max(0, min(ix, m->hf_nx - 2)); iy = max(0, min(iy, m->hf_ny - 2));
        float tx = fminf(fmaxf(fx - ix, 0.f), 1.f), ty = fminf(fmaxf(fy - iy, 0.f), 1.f);
        const int16_t *p = hf + (size_t)ix * m->hf_ny + iy;         // height samples: global memory, read-only path
        float h00 = __ldg(p) * m->hf_vscale, h01 = __ldg(p + 1) * m->hf_vscale;
        float h10 = __ldg(p + m->hf_ny) * m->hf_vscale, h11 = __ldg(p + m->hf_ny + 1) * m->hf_vscale;
        float dhx, dhy;
        if (tx + ty <= 1.f) { dhx = h10 - h00; dhy = h01 - h00; h = h00 + tx * dhx + ty * dhy; }
        else { dhx = h11 - h01; dhy = h11 - h10; h = h11 - (1.f - tx) * dhx - (1.f - ty) * dhy; }
        float gx = dhx * m->hf_inv_scale, gy = dhy * m->hf_inv_scale;
        float inv = rsqrtf(gx * gx + gy * gy + 1.f);
        n[0] = -gx * inv; n[1] = -gy * inv; n[2] = inv;
    }
};

// xor-butterfly sum over the L lanes of an env
template <int L>
__device__ __forceinline__ float lane_sum(float v) {
    if (L >= 2) v += __shfl_xor_sync(0xffffffffu, v, 1);
    if (L >= 4) v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (L >= 8) v += __shfl_xor_sync(0xffffffffu, v, 4);
    return v;
}

// ---------------------------------------------------------------------------------------------
// contact spheres of one link against the ground.  ACCUM: add the explicit force to the bias
// (pa, pl) and the implicit term h*J^T G J to IA.  !ACCUM (after the accelerations are known):
// accumulate the force actually applied over the sub-step, F = F0 - h*G*(J a), and its torque
// about the link origin.  HF=false folds the z=0 plane in (n = e_z): G = diag(gam, gam, gn).
template <bool ACCUM, bool HF>
__device__ __forceinline__ void link_contacts(const DevModel *m, const Ground &gr, const LinkC &lk, const float rp[3],
                                              const float R[9], const float x[3], const float vw[3], const float vl[3],
                                              float IA[21], float pa[3], float pl[3],
                                              const float aw[3], const float al[3], float F[3], float T[3],
                                              int cp_first, int cp_step) {
    const float h = m->h;
    const float gn = m->cn + h * m->kn;
#pragma unroll 1
    for (int k = lk.cp_begin + cp_first; k < lk.cp_end; k += cp_step) {
        const CpC &cp = gr.cps[k];
        float pc[3], lp[3] = {cp.pos[0], cp.pos[1], cp.pos[2]};
        matvec(R, lp, pc);
        pc[0] += x[0]; pc[1] += x[1]; pc[2] += x[2];          // sphere centre relative to O
        float hg = 0.f, n[3] = {0.f, 0.f, 1.f};
        if (HF) gr.sample(rp[0] + pc[0], rp[1] + pc[1], hg, n);
        const float d = HF ? cp.radius - (rp[2] + pc[2] - hg) * n[2] : cp.radius - (rp[2] + pc[2]);
        if (d <= 0.f) continue;
        float r[3];
        if (HF) { r[0] = pc[0] - cp.radius * n[0]; r[1] = pc[1] - cp.radius * n[1]; r[2] = pc[2] - cp.radius * n[2]; }
        else { r[0] = pc[0]; r[1] = pc[1]; r[2] = pc[2] - cp.radius; }
        float wxr[3]; cross(vw, r, wxr);
        const float u[3] = {vl[0] + wxr[0], vl[1] + wxr[1], vl[2] + wxr[2]};
        const float un = HF ? dot3(u, n) : u[2];
        const float Fn = m->kn * d - gn * un;
        if (Fn <= 0.f) continue;
        float ut[3];
        if (HF) { ut[0] = u[0] - un * n[0]; ut[1] = u[1] - un * n[1]; ut[2] = u[2] - un * n[2]; }
        else { ut[0] = u[0]; ut[1] = u[1]; ut[2] = 0.f; }
        const float gam = (gr.env_mu >= 0.f ? gr.env_mu : cp.mu) * Fn * rsqrtf(dot3(ut, ut) + m->vs2);
        float F0[3];
        if (HF) { F0[0] = Fn * n[0] - gam * ut[0]; F0[1] = Fn * n[1] - gam * ut[1]; F0[2] = Fn * n[2] - gam * ut[2]; }
        else { F0[0] = -gam * ut[0]; F0[1] = -gam * ut[1]; F0[2] = Fn; }
        if (ACCUM) {
            float rxF[3]; cross(r, F0, rxF);
            pa[0] -= rxF[0]; pa[1] -= rxF[1]; pa[2] -= rxF[2];
            pl[0] -= F0[0]; pl[1] -= F0[1]; pl[2] -= F0[2];
            const float hgam = h * gam;
            if (HF) {
                // J^T G J with G = gam*1 + (gn-gam) n n^T ; rows of J: j_k = (r x e_k ; e_k)
                const float jx[3] = {0.f, r[2], -r[1]}, jy[3] = {-r[2], 0.f, r[0]}, jz[3] = {r[1], -r[0], 0.f};
                const float ex[3] = {1.f, 0.f, 0.f}, ey[3] = {0.f, 1.f, 0.f}, ez[3] = {0.f, 0.f, 1.f};
                sym6_rank1(IA, hgam, jx, ex); sym6_rank1(IA, hgam, jy, ey); sym6_rank1(IA, hgam, jz, ez);
                float rxn[3]; cross(r, n, rxn);
                sym6_rank1(IA, h * (gn - gam), rxn, n);
            } else {
                // the same three rank-1 terms with G = diag(gam, gam, gn), zeros folded away
                const float hgn = h * gn, rx = r[0], ry = r[1], rz = r[2];
                IA[0] += hgam * rz * rz + hgn * ry * ry;
                IA[1] += hgam * rz * rz + hgn * rx * rx;
                IA[2] += hgam * (rx * rx + ry * ry);
                IA[3] -= hgn * rx * ry; IA[4] -= hgam * rx * rz; IA[5] -= hgam * ry * rz;
                IA[7] -= hgam * rz; IA[8] += hgn * ry;
                IA[9] += hgam * rz; IA[11] -= hgn * rx;
                IA[12] -= hgam * ry; IA[13] += hgam * rx;
                IA[15] += hgam; IA[16] += hgam; IA[17] += hgn;
            }
        } else {
            float axr[3]; cross(aw, r, axr);
            const float Ja[3] = {al[0] + axr[0], al[1] + axr[1], al[2] + axr[2]};
            float Fk[3];
            if (HF) {
                const float Jan = dot3(Ja, n);
#pragma unroll
                for (int c = 0; c < 3; c++) Fk[c] = F0[c] - h * (gam * Ja[c] + (gn - gam) * Jan * n[c]);
            } else {
                Fk[0] = F0[0] - h * gam * Ja[0]; Fk[1] = F0[1] - h * gam * Ja[1]; Fk[2] = F0[2] - h * gn * Ja[2];
            }
            const float rl[3] = {r[0] - x[0], r[1] - x[1], r[2] - x[2]};
            float t[3]; cross(rl, Fk, t);
#pragma unroll
            for (int c = 0; c < 3; c++) { F[c] += Fk[c]; T[c] += t[c]; }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// per-slot state in shared memory: 10 float4 per slot per thread, [slot][k][thread]
//  k0: R0..R3   k1: R4..R7   k2: R8 x0 x1 x2   k3: vw0 vw1 vw2 vl0   k4: vl1 vl2 w0 w1   k5: w2 sl0 sl1 sl2
//  k6: tau diag q qd   k7: act Dinv u -   k8: U0..U3   k9: U4 U5 - -
//  after pass 3 the link acceleration (aw, al) overlays k0 / k1.xy for slots with non-adjacent children
constexpr int SLOT_F4 = 10;
constexpr int ACC_F4 = 7;     // a parked articulated inertia + bias: 27 floats

struct RootState {            // replicated on the L lanes of the env
    float rp[3], rq[4], rv[3], rw[3];
};
struct ObjState {             // the free object (world frame, at its COM), replicated on the L lanes
    float p[3], q[4], v[3], w[3];
};
struct ObjPose {              // the object at the start of the sub-step, as the contacts see it: about O, world axes
    float Ro[9], c[3], w[3], vO[3];
};

// SELF: link-link contact code compiled in (the kernels instantiate it separately: the default path carries none of it)
template <int L, bool HF, int BLOCK, bool OBJ = false, bool SELF = false>
struct Stepper {
    const DevModel *m;        // header (scalars, sensor tables)
    const SlotRec *slots;     // [ns][MAX_LANES]
    const LinkC *links;
    Ground gr;
    float4 *ss;               // this thread's column of the slot-state array
    float4 *acc;              // this thread's column of the accumulator pool
    int lane;
    const DevModel *gmodel;   // the model's copy in global memory (self-collision tables), may be null when self_on == 0
    const float *dr_mass;     // per-env physical parameters (vec_task.py:720-828 as arrays; null = the model's own): this env's link-mass
    const float4 *dr_dof;     // factors [nl] (inertia scales with the mass), and per DOF (damping, stiffness, lower, upper)
    float4 *scen;             // this ENV's self-collision scratch, element i at scen[i * scs]: [0, ncp) sphere centres about O +
    int scs;                  // radius, [ncp].x hit count, [ncp + 1, ncp + 5) the overlapping pairs of this sub-step (SELF_HITS x uint16)

    // Two layouts of the per-slot state.  Default: [slot][k][thread] -- every thread owns ns rows (idle slots included),
    // 128-bit accesses are conflict-free.  OBJ (few, large environments: the shared memory per env decides how many
    // fit on the chip): [link][k][env] -- one row per LINK of the env, whichever lane processes it, so no storage
    // for idle slots; ss / acc then point at the ENV's column and accumulators carry env-wide ids.
    static constexpr int EPB = BLOCK / L;
    static constexpr int KS = OBJ ? (EPB | 1) : BLOCK;       // float4 stride between consecutive k (odd in OBJ mode: banks)
    __device__ __forceinline__ const SlotRec &rec(int s) const { return slots[s * MAX_LANES + lane]; }
    __device__ __forceinline__ int link_of(int s) const { return slots[s * MAX_LANES + lane].link; }
    __device__ __forceinline__ float4 &S4(int s, int k) const {
        return OBJ ? ss[((link_of(s) - 1) * SLOT_F4 + k) * KS] : ss[(s * SLOT_F4 + k) * KS];
    }
    // slot state of another lane of the same env (cross-lane parents)
    __device__ __forceinline__ const float4 &S4x(int ln, int s, int k) const {
        return OBJ ? ss[((slots[s * MAX_LANES + ln].link - 1) * SLOT_F4 + k) * KS] : ss[(s * SLOT_F4 + k) * KS + (ln - lane)];
    }
    __device__ __forceinline__ float4 &A4(int a, int k) const { return acc[(a * ACC_F4 + k) * KS]; }
    __device__ __forceinline__ const float4 &A4x(int ln, int a, int k) const { return OBJ ? acc[(a * ACC_F4 + k) * KS] : acc[(a * ACC_F4 + k) * KS + (ln - lane)]; }
    // accumulators every lane owns one of (OBJ layout: consecutive env-wide ids, one per lane)
    __device__ __forceinline__ int lane_acc(int a) const { return OBJ ? a + lane : a; }

    __device__ __forceinline__ void set_joint(int s, float q, float qd, float act) const {
        float4 v = S4(s, 6); v.z = q; v.w = qd; S4(s, 6) = v;
        S4(s, 7) = make_float4(act, 0.f, 0.f, 0.f);     // .w: extra explicit joint force (tendons), zero unless set per sub-step
    }
    __device__ __forceinline__ void set_act(int s, float act) const { float4 u = S4(s, 7); u.x = act; S4(s, 7) = u; }
    __device__ __forceinline__ void set_q(int s, float q, float qd) const { float4 v = S4(s, 6); v.z = q; v.w = qd; S4(s, 6) = v; }
    __device__ __forceinline__ float2 get_q(int s) const { const float4 v = S4(s, 6); return make_float2(v.z, v.w); }

    __device__ __forceinline__ void load_pose_x(int ln, int s, float R[9], float x[3], float vw[3], float vl[3]) const {
        const float4 a = S4x(ln, s, 0), b = S4x(ln, s, 1), c = S4x(ln, s, 2), d = S4x(ln, s, 3), e = S4x(ln, s, 4);
        R[0] = a.x; R[1] = a.y; R[2] = a.z; R[3] = a.w; R[4] = b.x; R[5] = b.y; R[6] = b.z; R[7] = b.w; R[8] = c.x;
        x[0] = c.y; x[1] = c.z; x[2] = c.w; vw[0] = d.x; vw[1] = d.y; vw[2] = d.z; vl[0] = d.w; vl[1] = e.x; vl[2] = e.y;
    }
    __device__ __forceinline__ void load_pose(int s, float R[9], float x[3], float vw[3], float vl[3]) const { load_pose_x(lane, s, R, x, vw, vl); }
    __device__ __forceinline__ void load_twist_x(int ln, int s, float vw[3], float vl[3]) const {
        const float4 d = S4x(ln, s, 3), e = S4x(ln, s, 4);
        vw[0] = d.x; vw[1] = d.y; vw[2] = d.z; vl[0] = d.w; vl[1] = e.x; vl[2] = e.y;
    }
    __device__ __forceinline__ void load_twist(int s, float vw[3], float vl[3]) const {
        const float4 d = S4(s, 3), e = S4(s, 4);
        vw[0] = d.x; vw[1] = d.y; vw[2] = d.z; vl[0] = d.w; vl[1] = e.x; vl[2] = e.y;
    }
    __device__ __forceinline__ void load_axis(int s, float w[3], float sl[3]) const {
        const float4 e = S4(s, 4), f = S4(s, 5);
        w[0] = e.z; w[1] = e.w; w[2] = f.x; sl[0] = f.y; sl[1] = f.z; sl[2] = f.w;
    }
    // velocity-product acceleration c = crm(v)(S qd) of a slot, from its twist and joint axis
    __device__ __forceinline__ static void bias_accel(const float vw[3], const float vl[3], const float w[3], const float sl[3],
                                                      float qd, float cw[3], float cl[3]) {
        float a1[3], a2[3], a3[3];
        cross(vw, w, a1); cross(vw, sl, a2); cross(vl, w, a3);
#pragma unroll
        for (int c = 0; c < 3; c++) { cw[c] = a1[c] * qd; cl[c] = (a2[c] + a3[c]) * qd; }
    }
    __device__ __forceinline__ void root_pose(const RootState &rs, float R[9], float vw[3], float vl[3]) const {
        quat_to_mat(rs.rq, R);
        const bool fixed = m->root_fixed != 0;
#pragma unroll
        for (int c = 0; c < 3; c++) { vw[c] = fixed ? 0.f : rs.rw[c]; vl[c] = fixed ? 0.f : rs.rv[c]; }
    }
    // lanes of an env exchange slot state through shared memory: order the accesses
    __device__ __forceinline__ void lane_sync() const { if (L > 1 && m->cross_lane) __syncwarp(); }

    // ---- self-collision (collision filter 0).  Detection once per sub-step, cooperatively: every lane writes the world centres
    // of its links' contact spheres into the env's scratch, then the lanes of the env share the flat list of candidate pairs
    // (uniform loop: no divergence between links) and append the overlapping ones -- typically none, a handful when limbs
    // touch -- to a short per-env list.  Application per link (self_apply): each link takes ITS side of a listed pair:
    // h J^T G J joins this link's inertia, -J^T F0 its bias -- implicit in its own acceleration, explicit in the partner's
    // velocity (block-Jacobi, like the hand-object contact).
    // element i of the env's scratch.  It lives in a run of slot cells that no link occupies (the [slot][k][thread] layout leaves
    // them idle: the Humanoid's arm lanes use 3 of 9 slots), i.e. at a float4 stride of BLOCK -- link-link contact then costs no
    // shared memory and no occupancy; models without such a run get it appended per env (stride 1).
    __device__ __forceinline__ float4 &SC(int i) const { return scen[i * scs]; }
    __device__ __forceinline__ void self_detect(const RootState &rs) const {
        const int ncp = m->ncp;
        if (L > 1) __syncwarp();                       // pass 1 of every lane is complete; last sub-step's readers are done
#pragma unroll 1
        for (int s = 0; s < m->ns; s++) {
            const int li = link_of(s);
            if (li < 0) continue;
            const LinkC &lk = links[li];
            if (lk.cp_end <= lk.cp_begin) continue;
            const float4 a = S4(s, 0), b = S4(s, 1), c = S4(s, 2);
            const float R[9] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x}, x[3] = {c.y, c.z, c.w};
#pragma unroll 1
            for (int n = lk.cp_begin; n < lk.cp_end; n++) {
                const CpC &cp = gr.cps[n];
                const float p[3] = {cp.pos[0], cp.pos[1], cp.pos[2]};
                float ci[3]; matvec_add(R, p, x, ci);
                SC(n) = make_float4(ci[0], ci[1], ci[2], cp.radius);
            }
        }
        if (lane == 0) {
            const LinkC &lk = links[0];
            float Rr[9]; quat_to_mat(rs.rq, Rr);
            const float xr[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
            for (int n = lk.cp_begin; n < lk.cp_end; n++) {
                const CpC &cp = gr.cps[n];
                const float p[3] = {cp.pos[0], cp.pos[1], cp.pos[2]};
                float ci[3]; matvec_add(Rr, p, xr, ci);
                SC(n) = make_float4(ci[0], ci[1], ci[2], cp.radius);
            }
            SC(ncp) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (L > 1) __syncwarp();
        unsigned *cnt = reinterpret_cast<unsigned *>(&SC(ncp));
        // 4 pairs per lane and iteration from one 64-bit load (the list is padded with (0, 0), which the d2 >= 1e-12 test rejects):
        // eight independent shared-memory loads in flight -- this loop runs at one warp per scheduler
        const int nq = __ldg(&gmodel->npairs);                       // quads
        const uint2 *quads = reinterpret_cast<const uint2 *>(gmodel->pair_list);
#pragma unroll 1
        for (int p = lane; p < nq; p += L) {
            const uint2 q = __ldg(&quads[p]);
            const unsigned pr[4] = {q.x & 0xffffu, q.x >> 16, q.y & 0xffffu, q.y >> 16};
            float4 ca[4], cb[4];
#pragma unroll
            for (int t = 0; t < 4; t++) { ca[t] = SC(pr[t] & 255u); cb[t] = SC(pr[t] >> 8); }
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const float dx = ca[t].x - cb[t].x, dy = ca[t].y - cb[t].y, dz = ca[t].z - cb[t].z, rsum = ca[t].w + cb[t].w;
                const float d2 = dx * dx + dy * dy + dz * dz;
                if (d2 < rsum * rsum && d2 >= 1e-12f) {
                    const unsigned idx = atomicAdd(cnt, 1u);
                    if (idx < (unsigned)SELF_HITS) reinterpret_cast<unsigned short *>(&SC(ncp + 1 + (idx >> 3)))[idx & 7] = (unsigned short)pr[t];
                }
            }
        }
        if (L > 1) __syncwarp();
    }
    // one side of one overlapping pair: sphere n (this link, twist vw / vl, origin x) against sphere k of link j
    template <bool ACCUM>
    __device__ __forceinline__ void self_pair(int n, int k, int j, const float x[3], const float vw[3], const float vl[3],
                                              float IA[21], float pa[3], float pl[3], const float aw[3], const float al[3],
                                              float F[3], float T[3], const RootState &rs) const {
        // gains from the reduced mass of the two links and the sub-step (dimensionless self_kn, self_cn): the half-explicit
        // block-Jacobi coupling is stable only while h^2 kn / m and h cn / m stay below ~1 for the lighter body
        const float h = m->h, smu = __ldg(&gmodel->self_mu);
        const float mi = links[gr.cps[n].pad].mass, mj = links[j].mass, mred = mi * mj / (mi + mj);
        const float skn = __ldg(&gmodel->self_kn) * mred / (h * h), gn = __ldg(&gmodel->self_cn) * mred / h + h * skn;
        const float4 ci = SC(n), cj = SC(k);
        float vwj[3], vlj[3];
        if (j == 0) {
            const bool fixed = m->root_fixed != 0;
#pragma unroll
            for (int c = 0; c < 3; c++) { vwj[c] = fixed ? 0.f : rs.rw[c]; vlj[c] = fixed ? 0.f : rs.rv[c]; }
        } else {
            const int ref = __ldg(&gmodel->link_slot[j]);
            load_twist_x(ref >> 8, ref & 255, vwj, vlj);
        }
        const float dv[3] = {ci.x - cj.x, ci.y - cj.y, ci.z - cj.z};
        const float d2 = dot3(dv, dv), rsum = ci.w + cj.w;
        const float inv = rsqrtf(d2), dist = d2 * inv, pen = rsum - dist;
        const float n_[3] = {dv[0] * inv, dv[1] * inv, dv[2] * inv};               // force on THIS link: away from the partner
        const float off = ci.w - 0.5f * pen;                                        // contact point: middle of the overlap
        const float r[3] = {ci.x - off * n_[0], ci.y - off * n_[1], ci.z - off * n_[2]};
        float ui[3], uj[3];
        cross_add(vw, r, vl, ui); cross_add(vwj, r, vlj, uj);
        const float rel[3] = {ui[0] - uj[0], ui[1] - uj[1], ui[2] - uj[2]};
        const float un = dot3(rel, n_);
        const float Fn = skn * pen - gn * un;
        if (Fn <= 0.f) return;
        const float ut[3] = {rel[0] - un * n_[0], rel[1] - un * n_[1], rel[2] - un * n_[2]};
        const float gam = smu * Fn * rsqrtf(dot3(ut, ut) + m->vs2);
        const float F0[3] = {Fn * n_[0] - gam * ut[0], Fn * n_[1] - gam * ut[1], Fn * n_[2] - gam * ut[2]};
        if (ACCUM) {
            contact_inertia(IA, h, gam, gn, r, n_);
            float rxF[3]; cross(r, F0, rxF);
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] -= rxF[c]; pl[c] -= F0[c]; }
        } else {
            float Ja[3]; cross_add(aw, r, al, Ja);
            const float Jan = dot3(Ja, n_);
            float Fk[3];
#pragma unroll
            for (int c = 0; c < 3; c++) Fk[c] = F0[c] - h * (gam * Ja[c] + (gn - gam) * Jan * n_[c]);
            const float rl[3] = {r[0] - x[0], r[1] - x[1], r[2] - x[2]};
            float tq[3]; cross(rl, Fk, tq);
#pragma unroll
            for (int c = 0; c < 3; c++) { F[c] += Fk[c]; T[c] += tq[c]; }
        }
    }
    // every listed pair one of whose spheres rides on link li
    template <bool ACCUM>
    __device__ __forceinline__ void self_apply(int li, const float x[3], const float vw[3], const float vl[3],
                                               float IA[21], float pa[3], float pl[3], const float aw[3], const float al[3],
                                               float F[3], float T[3], const RootState &rs) const {
        const int ncp = m->ncp;
        const unsigned cnt = min(*reinterpret_cast<const unsigned *>(&SC(ncp)), (unsigned)SELF_HITS);
#pragma unroll 1
        for (unsigned e = 0; e < cnt; e++) {
            const unsigned pr = reinterpret_cast<const unsigned short *>(&SC(ncp + 1 + (e >> 3)))[e & 7];
            const int a = pr & 255u, b = pr >> 8;
            const int la = gr.cps[a].pad, lb = gr.cps[b].pad;
            if (la == li) self_pair<ACCUM>(a, b, lb, x, vw, vl, IA, pa, pl, aw, al, F, T, rs);
            if (lb == li) self_pair<ACCUM>(b, a, la, x, vw, vl, IA, pa, pl, aw, al, F, T, rs);
        }
    }

    // ---- one sub-step.  LAST: also produce contact wrench / joint force outputs (see Outputs)
    struct Outputs {
        float *sensor;      // (nsens, 6) of this env or null
        float *dof_force;   // (nd) of this env or null
        float *net_contact; // (nb, 3) of this env or null
        bool write;         // env index valid
    };

    // ================= pass 1: kinematics, velocities, joint forces (root -> leaves).  Also run on its own after
    // the last sub-step by tasks that read link poses (fingertip states, shadow_hand.py:456-457)
    __device__ __forceinline__ void pass1(const RootState &rs) const {
        const float h = m->h;
        const int NS = m->ns;
        if (OBJ && m->nten > 0) {
            // fixed tendons (shared.xml:54-69): penalty spring-damper on the tendon length outside its range,
            // explicit; each end's lane computes the force of its own joint
            lane_sync();
#pragma unroll 1
            for (int t = 0; t < m->nten; t++) {
                const int r0 = m->ten_ref[t][0], r1 = m->ten_ref[t][1];
                if ((r0 >> 8) != lane && (r1 >> 8) != lane) continue;
                const float4 a = S4x(r0 >> 8, r0 & 255, 6), b = S4x(r1 >> 8, r1 & 255, 6);
                const float c0 = m->ten_coef[t][0], c1 = m->ten_coef[t][1];
                const float len = c0 * a.z + c1 * b.z, rate = c0 * a.w + c1 * b.w;
                float f = 0.f;
                if (len > m->ten_range[t][1]) f = -m->ten_k * (len - m->ten_range[t][1]) - m->ten_d * rate;
                else if (len < m->ten_range[t][0]) f = -m->ten_k * (len - m->ten_range[t][0]) - m->ten_d * rate;
                if ((r0 >> 8) == lane) { float4 u = S4(r0 & 255, 7); u.w = c0 * f; S4(r0 & 255, 7) = u; }
                if ((r1 >> 8) == lane) { float4 u = S4(r1 & 255, 7); u.w = c1 * f; S4(r1 & 255, 7) = u; }
            }
        }
        {
            float Rc[9], xc[3], vwc[3], vlc[3];      // the slot just finished; starts as the root (parent of slot 0)
            root_pose(rs, Rc, vwc, vlc);
            xc[0] = xc[1] = xc[2] = 0.f;
#pragma unroll 1
            for (int s = 0; s < NS; s++) {
                const SlotRec &sr = rec(s);
                if (sr.link >= 0) {
                    const LinkC &lk = links[sr.link];
                    const int pl_ = sr.parent >> 8, ps = (sr.parent & 255) - 1;   // parent lane / slot (ps = -1: root)
                    float Rp[9], xp[3], vwp[3], vlp[3];
                    if (ps == s - 1 && (ps < 0 || pl_ == lane)) {                 // previous slot of this lane (or root before slot 0)
#pragma unroll
                        for (int c = 0; c < 9; c++) Rp[c] = Rc[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { xp[c] = xc[c]; vwp[c] = vwc[c]; vlp[c] = vlc[c]; }
                    } else if (ps < 0) {
                        root_pose(rs, Rp, vwp, vlp);
                        xp[0] = xp[1] = xp[2] = 0.f;
                    } else {
                        load_pose_x(pl_, ps, Rp, xp, vwp, vlp);
                    }
                    const float4 jq = S4(s, 6);
                    const float q = jq.z, qd = jq.w;
                    const float4 k7in = S4(s, 7);
                    const float act = k7in.x;
                    float Rt[9], w[3], sl[3];
                    if (lk.flags & LF_R0_IDENTITY) {
#pragma unroll
                        for (int c = 0; c < 9; c++) Rt[c] = Rp[c];
                    } else {
                        matmul(Rp, lk.R0, Rt);
                    }
                    const float ax[3] = {lk.axis[0], lk.axis[1], lk.axis[2]};
                    matvec(Rt, ax, w);
                    const float lp[3] = {lk.lpos[0], lk.lpos[1], lk.lpos[2]};
                    float d[3]; matvec(Rp, lp, d);
                    if (!(lk.flags & LF_SLIDE)) {
                        float sn, cs; b2g_sincos(q, &sn, &cs);
                        const float oc = 1.f - cs;
#pragma unroll
                        for (int j = 0; j < 3; j++) {   // rotate column j of Rt about the world axis w by q
                            const float col[3] = {Rt[j], Rt[3 + j], Rt[6 + j]};
                            float wxc[3]; cross(w, col, wxc);
                            const float wd = dot3(w, col) * oc;
                            Rc[j] = col[0] * cs + wxc[0] * sn + w[0] * wd;
                            Rc[3 + j] = col[1] * cs + wxc[1] * sn + w[1] * wd;
                            Rc[6 + j] = col[2] * cs + wxc[2] * sn + w[2] * wd;
                        }
#pragma unroll
                        for (int c = 0; c < 3; c++) xc[c] = xp[c] + d[c];
                        cross(xc, w, sl);                                 // S = (w ; x x w)
#pragma unroll
                        for (int c = 0; c < 3; c++) { vwc[c] = vwp[c] + w[c] * qd; vlc[c] = vlp[c] + sl[c] * qd; }
                    } else {
#pragma unroll
                        for (int c = 0; c < 9; c++) Rc[c] = Rt[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { xc[c] = xp[c] + d[c] + w[c] * q; sl[c] = w[c]; vwc[c] = vwp[c]; vlc[c] = vlp[c] + w[c] * qd; w[c] = 0.f; }
                    }
                    // joint force: explicit part + implicit diagonal (linear terms at the end of the sub-step)
                    const float qp = q + h * qd;
                    float jd = lk.damping, jk = lk.stiffness, jlo = lk.lower, jhi = lk.upper;
                    if (dr_dof) { const float4 v = dr_dof[sr.link - 1]; jd = v.x; jk = v.y; jlo = v.z; jhi = v.w; }
                    float f = -jd * qd - jk * qp;
                    float dg = lk.armature + h * jd + h * h * jk;
                    if (lk.flags & LF_POSDRIVE) {
                        float pd = lk.kp * (act - qp) - lk.kd * qd;
                        pd = fminf(fmaxf(pd, -lk.effort), lk.effort);
                        f += pd; dg += h * lk.kd + h * h * lk.kp;
                    } else {
                        f += fminf(fmaxf(act, -lk.effort), lk.effort);
                    }
                    if (OBJ) f += k7in.w;
                    if (lk.flags & LF_LIMITED) {
                        if (q < jlo) { f += lk.limit_k * (jlo - qp) - lk.limit_d * qd; dg += h * lk.limit_d + h * h * lk.limit_k; }
                        else if (q > jhi) { f += lk.limit_k * (jhi - qp) - lk.limit_d * qd; dg += h * lk.limit_d + h * h * lk.limit_k; }
                    }
                    S4(s, 0) = make_float4(Rc[0], Rc[1], Rc[2], Rc[3]);
                    S4(s, 1) = make_float4(Rc[4], Rc[5], Rc[6], Rc[7]);
                    S4(s, 2) = make_float4(Rc[8], xc[0], xc[1], xc[2]);
                    S4(s, 3) = make_float4(vwc[0], vwc[1], vwc[2], vlc[0]);
                    S4(s, 4) = make_float4(vlc[1], vlc[2], w[0], w[1]);
                    S4(s, 5) = make_float4(w[2], sl[0], sl[1], sl[2]);
                    S4(s, 6) = make_float4(f, dg, q, qd);
                }
                lane_sync();
            }
        }
    }

    // ---- the free object as the sub-step's contacts see it (kept in this thread's accumulator column)
    __device__ __forceinline__ void obj_store_pose(const RootState &rs, const ObjState &ob) const {
        float Ro[9]; quat_to_mat(ob.q, Ro);
        const float c[3] = {ob.p[0] - rs.rp[0], ob.p[1] - rs.rp[1], ob.p[2] - rs.rp[2]};
        float wxc[3]; cross(ob.w, c, wxc);
        const int a = m->obj_pose_acc;                       // one copy per env: lane 0 writes, every lane reads
        if (L > 1) __syncwarp();                             // the previous sub-step's readers are done
        if (lane == 0) {
            A4(a, 0) = make_float4(Ro[0], Ro[1], Ro[2], Ro[3]);
            A4(a, 1) = make_float4(Ro[4], Ro[5], Ro[6], Ro[7]);
            A4(a, 2) = make_float4(Ro[8], c[0], c[1], c[2]);
            A4(a, 3) = make_float4(ob.w[0], ob.w[1], ob.w[2], ob.v[0] - wxc[0]);
            A4(a, 4) = make_float4(ob.v[1] - wxc[1], ob.v[2] - wxc[2], 0.f, 0.f);
        }
        if (L > 1) __syncwarp();
    }
    // external force on the free object, in ITS frame, at its COM (gym.apply_rigid_body_force_tensors LOCAL_SPACE), held over the
    // sub-steps that follow: parked in the free row 5 of the pose accumulator (not in registers: the hand kernels sit at the
    // register cap).  Call before the first substep(); obj_store_pose's barriers publish it to the env's lanes.
    __device__ __forceinline__ void set_obj_force(float fx, float fy, float fz) const {
        if (lane == 0) A4(m->obj_pose_acc, 5) = make_float4(fx, fy, fz, 0.f);
    }
    __device__ __forceinline__ void obj_load_pose(ObjPose &P) const {
        const int ai = m->obj_pose_acc;
        const float4 a = A4(ai, 0), b = A4(ai, 1), c = A4(ai, 2), d = A4(ai, 3), e = A4(ai, 4);
        P.Ro[0] = a.x; P.Ro[1] = a.y; P.Ro[2] = a.z; P.Ro[3] = a.w; P.Ro[4] = b.x; P.Ro[5] = b.y; P.Ro[6] = b.z; P.Ro[7] = b.w; P.Ro[8] = c.x;
        P.c[0] = c.y; P.c[1] = c.z; P.c[2] = c.w; P.w[0] = d.x; P.w[1] = d.y; P.w[2] = d.z; P.vO[0] = d.w; P.vO[1] = e.x; P.vO[2] = e.y;
    }
    // one hand-object contact at r (about O), n = unit normal of the force on the LINK, pen = penetration.
    // ACCUM: the link gets h J^T G J and -J^T F0 (IA, pa, pl); the object, whose J about O is the same, gets the same
    // inertia term and the opposite force in its accumulator (block-Jacobi: each body implicit in its own acceleration).
    // !ACCUM: the force applied to the link over the sub-step, F0 - h G (J a_link), and its torque about the link origin.
    template <bool ACCUM>
    __device__ __forceinline__ void obj_contact_point(const ObjPose &P, const float r[3], const float n[3], float pen,
                                                      const float x[3], const float vw[3], const float vl[3],
                                                      float IA[21], float pa[3], float pl[3],
                                                      const float aw[3], const float al[3], float F[3], float T[3]) const {
        const float h = m->h, gn = m->obj_cn + h * m->obj_kn;
        float wxr[3], oxr[3]; cross(vw, r, wxr); cross(P.w, r, oxr);
        const float rel[3] = {vl[0] + wxr[0] - P.vO[0] - oxr[0], vl[1] + wxr[1] - P.vO[1] - oxr[1], vl[2] + wxr[2] - P.vO[2] - oxr[2]};
        const float un = dot3(rel, n);
        const float Fn = m->obj_kn * pen - gn * un;
        if (Fn <= 0.f) return;
        const float ut[3] = {rel[0] - un * n[0], rel[1] - un * n[1], rel[2] - un * n[2]};
        const float gam = m->obj_mu * Fn * rsqrtf(dot3(ut, ut) + m->vs2);
        const float F0[3] = {Fn * n[0] - gam * ut[0], Fn * n[1] - gam * ut[1], Fn * n[2] - gam * ut[2]};
        if (ACCUM) {
            float dM[21];
#pragma unroll
            for (int c = 0; c < 21; c++) dM[c] = 0.f;
            contact_inertia(dM, h, gam, gn, r, n);
            float rxF[3]; cross(r, F0, rxF);
#pragma unroll
            for (int c = 0; c < 21; c++) IA[c] += dM[c];
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] -= rxF[c]; pl[c] -= F0[c]; }
            const int ai = lane_acc(m->obj_acc);
            float t[28];
#pragma unroll
            for (int c = 0; c < 21; c++) t[c] = dM[c];
            t[21] = rxF[0]; t[22] = rxF[1]; t[23] = rxF[2]; t[24] = F0[0]; t[25] = F0[1]; t[26] = F0[2]; t[27] = 0.f;
#pragma unroll
            for (int k = 0; k < ACC_F4; k++) {
                float4 v = A4(ai, k);
                v.x += t[4 * k]; v.y += t[4 * k + 1]; v.z += t[4 * k + 2]; v.w += t[4 * k + 3];
                A4(ai, k) = v;
            }
        } else {
            float axr[3]; cross(aw, r, axr);
            const float Ja[3] = {al[0] + axr[0], al[1] + axr[1], al[2] + axr[2]};
            const float Jan = dot3(Ja, n);
            float Fk[3];
#pragma unroll
            for (int c = 0; c < 3; c++) Fk[c] = F0[c] - h * (gam * Ja[c] + (gn - gam) * Jan * n[c]);
            const float rl[3] = {r[0] - x[0], r[1] - x[1], r[2] - x[2]};
            float tq[3]; cross(rl, Fk, tq);
#pragma unroll
            for (int c = 0; c < 3; c++) { F[c] += Fk[c]; T[c] += tq[c]; }
        }
    }
    // all contacts between one link and the object: the link's spheres against the object's box, the object's
    // corners against the link's box primitives
    template <bool ACCUM>
    __device__ __forceinline__ void obj_link_contacts(const LinkC &lk, int li, const float R[9], const float x[3],
                                                      const float vw[3], const float vl[3], float IA[21], float pa[3], float pl[3],
                                                      const float aw[3], const float al[3], float F[3], float T[3],
                                                      int cp_first, int cp_step) const {
        ObjPose P; obj_load_pose(P);
        const float hb[3] = {m->obj_half[0], m->obj_half[1], m->obj_half[2]};
        const float orad = m->obj_round;                   // read once: the sphere loop below is the hot loop of the hand kernels
#pragma unroll 1
        for (int k = lk.cp_begin + cp_first; k < lk.cp_end; k += cp_step) {
            const CpC &cp = gr.cps[k];
            float pc[3]; const float lp[3] = {cp.pos[0], cp.pos[1], cp.pos[2]};
            matvec(R, lp, pc);
            pc[0] += x[0]; pc[1] += x[1]; pc[2] += x[2];
            float pen, n[3];
            if (!sphere_box(pc, cp.radius + orad, P.c, P.Ro, hb, pen, n)) continue;     // rounded box: inflate the sphere instead
            const float r[3] = {pc[0] - cp.radius * n[0], pc[1] - cp.radius * n[1], pc[2] - cp.radius * n[2]};
            obj_contact_point<ACCUM>(P, r, n, pen, x, vw, vl, IA, pa, pl, aw, al, F, T);
        }
        if (cp_first != 0 || !(lk.flags & LF_HAS_BOX)) return;
#pragma unroll 1
        for (int b = 0; b < m->nbox; b++) {
            if (m->box_link[b] != li) continue;
            float Rwb[9], xb[3];
            matmul(R, m->box_R[b], Rwb);
            const float bp[3] = {m->box_pos[b][0], m->box_pos[b][1], m->box_pos[b][2]};
            matvec(R, bp, xb);
            xb[0] += x[0]; xb[1] += x[1]; xb[2] += x[2];
            const float bh[3] = {m->box_half[b][0], m->box_half[b][1], m->box_half[b][2]};
#pragma unroll 1
            for (int cn = 0; cn < 8; cn++) {
                if (obj_corner_dup(cn, hb)) continue;
                const float lc[3] = {(cn & 1) ? hb[0] : -hb[0], (cn & 2) ? hb[1] : -hb[1], (cn & 4) ? hb[2] : -hb[2]};
                float pc[3]; matvec(P.Ro, lc, pc);
                pc[0] += P.c[0]; pc[1] += P.c[1]; pc[2] += P.c[2];
                float pen, nout[3];
                if (!sphere_box(pc, orad, xb, Rwb, bh, pen, nout)) continue; // the corner (sphere) is inside the link's box
                const float n[3] = {-nout[0], -nout[1], -nout[2]};              // the link is pushed away from the corner
                const float rc[3] = {pc[0] + orad * n[0], pc[1] + orad * n[1], pc[2] + orad * n[2]};
                obj_contact_point<ACCUM>(P, rc, n, pen, x, vw, vl, IA, pa, pl, aw, al, F, T);
            }
        }
    }
    // corners of a degenerate box (a zero half extent: the capsule's segment has two distinct corners): keep one of each
    __device__ __forceinline__ static bool obj_corner_dup(int cn, const float hb[3]) {
        return ((cn & 1) && hb[0] == 0.f) || ((cn & 2) && hb[1] == 0.f) || ((cn & 4) && hb[2] == 0.f);
    }
    // the object's own dynamics for this sub-step: summed contact terms + ground + rigid-body terms -> 6x6 solve -> integrate
    __device__ __forceinline__ void obj_advance(const RootState &rs, ObjState &ob) const {
        const float h = m->h;
        ObjPose P; obj_load_pose(P);
        float Io[21], pao[3], plo[3];
        {
            float t[28];
#pragma unroll
            for (int k = 0; k < ACC_F4; k++) { const float4 v = A4(lane_acc(m->obj_acc), k); t[4 * k] = v.x; t[4 * k + 1] = v.y; t[4 * k + 2] = v.z; t[4 * k + 3] = v.w; }
#pragma unroll
            for (int c = 0; c < 21; c++) Io[c] = t[c];
#pragma unroll
            for (int c = 0; c < 3; c++) { pao[c] = t[21 + c]; plo[c] = t[24 + c]; }
        }
        // corners against the ground plane, dealt round-robin to the lanes
        const float gn = m->obj_cn + h * m->obj_kn, orad = m->obj_round;
        const float hbo[3] = {m->obj_half[0], m->obj_half[1], m->obj_half[2]};
#pragma unroll 1
        for (int cn = lane; cn < 8; cn += L) {
            if (obj_corner_dup(cn, hbo)) continue;
            const float lc[3] = {(cn & 1) ? hbo[0] : -hbo[0], (cn & 2) ? hbo[1] : -hbo[1], (cn & 4) ? hbo[2] : -hbo[2]};
            float r[3]; matvec(P.Ro, lc, r);
            r[0] += P.c[0]; r[1] += P.c[1]; r[2] += P.c[2];
            const float d = orad - (rs.rp[2] + r[2]);                     // the corner carries a sphere of the rounding radius
            if (d <= 0.f) continue;
            r[2] -= orad;                                                // contact point: the sphere's lowest point
            float oxr[3]; cross(P.w, r, oxr);
            const float u[3] = {P.vO[0] + oxr[0], P.vO[1] + oxr[1], P.vO[2] + oxr[2]};
            const float Fn = m->obj_kn * d - gn * u[2];
            if (Fn <= 0.f) continue;
            const float gam = m->obj_mu * Fn * rsqrtf(u[0] * u[0] + u[1] * u[1] + m->vs2);
            const float F0[3] = {-gam * u[0], -gam * u[1], Fn}, ez[3] = {0.f, 0.f, 1.f};
            contact_inertia(Io, h, gam, gn, r, ez);
            float rxF[3]; cross(r, F0, rxF);
#pragma unroll
            for (int c = 0; c < 3; c++) { pao[c] -= rxF[c]; plo[c] -= F0[c]; }
        }
#pragma unroll
        for (int c = 0; c < 21; c++) Io[c] = lane_sum<L>(Io[c]);
#pragma unroll
        for (int c = 0; c < 3; c++) { pao[c] = lane_sum<L>(pao[c]); plo[c] = lane_sum<L>(plo[c]); }
        {   // rigid-body terms about O: Icw = Ro diag(I) Ro^T
            const float *Ro = P.Ro, i0 = m->obj_I[0], i1 = m->obj_I[1], i2 = m->obj_I[2];
            float Icw[6];
            Icw[0] = i0 * Ro[0] * Ro[0] + i1 * Ro[1] * Ro[1] + i2 * Ro[2] * Ro[2];
            Icw[1] = i0 * Ro[3] * Ro[3] + i1 * Ro[4] * Ro[4] + i2 * Ro[5] * Ro[5];
            Icw[2] = i0 * Ro[6] * Ro[6] + i1 * Ro[7] * Ro[7] + i2 * Ro[8] * Ro[8];
            Icw[3] = i0 * Ro[0] * Ro[3] + i1 * Ro[1] * Ro[4] + i2 * Ro[2] * Ro[5];
            Icw[4] = i0 * Ro[0] * Ro[6] + i1 * Ro[1] * Ro[7] + i2 * Ro[2] * Ro[8];
            Icw[5] = i0 * Ro[3] * Ro[6] + i1 * Ro[4] * Ro[7] + i2 * Ro[5] * Ro[8];
            const float go[3] = {m->obj_g[0], m->obj_g[1], m->obj_g[2]};
            float I[21], qa[3], ql[3];
            spatial_inertia(m->obj_mass, 1.f, Icw, P.c, P.w, P.vO, go, I, qa, ql, m->obj_ang_damp, m->obj_lin_damp);
#pragma unroll
            for (int c = 0; c < 21; c++) Io[c] += I[c];
#pragma unroll
            for (int c = 0; c < 3; c++) { pao[c] += qa[c]; plo[c] += ql[c]; }
            // external force (object frame -> world) at the COM: wrench about O is (c x F ; F); biases carry minus the applied wrench
            const float4 fe = A4(m->obj_pose_acc, 5);
            const float fl[3] = {fe.x, fe.y, fe.z};
            float Fw[3], cxF[3];
            matvec(Ro, fl, Fw); cross(P.c, Fw, cxF);
#pragma unroll
            for (int c = 0; c < 3; c++) { pao[c] -= cxF[c]; plo[c] -= Fw[c]; }
        }
        float ao_w[3], ao_l[3];
        const float ba[3] = {-pao[0], -pao[1], -pao[2]}, bl[3] = {-plo[0], -plo[1], -plo[2]};
        sym6_solve(Io, ba, bl, ao_w, ao_l);
        // classical acceleration of the COM: a_c = a_O + alpha x c + w x v_c
        float axc[3], wxv[3]; cross(ao_w, P.c, axc); cross(ob.w, ob.v, wxv);
#pragma unroll
        for (int c = 0; c < 3; c++) { ob.w[c] += h * ao_w[c]; ob.v[c] += h * (ao_l[c] + axc[c] + wxv[c]); }
        if (m->obj_max_angvel > 0.f) {                              // the object's AssetOptions.max_angular_velocity
            const float wn2 = dot3(ob.w, ob.w);
            if (wn2 > m->obj_max_angvel * m->obj_max_angvel) { const float k = m->obj_max_angvel * rsqrtf(wn2); ob.w[0] *= k; ob.w[1] *= k; ob.w[2] *= k; }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) ob.p[c] += h * ob.v[c];
        integrate_quat(ob.q, ob.w, h);
    }
    __device__ __forceinline__ static void integrate_quat(float q[4], const float w[3], float h) {
        const float wn2 = dot3(w, w);
        float dq[4];
        if (wn2 > 1e-24f) {
            const float wn = sqrtf(wn2);
            float sn, cs; b2g_sincos(0.5f * wn * h, &sn, &cs);
            const float k = sn / wn;
            dq[0] = w[0] * k; dq[1] = w[1] * k; dq[2] = w[2] * k; dq[3] = cs;
        } else { dq[0] = 0.5f * h * w[0]; dq[1] = 0.5f * h * w[1]; dq[2] = 0.5f * h * w[2]; dq[3] = 1.f; }
        const float qx = q[0], qy = q[1], qz = q[2], qw = q[3];
        const float nq[4] = {dq[3] * qx + dq[0] * qw + dq[1] * qz - dq[2] * qy,
                             dq[3] * qy - dq[0] * qz + dq[1] * qw + dq[2] * qx,
                             dq[3] * qz + dq[0] * qy - dq[1] * qx + dq[2] * qw,
                             dq[3] * qw - dq[0] * qx - dq[1] * qy - dq[2] * qz};
        const float inv = rsqrtf(nq[0] * nq[0] + nq[1] * nq[1] + nq[2] * nq[2] + nq[3] * nq[3]);
#pragma unroll
        for (int c = 0; c < 4; c++) q[c] = nq[c] * inv;
    }

    __device__ __forceinline__ void substep(RootState &rs, const bool LAST, const Outputs &o, ObjState *ob = nullptr) const {
        const float h = m->h;
        const int NS = m->ns;
        const float g[3] = {m->g[0], m->g[1], m->g[2]};
        const bool fixed = m->root_fixed != 0;

        pass1(rs);
        // OBJ kernels (table-top manipulators): when the root is higher than the articulation can reach, skip the
        // ground scan of every link
        const bool ground = !OBJ || HF || rs.rp[2] < m->reach;
        if (OBJ) {
            obj_store_pose(rs, *ob);
#pragma unroll
            for (int k = 0; k < ACC_F4; k++) A4(lane_acc(m->obj_acc), k) = make_float4(0.f, 0.f, 0.f, 0.f);
        }

        // ================= pass 2: articulated inertias (leaves -> root)
        // A slot's projected inertia either travels in registers to the next-lower slot of the lane
        // (chains; finally from slot 0 to the root) or is parked in one of this thread's accumulators,
        // from where its parent -- possibly in another lane -- collects it (SlotRec::child).
        if (SELF && m->self_on) self_detect(rs);
        const int racc = m->root_acc >= 0 ? lane_acc(m->root_acc) : -1;
        if (racc >= 0) {
#pragma unroll
            for (int k = 0; k < ACC_F4; k++) A4(racc, k) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float IA[21], pa[3], pl[3];
#pragma unroll
        for (int c = 0; c < 21; c++) IA[c] = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) { pa[c] = 0.f; pl[c] = 0.f; }
        {
            bool carry = false;
#pragma unroll 1
            for (int s = NS - 1; s >= 0; s--) {
                const SlotRec &sr = rec(s);
                if (sr.link >= 0) {
                    const LinkC &lk = links[sr.link];
                    float R[9], x[3], vw[3], vl[3], w[3], sl[3];
                    load_pose(s, R, x, vw, vl);
                    load_axis(s, w, sl);
                    float I[21], qa[3], ql[3];
                    const float msc = dr_mass ? dr_mass[sr.link] : 1.f;
                    link_inertia(lk, lk.mass * msc, msc, R, x, vw, vl, g, I, qa, ql, m->ang_damp, m->lin_damp);
                    float dummy[3];
                    if (ground) link_contacts<true, HF>(m, gr, lk, rs.rp, R, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy, 0, 1);
                    if (OBJ) obj_link_contacts<true>(lk, sr.link, R, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy, 0, 1);
                    if (SELF && m->self_on) self_apply<true>(sr.link, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy, rs);
                    if (carry) {
#pragma unroll
                        for (int c = 0; c < 21; c++) I[c] += IA[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { qa[c] += pa[c]; ql[c] += pl[c]; }
                    }
#pragma unroll 1
                    for (int ci = 0; ci < MAX_CHILD_REFS; ci++) {
                        const int cr = sr.child[ci];
                        if (cr < 0) break;
                        float t[28];
#pragma unroll
                        for (int k = 0; k < ACC_F4; k++) { const float4 v = A4x(cr >> 8, cr & 255, k); t[4 * k] = v.x; t[4 * k + 1] = v.y; t[4 * k + 2] = v.z; t[4 * k + 3] = v.w; }
#pragma unroll
                        for (int c = 0; c < 21; c++) I[c] += t[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { qa[c] += t[21 + c]; ql[c] += t[24 + c]; }
                    }
                    const float4 k6 = S4(s, 6);
                    const float tau = k6.x, dg = k6.y;
                    float cw[3], cl[3];
                    bias_accel(vw, vl, w, sl, k6.w, cw, cl);
                    float Ua[3], Ul[3];
                    sym6_mul(I, w, sl, Ua, Ul);
                    const float D = dot3(w, Ua) + dot3(sl, Ul) + dg;
                    const float di = 1.f / D;
                    const float u_ = tau - (dot3(w, qa) + dot3(sl, ql));
                    S4(s, 8) = make_float4(Ua[0], Ua[1], Ua[2], Ul[0]);
                    S4(s, 9) = make_float4(Ul[1], Ul[2], 0.f, 0.f);
                    { float4 v = S4(s, 7); v.y = di; v.z = u_; S4(s, 7) = v; }
                    sym6_rank1(I, -di, Ua, Ul);                           // Ia = IA - U U^T / D
                    float ya[3], yl[3];
                    sym6_mul(I, cw, cl, ya, yl);
                    const float ud = u_ * di;
#pragma unroll
                    for (int c = 0; c < 3; c++) { qa[c] += ya[c] + Ua[c] * ud; ql[c] += yl[c] + Ul[c] * ud; }
                    carry = (sr.out == -1);
                    if (sr.out == -2) {
                        // child of a fixed root: nothing collects its inertia
                    } else if (carry) {
#pragma unroll
                        for (int c = 0; c < 21; c++) IA[c] = I[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { pa[c] = qa[c]; pl[c] = ql[c]; }
                    } else {
                        float t[28];
#pragma unroll
                        for (int c = 0; c < 21; c++) t[c] = I[c];
#pragma unroll
                        for (int c = 0; c < 3; c++) { t[21 + c] = qa[c]; t[24 + c] = ql[c]; }
                        t[27] = 0.f;
                        if (sr.out == m->root_acc) {                      // several root children share the root accumulator
#pragma unroll
                            for (int k = 0; k < ACC_F4; k++) {
                                float4 v = A4(racc, k);
                                v.x += t[4 * k]; v.y += t[4 * k + 1]; v.z += t[4 * k + 2]; v.w += t[4 * k + 3];
                                A4(racc, k) = v;
                            }
                        } else {
#pragma unroll
                            for (int k = 0; k < ACC_F4; k++) A4(sr.out, k) = make_float4(t[4 * k], t[4 * k + 1], t[4 * k + 2], t[4 * k + 3]);
                        }
                    }
                } else {
                    carry = false;
                }
                lane_sync();
            }
            if (!carry) {
#pragma unroll
                for (int c = 0; c < 21; c++) IA[c] = 0.f;
#pragma unroll
                for (int c = 0; c < 3; c++) { pa[c] = 0.f; pl[c] = 0.f; }
            }
        }
        // ---- root: own inertia (lane 0), its contact spheres (dealt round-robin to the lanes), butterfly, solve
        float awr[3], alr[3];
        {
            const LinkC &lk = links[0];
            const bool mine = (lane == 0);
            float I[21], qa[3], ql[3], dummy[3], Rr[9], vwr[3], vlr[3];
            const float xr[3] = {0.f, 0.f, 0.f};
            root_pose(rs, Rr, vwr, vlr);
            const float msc0 = dr_mass ? dr_mass[0] : 1.f;
            link_inertia(lk, mine ? lk.mass * msc0 : 0.f, mine ? msc0 : 0.f, Rr, xr, vwr, vlr, g, I, qa, ql, m->ang_damp, m->lin_damp);
            if (ground) link_contacts<true, HF>(m, gr, lk, rs.rp, Rr, xr, vwr, vlr, I, qa, ql, dummy, dummy, dummy, dummy, lane, L);
            if (OBJ) obj_link_contacts<true>(lk, 0, Rr, xr, vwr, vlr, I, qa, ql, dummy, dummy, dummy, dummy, lane, L);
            if (SELF && m->self_on && mine) self_apply<true>(0, xr, vwr, vlr, I, qa, ql, dummy, dummy, dummy, dummy, rs);
#pragma unroll
            for (int c = 0; c < 21; c++) IA[c] += I[c];               // IA holds slot 0's contribution (or zeros)
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] += qa[c]; pl[c] += ql[c]; }
            if (racc >= 0) {
                float t[28];
#pragma unroll
                for (int k = 0; k < ACC_F4; k++) { const float4 v = A4(racc, k); t[4 * k] = v.x; t[4 * k + 1] = v.y; t[4 * k + 2] = v.z; t[4 * k + 3] = v.w; }
#pragma unroll
                for (int c = 0; c < 21; c++) IA[c] += t[c];
#pragma unroll
                for (int c = 0; c < 3; c++) { pa[c] += t[21 + c]; pl[c] += t[24 + c]; }
            }
#pragma unroll
            for (int c = 0; c < 21; c++) IA[c] = lane_sum<L>(IA[c]);
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] = lane_sum<L>(pa[c]); pl[c] = lane_sum<L>(pl[c]); }
            if (fixed) {
#pragma unroll
                for (int c = 0; c < 3; c++) { awr[c] = 0.f; alr[c] = 0.f; }
            } else {
                const float ba[3] = {-pa[0], -pa[1], -pa[2]}, bl[3] = {-pl[0], -pl[1], -pl[2]};
                sym6_solve(IA, ba, bl, awr, alr);
            }
            if (LAST) {
                float F[3] = {0.f, 0.f, 0.f}, T[3] = {0.f, 0.f, 0.f};
                if (ground) link_contacts<false, HF>(m, gr, lk, rs.rp, Rr, xr, vwr, vlr, I, qa, ql, awr, alr, F, T, lane, L);
                if (OBJ) obj_link_contacts<false>(lk, 0, Rr, xr, vwr, vlr, I, qa, ql, awr, alr, F, T, lane, L);
                if (SELF && m->self_on && mine) self_apply<false>(0, xr, vwr, vlr, I, qa, ql, awr, alr, F, T, rs);
#pragma unroll
                for (int c = 0; c < 3; c++) { F[c] = lane_sum<L>(F[c]); T[c] = lane_sum<L>(T[c]); }
                if (lane == 0) emit_wrench(0, lk, Rr, F, T, o);
            }
        }

        // ================= pass 3: accelerations (root -> leaves), joint integration, outputs
        {
            float awc[3] = {awr[0], awr[1], awr[2]}, alc[3] = {alr[0], alr[1], alr[2]};
#pragma unroll 1
            for (int s = 0; s < NS; s++) {
                const SlotRec &sr = rec(s);
                if (sr.link >= 0) {
                    const int pl_ = sr.parent >> 8, ps = (sr.parent & 255) - 1;
                    float ap_w[3], ap_l[3];
                    if (ps == s - 1 && (ps < 0 || pl_ == lane)) {
#pragma unroll
                        for (int c = 0; c < 3; c++) { ap_w[c] = awc[c]; ap_l[c] = alc[c]; }
                    } else if (ps < 0) {
#pragma unroll
                        for (int c = 0; c < 3; c++) { ap_w[c] = awr[c]; ap_l[c] = alr[c]; }
                    } else {
                        const float4 a = S4x(pl_, ps, 8), b = S4x(pl_, ps, 9);   // parent's parked acceleration (overlays its U)
                        ap_w[0] = a.x; ap_w[1] = a.y; ap_w[2] = a.z; ap_l[0] = a.w; ap_l[1] = b.x; ap_l[2] = b.y;
                    }
                    float w[3], sl[3], vw[3], vl[3];
                    load_axis(s, w, sl);
                    load_twist(s, vw, vl);
                    const float4 k6 = S4(s, 6), k7 = S4(s, 7), k8 = S4(s, 8), k9 = S4(s, 9);
                    float cw[3], cl[3];
                    bias_accel(vw, vl, w, sl, k6.w, cw, cl);
                    const float a_w[3] = {ap_w[0] + cw[0], ap_w[1] + cw[1], ap_w[2] + cw[2]};
                    const float a_l[3] = {ap_l[0] + cl[0], ap_l[1] + cl[1], ap_l[2] + cl[2]};
                    const float Ua_ = k8.x * a_w[0] + k8.y * a_w[1] + k8.z * a_w[2] + k8.w * a_l[0] + k9.x * a_l[1] + k9.y * a_l[2];
                    const float qdd = (k7.z - Ua_) * k7.y;
#pragma unroll
                    for (int c = 0; c < 3; c++) { awc[c] = a_w[c] + w[c] * qdd; alc[c] = a_l[c] + sl[c] * qdd; }
                    const float qd = k6.w + h * qdd;
                    const float q = k6.z + h * qd;
                    S4(s, 6) = make_float4(k6.x, k6.y, q, qd);
                    if (LAST) {
                        const LinkC &lk = links[sr.link];
                        const int li = sr.link;
                        if (o.dof_force && o.write) o.dof_force[li - 1] = k6.x - (k6.y - lk.armature) * qdd;
                        if (lk.cp_end > lk.cp_begin && (lk.sensor >= 0 || o.net_contact)) {
                            float R[9], x[3], F[3] = {0.f, 0.f, 0.f}, T[3] = {0.f, 0.f, 0.f}, dI[1], d3[3];
                            load_pose(s, R, x, vw, vl);
                            if (ground) link_contacts<false, HF>(m, gr, lk, rs.rp, R, x, vw, vl, dI, d3, d3, awc, alc, F, T, 0, 1);
                            if (OBJ) obj_link_contacts<false>(lk, li, R, x, vw, vl, dI, d3, d3, awc, alc, F, T, 0, 1);
                            if (SELF && m->self_on) self_apply<false>(li, x, vw, vl, dI, d3, d3, awc, alc, F, T, rs);
                            emit_wrench(li, lk, R, F, T, o);
                        } else if (lk.sensor >= 0 || (o.net_contact && m->link_body[li] >= 0)) {
                            float R[9], x[3]; const float z[3] = {0.f, 0.f, 0.f};
                            load_pose(s, R, x, vw, vl);
                            emit_wrench(li, lk, R, z, z, o);
                        }
                    }
                    if (sr.flags & 1) {                                // a child is not the next slot of this lane: park a over U
                        S4(s, 8) = make_float4(awc[0], awc[1], awc[2], alc[0]);
                        S4(s, 9) = make_float4(alc[1], alc[2], 0.f, 0.f);
                    }
                }
                lane_sync();
            }
        }

        if (OBJ) obj_advance(rs, *ob);

        // ================= root integration (classical acceleration of the origin = spatial + w x v)
        if (!fixed) {
            float wxv[3]; cross(rs.rw, rs.rv, wxv);
#pragma unroll
            for (int c = 0; c < 3; c++) { rs.rw[c] += h * awr[c]; rs.rv[c] += h * (alr[c] + wxv[c]); }
#pragma unroll
            for (int c = 0; c < 3; c++) rs.rp[c] += h * rs.rv[c];
            if (m->max_angvel > 0.f) {                                 // AssetOptions.max_angular_velocity
                const float wn2 = dot3(rs.rw, rs.rw);
                if (wn2 > m->max_angvel * m->max_angvel) { const float k = m->max_angvel * rsqrtf(wn2); rs.rw[0] *= k; rs.rw[1] *= k; rs.rw[2] *= k; }
            }
            integrate_quat(rs.rq, rs.rw, h);
        }
    }

    // spatial inertia about O in world axes (scaled by `sc`, mass given) and the bias force
    // p = v x* (I v) - gravity wrench
    __device__ __forceinline__ static void link_inertia(const LinkC &lk, float mass, float sc, const float R[9], const float x[3],
                                                         const float vw[3], const float vl[3], const float g[3],
                                                         float I[21], float pa[3], float pl[3], float da = 0.f, float dl = 0.f) {
        const float cl_[3] = {lk.com[0], lk.com[1], lk.com[2]};
        float cw_[3]; matvec(R, cl_, cw_);
#pragma unroll
        for (int c = 0; c < 3; c++) cw_[c] += x[c];
        const float *I6 = lk.Ic;
        const float Im[9] = {I6[0], I6[3], I6[4], I6[3], I6[1], I6[5], I6[4], I6[5], I6[2]};
        float T_[9]; matmul(R, Im, T_);
        float Icw[6];
        Icw[0] = T_[0] * R[0] + T_[1] * R[1] + T_[2] * R[2];
        Icw[1] = T_[3] * R[3] + T_[4] * R[4] + T_[5] * R[5];
        Icw[2] = T_[6] * R[6] + T_[7] * R[7] + T_[8] * R[8];
        Icw[3] = T_[0] * R[3] + T_[1] * R[4] + T_[2] * R[5];
        Icw[4] = T_[0] * R[6] + T_[1] * R[7] + T_[2] * R[8];
        Icw[5] = T_[3] * R[6] + T_[4] * R[7] + T_[5] * R[8];
        spatial_inertia(mass, sc, Icw, cw_, vw, vl, g, I, pa, pl, da, dl);
    }
    // same from the rotational inertia about the COM in world axes (Icw) and the COM position about O (cw_)
    // da / dl: damping accelerations of the COM twist (AssetOptions.angular_damping / linear_damping): wrench
    // (-da Icw w ; -dl m v_c) at the COM, explicit
    __device__ __forceinline__ static void spatial_inertia(float mass, float sc, const float Icw[6], const float cw_[3],
                                                           const float vw[3], const float vl[3], const float g[3],
                                                           float I[21], float pa[3], float pl[3], float da = 0.f, float dl = 0.f) {
        const float hm[3] = {mass * cw_[0], mass * cw_[1], mass * cw_[2]};
        const float c2 = dot3(cw_, cw_);
        I[0] = sc * Icw[0] + mass * (c2 - cw_[0] * cw_[0]);
        I[1] = sc * Icw[1] + mass * (c2 - cw_[1] * cw_[1]);
        I[2] = sc * Icw[2] + mass * (c2 - cw_[2] * cw_[2]);
        I[3] = sc * Icw[3] - mass * cw_[0] * cw_[1];
        I[4] = sc * Icw[4] - mass * cw_[0] * cw_[2];
        I[5] = sc * Icw[5] - mass * cw_[1] * cw_[2];
        I[6] = 0.f; I[7] = -hm[2]; I[8] = hm[1];
        I[9] = hm[2]; I[10] = 0.f; I[11] = -hm[0];
        I[12] = -hm[1]; I[13] = hm[0]; I[14] = 0.f;
        I[15] = mass; I[16] = mass; I[17] = mass; I[18] = 0.f; I[19] = 0.f; I[20] = 0.f;
        float na[3], nf[3];
        sym6_mul(I, vw, vl, na, nf);
        float t1[3], t2[3], t3[3], hxg[3];
        cross(vw, na, t1); cross(vl, nf, t2); cross(vw, nf, t3); cross(hm, g, hxg);
#pragma unroll
        for (int c = 0; c < 3; c++) { pa[c] = t1[c] + t2[c] - hxg[c]; pl[c] = t3[c] - mass * g[c]; }
        if (da != 0.f || dl != 0.f) {
            float vxc[3]; cross(vw, cw_, vxc);
            const float f[3] = {dl * mass * (vl[0] + vxc[0]), dl * mass * (vl[1] + vxc[1]), dl * mass * (vl[2] + vxc[2])};   // minus the damping force
            const float hc[3] = {sc * (Icw[0] * vw[0] + Icw[3] * vw[1] + Icw[4] * vw[2]), sc * (Icw[3] * vw[0] + Icw[1] * vw[1] + Icw[5] * vw[2]),
                                 sc * (Icw[4] * vw[0] + Icw[5] * vw[1] + Icw[2] * vw[2])};
            float cxf[3]; cross(cw_, f, cxf);
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] += da * hc[c] + cxf[c]; pl[c] += f[c]; }
        }
    }

    // contact wrench of a link (world axes, torque about the link origin) -> force sensor (body
    // frame, torque about the body origin) and net contact force tensors
    __device__ __forceinline__ void emit_wrench(int li, const LinkC &lk, const float R[9], const float F[3], const float T[3],
                                                const Outputs &o) const {
        if (!o.write) return;
        if (lk.sensor >= 0 && o.sensor) {
            const float bp[3] = {m->sensor_bpos[lk.sensor][0], m->sensor_bpos[lk.sensor][1], m->sensor_bpos[lk.sensor][2]};
            float wb[3], bxF[3], Tb_[3], Fb[3], Tb[3];
            matvec(R, bp, wb); cross(wb, F, bxF);
            Tb_[0] = T[0] - bxF[0]; Tb_[1] = T[1] - bxF[1]; Tb_[2] = T[2] - bxF[2];
            matTvec(R, F, Fb); matTvec(R, Tb_, Tb);
            float *d = o.sensor + 6 * lk.sensor;
            d[0] = Fb[0]; d[1] = Fb[1]; d[2] = Fb[2]; d[3] = Tb[0]; d[4] = Tb[1]; d[5] = Tb[2];
        }
        if (o.net_contact && m->link_body[li] >= 0) {
            float *d = o.net_contact + 3 * m->link_body[li];
            d[0] = F[0]; d[1] = F[1]; d[2] = F[2];
        }
    }
};

}  // namespace b2g

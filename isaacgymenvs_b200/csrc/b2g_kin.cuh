// b2g_kin.cuh -- Jacobian and joint-space mass-matrix tensors (sm_90a).
//
// Stands behind gym.acquire_jacobian_tensor / acquire_mass_matrix_tensor + refresh_jacobian_tensors /
// refresh_mass_matrix_tensors (reference call sites tasks/franka_cube_stack.py:388-392,439-440; consumer: the
// operational-space controller :600-627, which reads the end effector's rows of J and the arm's block of M).
//
// Layouts (DESIGN.md 3b; the closed binary defines them, the call sites fix the fixed-base case):
//   J  (N, rows, 6, nc)   row = body (a fixed base has no row for its base body 0: `jacobian[:, joint_index]`),
//                         6 = world linear velocity of the body-frame origin (3) | world angular velocity (3),
//                         nc = nd joint columns, preceded for a FLOATING base by 6 base columns: world linear then
//                         world angular velocity of the root origin (the order the root-state tensor carries them);
//   M  (N, nc, nc)        composite-rigid-body inertia in the same coordinates, + joint armature on the diagonal.
//
// Formulation (differs on purpose from the oracle's body-coordinate CRBA with 6x6 Pluecker transforms): everything in
// WORLD-ALIGNED axes about the root origin O.  There a rigid body's inertia is ten additive numbers -- the inertia tensor
// about O (6), mass x COM offset (3), mass (1) -- so the composite inertia of a sub-tree is a plain sum over descendants,
// and M[i][j] = S_j . (Ic_i S_i) needs no transforms at all.  A joint's motion subspace about O is S = (sa ; sb) -- hinge (w ; x cross w),
// slide (0 ; w), base coordinates (unit vectors) -- so the twist of a body origin p is (sa x p + sb ; sa) for every column kind.
//
// Work decomposition: ONE WARP PER ENVIRONMENT (half a warp when links and bodies fit 16 lanes), lane = link (nl <= 32) for the kinematics / inertias, lane = body for the
// body origins, lane = output column for the fills, so every global store is a contiguous run of one output row.  Lanes
// exchange through a per-warp shared-memory scratch ordered by __syncwarp; every phase is a __host__ __device__ function
// of (lane, tables, scratch), so tests/kin_host.cu runs the exact device arithmetic on the CPU against the fp64 oracle.
#pragma once
#include "b2g_device.cuh"

namespace b2g {

constexpr int KIN_MAX_CHILD = 8;

// constant tables of one articulation (built on the host by kin_build, b2g_kin_host.h)
struct alignas(16) KinModel {
    int nl, nb, nbase, nc;          // links, bodies, base columns (0 fixed / 6 floating), columns
    int rows, row0;                 // Jacobian rows, first body with a row (1 for a fixed base)
    int maxdepth, root_stride;      // tree depth; actors per env in the root-state tensor
    int parent[MAX_LINKS], depth[MAX_LINKS], slide[MAX_LINKS], body_link[MAX_LINKS];
    unsigned anc[MAX_LINKS];        // bit j set: link j (j >= 1) is link i itself or one of its ancestors
    int nchild[MAX_LINKS], child[MAX_LINKS][KIN_MAX_CHILD];
    float R0[MAX_LINKS][9], lpos[MAX_LINKS][3], axis[MAX_LINKS][3], com[MAX_LINKS][3], Ic[MAX_LINKS][6];
    float mass[MAX_LINKS], armature[MAX_LINKS], body_pos[MAX_LINKS][3];
};

// per-warp scratch.  Everything a phase hands to another lane is packed into float4 rows: the first version
// kept the LSU pipe busy with 32-bit shared loads -- one 128-bit load moves four of them.  Lane-indexed accesses at a stride of 3 float4 (12 words) are conflict-free per quarter-warp.
struct KinScratch {
    float4 Rx[MAX_LINKS][3];        // row k: (R[k][0], R[k][1], R[k][2], x[k]) -- link frame in world axes, origin relative to the root origin O
    float4 S[MAX_LINKS][3];         // (n.xyz, f.x) (f.yz, sa.xy) (sa.z, sb.xyz): Ic_i S_i = (n ; f) and the motion subspace S = (sa ; sb) about O
    float4 in[MAX_LINKS][3];        // inertia about O: (Ixx Iyy Izz Ixy) (Ixz Iyz mcx mcy) (mcz m - -) -- the link's own, then its sub-tree's
    float4 pb[MAX_LINKS];           // body-frame origin relative to O; .w = the ancestor mask of the body's link (bits)
    float4 cb[3];                   // composite inertia of the whole articulation (base block of M), layout of `in`
};

B2G_HD float kin_u2f(unsigned u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
B2G_HD unsigned kin_f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    unsigned u; memcpy(&u, &f, 4); return u;
#endif
}
B2G_HD void kin_load_Rx(const KinScratch &s, int i, float R[9], float x[3]) {
    const float4 a = s.Rx[i][0], b = s.Rx[i][1], c = s.Rx[i][2];
    R[0] = a.x; R[1] = a.y; R[2] = a.z; R[3] = b.x; R[4] = b.y; R[5] = b.z; R[6] = c.x; R[7] = c.y; R[8] = c.z;
    x[0] = a.w; x[1] = b.w; x[2] = c.w;
}
B2G_HD void kin_store_Rx(KinScratch &s, int i, const float R[9], const float x[3]) {
    s.Rx[i][0] = make_float4(R[0], R[1], R[2], x[0]);
    s.Rx[i][1] = make_float4(R[3], R[4], R[5], x[1]);
    s.Rx[i][2] = make_float4(R[6], R[7], R[8], x[2]);
}
B2G_HD void kin_load_in(const float4 v[3], float a[10]) {
    a[0] = v[0].x; a[1] = v[0].y; a[2] = v[0].z; a[3] = v[0].w; a[4] = v[1].x; a[5] = v[1].y; a[6] = v[1].z; a[7] = v[1].w; a[8] = v[2].x; a[9] = v[2].y;
}
B2G_HD void kin_store_in(float4 v[3], const float a[10]) {
    v[0] = make_float4(a[0], a[1], a[2], a[3]); v[1] = make_float4(a[4], a[5], a[6], a[7]); v[2] = make_float4(a[8], a[9], 0.f, 0.f);
}
// the packed (n ; f ; sa ; sb) of link i
struct KinS { float n[3], f[3], sa[3], sb[3]; };
B2G_HD KinS kin_load_S(const KinScratch &s, int i) {
    const float4 a = s.S[i][0], b = s.S[i][1], c = s.S[i][2];
    KinS r;
    r.n[0] = a.x; r.n[1] = a.y; r.n[2] = a.z; r.f[0] = a.w; r.f[1] = b.x; r.f[2] = b.y;
    r.sa[0] = b.z; r.sa[1] = b.w; r.sa[2] = c.x; r.sb[0] = c.y; r.sb[1] = c.z; r.sb[2] = c.w;
    return r;
}
B2G_HD void kin_store_S(KinScratch &s, int i, const KinS &r) {
    s.S[i][0] = make_float4(r.n[0], r.n[1], r.n[2], r.f[0]);
    s.S[i][1] = make_float4(r.f[1], r.f[2], r.sa[0], r.sa[1]);
    s.S[i][2] = make_float4(r.sa[2], r.sb[0], r.sb[1], r.sb[2]);
}

// ---- phase 0: joint transform of link i in its parent's frame -> scratch (overwritten by the world frame in phase 1)
B2G_HD void kin_local(int i, const KinModel &t, KinScratch &s, const float *root, float q) {
    if (i == 0) {
        const float rq[4] = {root[3], root[4], root[5], root[6]};
        float R[9];
        // plain normalisation (not the raw rsqrt of the step kernels: this is not a hot loop)
        const float n = 1.0f / sqrtf(rq[0] * rq[0] + rq[1] * rq[1] + rq[2] * rq[2] + rq[3] * rq[3]);
        const float x = rq[0] * n, y = rq[1] * n, z = rq[2] * n, w = rq[3] * n;
        R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - z * w); R[2] = 2.f * (x * z + y * w);
        R[3] = 2.f * (x * y + z * w); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - x * w);
        R[6] = 2.f * (x * z - y * w); R[7] = 2.f * (y * z + x * w); R[8] = 1.f - 2.f * (x * x + y * y);
        const float zero[3] = {0.f, 0.f, 0.f};
        kin_store_Rx(s, 0, R, zero);
        return;
    }
    const float *R0 = t.R0[i], *ax = t.axis[i];
    if (!t.slide[i]) {
        float sn, cs; sincosf(q, &sn, &cs);
        const float oc = 1.f - cs, ux = ax[0], uy = ax[1], uz = ax[2];
        const float Rj[9] = {cs + ux * ux * oc, ux * uy * oc - uz * sn, ux * uz * oc + uy * sn,
                             uy * ux * oc + uz * sn, cs + uy * uy * oc, uy * uz * oc - ux * sn,
                             uz * ux * oc - uy * sn, uz * uy * oc + ux * sn, cs + uz * uz * oc};
        float R[9]; matmul(R0, Rj, R);
        const float lp[3] = {t.lpos[i][0], t.lpos[i][1], t.lpos[i][2]};
        kin_store_Rx(s, i, R, lp);
    } else {
        float d[3]; matvec(R0, ax, d);
        const float R[9] = {R0[0], R0[1], R0[2], R0[3], R0[4], R0[5], R0[6], R0[7], R0[8]};
        const float lp[3] = {t.lpos[i][0] + d[0] * q, t.lpos[i][1] + d[1] * q, t.lpos[i][2] + d[2] * q};
        kin_store_Rx(s, i, R, lp);
    }
}

// ---- phase 1 (once per tree level d = 1 .. maxdepth): compose with the parent's world frame
B2G_HD void kin_level_do(int i, int p, KinScratch &s) {
    float Rp[9], xp[3], Rl[9], r[3], R[9], wr[3];
    kin_load_Rx(s, p, Rp, xp); kin_load_Rx(s, i, Rl, r);
    matmul(Rp, Rl, R); matvec(Rp, r, wr);
    const float x[3] = {xp[0] + wr[0], xp[1] + wr[1], xp[2] + wr[2]};
    kin_store_Rx(s, i, R, x);
}
B2G_HD void kin_level(int i, int d, const KinModel &t, KinScratch &s) {
    if (i < t.nl && t.depth[i] == d) kin_level_do(i, t.parent[i], s);
}

// ---- phase 2: world joint axis, motion subspace, the link's own inertia about O
B2G_HD void kin_link(int i, const KinModel &t, KinScratch &s) {
    float R[9], x[3], w[3];
    KinS S;
#pragma unroll
    for (int c = 0; c < 3; c++) { S.n[c] = S.f[c] = S.sa[c] = S.sb[c] = 0.f; }
    kin_load_Rx(s, i, R, x);
    if (i > 0) {
        const float ax[3] = {t.axis[i][0], t.axis[i][1], t.axis[i][2]};
        matvec(R, ax, w);
        if (!t.slide[i]) { cross(x, w, S.sb); S.sa[0] = w[0]; S.sa[1] = w[1]; S.sa[2] = w[2]; }
        else { S.sb[0] = w[0]; S.sb[1] = w[1]; S.sb[2] = w[2]; }
    }
    kin_store_S(s, i, S);
    // inertia about the COM in world axes: R Ic R^T, then the parallel-axis term to O
    const float *I6 = t.Ic[i];
    const float Il[9] = {I6[0], I6[3], I6[4], I6[3], I6[1], I6[5], I6[4], I6[5], I6[2]};
    float T[9], Rt[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]}, Iw[9];
    matmul(R, Il, T); matmul(T, Rt, Iw);
    const float lc[3] = {t.com[i][0], t.com[i][1], t.com[i][2]};
    float c[3]; matvec(R, lc, c);
#pragma unroll
    for (int k = 0; k < 3; k++) c[k] += x[k];
    const float m = t.mass[i], cc = dot3(c, c);
    const float a[10] = {Iw[0] + m * (cc - c[0] * c[0]), Iw[4] + m * (cc - c[1] * c[1]), Iw[8] + m * (cc - c[2] * c[2]),
                         Iw[1] - m * c[0] * c[1], Iw[2] - m * c[0] * c[2], Iw[5] - m * c[1] * c[2], m * c[0], m * c[1], m * c[2], m};
    kin_store_in(s.in[i], a);
}

// ---- phase 3 (once per tree level d = maxdepth - 1 .. 0): composite inertia of the sub-tree rooted at link i = its own + its
// children's (already complete: they are one level deeper).  In place; a fixed order of the children keeps the sums reproducible.
B2G_HD void kin_composite_do(int i, int nchild, const KinModel &t, KinScratch &s) {
    float a[10];
    kin_load_in(s.in[i], a);
    for (int q = 0; q < nchild; q++) {
        float b[10];
        kin_load_in(s.in[t.child[i][q]], b);
#pragma unroll
        for (int c = 0; c < 10; c++) a[c] += b[c];
    }
    kin_store_in(s.in[i], a);
}
B2G_HD void kin_composite_level(int i, int d, const KinModel &t, KinScratch &s) {
    if (i < t.nl && t.depth[i] == d && t.nchild[i] > 0) kin_composite_do(i, t.nchild[i], t, s);
}
// ---- phase 4: Ic_i S_i = (angular momentum about O ; linear momentum) of the sub-tree moving with joint i at unit rate
B2G_HD void kin_momentum(int i, const KinModel &t, KinScratch &s) {
    if (i == 0) {
        s.cb[0] = s.in[0][0]; s.cb[1] = s.in[0][1]; s.cb[2] = s.in[0][2];
        return;
    }
    float a[10];
    kin_load_in(s.in[i], a);
    KinS S = kin_load_S(s, i);
    const float mc[3] = {a[6], a[7], a[8]};
    // n = I_O sa + mc x sb,  f = m sb - mc x sa
    float t1[3], t2[3];
    cross(mc, S.sb, t1); cross(mc, S.sa, t2);
    S.n[0] = a[0] * S.sa[0] + a[3] * S.sa[1] + a[4] * S.sa[2] + t1[0];
    S.n[1] = a[3] * S.sa[0] + a[1] * S.sa[1] + a[5] * S.sa[2] + t1[1];
    S.n[2] = a[4] * S.sa[0] + a[5] * S.sa[1] + a[2] * S.sa[2] + t1[2];
#pragma unroll
    for (int c = 0; c < 3; c++) S.f[c] = a[9] * S.sb[c] - t2[c];
    kin_store_S(s, i, S);
}

// ---- phase 2b: origin of body b's frame relative to O, with the ancestor mask of its link
B2G_HD void kin_body(int b, const KinModel &t, KinScratch &s) {
    const int l = t.body_link[b];
    float R[9], x[3], o[3];
    kin_load_Rx(s, l, R, x);
    const float bp[3] = {t.body_pos[b][0], t.body_pos[b][1], t.body_pos[b][2]};
    matvec(R, bp, o);
    s.pb[b] = make_float4(x[0] + o[0], x[1] + o[1], x[2] + o[2], kin_u2f(t.anc[l]));
}

// ---- fills.  A lane owns one COLUMN c of both tensors for the whole env, so what belongs to the column -- the joint's world
// axis, origin, motion subspace, Ic S and ancestor mask -- is fetched once (KinCol) and every output row costs a few
// multiply-adds; the stores of a warp are one contiguous run of an output row.
struct KinCol {
    int base;               // 0..5: base column (world linear 0..2, world angular 3..5), -1: joint column
    int link;               // joint column: its link
    unsigned anc;
    float sa[3], sb[3], n[3], f[3], arm;      // the column's motion subspace about O and Ic S
};
B2G_HD KinCol kin_col(int c, const KinModel &t, const KinScratch &s) {
    KinCol k;
    k.base = c < t.nbase ? c : -1;
    const int j = c < t.nbase ? 0 : c - t.nbase + 1;
    k.link = j; k.anc = t.anc[j]; k.arm = t.armature[j];
    const KinS S = kin_load_S(s, j);                                 // base columns read the root's row (zeros), overwritten below
#pragma unroll
    for (int a = 0; a < 3; a++) {
        k.sa[a] = c < t.nbase ? ((c >= 3 && c - 3 == a) ? 1.f : 0.f) : S.sa[a];      // base: (0 ; e_c) linear, (e_c ; 0) angular
        k.sb[a] = c < t.nbase ? ((c < 3 && c == a) ? 1.f : 0.f) : S.sb[a];
        k.n[a] = S.n[a]; k.f[a] = S.f[a];
    }
    return k;
}

B2G_HD float kin_pick(const float v[3], int a) { return a == 0 ? v[0] : (a == 1 ? v[1] : v[2]); }   // no dynamic register indexing

// the six entries (linear 3, angular 3) of body b's Jacobian block in column k.  With S = (sa ; sb) about O the twist of a point p
// riding on the joint's sub-tree is (sa x p + sb ; sa) -- hinge, slide and the six base coordinates alike (base: S = unit vectors,
// every body rides on it) -- so the lanes of a warp run one branch-free expression.
B2G_HD void kin_jac_col(int b, const KinCol &k, const KinModel &t, const KinScratch &s, float o[6]) {
    const float4 pw = s.pb[b];                                                    // one 128-bit broadcast: origin + ancestor mask
    const float pb[3] = {pw.x, pw.y, pw.z};
    const bool on = k.base >= 0 || ((kin_f2u(pw.w) >> k.link) & 1u);             // the joint lies between the base and this body
    float v[3]; cross(k.sa, pb, v);
#pragma unroll
    for (int c = 0; c < 3; c++) { o[c] = on ? v[c] + k.sb[c] : 0.f; o[3 + c] = on ? k.sa[c] : 0.f; }
}

// entry (row a, column k) of the mass matrix
B2G_HD float kin_mass_col(int a, const KinCol &k, const KinModel &t, const KinScratch &s) {
    const int nb = t.nbase;
    if (a < nb) {
        const int ax = a < 3 ? a : a - 3;
        if (k.base < 0) return a < 3 ? kin_pick(k.f, ax) : kin_pick(k.n, ax);           // base row against a joint column: Ic_j S_j
        float cb[10]; kin_load_in(s.cb, cb);
        const int kx = k.base < 3 ? k.base : k.base - 3;
        if (a < 3 && k.base < 3) return ax == kx ? cb[9] : 0.f;     // m 1
        if (a >= 3 && k.base >= 3) {                                 // I_O: (0,1) -> 3, (0,2) -> 4, (1,2) -> 5
            const int q = ax == kx ? ax : 2 + ax + kx;
            return q == 0 ? cb[0] : q == 1 ? cb[1] : q == 2 ? cb[2] : q == 3 ? cb[3] : q == 4 ? cb[4] : cb[5];
        }
        // linear row i, angular column j: p = w x (m c) -> -[mc]x [i][j]; the (angular, linear) entry is its transpose
        const int i = a < 3 ? ax : kx, j = a < 3 ? kx : ax;
        if (i == j) return 0.f;
        const float mc[3] = {cb[6], cb[7], cb[8]};
        const float v = kin_pick(mc, 3 - i - j);
        return ((j - i + 3) % 3 == 1) ? v : -v;
    }
    const int i = a - nb + 1;
    const KinS R = kin_load_S(s, i);                                // the row link's (Ic S ; S): three 128-bit broadcasts
    const int j = k.link;
    // S_deeper-or-equal's Ic S against the other's S: column joint j on row link i's path -> S_j . (Ic_i S_i); row link i on column
    // joint j's path -> S_i . (Ic_j S_j); different branches of the tree -> 0.  Selected without branching: the lanes of a warp
    // (columns) fall into all three cases in the same row.
    // A base column is the same expression with S = unit vectors (every link rides on the base), so it takes the first case.
    const bool ja = k.base >= 0 || ((t.anc[i] >> j) & 1u), ib = (k.anc >> i) & 1u;
    float v = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float sa = ja ? k.sa[c] : R.sa[c], sb = ja ? k.sb[c] : R.sb[c];
        const float n = ja ? R.n[c] : k.n[c], f = ja ? R.f[c] : k.f[c];
        v += sa * n + sb * f;
    }
    if (!(ja || ib)) v = 0.f;
    return i == j ? v + k.arm : v;
}

#ifdef __CUDACC__
// G lanes per env (32: one warp per env; 16 / 8: two / four small articulations per warp -- an arm or a quadruped leaves most
// of a warp idle otherwise), grid-stride over groups of 32 / G envs.  jac / mass may be null (only the other tensor is refreshed).
template <int WARPS, int G>
__global__ void __launch_bounds__(WARPS * 32) kin_tensors_kernel(const KinModel *__restrict__ gm, const float *__restrict__ g_root,
                                                                 const float *__restrict__ g_dof, float *__restrict__ jac,
                                                                 float *__restrict__ mass, int N) {
    constexpr int EPW = 32 / G;                              // envs per warp
    __shared__ KinModel t;
    __shared__ KinScratch sc[WARPS * EPW];
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(gm);
        uint4 *dst = reinterpret_cast<uint4 *>(&t);
        for (int i = threadIdx.x; i < (int)(sizeof(KinModel) / 16); i += blockDim.x) dst[i] = src[i];
        __syncthreads();
    }
    const int lane = (threadIdx.x & 31) % G, grp = (threadIdx.x & 31) / G, warp = threadIdx.x >> 5;
    KinScratch &s = sc[warp * EPW + grp];
    const int nl = t.nl, nd = nl - 1, nc = t.nc;
    // what a lane needs of the tables in the level loops, read once for all the envs this warp processes
    const int my_depth = lane < nl ? t.depth[lane] : -1, my_parent = lane < nl ? t.parent[lane] : 0, my_nchild = lane < nl ? t.nchild[lane] : 0;
    for (int e0 = (blockIdx.x * WARPS + warp) * EPW; e0 < N; e0 += gridDim.x * WARPS * EPW) {
        const int e = e0 + grp;
        const bool valid = e < N;                            // the groups of a warp run in step (warp-wide barriers): a tail group idles
        const float *root = g_root + 13 * (size_t)(valid ? e : 0) * t.root_stride;
        const float2 *dof = reinterpret_cast<const float2 *>(g_dof) + (size_t)(valid ? e : 0) * nd;
        __syncwarp();                                        // the previous env's readers are done with the scratch
        if (lane < nl) kin_local(lane, t, s, root, lane > 0 ? dof[lane - 1].x : 0.f);
        for (int d = 1; d <= t.maxdepth; d++) { __syncwarp(); if (my_depth == d) kin_level_do(lane, my_parent, s); }
        __syncwarp();
        if (lane < nl) kin_link(lane, t, s);
        if (jac && lane < t.nb) kin_body(lane, t, s);
        __syncwarp();
        if (mass) {
            for (int d = t.maxdepth - 1; d >= 0; d--) { if (my_depth == d && my_nchild > 0) kin_composite_do(lane, my_nchild, t, s); __syncwarp(); }
            if (lane < nl) kin_momentum(lane, t, s);
            __syncwarp();
        }
        if (!valid) continue;
        for (int c = lane; c < nc; c += G) {                 // one pass when the columns fit the group
            const KinCol k = kin_col(c, t, s);
            if (mass) {
                float *M = mass + (size_t)e * nc * nc + c;
                for (int a = 0; a < nc; a++, M += nc) *M = kin_mass_col(a, k, t, s);
            }
            if (jac) {
                float *J = jac + (size_t)e * t.rows * 6 * nc + c;
                const size_t st = (size_t)nc;
                for (int b = 0; b < t.rows; b++) {
                    float o[6]; kin_jac_col(t.row0 + b, k, t, s, o);
                    J[0] = o[0]; J[st] = o[1]; J[2 * st] = o[2]; J[3 * st] = o[3]; J[4 * st] = o[4]; J[5 * st] = o[5];
                    J += 6 * st;
                }
            }
        }
    }
}
#endif

}   // namespace b2g

// b2g_quad.cuh -- the specialised sub-step of "four chains on a free base" articulations (Ant: 4 legs x 2 hinges,
// ANYmal: 4 legs x 3 hinges): the same physics as Stepper::substep (b2g_device.cuh; replaces gym.simulate,
// reference call sites tasks/base/vec_task.py:379-382, tasks/anymal_terrain.py:448) as STRAIGHT-LINE code.
//
// Why a second formulation of the same sub-step: the generic Stepper interprets a slot program (rolled loops,
// per-slot records, 10 float4 of shared-memory state per link and pass, runtime joint-type flags).  In its Ant
// kernel the floating-point work is about half of the instructions -- the rest is addressing, loop control, flag tests and shared-memory
// traffic.  Here the chain length NS is a template parameter, everything a lane needs between the sweeps stays
// in registers, the model constants arrive as conflict-free 128-bit shared-memory loads ([k][leg] layout), the
// joint rotation is three constant matrices (Rj = M0 + cos q M1 + sin q M2, so no per-joint Rodrigues on matrix
// columns), and the link-local work (inertia, bias force, contacts) is fused into the root->leaf sweep.
//
// Work decomposition (unchanged): one env = 4 lanes of a warp, lane = leg; the base is replicated on the four
// lanes and the legs' articulated inertias meet in an xor-butterfly of warp shuffles.
//
// Everything that is plain arithmetic is __host__ __device__: tests/quad_host.cu compiles this header for the
// host and runs the identical code path lane by lane against the fp64 oracle (no GPU needed for that test).
#pragma once
#include <string.h>
#include <math.h>
#include "b2g_device.cuh"

namespace b2g {

// ---------------------------------------------------------------------------------------------
// Quad model blob (float4 units).  Header (broadcast reads) then the link table [(s * QL_F4 + k) * 4 + leg].
//  H0: h g0 g1 g2            H1: kn cn vs2 gn(=cn+h*kn)      H2: hf_inv_scale hf_vscale hf_ox hf_oy
//  H3: (int) hf_nx hf_ny ncp_root root_sensor                H4: root com xyz, mass
//  H5: root Ab xx yy zz xy   H6: Ab xz yz, (int) root_body, (int) substeps  (Ab: rotational inertia about the ROOT ORIGIN, root axes)
//  H7: root sensor body origin xyz (link frame), (int) nsens | nb << 8           H8..15: root spheres (pos, radius)   H16,17: their friction (combined)  H18: ground_mu ang_damp lin_damp max_angvel
// link block k: 0..6 M0 M1 M2 axp[0] | 7: axp[1] axp[2] lpos[0] lpos[1] | 8: lpos[2] com xyz | 9: Ic xx yy zz xy
//  10: Ic xz yz, mass, dg0 | 11: damping stiffness lower upper | 12: effort limit_k limit_d limit_dg | 13,14: spheres (pos, radius; radius<0 unused)
//  15: mu0 mu1 sbpos.x sbpos.y | 16: sbpos.z (int)sensor (int)body (int)dof | 17: armature - - -
constexpr int QHDR_F4 = 19;
constexpr int QL_F4 = 18;
constexpr int QROOT_CP = 8;
constexpr int QLINK_CP = 2;
constexpr int QPOSE_F4 = 5;      // parked pose of a link: R(9) x(3) vw(3) vl(3)
__host__ __device__ constexpr int quad_model_f4(int ns) { return QHDR_F4 + ns * QL_F4 * 4; }
__host__ __device__ constexpr int quad_park_f4(int ns) { return ns * QPOSE_F4 + (ns - 1) * ACC_F4; }

B2G_HD float q_rsqrt(float x) {
#ifdef __CUDA_ARCH__
    return b2g_rsqrt(x);                                     // arguments are sums of squares + a positive floor: never denormal
#else
    return 1.0f / sqrtf(x);
#endif
}
B2G_HD float q_rcp(float x) {
#ifdef __CUDA_ARCH__
    float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
#else
    return 1.0f / x;
#endif
}
B2G_HD int q_f2i(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_int(f);
#else
    int i; memcpy(&i, &f, 4); return i;
#endif
}

struct QOutputs {
    float *sensor;      // (nsens, 6) of this env or null
    float *dof_force;   // (nd) of this env or null
    float *net_contact; // (nb, 3) of this env or null
    bool write;
};

// SP: specialisation flags decided on the host from the model (quad_build):
//   bit 0  every chain link's inertia about its COM is axisymmetric (a 1 + bm u u^T: capsules, spheres, cylinders) --
//          rows 9/10 of the link block then hold (u, a | bm) and the congruence R Ic R^T (45 ops) becomes a 1 + bm (R u)(R u)^T (18);
//   bit 1  the base's inertia is axisymmetric AND its COM is at its origin: no first-moment terms at all.
template <int NS, bool HF, int SP = 0>
struct QLane {
    // accumulate-into-FMA forms: on for the 3-link chains (ANYmal: 196 registers, nothing spills), off for the 2-link Ant
    // kernel whose 128-register cap (14 warps per SM = one wave of 16384 envs) turns the longer live ranges into spills
    static constexpr bool FACC = (B2G_FUSE_ACC != 0) && (NS >= 3);
    const float4 *qm;         // quad model (shared memory on the device)
    const int16_t *hf;        // height samples (global) or null
    float4 *park;             // this thread's parking column: rows at stride `pstride` float4
    int pstride;
    int lane;
    float env_mu;             // >= 0: this env's combined friction (friction buckets), else the sphere's own
    // physical domain randomisation (null = the model's values): this env's per-link mass factors (nl) and per-DOF
    // (damping, stiffness, lower, upper) (nd float4)
    const float *dr_mass;
    const float4 *dr_dof;
    // joint state and actuation of this lane's chain
    float q[NS], qd[NS], act[NS];
    // carried from the sweeps to the acceleration pass
    float w[NS][3], sl[NS][3], cw[NS][3], cl[NS][3], U[NS][6], Dinv[NS], u[NS], tau[NS], dgv[NS];

    B2G_HD float4 LK(int s, int k) const { return qm[QHDR_F4 + (s * QL_F4 + k) * 4 + lane]; }
    B2G_HD float4 &PK(int r) const { return park[r * pstride]; }

    // ---- ground height and unit normal at world (x, y)
    B2G_HD void ground(float x, float y, float &hgt, float n[3]) const {
        if (!HF) { hgt = 0.f; n[0] = 0.f; n[1] = 0.f; n[2] = 1.f; return; }
        const float4 H2 = qm[2], H3 = qm[3];
        const int nx = q_f2i(H3.x), ny = q_f2i(H3.y);
        const float fx = (x - H2.z) * H2.x, fy = (y - H2.w) * H2.x;
        int ix = (int)floorf(fx), iy = (int)floorf(fy);
        ix = max(0, min(ix, nx - 2)); iy = max(0, min(iy, ny - 2));
        const float tx = fminf(fmaxf(fx - ix, 0.f), 1.f), ty = fminf(fmaxf(fy - iy, 0.f), 1.f);
        const int16_t *p = hf + (size_t)ix * ny + iy;
#ifdef __CUDA_ARCH__
        const float h00 = __ldg(p) * H2.y, h01 = __ldg(p + 1) * H2.y, h10 = __ldg(p + ny) * H2.y, h11 = __ldg(p + ny + 1) * H2.y;
#else
        const float h00 = p[0] * H2.y, h01 = p[1] * H2.y, h10 = p[ny] * H2.y, h11 = p[ny + 1] * H2.y;
#endif
        float dhx, dhy;
        if (tx + ty <= 1.f) { dhx = h10 - h00; dhy = h01 - h00; hgt = h00 + tx * dhx + ty * dhy; }
        else { dhx = h11 - h01; dhy = h11 - h10; hgt = h11 - (1.f - tx) * dhx - (1.f - ty) * dhy; }
        const float gx = dhx * H2.x, gy = dhy * H2.x;
        const float inv = q_rsqrt(gx * gx + gy * gy + 1.f);
        n[0] = -gx * inv; n[1] = -gy * inv; n[2] = inv;
    }

    // ---- one contact sphere (link-frame centre cp.xyz, radius cp.w) of a link posed at (R, x) with twist (vw, vl).
    // Split in two so that the height-field samples of several spheres (4 global loads each) are in flight together and
    // overlap the link's inertia arithmetic: sphere_geom = centre about O + ground height / normal under it,
    // sphere = the contact itself.
    // ACCUM: explicit force into the bias (pa, pl), implicit term h J^T G J into I.  !ACCUM: the force applied over
    // the sub-step, F0 - h G (J a), and its torque about the link origin, added to (F, T).
    struct SphereGeom { float pc[3], hg, n[3]; };
    B2G_HD void sphere_geom(const float4 cp, const float rp[3], const float R[9], const float x[3], SphereGeom &g) const {
        const float cpl[3] = {cp.x, cp.y, cp.z};
        matvec_add(R, cpl, x, g.pc);
        g.hg = 0.f; g.n[0] = 0.f; g.n[1] = 0.f; g.n[2] = 1.f;
        if (HF) ground(rp[0] + g.pc[0], rp[1] + g.pc[1], g.hg, g.n);
    }
    template <bool ACCUM>
    B2G_HD void sphere(const float4 cp, float mu, const float rp[3], const float R[9], const float x[3],
                       const float vw[3], const float vl[3], float I[21], float pa[3], float pl[3],
                       const float aw[3], const float al[3], float F[3], float T[3]) const {
        SphereGeom g; sphere_geom(cp, rp, R, x, g);
        sphere<ACCUM>(cp, mu, g, rp, x, vw, vl, I, pa, pl, aw, al, F, T);
    }
    template <bool ACCUM>
    B2G_HD void sphere(const float4 cp, float mu, const SphereGeom &g, const float rp[3], const float x[3],
                       const float vw[3], const float vl[3], float I[21], float pa[3], float pl[3],
                       const float aw[3], const float al[3], float F[3], float T[3]) const {
        const float4 H0 = qm[0], H1 = qm[1];
        const float h = H0.x, kn = H1.x, vs2 = H1.z, gn = H1.w;
        const float *pc = g.pc, *n = g.n;
        const float hg = g.hg;
        const float d = HF ? cp.w - (rp[2] + pc[2] - hg) * n[2] : cp.w - (rp[2] + pc[2]);
        if (d <= 0.f) return;
        float r[3];
        if (HF) { r[0] = pc[0] - cp.w * n[0]; r[1] = pc[1] - cp.w * n[1]; r[2] = pc[2] - cp.w * n[2]; }
        else { r[0] = pc[0]; r[1] = pc[1]; r[2] = pc[2] - cp.w; }
        float uv[3]; cross_add(vw, r, vl, uv);
        const float un = HF ? dot3(uv, n) : uv[2];
        const float Fn = kn * d - gn * un;
        if (Fn <= 0.f) return;
        float ut[3];
        if (HF) { ut[0] = uv[0] - un * n[0]; ut[1] = uv[1] - un * n[1]; ut[2] = uv[2] - un * n[2]; }
        else { ut[0] = uv[0]; ut[1] = uv[1]; ut[2] = 0.f; }
        const float gam = (env_mu >= 0.f ? env_mu : mu) * Fn * q_rsqrt(dot3(ut, ut) + vs2);
        float F0[3];
        if (HF) { F0[0] = Fn * n[0] - gam * ut[0]; F0[1] = Fn * n[1] - gam * ut[1]; F0[2] = Fn * n[2] - gam * ut[2]; }
        else { F0[0] = -gam * ut[0]; F0[1] = -gam * ut[1]; F0[2] = Fn; }
        if (ACCUM) {
            cross_sub<FACC>(r, F0, pa);
            pl[0] -= F0[0]; pl[1] -= F0[1]; pl[2] -= F0[2];
            const float hgam = h * gam;
            if (HF) {
                const float jx[3] = {0.f, r[2], -r[1]}, jy[3] = {-r[2], 0.f, r[0]}, jz[3] = {r[1], -r[0], 0.f};
                const float ex[3] = {1.f, 0.f, 0.f}, ey[3] = {0.f, 1.f, 0.f}, ez[3] = {0.f, 0.f, 1.f};
                sym6_rank1(I, hgam, jx, ex); sym6_rank1(I, hgam, jy, ey); sym6_rank1(I, hgam, jz, ez);
                float rxn[3]; cross(r, n, rxn);
                sym6_rank1(I, h * (gn - gam), rxn, n);
            } else {
                const float hgn = h * gn, rx = r[0], ry = r[1], rz = r[2];
                I[0] += hgam * rz * rz + hgn * ry * ry;
                I[1] += hgam * rz * rz + hgn * rx * rx;
                I[2] += hgam * (rx * rx + ry * ry);
                I[3] -= hgn * rx * ry; I[4] -= hgam * rx * rz; I[5] -= hgam * ry * rz;
                I[7] -= hgam * rz; I[8] += hgn * ry;
                I[9] += hgam * rz; I[11] -= hgn * rx;
                I[12] -= hgam * ry; I[13] += hgam * rx;
                I[15] += hgam; I[16] += hgam; I[17] += hgn;
            }
        } else {
            float Ja[3]; cross_add(aw, r, al, Ja);
            float Fk[3];
            if (HF) {
                const float Jan = dot3(Ja, n);
#pragma unroll
                for (int c = 0; c < 3; c++) Fk[c] = F0[c] - h * (gam * Ja[c] + (gn - gam) * Jan * n[c]);
            } else {
                Fk[0] = F0[0] - h * gam * Ja[0]; Fk[1] = F0[1] - h * gam * Ja[1]; Fk[2] = F0[2] - h * gn * Ja[2];
            }
            const float rl[3] = {r[0] - x[0], r[1] - x[1], r[2] - x[2]};
            cross_acc<FACC>(rl, Fk, T);
#pragma unroll
            for (int c = 0; c < 3; c++) F[c] += Fk[c];
        }
    }

    // rigid-body spatial inertia about O (world axes) and bias force p = v x* (I v) - gravity wrench, from the
    // rotational inertia about the COM in world axes (Icw), the COM about O (c) and the twist about O
    // da, dl: AssetOptions.angular_damping / linear_damping -- wrench (-da Icw w ; -dl m v_c) at the COM, explicit
    template <bool FUSE>
    B2G_HD static void rigid_terms(float mass, const float Icw[6], const float c[3], const float vw[3], const float vl[3],
                                   const float g[3], float da, float dl, float I[21], float pa[3], float pl[3]) {
        float vc[3]; cross_add(vw, c, vl, vc);
        const float l[3] = {mass * vc[0], mass * vc[1], mass * vc[2]};                                    // linear momentum
        const float hc[3] = {Icw[0] * vw[0] + Icw[3] * vw[1] + Icw[4] * vw[2],
                             Icw[3] * vw[0] + Icw[1] * vw[1] + Icw[5] * vw[2],
                             Icw[4] * vw[0] + Icw[5] * vw[1] + Icw[2] * vw[2]};                           // angular momentum about the COM
        if (FUSE) {
        pl[0] = fmaf(dl, l[0], -mass * g[0]); pl[1] = fmaf(dl, l[1], -mass * g[1]); pl[2] = fmaf(dl, l[2], -mass * g[2]);
        cross_acc<true>(vw, l, pl);
        pa[0] = da * hc[0]; pa[1] = da * hc[1]; pa[2] = da * hc[2];
        cross_acc<true>(vw, hc, pa); cross_acc<true>(c, pl, pa);
        } else {
        float t1[3], t2[3];
        cross(vw, l, t1);
        pl[0] = t1[0] - mass * g[0] + dl * l[0]; pl[1] = t1[1] - mass * g[1] + dl * l[1]; pl[2] = t1[2] - mass * g[2] + dl * l[2];
        cross(vw, hc, t1); cross(c, pl, t2);
        pa[0] = t1[0] + t2[0] + da * hc[0]; pa[1] = t1[1] + t2[1] + da * hc[1]; pa[2] = t1[2] + t2[2] + da * hc[2];
        }
        const float hm[3] = {mass * c[0], mass * c[1], mass * c[2]};
        const float c2 = dot3(c, c);
        I[0] = Icw[0] + mass * c2 - hm[0] * c[0];
        I[1] = Icw[1] + mass * c2 - hm[1] * c[1];
        I[2] = Icw[2] + mass * c2 - hm[2] * c[2];
        I[3] = Icw[3] - hm[0] * c[1]; I[4] = Icw[4] - hm[0] * c[2]; I[5] = Icw[5] - hm[1] * c[2];
        I[6] = 0.f; I[7] = -hm[2]; I[8] = hm[1];
        I[9] = hm[2]; I[10] = 0.f; I[11] = -hm[0];
        I[12] = -hm[1]; I[13] = hm[0]; I[14] = 0.f;
        I[15] = mass; I[16] = mass; I[17] = mass; I[18] = 0.f; I[19] = 0.f; I[20] = 0.f;
    }
    // R diag-free congruence: Icw = R Ic R^T for a symmetric Ic (xx yy zz xy xz yz)
    B2G_HD static void rotate_inertia(const float R[9], const float a, const float b, const float c, const float d, const float e, const float f,
                                      float Icw[6]) {
        const float T0 = R[0] * a + R[1] * d + R[2] * e, T1 = R[0] * d + R[1] * b + R[2] * f, T2 = R[0] * e + R[1] * f + R[2] * c;
        const float T3 = R[3] * a + R[4] * d + R[5] * e, T4 = R[3] * d + R[4] * b + R[5] * f, T5 = R[3] * e + R[4] * f + R[5] * c;
        const float T6 = R[6] * a + R[7] * d + R[8] * e, T7 = R[6] * d + R[7] * b + R[8] * f, T8 = R[6] * e + R[7] * f + R[8] * c;
        Icw[0] = T0 * R[0] + T1 * R[1] + T2 * R[2];
        Icw[1] = T3 * R[3] + T4 * R[4] + T5 * R[5];
        Icw[2] = T6 * R[6] + T7 * R[7] + T8 * R[8];
        Icw[3] = T0 * R[3] + T1 * R[4] + T2 * R[5];
        Icw[4] = T0 * R[6] + T1 * R[7] + T2 * R[8];
        Icw[5] = T3 * R[6] + T4 * R[7] + T5 * R[8];
    }

    B2G_HD void park_pose(int s, const float R[9], const float x[3], const float vw[3], const float vl[3]) const {
        PK(s * QPOSE_F4 + 0) = make_float4(R[0], R[1], R[2], R[3]);
        PK(s * QPOSE_F4 + 1) = make_float4(R[4], R[5], R[6], R[7]);
        PK(s * QPOSE_F4 + 2) = make_float4(R[8], x[0], x[1], x[2]);
        PK(s * QPOSE_F4 + 3) = make_float4(vw[0], vw[1], vw[2], vl[0]);
        PK(s * QPOSE_F4 + 4) = make_float4(vl[1], vl[2], 0.f, 0.f);
    }
    B2G_HD void load_pose(int s, float R[9], float x[3], float vw[3], float vl[3]) const {
        const float4 a = PK(s * QPOSE_F4 + 0), b = PK(s * QPOSE_F4 + 1), c = PK(s * QPOSE_F4 + 2), d = PK(s * QPOSE_F4 + 3), e = PK(s * QPOSE_F4 + 4);
        R[0] = a.x; R[1] = a.y; R[2] = a.z; R[3] = a.w; R[4] = b.x; R[5] = b.y; R[6] = b.z; R[7] = b.w; R[8] = c.x;
        x[0] = c.y; x[1] = c.z; x[2] = c.w; vw[0] = d.x; vw[1] = d.y; vw[2] = d.z; vl[0] = d.w; vl[1] = e.x; vl[2] = e.y;
    }

    // ================= sweeps root -> leaves -> root of this lane's chain, plus this lane's share of the base.
    // Out: the lane's contribution to the base's articulated inertia and bias (to be summed over the 4 lanes).
    // park_poses: the acceleration pass of this sub-step will need the link poses again (contact wrench outputs).
    B2G_HD void sweep(const RootState &rs, bool park_poses, float IA[21], float pa[3], float pl[3]) {
        const float4 H0 = qm[0];
        const float h = H0.x;
        const float g[3] = {H0.y, H0.z, H0.w};
        const float da = qm[18].y, dl = qm[18].z;
        float Rr[9]; quat_to_mat(rs.rq, Rr);
        constexpr int IROW = NS * QPOSE_F4;           // first parked-inertia row
        {
            float Rp[9], xp[3] = {0.f, 0.f, 0.f}, vwp[3] = {rs.rw[0], rs.rw[1], rs.rw[2]}, vlp[3] = {rs.rv[0], rs.rv[1], rs.rv[2]};
#pragma unroll
            for (int c = 0; c < 9; c++) Rp[c] = Rr[c];
            float I[21], qa[3], ql[3];
#pragma unroll
            for (int s = 0; s < NS; s++) {
                // ---- kinematics
                const float4 k0 = LK(s, 0), k1 = LK(s, 1), k2 = LK(s, 2), k3 = LK(s, 3), k4 = LK(s, 4), k5 = LK(s, 5), k6 = LK(s, 6), k7 = LK(s, 7), k8 = LK(s, 8);
                float sn, cs; b2g_sincos(q[s], &sn, &cs);
                const float Rj[9] = {k0.x + cs * k2.y + sn * k4.z, k0.y + cs * k2.z + sn * k4.w, k0.z + cs * k2.w + sn * k5.x,
                                     k0.w + cs * k3.x + sn * k5.y, k1.x + cs * k3.y + sn * k5.z, k1.y + cs * k3.z + sn * k5.w,
                                     k1.z + cs * k3.w + sn * k6.x, k1.w + cs * k4.x + sn * k6.y, k2.x + cs * k4.y + sn * k6.z};
                float R[9]; matmul(Rp, Rj, R);
                const float axp[3] = {k6.w, k7.x, k7.y}, lp[3] = {k7.z, k7.w, k8.x};
                float x[3];
                matvec(Rp, axp, w[s]);
                matvec_add(Rp, lp, xp, x);
                cross(x, w[s], sl[s]);
                const float qds = qd[s];
                const float wq[3] = {w[s][0] * qds, w[s][1] * qds, w[s][2] * qds}, slq[3] = {sl[s][0] * qds, sl[s][1] * qds, sl[s][2] * qds};
                {   // velocity-product acceleration c = crm(v)(S qd)
                    cross(vwp, wq, cw[s]); cross(vwp, slq, cl[s]); cross_acc<FACC>(vlp, wq, cl[s]);
                }
                float vw[3], vl[3];
#pragma unroll
                for (int c = 0; c < 3; c++) { vw[c] = vwp[c] + wq[c]; vl[c] = vlp[c] + slq[c]; }
                // ---- joint force: explicit part + implicit diagonal (linear terms at the end of the sub-step)
                float4 k10 = LK(s, 10), k11 = LK(s, 11);
                const float4 k12 = LK(s, 12);
                float mfac = 1.f;                                     // link-mass factor: mass AND rotational inertia (recomputeInertia, vec_task.py:773)
                if (dr_dof || dr_mass) {                              // per-env joint properties / link mass (domain randomisation)
                    const int dof = q_f2i(LK(s, 16).w);
                    if (dr_dof) { k11 = dr_dof[dof]; k10.w = LK(s, 17).x + h * k11.x + h * h * k11.y; }
                    if (dr_mass) { mfac = dr_mass[dof + 1]; k10.z *= mfac; }
                }
                {
                    const float qp = q[s] + h * qds;
                    float f = -k11.x * qds - k11.y * qp + fminf(fmaxf(act[s], -k12.x), k12.x);
                    float dg = k10.w;
                    const bool lo = q[s] < k11.z, hi = q[s] > k11.w;
                    if (lo || hi) { f += k12.y * ((lo ? k11.z : k11.w) - qp) - k12.z * qds; dg += k12.w; }
                    tau[s] = f; dgv[s] = dg;
                }
                // ---- link-local terms: rigid-body inertia and bias about O, contacts (ground samples requested first)
                const float4 c0 = LK(s, 13), c1 = LK(s, 14), k15 = LK(s, 15);
                SphereGeom g0, g1;
                if (HF) {
                    if (c0.w >= 0.f) sphere_geom(c0, rs.rp, R, x, g0);
                    if (c1.w >= 0.f) sphere_geom(c1, rs.rp, R, x, g1);
                }
                const float4 k9 = LK(s, 9);
                const float cm_[3] = {k8.y, k8.z, k8.w};
                float c_[3]; matvec_add(R, cm_, x, c_);
                float Icw[6];
                if (SP & 1) {
                    const float ul[3] = {k9.x, k9.y, k9.z};
                    float uw[3]; matvec(R, ul, uw);
                    const float bmf = k10.x * mfac, af = k9.w * mfac;
                    const float b0 = bmf * uw[0], b1 = bmf * uw[1], b2 = bmf * uw[2];
                    Icw[0] = af + b0 * uw[0]; Icw[1] = af + b1 * uw[1]; Icw[2] = af + b2 * uw[2];
                    Icw[3] = b0 * uw[1]; Icw[4] = b0 * uw[2]; Icw[5] = b1 * uw[2];
                } else {
                    rotate_inertia(R, k9.x, k9.y, k9.z, k9.w, k10.x, k10.y, Icw);
                    if (dr_mass) {
#pragma unroll
                        for (int c = 0; c < 6; c++) Icw[c] *= mfac;
                    }
                }
                rigid_terms<FACC>(k10.z, Icw, c_, vw, vl, g, da, dl, I, qa, ql);
                {
                    float dummy[3];
                    if (HF) {
                        if (c0.w >= 0.f) sphere<true>(c0, k15.x, g0, rs.rp, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy);
                        if (c1.w >= 0.f) sphere<true>(c1, k15.y, g1, rs.rp, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy);
                    } else {                                          // plane: nothing to prefetch, one sphere at a time
                        if (c0.w >= 0.f) sphere<true>(c0, k15.x, rs.rp, R, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy);
                        if (c1.w >= 0.f) sphere<true>(c1, k15.y, rs.rp, R, x, vw, vl, I, qa, ql, dummy, dummy, dummy, dummy);
                    }
                }
                if (park_poses) park_pose(s, R, x, vw, vl);
                if (s < NS - 1) {     // park the link's own terms until the leaf->root sweep comes back
                    float t[28];
#pragma unroll
                    for (int c = 0; c < 21; c++) t[c] = I[c];
#pragma unroll
                    for (int c = 0; c < 3; c++) { t[21 + c] = qa[c]; t[24 + c] = ql[c]; }
                    t[27] = 0.f;
#pragma unroll
                    for (int k = 0; k < ACC_F4; k++) PK(IROW + s * ACC_F4 + k) = make_float4(t[4 * k], t[4 * k + 1], t[4 * k + 2], t[4 * k + 3]);
#pragma unroll
                    for (int c = 0; c < 9; c++) Rp[c] = R[c];
#pragma unroll
                    for (int c = 0; c < 3; c++) { xp[c] = x[c]; vwp[c] = vw[c]; vlp[c] = vl[c]; }
                }
            }
            // ---- leaves -> root: project the joint out of the articulated inertia, hand it to the parent
#pragma unroll
            for (int s = NS - 1; s >= 0; s--) {
                if (s < NS - 1) {
                    float t[28];
#pragma unroll
                    for (int k = 0; k < ACC_F4; k++) { const float4 v = PK(IROW + s * ACC_F4 + k); t[4 * k] = v.x; t[4 * k + 1] = v.y; t[4 * k + 2] = v.z; t[4 * k + 3] = v.w; }
#pragma unroll
                    for (int c = 0; c < 21; c++) I[c] += t[c];
#pragma unroll
                    for (int c = 0; c < 3; c++) { qa[c] += t[21 + c]; ql[c] += t[24 + c]; }
                }
                float Ua[3], Ul[3];
                sym6_mul(I, w[s], sl[s], Ua, Ul);
                float D, u_;
                if (FACC) {
                D = fmaf(w[s][0], Ua[0], fmaf(w[s][1], Ua[1], fmaf(w[s][2], Ua[2], fmaf(sl[s][0], Ul[0], fmaf(sl[s][1], Ul[1], fmaf(sl[s][2], Ul[2], dgv[s]))))));
                u_ = fmaf(-w[s][0], qa[0], fmaf(-w[s][1], qa[1], fmaf(-w[s][2], qa[2], fmaf(-sl[s][0], ql[0], fmaf(-sl[s][1], ql[1], fmaf(-sl[s][2], ql[2], tau[s]))))));
                } else {
                D = dot3(w[s], Ua) + dot3(sl[s], Ul) + dgv[s];
                u_ = tau[s] - (dot3(w[s], qa) + dot3(sl[s], ql));
                }
                const float di = q_rcp(D);
                U[s][0] = Ua[0]; U[s][1] = Ua[1]; U[s][2] = Ua[2]; U[s][3] = Ul[0]; U[s][4] = Ul[1]; U[s][5] = Ul[2];
                Dinv[s] = di; u[s] = u_;
                sym6_rank1(I, -di, Ua, Ul);                           // Ia = IA - U U^T / D
                const float ud = u_ * di;
#pragma unroll
                for (int c = 0; c < 3; c++) { qa[c] = fmaf(Ua[c], ud, qa[c]); ql[c] = fmaf(Ul[c], ud, ql[c]); }
                sym6_mul_acc<FACC>(I, cw[s], cl[s], qa, ql);
            }
#pragma unroll
            for (int c = 0; c < 21; c++) IA[c] = I[c];
#pragma unroll
            for (int c = 0; c < 3; c++) { pa[c] = qa[c]; pl[c] = ql[c]; }
        }
        // ---- the base: its own rigid-body terms (lane 0 contributes them), its spheres dealt round-robin to the lanes;
        // everything is accumulated straight onto the chain's contribution (no separate 27-value sum, no adds of zeros)
        {
            const float4 H3 = qm[3], H4 = qm[4], H5 = qm[5], H6 = qm[6];
            const float xr[3] = {0.f, 0.f, 0.f};
            const float on = (lane == 0) ? 1.f : 0.f;
            const float *vw = rs.rw, *vl = rs.rv;
            const float msc = dr_mass ? dr_mass[0] : 1.f;             // domain randomisation: the base's mass factor
            if (SP & 2) {
                // axisymmetric base with its COM at the origin: A = a 1 + bm (R u)(R u)^T, no first moment
                const float ul[3] = {H5.x, H5.y, H5.z};
                float uw[3]; matvec(Rr, ul, uw);
                const float am = on * H5.w * msc, bm = on * H6.x * msc, mo = on * H4.w * msc;
                const float s_ = bm * dot3(uw, vw);
                const float nO[3] = {am * vw[0] + s_ * uw[0], am * vw[1] + s_ * uw[1], am * vw[2] + s_ * uw[2]};     // A vw
                float a3[3];
                cross_acc<FACC>(vw, nO, pa); cross(vw, vl, a3);
#pragma unroll
                for (int c = 0; c < 3; c++) { pa[c] = fmaf(da, nO[c], pa[c]); pl[c] += mo * (a3[c] - g[c] + dl * vl[c]); }
                const float b0 = bm * uw[0], b1 = bm * uw[1], b2 = bm * uw[2];
                IA[0] += am + b0 * uw[0]; IA[1] += am + b1 * uw[1]; IA[2] += am + b2 * uw[2];
                IA[3] += b0 * uw[1]; IA[4] += b0 * uw[2]; IA[5] += b1 * uw[2];
                IA[15] += mo; IA[16] += mo; IA[17] += mo;
            } else {
                // about the root origin directly: A = R Ab R^T, first moment hm = R (m com)
                float Ab[6] = {H5.x, H5.y, H5.z, H5.w, H6.x, H6.y};
                const float mass = H4.w * msc;
                if (dr_mass) {                                        // Ab = Ic + m (c^2 1 - c c^T): both parts follow the mass factor
#pragma unroll
                    for (int c = 0; c < 6; c++) Ab[c] *= msc;
                }
                float A[6]; rotate_inertia(Rr, Ab[0], Ab[1], Ab[2], Ab[3], Ab[4], Ab[5], A);
                const float cb[3] = {H4.x * mass, H4.y * mass, H4.z * mass};
                float hm[3]; matvec(Rr, cb, hm);
                // momentum about O: n = A vw + hm x vl ; l = m vl - hm x vw
                float t1[3], t2[3];
                cross(hm, vl, t1); cross(hm, vw, t2);
                const float nO[3] = {A[0] * vw[0] + A[3] * vw[1] + A[4] * vw[2] + t1[0],
                                     A[3] * vw[0] + A[1] * vw[1] + A[5] * vw[2] + t1[1],
                                     A[4] * vw[0] + A[5] * vw[1] + A[2] * vw[2] + t1[2]};
                const float l[3] = {mass * vl[0] - t2[0], mass * vl[1] - t2[1], mass * vl[2] - t2[2]};
                float a1[3], a2[3], a3[3], a4[3];
                cross(vw, nO, a1); cross(vl, l, a2); cross(vw, l, a3); cross(hm, g, a4);
                // damping wrench at the COM moved to O: linear momentum l = m v_c; angular momentum about the COM hc = nO - c x l
                float dpa[3] = {0.f, 0.f, 0.f}, dpl[3] = {0.f, 0.f, 0.f};
                if (da != 0.f || dl != 0.f) {
                    const float inv_m = 1.f / mass;
                    const float cc[3] = {hm[0] * inv_m, hm[1] * inv_m, hm[2] * inv_m};
                    float cxl[3], cxf[3]; cross(cc, l, cxl);
#pragma unroll
                    for (int c = 0; c < 3; c++) dpl[c] = dl * l[c];
                    cross(cc, dpl, cxf);
#pragma unroll
                    for (int c = 0; c < 3; c++) dpa[c] = da * (nO[c] - cxl[c]) + cxf[c];
                }
#pragma unroll
                for (int c = 0; c < 3; c++) { pa[c] += on * (a1[c] + a2[c] - a4[c] + dpa[c]); pl[c] += on * (a3[c] - mass * g[c] + dpl[c]); }
#pragma unroll
                for (int c = 0; c < 6; c++) IA[c] += on * A[c];
                IA[7] -= on * hm[2]; IA[8] += on * hm[1];
                IA[9] += on * hm[2]; IA[11] -= on * hm[0];
                IA[12] -= on * hm[1]; IA[13] += on * hm[0];
                IA[15] += on * mass; IA[16] += on * mass; IA[17] += on * mass;
            }
            const int ncp = q_f2i(H3.z);
            float dummy[3];
            // software-pipelined: the next sphere's constants are in flight while this one is processed
            float4 cp = qm[8 + lane];
            float mu = reinterpret_cast<const float *>(qm + 16)[lane];
#pragma unroll 1
            for (int k = lane; k < ncp; k += 4) {
                const float4 cpn = qm[8 + ((k + 4) & (QROOT_CP - 1))];
                const float mun = reinterpret_cast<const float *>(qm + 16)[(k + 4) & (QROOT_CP - 1)];
                sphere<true>(cp, mu, rs.rp, Rr, xr, rs.rw, rs.rv, IA, pa, pl, dummy, dummy, dummy, dummy);
                cp = cpn; mu = mun;
            }
        }
    }

    // contact wrench of this lane's share of the base's spheres over the sub-step (to be summed over the lanes)
    B2G_HD void root_wrench(const RootState &rs, const float awr[3], const float alr[3], float F[3], float T[3]) const {
        float Rr[9]; quat_to_mat(rs.rq, Rr);
        const float xr[3] = {0.f, 0.f, 0.f};
        const int ncp = q_f2i(qm[3].z);
        float dI[1], d3[3];
        F[0] = F[1] = F[2] = 0.f; T[0] = T[1] = T[2] = 0.f;
#pragma unroll 1
        for (int k = lane; k < ncp; k += 4) {
            const float4 cp = qm[8 + k];
            const float mu = reinterpret_cast<const float *>(qm + 16)[k];
            sphere<false>(cp, mu, rs.rp, Rr, xr, rs.rw, rs.rv, dI, d3, d3, awr, alr, F, T);
        }
    }
    // force sensor (body frame, torque about the body origin) / net contact force of one link
    // keep (optional, 6 floats): the sensor reading also stays with the caller (the fused step kernels put it into the
    // observation without reading the tensor back)
    B2G_HD static void emit(const QOutputs &o, int sensor, int body, const float sb[3], const float R[9], const float F[3], const float T[3],
                            float *keep = nullptr) {
        if (!o.write) return;
        if (sensor >= 0 && o.sensor) {
            float wb[3], Tb_[3] = {T[0], T[1], T[2]}, Fb[3], Tb[3];
            matvec(R, sb, wb); cross_sub<true>(wb, F, Tb_);
            matTvec(R, F, Fb); matTvec(R, Tb_, Tb);
            float *d = o.sensor + 6 * sensor;
            d[0] = Fb[0]; d[1] = Fb[1]; d[2] = Fb[2]; d[3] = Tb[0]; d[4] = Tb[1]; d[5] = Tb[2];
            if (keep) { keep[0] = Fb[0]; keep[1] = Fb[1]; keep[2] = Fb[2]; keep[3] = Tb[0]; keep[4] = Tb[1]; keep[5] = Tb[2]; }
        }
        if (o.net_contact && body >= 0) {
            float *d = o.net_contact + 3 * body;
            d[0] = F[0]; d[1] = F[1]; d[2] = F[2];
        }
    }
    B2G_HD void emit_root(const RootState &rs, const QOutputs &o, const float F[3], const float T[3]) const {
        float Rr[9]; quat_to_mat(rs.rq, Rr);
        const float4 H7 = qm[7];
        const float sb[3] = {H7.x, H7.y, H7.z};
        emit(o, q_f2i(qm[3].w), q_f2i(qm[6].z), sb, Rr, F, T);
    }

    // ================= accelerations root -> leaves, joint integration; LAST: joint force / contact wrench outputs
    B2G_HD void accelerate(const RootState &rs, const float awr[3], const float alr[3], bool LAST, const QOutputs &o) {
        const float h = qm[0].x;
        float aw[3] = {awr[0], awr[1], awr[2]}, al[3] = {alr[0], alr[1], alr[2]};
#pragma unroll
        for (int s = 0; s < NS; s++) {
#pragma unroll
            for (int c = 0; c < 3; c++) { aw[c] += cw[s][c]; al[c] += cl[s][c]; }
            const float r_ = FACC ? fmaf(-U[s][0], aw[0], fmaf(-U[s][1], aw[1], fmaf(-U[s][2], aw[2], fmaf(-U[s][3], al[0], fmaf(-U[s][4], al[1], fmaf(-U[s][5], al[2], u[s]))))))
                                  : u[s] - (U[s][0] * aw[0] + U[s][1] * aw[1] + U[s][2] * aw[2] + U[s][3] * al[0] + U[s][4] * al[1] + U[s][5] * al[2]);
            const float qdd = r_ * Dinv[s];
#pragma unroll
            for (int c = 0; c < 3; c++) { aw[c] += w[s][c] * qdd; al[c] += sl[s][c] * qdd; }
            qd[s] += h * qdd;
            q[s] += h * qd[s];
            if (LAST) {
                const float4 k16 = LK(s, 16);
                const int sensor = q_f2i(k16.y), body = q_f2i(k16.z), dof = q_f2i(k16.w);
                if (o.dof_force && o.write) o.dof_force[dof] = tau[s] - (dgv[s] - LK(s, 17).x) * qdd;
                if (sensor >= 0 || (o.net_contact && body >= 0)) {
                    const float4 c0 = LK(s, 13), c1 = LK(s, 14), k15 = LK(s, 15);
                    float R[9], x[3], vw[3], vl[3], F[3] = {0.f, 0.f, 0.f}, T[3] = {0.f, 0.f, 0.f}, dI[1], d3[3];
                    load_pose(s, R, x, vw, vl);
                    if (c0.w >= 0.f) sphere<false>(c0, k15.x, rs.rp, R, x, vw, vl, dI, d3, d3, aw, al, F, T);
                    if (c1.w >= 0.f) sphere<false>(c1, k15.y, rs.rp, R, x, vw, vl, dI, d3, d3, aw, al, F, T);
                    const float sb[3] = {k15.z, k15.w, k16.x};
                    emit(o, sensor, body, sb, R, F, T);
                }
            }
        }
    }
    // does the acceleration pass of the last sub-step read link poses back?
    B2G_HD bool needs_poses(const QOutputs &o) const {
        bool need = false;
#pragma unroll
        for (int s = 0; s < NS; s++) { const float4 k16 = LK(s, 16); need = need || q_f2i(k16.y) >= 0 || (o.net_contact && q_f2i(k16.z) >= 0); }
        return need;
    }
    B2G_HD bool root_emits(const QOutputs &o) const { return q_f2i(qm[3].w) >= 0 || (o.net_contact && q_f2i(qm[6].z) >= 0); }

    // base: 6x6 solve, then semi-implicit Euler of the base (classical acceleration of the origin = spatial + w x v)
    B2G_HD static void solve_base(const float IA[21], const float pa[3], const float pl[3], float awr[3], float alr[3]) {
        const float ba[3] = {-pa[0], -pa[1], -pa[2]}, bl[3] = {-pl[0], -pl[1], -pl[2]};
        sym6_solve(IA, ba, bl, awr, alr);
    }
    B2G_HD void integrate_base(RootState &rs, const float awr[3], const float alr[3]) const {
        const float h = qm[0].x;
        float av[3]; cross_add(rs.rw, rs.rv, alr, av);
#pragma unroll
        for (int c = 0; c < 3; c++) { rs.rw[c] += h * awr[c]; rs.rv[c] += h * av[c]; }
#pragma unroll
        for (int c = 0; c < 3; c++) rs.rp[c] += h * rs.rv[c];
        float wn2 = dot3(rs.rw, rs.rw);
        const float mx = qm[18].w;                                   // AssetOptions.max_angular_velocity (0: no clamp)
        if (mx > 0.f && wn2 > mx * mx) { const float k = mx * q_rsqrt(wn2); rs.rw[0] *= k; rs.rw[1] *= k; rs.rw[2] *= k; wn2 = mx * mx; }
        float dq[4];
        if (wn2 > 1e-24f) {
            const float inv = q_rsqrt(wn2), wn = wn2 * inv;
            float sn, cs; b2g_sincos(0.5f * wn * h, &sn, &cs);
            const float k = sn * inv;
            dq[0] = rs.rw[0] * k; dq[1] = rs.rw[1] * k; dq[2] = rs.rw[2] * k; dq[3] = cs;
        } else { dq[0] = 0.5f * h * rs.rw[0]; dq[1] = 0.5f * h * rs.rw[1]; dq[2] = 0.5f * h * rs.rw[2]; dq[3] = 1.f; }
        const float qx = rs.rq[0], qy = rs.rq[1], qz = rs.rq[2], qw = rs.rq[3];
        const float nq[4] = {dq[3] * qx + dq[0] * qw + dq[1] * qz - dq[2] * qy,
                             dq[3] * qy - dq[0] * qz + dq[1] * qw + dq[2] * qx,
                             dq[3] * qz + dq[0] * qy - dq[1] * qx + dq[2] * qw,
                             dq[3] * qw - dq[0] * qx - dq[1] * qy - dq[2] * qz};
        const float inv = q_rsqrt(nq[0] * nq[0] + nq[1] * nq[1] + nq[2] * nq[2] + nq[3] * nq[3]);
#pragma unroll
        for (int c = 0; c < 4; c++) rs.rq[c] = nq[c] * inv;
    }

#ifdef __CUDACC__
    // ================= one sub-step on the device: the four lanes of the env run in lock-step
    __device__ __forceinline__ void substep(RootState &rs, const bool LAST, const QOutputs &o) {
        float IA[21], pa[3], pl[3];
        const bool poses = LAST && needs_poses(o);
        sweep(rs, poses, IA, pa, pl);
#pragma unroll
        for (int c = 0; c < 21; c++) IA[c] = lane_sum<4>(IA[c]);
#pragma unroll
        for (int c = 0; c < 3; c++) { pa[c] = lane_sum<4>(pa[c]); pl[c] = lane_sum<4>(pl[c]); }
        float awr[3], alr[3];
        solve_base(IA, pa, pl, awr, alr);
        if (LAST && root_emits(o)) {
            float F[3], T[3];
            root_wrench(rs, awr, alr, F, T);
#pragma unroll
            for (int c = 0; c < 3; c++) { F[c] = lane_sum<4>(F[c]); T[c] = lane_sum<4>(T[c]); }
            if (lane == 0) emit_root(rs, o, F, T);
        }
        accelerate(rs, awr, alr, LAST, o);
        integrate_base(rs, awr, alr);
    }
#endif
};

}  // namespace b2g

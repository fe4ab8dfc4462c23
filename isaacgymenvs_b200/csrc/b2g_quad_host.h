// b2g_quad_host.h -- host side of the quad path (b2g_quad.cuh): decides whether an articulation is "four equal
// hinge chains on a free base" and packs its constants into the quad model blob.  Plain C++ (no CUDA), shared by
// b2g_model_host.h (b2g_create) and tests/quad_host.cu (the CPU run of the same arithmetic against the oracle).
#pragma once
#include <math.h>
#include <string.h>
#include <vector>
#include "../../include/b200gym.h"
#include "b2g_quad.cuh"
#include "b2g_kin_host.h"

namespace b2g {

static inline float q_i2f(int i) { float f; memcpy(&f, &i, 4); return f; }

// Is the symmetric inertia (xx yy zz xy xz yz) of the form a 1 + bm u u^T (two equal principal moments)?  Jacobi
// eigen-decomposition in double; equal within 1e-6 of the largest moment.
static inline bool quad_axisymmetric(const float I6[6], float u[3], float *a, float *bm) {
    double A[3][3] = {{I6[0], I6[3], I6[4]}, {I6[3], I6[1], I6[5]}, {I6[4], I6[5], I6[2]}}, V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 32; sweep++) {
        double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        if (off < 1e-300) break;
        for (int p_ = 0; p_ < 2; p_++) for (int q_ = p_ + 1; q_ < 3; q_++) {
            if (fabs(A[p_][q_]) < 1e-300) continue;
            const double th = (A[q_][q_] - A[p_][p_]) / (2 * A[p_][q_]);
            const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1)), c = 1 / sqrt(t * t + 1), s_ = t * c;
            for (int k = 0; k < 3; k++) { const double x = A[k][p_], y = A[k][q_]; A[k][p_] = c * x - s_ * y; A[k][q_] = s_ * x + c * y; }
            for (int k = 0; k < 3; k++) { const double x = A[p_][k], y = A[q_][k]; A[p_][k] = c * x - s_ * y; A[q_][k] = s_ * x + c * y; }
            for (int k = 0; k < 3; k++) { const double x = V[k][p_], y = V[k][q_]; V[k][p_] = c * x - s_ * y; V[k][q_] = s_ * x + c * y; }
        }
    }
    const double l[3] = {A[0][0], A[1][1], A[2][2]};
    const double big = fmax(fabs(l[0]), fmax(fabs(l[1]), fabs(l[2])));
    int odd = -1;
    if (fabs(l[0] - l[1]) <= 1e-6 * big) odd = 2;
    else if (fabs(l[0] - l[2]) <= 1e-6 * big) odd = 1;
    else if (fabs(l[1] - l[2]) <= 1e-6 * big) odd = 0;
    if (odd < 0) return false;
    const double aa = 0.5 * (l[(odd + 1) % 3] + l[(odd + 2) % 3]);
    *a = (float)aa; *bm = (float)(l[odd] - aa);
    for (int k = 0; k < 3; k++) u[k] = (float)V[k][odd];
    return true;
}

// Returns the chain length NS (2 or 3) and fills `qm` (quad_model_f4(NS, self) float4, as floats) when the model fits the
// quad path; 0 otherwise (the generic Stepper handles it).  leg_link[l * NS + s] = link of lane l, slot s.
// *spec receives the QLane specialisation flags the packed constants are laid out for (0 or 3; want_spec = 0 forces the
// general layout).  A self-colliding model (m->self_collide) fits for chain length 3 only, in the general layout, and only
// when no candidate pair lies within one leg; its self-collision table follows the link table (b2g_quad.cuh).
static inline int quad_build(const b2g_model *m, const b2g_sim_params *sp, std::vector<float> &qm, int leg_link[12], int *spec = nullptr, int want_spec = 3) {
    if (m->root_fixed || m->nl < 9) return 0;
    const int nd = m->nl - 1;
    if (nd != 8 && nd != 12) return 0;
    const int NS = nd / 4;
    const bool self = m->self_collide && m->self_pairs;
    if (self && NS != 3) return 0;
    if (self) want_spec = 0;
    int roots[4], nroot = 0;
    for (int i = 1; i < m->nl; i++) if (m->parent[i] == 0) { if (nroot == 4) return 0; roots[nroot++] = i; }
    if (nroot != 4) return 0;
    for (int l = 0; l < 4; l++) {
        int cur = roots[l];
        for (int s = 0; s < NS; s++) {
            leg_link[l * NS + s] = cur;
            int child = -1, nchild = 0;
            for (int i = 1; i < m->nl; i++) if (m->parent[i] == cur) { child = i; nchild++; }
            if (s < NS - 1) { if (nchild != 1) return 0; cur = child; }
            else if (nchild != 0) return 0;
        }
    }
    for (int i = 1; i < m->nl; i++) if (m->jtype[i] != 0 || m->drive_mode[i] == 1) return 0;   // hinges, effort-driven
    std::vector<int> ncp(m->nl, 0);
    for (int k = 0; k < m->ncp; k++) ncp[m->cp_link[k]]++;
    if (ncp[0] > QROOT_CP) return 0;
    for (int i = 1; i < m->nl; i++) if (ncp[i] > QLINK_CP) return 0;
    std::vector<int> link_sensor(m->nl, -1), link_body(m->nl, -1);
    for (int k = 0; k < m->nsens; k++) {
        const int li = m->body_link[m->sensor_body[k]];
        if (link_sensor[li] >= 0) return 0;                       // one sensor per link
        link_sensor[li] = k;
    }
    for (int b = m->nb - 1; b >= 0; b--) link_body[m->body_link[b]] = b;

    // specialisation: every chain link axisymmetric about its COM (bit 0) and an axisymmetric base with its COM at its origin (bit 1)
    int sflags = want_spec;
    std::vector<float> ax(4 * 5 * 3 + 5, 0.f);            // per link (u, a, bm), link order of leg_link; last 5: the base
    if (sflags) {
        for (int k = 0; k < 4 * NS && sflags; k++) {
            const int li = leg_link[k];
            if (!quad_axisymmetric(m->inertia + 6 * li, &ax[5 * k], &ax[5 * k + 3], &ax[5 * k + 4])) sflags = 0;
        }
        float *rb = &ax[5 * 12];
        if (sflags && !(quad_axisymmetric(m->inertia, rb, rb + 3, rb + 4) && m->com[0] == 0.f && m->com[1] == 0.f && m->com[2] == 0.f)) sflags = 0;
    }
    if (spec) *spec = sflags;

    qm.assign((size_t)quad_model_f4(NS, self) * 4, 0.f);
    std::vector<int> sph_lane(m->ncp, -1), sph_slot(m->ncp, 0);     // contact sphere -> (lane, 2 s + c), or (-1, base slot)
    auto F4 = [&](int idx) { return qm.data() + 4 * (size_t)idx; };
    const float h = sp->dt / (float)sp->substeps;
    float g[3];
    for (int c = 0; c < 3; c++) g[c] = m->gravity_on ? sp->gravity[c] : 0.f;
    { float *H = F4(0); H[0] = h; H[1] = g[0]; H[2] = g[1]; H[3] = g[2]; }
    { float *H = F4(1); H[0] = m->contact_kn; H[1] = m->contact_cn; H[2] = m->contact_vs * m->contact_vs; H[3] = m->contact_cn + h * m->contact_kn; }
    if (sp->hf_samples) {
        float *H = F4(2); H[0] = 1.f / sp->hf_horizontal_scale; H[1] = sp->hf_vertical_scale; H[2] = sp->hf_origin_x; H[3] = sp->hf_origin_y;
    }
    {
        float *H = F4(3);
        H[0] = q_i2f(sp->hf_samples ? sp->hf_nx : 0); H[1] = q_i2f(sp->hf_samples ? sp->hf_ny : 0);
        H[2] = q_i2f(ncp[0]); H[3] = q_i2f(link_sensor[0]);
    }
    {   // the base
        const float *c = m->com, *I6 = m->inertia;
        const float ms = m->mass[0], c2 = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
        float *H = F4(4); H[0] = c[0]; H[1] = c[1]; H[2] = c[2]; H[3] = ms;
        float *A = F4(5);
        A[0] = I6[0] + ms * (c2 - c[0] * c[0]); A[1] = I6[1] + ms * (c2 - c[1] * c[1]); A[2] = I6[2] + ms * (c2 - c[2] * c[2]);
        A[3] = I6[3] - ms * c[0] * c[1];
        float *B = F4(6);
        B[0] = I6[4] - ms * c[0] * c[2]; B[1] = I6[5] - ms * c[1] * c[2]; B[2] = q_i2f(link_body[0]); B[3] = q_i2f(sp->substeps);
        if (sflags & 2) { const float *rb = &ax[5 * 12]; A[0] = rb[0]; A[1] = rb[1]; A[2] = rb[2]; A[3] = rb[3]; B[0] = rb[4]; B[1] = 0.f; }
        if (link_sensor[0] >= 0) { const float *bp = m->body_pos + 3 * m->sensor_body[link_sensor[0]]; float *S = F4(7); S[0] = bp[0]; S[1] = bp[1]; S[2] = bp[2]; }
        F4(7)[3] = q_i2f(m->nsens | (m->nb << 8));
        F4(18)[0] = sp->ground_friction; F4(18)[1] = m->angular_damping; F4(18)[2] = m->linear_damping; F4(18)[3] = m->max_angular_velocity;
        int k0 = 0;
        for (int k = 0; k < m->ncp; k++) if (m->cp_link[k] == 0) {
            float *P = F4(8 + k0);
            P[0] = m->cp_pos[3 * k]; P[1] = m->cp_pos[3 * k + 1]; P[2] = m->cp_pos[3 * k + 2]; P[3] = m->cp_radius[k];
            F4(16)[k0] = 0.5f * (m->cp_mu[k] + sp->ground_friction);
            sph_slot[k] = k0;
            k0++;
        }
    }
    for (int l = 0; l < 4; l++) for (int s = 0; s < NS; s++) {
        const int li = leg_link[l * NS + s];
        float L[QL_F4 * 4];
        memset(L, 0, sizeof(L));
        float R0[9];
        host_quat_to_mat(m->lquat + 4 * li, R0);
        float a[3] = {m->axis[3 * li], m->axis[3 * li + 1], m->axis[3 * li + 2]};
        const float an = sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
        if (!(an > 0.f)) return 0;
        a[0] /= an; a[1] /= an; a[2] /= an;
        // Rodrigues in the link frame: Rot(a, q) = a a^T + cos q (1 - a a^T) + sin q [a]x ; Rj = R0 Rot
        const float aaT[9] = {a[0] * a[0], a[0] * a[1], a[0] * a[2], a[1] * a[0], a[1] * a[1], a[1] * a[2], a[2] * a[0], a[2] * a[1], a[2] * a[2]};
        const float K[9] = {0.f, -a[2], a[1], a[2], 0.f, -a[0], -a[1], a[0], 0.f};
        float M0[9], M1[9], M2[9];
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
            float s0 = 0.f, s1 = 0.f, s2 = 0.f;
            for (int k = 0; k < 3; k++) {
                s0 += R0[3 * i + k] * aaT[3 * k + j];
                s1 += R0[3 * i + k] * ((k == j ? 1.f : 0.f) - aaT[3 * k + j]);
                s2 += R0[3 * i + k] * K[3 * k + j];
            }
            M0[3 * i + j] = s0; M1[3 * i + j] = s1; M2[3 * i + j] = s2;
        }
        for (int c = 0; c < 9; c++) { L[c] = M0[c]; L[9 + c] = M1[c]; L[18 + c] = M2[c]; }
        for (int i = 0; i < 3; i++) L[27 + i] = R0[3 * i] * a[0] + R0[3 * i + 1] * a[1] + R0[3 * i + 2] * a[2];   // axis in the parent frame
        for (int c = 0; c < 3; c++) { L[30 + c] = m->lpos[3 * li + c]; L[33 + c] = m->com[3 * li + c]; }
        for (int c = 0; c < 6; c++) L[36 + c] = m->inertia[6 * li + c];
        if (sflags & 1) { const float *a5 = &ax[5 * (l * NS + s)]; L[36] = a5[0]; L[37] = a5[1]; L[38] = a5[2]; L[39] = a5[3]; L[40] = a5[4]; L[41] = 0.f; }
        L[42] = m->mass[li];
        L[43] = m->armature[li] + h * m->damping[li] + h * h * m->stiffness[li];           // dg0
        L[44] = m->damping[li]; L[45] = m->stiffness[li];
        L[46] = m->limited[li] ? m->lower[li] : -3e38f; L[47] = m->limited[li] ? m->upper[li] : 3e38f;
        L[48] = m->effort[li]; L[49] = m->limit_k[li]; L[50] = m->limit_d[li];
        L[51] = h * m->limit_d[li] + h * h * m->limit_k[li];                                 // limit_dg
        L[52 + 3] = -1.f; L[56 + 3] = -1.f;                                                  // unused sphere slots
        int k0 = 0;
        for (int k = 0; k < m->ncp; k++) if (m->cp_link[k] == li) {
            float *P = L + 52 + 4 * k0;
            P[0] = m->cp_pos[3 * k]; P[1] = m->cp_pos[3 * k + 1]; P[2] = m->cp_pos[3 * k + 2]; P[3] = m->cp_radius[k];
            L[60 + k0] = 0.5f * (m->cp_mu[k] + sp->ground_friction);
            sph_lane[k] = l; sph_slot[k] = 2 * s + k0;
            k0++;
        }
        if (link_sensor[li] >= 0) { const float *bp = m->body_pos + 3 * m->sensor_body[link_sensor[li]]; L[62] = bp[0]; L[63] = bp[1]; L[64] = bp[2]; }
        L[65] = q_i2f(link_sensor[li]); L[66] = q_i2f(link_body[li]); L[67] = q_i2f(li - 1);
        L[68] = m->armature[li];
        for (int k = 0; k < QL_F4; k++) memcpy(F4(QHDR_F4 + (s * QL_F4 + k) * 4 + l), L + 4 * k, 16);
    }
    if (self) {
        const int QS = QHDR_F4 + NS * QL_F4 * 4;
        { float *S = F4(QS); S[0] = m->self_kn; S[1] = m->self_cn; S[2] = m->self_mu; }
        unsigned word[4][8] = {};
        for (int i = 0; i < m->ncp; i++) for (int j = i + 1; j < m->ncp; j++) {
            if (!m->self_pairs[(size_t)i * m->ncp + j] && !m->self_pairs[(size_t)j * m->ncp + i]) continue;
            const int li = sph_lane[i], lj = sph_lane[j], ai = sph_slot[i], aj = sph_slot[j];
            if (li < 0 && lj < 0) continue;                                  // both on the base: one link
            if (li == lj) return 0;                                          // within one leg: the generic Stepper
            if (li < 0) word[lj][aj] |= 1u << (18 + ai);
            else if (lj < 0) word[li][ai] |= 1u << (18 + aj);
            else {
                const int p = li ^ lj;
                word[li][ai] |= 1u << (6 * (p - 1) + aj);
                word[lj][aj] |= 1u << (6 * (p - 1) + ai);
            }
        }
        for (int l = 0; l < 4; l++) for (int a = 0; a < 2 * NS; a++) F4(QS + 1 + (a >> 2) * 4 + l)[a & 3] = q_i2f((int)word[l][a]);
    }
    return NS;
}

}  // namespace b2g

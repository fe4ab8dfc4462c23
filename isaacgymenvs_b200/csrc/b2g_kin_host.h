// b2g_kin_host.h -- host-side construction of the constant tables of the Jacobian / mass-matrix kernel (b2g_kin.cuh)
// from the importer's articulation model.  Included by b200gym.cu (the product) and by tests/kin_host.cu (the CPU twin).
#pragma once
#include <math.h>
#include <string.h>
#include "../../include/b200gym.h"
#include "b2g_kin.cuh"

namespace b2g {

// Unit quaternion (x, y, z, w) -> row-major rotation matrix, for the model constants built on the host (here, b2g_quad_host.h,
// b2g_model_host.h).  Not the device quat_to_mat: that one scales by b2g_rsqrt, which moves the constants in the last bit.
static inline void host_quat_to_mat(const float *q, float R[9]) {
    float x = q[0], y = q[1], z = q[2], w = q[3], n = sqrtf(x * x + y * y + z * z + w * w);
    x /= n; y /= n; z /= n; w /= n;
    const float M[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    memcpy(R, M, sizeof(M));
}

// returns 0, or -1 when the articulation exceeds the kernel's limits (one lane per link and per body)
static inline int kin_build(const b2g_model *m, int root_stride, KinModel &k) {
    memset(&k, 0, sizeof(k));
    if (m->nl < 1 || m->nl > MAX_LINKS || m->nb < 1 || m->nb > MAX_LINKS) return -1;
    k.nl = m->nl; k.nb = m->nb;
    k.nbase = m->root_fixed ? 0 : 6;
    k.nc = m->nl - 1 + k.nbase;
    k.row0 = m->root_fixed ? 1 : 0;
    k.rows = m->nb - k.row0;
    k.root_stride = root_stride;
    for (int i = 0; i < m->nl; i++) {
        const int p = i ? m->parent[i] : 0;
        k.parent[i] = p;
        k.depth[i] = i ? k.depth[p] + 1 : 0;
        k.anc[i] = i ? (k.anc[p] | (1u << i)) : 0u;
        if (k.depth[i] > k.maxdepth) k.maxdepth = k.depth[i];
        k.slide[i] = (i && m->jtype[i] == 1) ? 1 : 0;
        if (i) { if (k.nchild[p] == KIN_MAX_CHILD) return -1; k.child[p][k.nchild[p]++] = i; }
        host_quat_to_mat(m->lquat + 4 * i, k.R0[i]);
        for (int c = 0; c < 3; c++) { k.lpos[i][c] = m->lpos[3 * i + c]; k.axis[i][c] = m->axis[3 * i + c]; k.com[i][c] = m->com[3 * i + c]; }
        for (int c = 0; c < 6; c++) k.Ic[i][c] = m->inertia[6 * i + c];
        k.mass[i] = m->mass[i]; k.armature[i] = m->armature[i];
    }
    for (int b = 0; b < m->nb; b++) {
        k.body_link[b] = m->body_link[b];
        for (int c = 0; c < 3; c++) k.body_pos[b][c] = m->body_pos[3 * b + c];
    }
    return 0;
}

}   // namespace b2g

// b2g_model_host.h -- host side of b2g_create / b2g_create_ext: validates the articulation, builds its slot program and
// the generic model (DevModel), picks the CTA size and dynamic shared memory, places the self-collision scratch, builds
// the Jacobian tables and decides whether the quad path takes the model.  Plain C++ (no CUDA calls), shared by
// b200gym.cu and tests/model_host.cu (the CPU test of these decisions).
#pragma once
#include <math.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../include/b200gym.h"
#include "b2g_device.cuh"
#include "b2g_kin_host.h"
#include "b2g_quad_host.h"

namespace b2g {

// What a sim is built from, all of it decided on the host before the first CUDA call.
struct SimModel {
    int lanes = 1;
    int block = 128;             // threads per CTA, chosen so the slot state fits in shared memory
    size_t dyn_smem = 0;
    DevModel hm;                 // host copy of the generic model
    KinModel hk;                 // constant tables of the Jacobian / mass-matrix kernel (b2g_kin.cuh)
    bool kin_ok = false;
    // quad path (b2g_quad.cuh): chain length (2 Ant-like, 3 ANYmal-like) or 0 = generic Stepper; the packed constants
    int quad_ns = 0;
    int quad_spec = 0;           // QLane specialisation flags the constants are packed for (b2g_quad.cuh)
    std::vector<float> qm;
};

// (lane << 8) | slot of the slot that holds `link`, or -1
static inline int slot_of_link(const DevModel &h, int link) {
    for (int sl = 0; sl < h.ns; sl++)
        for (int l = 0; l < h.lanes; l++)
            if (h.slots[sl][l].link == link) return (l << 8) | sl;
    return -1;
}

// Build the lanes' slot programs: list-schedule the links over `L` lanes, critical path first; a lane
// keeps following a chain (parent at step s-1 in the same lane -> state travels in registers), any
// other parent/child relation goes through shared memory (parked inertia / pose / acceleration).
static inline int schedule(const b2g_model *m, int L, DevModel &h, bool compact = false) {
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

static inline int pick_lanes(const b2g_model *m, bool single) {
    if (single) return 1;
    int root_children = 0;
    for (int i = 1; i < m->nl; i++) if (m->parent[i] == 0) root_children++;
    if (m->nl - 1 >= 16) return 4;                 // long trees (Humanoid, hands): chains run in parallel lanes
    if (root_children >= 4) return 4;              // quadrupeds
    if (root_children >= 2) return 2;
    return 1;
}

// Everything a sim is built from (SimModel), from the importer's articulation, its optional extra actors and the sim
// parameters.  single_lane: one thread per env (the reference the 4-lane kernels are compared with); no_quad: the generic
// Stepper even where the quad path would take the model.  Returns B2G_OK, or an error code with *err set.
static inline int build_sim_model(const b2g_model *m, const b2g_model_ext *ext, const b2g_sim_params *sp, bool single_lane,
                                  bool no_quad, SimModel &out, const char **err) {
    auto bad = [&](int code, const char *msg) { *err = msg; return code; };
    if (ext && (ext->actors_per_env < 1 || ext->obj_actor >= ext->actors_per_env || ext->obj_actor == 0 || ext->nbox < 0 ||
                ext->nbox > MAX_BOX || ext->nten < 0 || ext->nten > MAX_TEN))
        return bad(B2G_E_INVALID, "b2g_create_ext: bad actor / box / tendon counts");
    if (ext && ext->obj_actor > 0 && sp->hf_samples) return bad(B2G_E_UNSUPPORTED, "b2g_create_ext: the free object needs the ground plane");
    if (m->nl < 1 || m->nl > MAX_LINKS || m->nl - 1 > MAX_SLOTS || m->ncp > MAX_CP || m->nsens > MAX_SENS || m->nb > MAX_LINKS)
        return bad(B2G_E_INVALID, "b2g_create: model exceeds compiled limits (links/contact points/sensors)");
    DevModel &h = out.hm;
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
    const bool compact = ext && ext->obj_actor > 0;                     // [link][k][env] state layout (Stepper<.., OBJ>)
    if (schedule(m, pick_lanes(m, single_lane), h, compact) != 0) return bad(B2G_E_INVALID, "b2g_create: the articulation does not fit the slot program limits");
    out.lanes = h.lanes;
    h.root_stride = ext ? ext->actors_per_env : 1;
    h.obj_on = 0; h.obj_acc = h.obj_pose_acc = -1;
    if (ext) {
        if (ext->obj_actor > 0) {
            h.obj_on = 1; h.obj_row = ext->obj_actor; h.obj_gravity_on = ext->obj_gravity_on;
            h.obj_mass = ext->obj_mass; h.obj_kn = ext->obj_kn; h.obj_cn = ext->obj_cn; h.obj_mu = ext->obj_mu;
            for (int c = 0; c < 3; c++) { h.obj_I[c] = ext->obj_inertia[c]; h.obj_half[c] = ext->obj_half[c]; }
            h.obj_round = ext->obj_round; h.obj_max_angvel = ext->obj_max_angular_velocity;
            if (ext->obj_round < 0.f || (ext->obj_round == 0.f && (ext->obj_half[0] <= 0.f || ext->obj_half[1] <= 0.f || ext->obj_half[2] <= 0.f)))
                return bad(B2G_E_INVALID, "b2g_create_ext: the object needs positive half extents, or a rounding radius");
            h.obj_acc = h.nacc; h.obj_pose_acc = h.nacc + h.lanes; h.nacc += h.lanes + 1;   // env-wide ids: one sum per lane, one pose
            // the object's gravity does not follow the articulation's disable_gravity flag (shadow_hand.py:239,279-282)
            for (int c = 0; c < 3; c++) h.obj_g[c] = ext->obj_gravity_on ? sp->gravity[c] : 0.f;
        }
        h.nbox = ext->nbox;
        for (int b = 0; b < ext->nbox; b++) {
            h.box_link[b] = ext->box_link[b];
            if (ext->box_link[b] < 0 || ext->box_link[b] >= m->nl) return bad(B2G_E_INVALID, "b2g_create_ext: box link out of range");
            host_quat_to_mat(ext->box_quat[b], h.box_R[b]);
            for (int c = 0; c < 3; c++) { h.box_pos[b][c] = ext->box_pos[b][c]; h.box_half[b][c] = ext->box_half[b][c]; }
        }
        h.nten = ext->nten; h.ten_k = ext->ten_k; h.ten_d = ext->ten_d;
        for (int t = 0; t < ext->nten; t++) for (int k = 0; k < 2; k++) {
            const int ref = slot_of_link(h, ext->ten_dof[t][k] + 1);
            if (ref < 0) return bad(B2G_E_INVALID, "b2g_create_ext: tendon joint index out of range");
            h.ten_ref[t][k] = ref; h.ten_coef[t][k] = ext->ten_coef[t][k]; h.ten_range[t][k] = ext->ten_range[t][k];
        }
        if (h.nten > 0 && !h.obj_on) return bad(B2G_E_UNSUPPORTED, "b2g_create_ext: tendons are only compiled into the object-enabled kernels");
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
        if (!best) return bad(B2G_E_INVALID, "b2g_create: articulation too large for shared-memory slot state");
        out.block = best; out.dyn_smem = rows * (size_t)((best / h.lanes) | 1) * sizeof(float4);
    } else {   // CTA size: the per-thread slot state must fit in shared memory, preferably several CTAs per SM
        const size_t per_thread = ((size_t)h.ns * SLOT_F4 + (size_t)h.nacc * ACC_F4) * sizeof(float4);
        // self-collision scratch per ENV: preferably in a run of consecutive slot cells of one lane that no link occupies
        // (10 float4 each; no extra shared memory, the CTA size is unchanged), else behind the accumulator pool: sphere
        // centres, hit count, hit list (odd float4 count: banks)
        h.self_on = (m->self_collide && m->self_pairs) ? 1 : 0;
        h.self_f4 = 0;
        if (h.self_on) {
            const int need = (m->ncp + 1 + SELF_HITS * 2 / 16 + SLOT_F4 - 1) / SLOT_F4;
            int found = -1;
            for (int l = 0; l < h.lanes && found < 0; l++) for (int s0 = 0; s0 + need <= h.ns && found < 0; s0++) {
                bool idle = true;
                for (int k = 0; k < need; k++) idle = idle && h.slots[s0 + k][l].link < 0;
                if (idle) found = (l << 8) | s0;
            }
            h.self_cell = found;
            if (found < 0) h.self_f4 = (m->ncp + 1 + SELF_HITS * 2 / 16) | 1;
        }
        auto bytes_of = [&](int b) { return per_thread * b + (size_t)(b / h.lanes) * h.self_f4 * sizeof(float4); };
        int blk = 128;
        while (blk > 32 && bytes_of(blk) > 104 * 1024) blk >>= 1;
        if (bytes_of(blk) > 200 * 1024) return bad(B2G_E_INVALID, "b2g_create: articulation too large for shared-memory slot state");
        out.block = blk; out.dyn_smem = bytes_of(blk);
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
        host_quat_to_mat(m->lquat + 4 * i, l.R0);
        const float *R = l.R0;
        for (int c = 0; c < 3; c++) { l.lpos[c] = m->lpos[3 * i + c]; l.axis[c] = m->axis[3 * i + c]; l.com[c] = m->com[3 * i + c]; }
        for (int c = 0; c < 6; c++) l.Ic[c] = m->inertia[6 * i + c];
        l.mass = m->mass[i];
        l.armature = m->armature[i]; l.damping = m->damping[i]; l.stiffness = m->stiffness[i];
        l.lower = m->lower[i]; l.upper = m->upper[i]; l.effort = m->effort[i];
        l.kp = m->kp[i]; l.kd = m->kd[i]; l.limit_k = m->limit_k[i]; l.limit_d = m->limit_d[i];
        const bool ident = fabsf(R[0] - 1.f) < 1e-7f && fabsf(R[4] - 1.f) < 1e-7f && fabsf(R[8] - 1.f) < 1e-7f;
        l.flags = (m->jtype[i] == 1 ? LF_SLIDE : 0) | (m->limited[i] ? LF_LIMITED : 0) | (m->drive_mode[i] == 1 ? LF_POSDRIVE : 0) | (ident ? LF_R0_IDENTITY : 0);
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
        if (compact || (ext && ext->obj_actor >= 0)) return bad(B2G_E_UNSUPPORTED, "b2g_create_ext: self-collision is not compiled into the object-enabled kernels");
        if (m->ncp > 64 || m->nl > MAX_LINKS) return bad(B2G_E_UNSUPPORTED, "b2g_create: self-collision supports at most 64 contact spheres / 32 links");
        h.self_kn = m->self_kn; h.self_cn = m->self_cn; h.self_mu = m->self_mu;
        std::vector<int> inv(m->ncp);
        for (int k = 0; k < m->ncp; k++) inv[order[k]] = k;
        h.npairs = 0;
        for (int a = 0; a < m->ncp; a++) for (int b = a + 1; b < m->ncp; b++) {
            if (!m->self_pairs[(size_t)a * m->ncp + b] && !m->self_pairs[(size_t)b * m->ncp + a]) continue;
            if (h.npairs >= MAX_PAIRS) return bad(B2G_E_UNSUPPORTED, "b2g_create: too many self-collision pairs");
            const int ia = std::min(inv[a], inv[b]), ib = std::max(inv[a], inv[b]);
            h.pair_list[h.npairs++] = (unsigned short)(ia | (ib << 8));
        }
        while (h.npairs % (4 * h.lanes)) { if (h.npairs >= MAX_PAIRS) return bad(B2G_E_UNSUPPORTED, "b2g_create: too many self-collision pairs"); h.pair_list[h.npairs++] = 0; }
        h.npairs /= 4;                                              // quads from here on
        for (int i = 0; i < MAX_LINKS; i++) h.link_slot[i] = i > 0 ? slot_of_link(h, i) : -1;
    }
    // height field (the caller uploads the samples)
    if (sp->hf_samples) {
        h.has_hf = 1; h.hf_nx = sp->hf_nx; h.hf_ny = sp->hf_ny;
        h.hf_scale = sp->hf_horizontal_scale; h.hf_inv_scale = 1.f / sp->hf_horizontal_scale; h.hf_vscale = sp->hf_vertical_scale;
        h.hf_ox = sp->hf_origin_x; h.hf_oy = sp->hf_origin_y;
    }
    out.kin_ok = kin_build(m, h.root_stride, out.hk) == 0;
    // the specialised path of "four hinge chains on a free base" (Ant, ANYmal): b2g_quad.cuh
    out.quad_ns = out.quad_spec = 0;
    out.qm.clear();
    if (!no_quad && !ext && !single_lane) {                              // a self-colliding model: ANYmal-class only (quad_build)
        int leg_link[12];
        out.quad_ns = quad_build(m, sp, out.qm, leg_link, &out.quad_spec);
    }
    return B2G_OK;
}

}  // namespace b2g

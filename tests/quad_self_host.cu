// tests/quad_self_host.cu -- TEST INFRASTRUCTURE: the quad sub-step with link-link contact (QLane<.., SELF = true>,
// isaacgymenvs_b200/csrc/b2g_quad.cuh) on the HOST, lane by lane, so the arithmetic the CUDA kernels execute can be compared
// with the fp64 oracle without a GPU.  The device runs the four lanes of an env in lock-step with a __syncwarp around the
// kinematics pre-pass; here every lane's pre-pass runs before any lane's sweep, which is the same order of reads and writes.
// Built by tests/test_quad_self_host.py (nvcc -shared, host code only is called; nothing here is part of the product library).
#include <vector>
#include <stdint.h>
#include "../isaacgymenvs_b200/csrc/b2g_quad_host.h"

using namespace b2g;

template <int NS, bool HF>
static void run(const std::vector<float> &qmv, const int16_t *hf, int N, int substeps, float *root, float *dof, const float *act,
                float *dof_force, float *net_contact, int nb, const int *leg_link, const float *mass_scale, const float *dof_props,
                const float *env_friction) {
    using QL = QLane<NS, HF, 0, true>;
    const float4 *qm = reinterpret_cast<const float4 *>(qmv.data());
    const int nd = 4 * NS;
    std::vector<float4> park((size_t)4 * quad_park_f4(NS, true));
    for (int e = 0; e < N; e++) {
        QL L[4];
        RootState rs;
        const float *r = root + 13 * (size_t)e;
        for (int c = 0; c < 3; c++) { rs.rp[c] = r[c]; rs.rv[c] = r[7 + c]; rs.rw[c] = r[10 + c]; }
        for (int c = 0; c < 4; c++) rs.rq[c] = r[3 + c];
        for (int l = 0; l < 4; l++) {
            L[l].qm = qm; L[l].hf = hf; L[l].park = park.data() + l; L[l].pstride = 4; L[l].lane = l; L[l].env_mu = -1.f;
            L[l].dr_mass = mass_scale ? mass_scale + (size_t)e * (nd + 1) : nullptr;
            L[l].dr_dof = dof_props ? reinterpret_cast<const float4 *>(dof_props) + (size_t)e * nd : nullptr;
            if (env_friction) L[l].env_mu = 0.5f * (env_friction[e] + qm[18].x);
            for (int s = 0; s < NS; s++) {
                const int d = leg_link[l * NS + s] - 1;
                L[l].q[s] = dof[((size_t)e * nd + d) * 2]; L[l].qd[s] = dof[((size_t)e * nd + d) * 2 + 1];
                L[l].act[s] = act ? act[(size_t)e * nd + d] : 0.f;
            }
        }
        QOutputs o;
        o.sensor = nullptr;
        o.dof_force = dof_force ? dof_force + (size_t)e * nd : nullptr;
        o.net_contact = net_contact ? net_contact + (size_t)e * nb * 3 : nullptr;
        o.write = true;
        for (int k = 0; k < substeps; k++) {
            const bool LAST = k == substeps - 1;
            for (int l = 0; l < 4; l++) L[l].self_prepass(rs);
            float IA[21] = {0}, pa[3] = {0}, pl[3] = {0};
            for (int l = 0; l < 4; l++) {
                float I[21], a[3], b[3];
                L[l].sweep(rs, false, I, a, b);
                for (int c = 0; c < 21; c++) IA[c] += I[c];
                for (int c = 0; c < 3; c++) { pa[c] += a[c]; pl[c] += b[c]; }
            }
            float awr[3], alr[3];
            QL::solve_base(IA, pa, pl, awr, alr);
            if (LAST && L[0].root_emits(o)) {
                float F[3] = {0, 0, 0}, T[3] = {0, 0, 0};
                for (int l = 0; l < 4; l++) {
                    float f[3], t[3];
                    L[l].root_wrench(rs, awr, alr, f, t);
                    for (int c = 0; c < 3; c++) { F[c] += f[c]; T[c] += t[c]; }
                }
                L[0].emit_root(rs, o, F, T);
            }
            for (int l = 0; l < 4; l++) L[l].accelerate(rs, awr, alr, LAST, o);
            L[0].integrate_base(rs, awr, alr);
        }
        float *rw = root + 13 * (size_t)e;
        for (int c = 0; c < 3; c++) { rw[c] = rs.rp[c]; rw[7 + c] = rs.rv[c]; rw[10 + c] = rs.rw[c]; }
        for (int c = 0; c < 4; c++) rw[3 + c] = rs.rq[c];
        for (int l = 0; l < 4; l++) for (int s = 0; s < NS; s++) {
            const int d = leg_link[l * NS + s] - 1;
            dof[((size_t)e * nd + d) * 2] = L[l].q[s]; dof[((size_t)e * nd + d) * 2 + 1] = L[l].qd[s];
        }
    }
}

// the self-colliding model on the quad path: returns NS (3), 0 when the quad path does not take the model (or it does not
// self-collide), <0 on error.  Outputs as quad_host_simulate (tests/quad_host.cu), without force sensors.
extern "C" int quad_self_host_simulate(const b2g_model *m, const b2g_sim_params *sp, int N, float *root, float *dof, const float *act,
                                       float *dof_force, float *net_contact, const float *mass_scale, const float *dof_props,
                                       const float *env_friction) {
    if (!m->self_collide || !m->self_pairs || m->nsens) return -1;
    std::vector<float> qm;
    int leg_link[12], spec = 0;
    const int NS = quad_build(m, sp, qm, leg_link, &spec);
    if (NS != 3) return NS;
    if (spec != 0 || qm.size() != (size_t)quad_model_f4(3, true) * 4) return -2;
    if (sp->hf_samples) run<3, true>(qm, sp->hf_samples, N, sp->substeps, root, dof, act, dof_force, net_contact, m->nb, leg_link, mass_scale, dof_props, env_friction);
    else run<3, false>(qm, nullptr, N, sp->substeps, root, dof, act, dof_force, net_contact, m->nb, leg_link, mass_scale, dof_props, env_friction);
    return NS;
}

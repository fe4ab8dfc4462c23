// tests/model_host.cu -- TEST INFRASTRUCTURE: runs the host-side model builder of b2g_create / b2g_create_ext
// (isaacgymenvs_b200/csrc/b2g_model_host.h) on the CPU, so its decisions can be checked on a machine without a GPU.
// Built by tests/test_model_host.py (nvcc -shared, host code only is called; nothing here is part of the product library).
#include "../isaacgymenvs_b200/csrc/b2g_model_host.h"

using namespace b2g;

// out: lanes, CTA size, dynamic shared memory, ns, nacc, self_cell, self_f4, quad_ns, quad_spec.  Returns the builder's code.
extern "C" int model_host_build(const b2g_model *m, const b2g_model_ext *ext, const b2g_sim_params *sp, int single_lane, int64_t out[9]) {
    SimModel *sm = new SimModel;
    const char *err = "";
    const int rc = build_sim_model(m, ext, sp, single_lane != 0, false, *sm, &err);
    const int64_t v[9] = {sm->lanes, sm->block, (int64_t)sm->dyn_smem, sm->hm.ns, sm->hm.nacc, sm->hm.self_cell, sm->hm.self_f4,
                          sm->quad_ns, sm->quad_spec};
    memcpy(out, v, sizeof(v));
    delete sm;
    return rc;
}

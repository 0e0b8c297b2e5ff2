// TEST INFRASTRUCTURE (never part of the product): host build of the device environment's validation and apply bodies with the
// action read from an action table by id (grid2op_b200/csrc/b200pf_env.cuh, ActIds), run over the batch in instance order, so that
// the tensor path's id action can be checked against the numpy BatchedEnv on a machine without a GPU.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int act_ids_emu_sizes(int *out) {
    out[0] = (int)sizeof(EnvArgs);
    out[1] = (int)sizeof(ActArgs);
    out[2] = (int)sizeof(ActIds);
    return 0;
}

// what: 0 validate (sets ctl[ENV_CTL_ERR]), 1 apply (nothing when ctl[ENV_CTL_ERR] is set)
extern "C" int act_ids_emu_run(const EnvArgs *a, const ActArgs *r, const ActIds *ids, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!act_input_ok(*a, *r, i, ids)) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i, nullptr, nullptr, nullptr, r, ids); break;
        default: return -1;
        }
    }
    return 0;
}

// TEST INFRASTRUCTURE (never part of the product): host build of the device environment bodies with the action rules and the vector
// action bound (grid2op_b200/csrc/b200pf_env.cuh, ActArgs), run over the batch in instance order, so that the tensor path's vector
// action can be checked against the numpy BatchedEnv on a machine without a GPU.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int act_emu_sizes(int *out) {
    out[0] = (int)sizeof(EnvArgs);
    out[1] = (int)sizeof(ActArgs);
    return 0;
}

// what: 0 validate (sets ctl[ENV_CTL_ERR]), 1 apply (nothing when ctl[ENV_CTL_ERR] is set), 2 post, 3 reset
extern "C" int act_emu_run(const EnvArgs *a, const ActArgs *r, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!(r->vec ? act_input_ok(*a, *r, i) : env_input_ok(*a, i))) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i, nullptr, nullptr, nullptr, r); break;
        case 2: env_post_instance(*a, i, nullptr, nullptr, r); break;
        case 3: env_reset_instance(*a, i, nullptr, nullptr, nullptr, nullptr, nullptr, r); break;
        default: return -1;
        }
    }
    return 0;
}

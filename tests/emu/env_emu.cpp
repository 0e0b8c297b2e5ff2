// TEST INFRASTRUCTURE (never part of the product): host build of the device environment bodies (grid2op_b200/csrc/b200pf_env.cuh:
// validation, apply, post, reset), run over the batch in instance order, so that BatchedEnv.step_tensors' bookkeeping can be checked
// against the numpy BatchedEnv on a machine without a GPU.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int env_emu_args_size(void) { return (int)sizeof(EnvArgs); }

// what: 0 validate (sets ctl[ENV_CTL_ERR]), 1 apply (nothing when ctl[ENV_CTL_ERR] is set), 2 post, 3 reset, 4 after an observe
extern "C" int env_emu_run(const EnvArgs *a, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!env_input_ok(*a, i)) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i); break;
        case 2: env_post_instance(*a, i); break;
        case 3: env_reset_instance(*a, i); break;
        case 4: env_observed_instance(*a, i); break;
        default: return -1;
        }
    }
    return 0;
}

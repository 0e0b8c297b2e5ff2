// TEST INFRASTRUCTURE (never part of the product): host build of the device GeometricOpponentMultiArea (grid2op_b200/csrc/b200pf_opp.cuh)
// inside the environment bodies (b200pf_env.cuh), run over the batch in instance order, so that BatchedEnv.step_tensors'
// multi-area opponent can be checked against the numpy path and grid2op on a machine without a GPU.  Built with libm's log1p.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int multi_emu_args_size(void) { return (int)sizeof(OppMultiArgs); }
extern "C" int multi_emu_opp_args_size(void) { return (int)sizeof(OppArgs); }
extern "C" int multi_emu_env_args_size(void) { return (int)sizeof(EnvArgs); }

// what: 0 validate, 1 apply (with the opponent), 2 post, 3 reset (with the opponent), 4 after an observe
extern "C" int multi_emu_run(const EnvArgs *a, const OppArgs *o, const OppMultiArgs *m, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!env_input_ok(*a, i)) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i, o, nullptr, m); break;
        case 2: env_post_instance(*a, i); break;
        case 3: env_reset_instance(*a, i, o, nullptr, m); break;
        case 4: env_observed_instance(*a, i); break;
        default: return -1;
        }
    }
    return 0;
}

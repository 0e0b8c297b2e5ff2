// TEST INFRASTRUCTURE (never part of the product): host build of the device opponent (grid2op_b200/csrc/b200pf_opp.cuh) inside the
// environment bodies (b200pf_env.cuh), run over the batch in instance order, and its numpy-legacy random draws one by one, so that
// BatchedEnv.step_tensors' opponent can be checked against the numpy path and np.random.RandomState on a machine without a GPU.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int opp_emu_args_size(void) { return (int)sizeof(OppArgs); }
extern "C" int opp_emu_env_args_size(void) { return (int)sizeof(EnvArgs); }

// what: 0 validate, 1 apply (with the opponent), 2 post, 3 reset (with the opponent), 4 after an observe
extern "C" int opp_emu_run(const EnvArgs *a, const OppArgs *o, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!env_input_ok(*a, i)) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i, o); break;
        case 2: env_post_instance(*a, i); break;
        case 3: env_reset_instance(*a, i, o); break;
        case 4: env_observed_instance(*a, i); break;
        default: return -1;
        }
    }
    return 0;
}

// RandomState draws on one state (mt [624], *pos)
extern "C" void opp_emu_randint(uint32_t *mt, int32_t *pos, uint32_t n, int count, uint32_t *out) {
    for (int k = 0; k < count; ++k) out[k] = opp_randint(mt, pos, n);
}
extern "C" void opp_emu_random_sample(uint32_t *mt, int32_t *pos, int count, double *out) {
    for (int k = 0; k < count; ++k) out[k] = opp_random_sample(mt, pos);
}
// choice(n, p=w / w.sum()) (w >= 0, positive sum); -1 when the sum is not positive
extern "C" int opp_emu_choice_weighted(uint32_t *mt, int32_t *pos, const double *w, int n) {
    const double s = opp_np_sum(w, n);
    if (!(s > 0.0)) return -1;
    return opp_choice_weighted(mt, pos, w, n, s);
}

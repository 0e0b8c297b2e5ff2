// TEST INFRASTRUCTURE (never part of the product): host build of the device GeometricOpponent (grid2op_b200/csrc/b200pf_opp.cuh)
// inside the environment bodies (b200pf_env.cuh), run over the batch in instance order, and its draws one by one, so that
// BatchedEnv.step_tensors' GeometricOpponent can be checked against the numpy path, np.random.RandomState and grid2op on a machine
// without a GPU.  Built with libm's log1p.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"

using namespace b200pf;

extern "C" int geo_emu_args_size(void) { return (int)sizeof(OppGeoArgs); }
extern "C" int geo_emu_opp_args_size(void) { return (int)sizeof(OppArgs); }
extern "C" int geo_emu_env_args_size(void) { return (int)sizeof(EnvArgs); }

// what: 0 validate, 1 apply (with the opponent), 2 post, 3 reset (with the opponent), 4 after an observe
extern "C" int geo_emu_run(const EnvArgs *a, const OppArgs *o, const OppGeoArgs *g, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 0: if (!env_input_ok(*a, i)) a->ctl[ENV_CTL_ERR] |= 1; break;
        case 1: if (a->ctl[ENV_CTL_ERR]) return 0; env_apply_instance(*a, i, o, g); break;
        case 2: env_post_instance(*a, i); break;
        case 3: env_reset_instance(*a, i, o, g); break;
        case 4: env_observed_instance(*a, i); break;
        default: return -1;
        }
    }
    return 0;
}

// RandomState.geometric(p) on one state (mt [624], *pos), count draws
extern "C" void geo_emu_geometric(uint32_t *mt, int32_t *pos, double p, double logq, int count, int64_t *out) {
    for (int k = 0; k < count; ++k) out[k] = opp_geometric(mt, pos, p, logq);
}

// one schedule (sample_attack_times_and_durations) on one state -> its length; wait / dur [cap]; *dropped: entries past the cap
extern "C" int geo_emu_sample(uint32_t *mt, int32_t *pos, double p_hazard, double logq_hazard, double p_recovery, double logq_recovery,
                              int recovery_min, int32_t episode_max_time, int cap, int32_t *wait, int32_t *dur, int32_t *dropped) {
    int32_t gctr[OPP_GEO_CTR] = {0, 0, 0, 0};
    OppGeoArgs g{};
    g.p_hazard = p_hazard; g.logq_hazard = logq_hazard; g.p_recovery = p_recovery; g.logq_recovery = logq_recovery;
    g.recovery_min = recovery_min; g.cap = cap; g.emt = &episode_max_time; g.wait = wait; g.dur = dur; g.gctr = gctr;
    opp_geo_sample(g, 0, mt, pos);
    *dropped = gctr[OPP_GEO_OVERFLOW];
    return gctr[OPP_GEO_N];
}

// the attack of an opponent whose first scheduled attack (duration 5) is due now, on n connected lines 0..n-1 with rho [n]:
// ranks, weight table and choice -> the attacked line; the draws advance the state
extern "C" int geo_emu_attack(uint32_t *mt, int32_t *pos, int n, const float *rho, const double *weights, int32_t *dur) {
    int32_t lines[OPP_MAX_ATTACK], lor[OPP_MAX_ATTACK], lex[OPP_MAX_ATTACK];
    int8_t tv[2 * OPP_MAX_ATTACK];
    for (int k = 0; k < n; ++k) { lines[k] = k; lor[k] = 2 * k; lex[k] = 2 * k + 1; tv[2 * k] = tv[2 * k + 1] = 1; }
    int32_t ctr[OPP_CTR] = {0, 0, -1, OPP_NEXT_UNSET}, gctr[OPP_GEO_CTR] = {1, 0, 0, 0}, wait = 0, d = 5, emt = 1;
    OppArgs o{};
    o.kind = OPP_GEOMETRIC; o.n_attack = n; o.lines = lines; o.mt = mt; o.mt_pos = pos; o.rho = rho;
    OppGeoArgs g{};
    g.weights = weights; g.cap = 1; g.emt = &emt; g.wait = &wait; g.dur = &d; g.gctr = gctr;
    return opp_geo_attack(o, g, 0, tv, lor, lex, n, ctr, gctr, dur);
}

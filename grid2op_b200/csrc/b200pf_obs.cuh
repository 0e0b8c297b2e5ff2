// b200pf_obs.cuh — grid2op observation vectors and rewards of a whole batch, assembled on the device from what a series step
// leaves in HBM (result record, rho, device topology, chronics row index) plus a few host-only values per instance.
//
// What one instance's body restates (reference, per env):
//   obs.to_vect()        grid2op/Observation/baseObservation.py (update :4360-4530, set_game_over :1551-1700) for the attribute
//                        list of the environment's observation class (CompleteObservation.attr_list_vect, completeObservation.py:140-212,
//                        or a subset); every attribute as float32, in the order given;
//   reward               RedispReward (grid2op/Reward/redispReward.py:141-211) or L2RPNReward (l2RPNReward.py:52-77).
// Without redispatching, curtailment, storage actions or detachment these attributes hold the values the
// reference produces when the features are unused.  The overflow counters timestep_overflow / timestep_protection_engaged
// (baseEnv.py:3361-3370, counted even under NO_OVERFLOW_DISCONNECTION) are kept here, per instance, because the series kernels
// only count while their protections are on.
//
// The body is __host__ __device__: the CUDA launch runs one warp per instance; a host build (tests/emu) runs the same source with
// one "lane".  Values are computed element by element in the same order on both, so the vector is bit-identical; only the sums of the
// reward are reduced in a different order (32 lane partials + butterfly on the device, one sequential sum on the host).
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define OBS_HD __host__ __device__
#else
#define OBS_HD
#endif

namespace b200pf {

// attribute sources of the observation vector (grid2op_b200/observation.py OBS_SOURCES has the same order)
enum ObsSrc : int32_t {
    OS_YEAR = 0, OS_MONTH, OS_DAY, OS_HOUR, OS_MINUTE, OS_WEEKDAY,
    OS_GEN_P, OS_GEN_Q, OS_GEN_V, OS_LOAD_P, OS_LOAD_Q, OS_LOAD_V,
    OS_P_OR, OS_Q_OR, OS_V_OR, OS_A_OR, OS_P_EX, OS_Q_EX, OS_V_EX, OS_A_EX,
    OS_RHO, OS_LINE_STATUS, OS_TS_OVERFLOW, OS_TOPO_VECT, OS_CD_LINE, OS_CD_SUB, OS_T_NEXT_MAINT, OS_D_NEXT_MAINT,
    OS_TARGET_DISPATCH, OS_ACTUAL_DISPATCH, OS_STORAGE_CHARGE, OS_STORAGE_POWER_TARGET, OS_STORAGE_POWER,
    OS_GEN_P_BEFORE_CURTAIL, OS_CURTAILMENT, OS_CURTAILMENT_LIMIT, OS_CURTAILMENT_LIMIT_EFFECTIVE,
    OS_IS_ALARM_ILLEGAL, OS_TIME_SINCE_LAST_ALARM, OS_LAST_ALARM, OS_ATTENTION_BUDGET, OS_WAS_ALARM_USED_AFTER_GAME_OVER,
    OS_SHUNT_P, OS_SHUNT_Q, OS_SHUNT_V, OS_SHUNT_BUS, OS_CURRENT_STEP, OS_MAX_STEP, OS_DELTA_TIME,
    OS_GEN_MARGIN_UP, OS_GEN_MARGIN_DOWN,
    OS_ACTIVE_ALERT, OS_ATTACK_UNDER_ALERT, OS_TIME_SINCE_LAST_ALERT, OS_ALERT_DURATION, OS_TOTAL_NUMBER_OF_ALERT,
    OS_TIME_SINCE_LAST_ATTACK, OS_WAS_ALERT_USED_AFTER_ATTACK,
    OS_GEN_P_DELTA, OS_LOAD_DETACHED, OS_GEN_DETACHED, OS_STORAGE_DETACHED, OS_LOAD_P_DETACHED, OS_LOAD_Q_DETACHED,
    OS_GEN_P_DETACHED, OS_STORAGE_P_DETACHED, OS_TS_PROTECTION_ENGAGED,
    OS_N_SOURCES
};

enum { OBS_REWARD_NONE = 0, OBS_REWARD_REDISP = 1, OBS_REWARD_L2RPN = 2 };

// per-instance host input word flags (last int32 of the instance's host record)
enum { OBS_F_ILLEGAL = 1, OBS_F_DONE = 2, OBS_F_RESET_COUNTERS = 4, OBS_F_AMBIGUOUS = 8 };

struct ObsArgs {
    int batch;
    // grid sizes
    int n_line, n_sub, n_gen, n_hidden, n_load, n_sto, n_shunt, dim_topo, n_topo_in, n_out;
    const int32_t *line_or_pos, *line_ex_pos;           // [n_line]
    // what the series step left on the device
    const float *out;                                   // [batch][n_out] result records
    const float *rho;                                   // [batch][n_line]
    const int8_t *topo;                                 // [batch][n_topo_in] device topology
    const int32_t *t;                                   // [batch] chronics row of the NEXT solve
    const int32_t *scen;                                // [batch]
    const float *chron;                                 // [n_scen][n_rows][2 n_load + 2 n_gen]
    int n_rows;
    const float *th_lim;                                // [n_line] A
    // static tables bound once (b200pf_obs_bind)
    const int32_t *calendar;                            // [n_scen][n_rows][6] year month day hour minute weekday of every row
    const int32_t *max_step;                            // [n_scen]
    float delta_time;                                   // minutes
    const int32_t *maint_time, *maint_dur;              // [n_scen][n_rows][n_line] or NULL (no maintenance table)
    const float *gen_pmin, *gen_pmax, *gen_ramp_up, *gen_ramp_down, *gen_cost;   // [n_gen]
    const int8_t *gen_renewable;                        // [n_gen]
    int redisp_available;
    const float *sto_charge0, *sto_loss_step;           // [n_sto]: charge after the reset step, loss withdrawn per step (MWh)
    const int32_t *seg;                                 // [n_seg][3] source, offset, length
    int n_seg, n_obs;
    int reward_kind;
    double max_regret, reward_min, reward_illegal, dts_hours;
    // per-instance host inputs: int32 [batch][host_stride] = cooldown_line[n_line] | cooldown_sub[n_sub] | current_step | stamp | flags,
    // then with line alerts (n_alert > 0) the 6 n_alert + 1 alert values of alert_obs_record (b200pf_alert.cuh), then with alarms
    // (n_alarm > 0) the n_alarm + 4 alarm values of alarm_obs_record (b200pf_alarm.cuh)
    const int32_t *host;
    int host_stride, n_alert, n_alarm;
    // device state of the observation layer
    int32_t *ts_over, *ts_prot;                         // [batch][n_line]
    int32_t *stamp;                                     // [batch]: host stamp of the step the counters were last advanced for
    int32_t *go_row;                                    // [batch]: row of the step that ended the episode (-1: running)
    float soft_thr;
    // outputs
    float *obs;                                         // [batch][n_obs]
    float *reward;                                      // [batch] (may be NULL)
};

OBS_HD inline float obs_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);               // no contraction into an FMA: the host build rounds the product too
#else
    return a * b;
#endif
}

// record offsets (include/b200pf.h "out" layout)
struct ObsRec {
    int p_or, q_or, v_or, a_or, p_ex, q_ex, v_ex, a_ex, unit_p, unit_q, unit_v, sto_v, sh_p, sh_q, sh_v;
    OBS_HD explicit ObsRec(const ObsArgs &a) {
        const int nl = a.n_line, nu = a.n_gen + a.n_hidden;
        p_or = 0; q_or = nl; v_or = 2 * nl; a_or = 3 * nl; p_ex = 5 * nl; q_ex = 6 * nl; v_ex = 7 * nl; a_ex = 8 * nl;
        unit_p = 10 * nl; unit_q = unit_p + nu; unit_v = unit_q + nu;
        sto_v = 10 * nl + 4 * nu + 2 * a.n_load;
        sh_p = sto_v + a.n_sto; sh_q = sh_p + a.n_shunt; sh_v = sh_q + a.n_shunt;
    }
};

// first alarm value of an instance's host record
OBS_HD inline int obs_alarm_off(const ObsArgs &a) { return a.n_line + a.n_sub + 3 + (a.n_alert ? 6 * a.n_alert + 1 : 0); }

// value j of attribute source `src` for one instance (go: the game-over observation, BaseObservation.set_game_over)
OBS_HD inline float obs_value(const ObsArgs &a, const ObsRec &R, int inst, int src, int j, bool go, int row, int sc,
                              const float *rec, const int32_t *hin, const int32_t *tsov, const int32_t *tspr) {
    const int8_t *tv = a.topo + (size_t)inst * a.n_topo_in;
    const float *crow = a.chron + ((size_t)sc * a.n_rows + row) * (size_t)(2 * a.n_load + 2 * a.n_gen);
    const int32_t *cal = a.calendar + ((size_t)sc * a.n_rows + row) * 6;
    switch (src) {
    case OS_YEAR: case OS_MONTH: case OS_DAY: case OS_HOUR: case OS_MINUTE: case OS_WEEKDAY:
        return (float)cal[src - OS_YEAR];
    case OS_GEN_P: return go ? 0.f : rec[R.unit_p + a.n_hidden + j];
    case OS_GEN_Q: return go ? 0.f : rec[R.unit_q + a.n_hidden + j];
    case OS_GEN_V: return go ? 0.f : rec[R.unit_v + a.n_hidden + j];
    case OS_LOAD_P: return go ? 0.f : crow[j];
    case OS_LOAD_Q: return go ? 0.f : crow[a.n_load + j];
    case OS_LOAD_V: return go ? 0.f : rec[10 * a.n_line + 4 * (a.n_gen + a.n_hidden) + j];
    case OS_P_OR: return go ? 0.f : rec[R.p_or + j];
    case OS_Q_OR: return go ? 0.f : rec[R.q_or + j];
    case OS_V_OR: return go ? 0.f : rec[R.v_or + j];
    case OS_A_OR: return go ? 0.f : rec[R.a_or + j];
    case OS_P_EX: return go ? 0.f : rec[R.p_ex + j];
    case OS_Q_EX: return go ? 0.f : rec[R.q_ex + j];
    case OS_V_EX: return go ? 0.f : rec[R.v_ex + j];
    case OS_A_EX: return go ? 0.f : rec[R.a_ex + j];
    case OS_RHO: return go ? 0.f : a.rho[(size_t)inst * a.n_line + j];
    case OS_LINE_STATUS: return (!go && tv[a.line_or_pos[j]] > 0 && tv[a.line_ex_pos[j]] > 0) ? 1.f : 0.f;
    case OS_TS_OVERFLOW: return go ? 0.f : (float)tsov[j];
    case OS_TOPO_VECT: return go ? -1.f : (float)(tv[j] > 0 ? tv[j] : -1);
    case OS_CD_LINE: return go ? 0.f : (float)hin[j];
    case OS_CD_SUB: return go ? 0.f : (float)hin[a.n_line + j];
    case OS_T_NEXT_MAINT:
        return (go || !a.maint_time) ? -1.f : (float)a.maint_time[((size_t)sc * a.n_rows + row) * a.n_line + j];
    case OS_D_NEXT_MAINT:
        return (go || !a.maint_dur) ? 0.f : (float)a.maint_dur[((size_t)sc * a.n_rows + row) * a.n_line + j];
    case OS_STORAGE_CHARGE: {
        if (go) return 0.f;
        const float c = a.sto_charge0[j] - obs_mul((float)hin[a.n_line + a.n_sub], a.sto_loss_step[j]);
        return c > 0.f ? c : 0.f;
    }
    case OS_GEN_P_BEFORE_CURTAIL: return (go || !a.gen_renewable[j]) ? 0.f : rec[R.unit_p + a.n_hidden + j];   // renewables only
    case OS_CURTAILMENT_LIMIT: case OS_CURTAILMENT_LIMIT_EFFECTIVE: return 1.f;
    // alarms (n_alarm > 0): the game-over observation shows no alarm (last_alarm 0, not -1), a budget of 0, and the reward's
    // is_alarm_used; an ordinary one never sets was_alarm_used_after_game_over (BaseObservation._update_alarm, set_game_over)
    case OS_IS_ALARM_ILLEGAL: return (go || !a.n_alarm) ? 0.f : (float)hin[obs_alarm_off(a)];
    case OS_TIME_SINCE_LAST_ALARM: return (go || !a.n_alarm) ? -1.f : (float)hin[obs_alarm_off(a) + 1];
    case OS_LAST_ALARM: return go ? 0.f : (float)hin[obs_alarm_off(a) + 2 + j];
    case OS_ATTENTION_BUDGET: {
        if (go || !a.n_alarm) return 0.f;
        union { int32_t u; float f; } b;
        b.u = hin[obs_alarm_off(a) + 2 + a.n_alarm];
        return b.f;
    }
    case OS_WAS_ALARM_USED_AFTER_GAME_OVER: return (go && a.n_alarm) ? (float)hin[obs_alarm_off(a) + 3 + a.n_alarm] : 0.f;
    // line alerts (n_alert > 0): the game-over observation clears the alerts, their durations and the total, shows no attack,
    // and keeps attack_under_alert / was_alert_used_after_attack (BaseObservation.set_game_over, then update_after_reward)
    case OS_ACTIVE_ALERT: return go ? 0.f : (float)hin[a.n_line + a.n_sub + 3 + j];
    case OS_ATTACK_UNDER_ALERT: return (float)hin[a.n_line + a.n_sub + 3 + a.n_alert + j];
    case OS_TIME_SINCE_LAST_ALERT: return go ? 0.f : (float)hin[a.n_line + a.n_sub + 3 + 2 * a.n_alert + j];
    case OS_ALERT_DURATION: return go ? 0.f : (float)hin[a.n_line + a.n_sub + 3 + 3 * a.n_alert + j];
    case OS_TOTAL_NUMBER_OF_ALERT: return go ? 0.f : (float)hin[a.n_line + a.n_sub + 3 + 4 * a.n_alert];
    case OS_TIME_SINCE_LAST_ATTACK: return go ? -1.f : (float)hin[a.n_line + a.n_sub + 4 + 4 * a.n_alert + j];
    case OS_WAS_ALERT_USED_AFTER_ATTACK: return (float)hin[a.n_line + a.n_sub + 4 + 5 * a.n_alert + j];
    case OS_SHUNT_P: return go ? 0.f : rec[R.sh_p + j];
    case OS_SHUNT_Q: return go ? 0.f : rec[R.sh_q + j];
    case OS_SHUNT_V: return go ? 0.f : rec[R.sh_v + j];
    case OS_SHUNT_BUS: { const int b = tv[a.dim_topo + j]; return (go || b <= 0) ? -1.f : (float)b; }
    case OS_CURRENT_STEP: return (float)hin[a.n_line + a.n_sub];
    case OS_MAX_STEP: return (float)a.max_step[sc];
    case OS_DELTA_TIME: return a.delta_time;
    case OS_GEN_MARGIN_UP: case OS_GEN_MARGIN_DOWN: {
        if (go || !a.redisp_available || a.gen_renewable[j]) return 0.f;
        const float p = rec[R.unit_p + a.n_hidden + j];
        float m = src == OS_GEN_MARGIN_UP ? a.gen_pmax[j] - p : p - a.gen_pmin[j];
        const float r = src == OS_GEN_MARGIN_UP ? a.gen_ramp_up[j] : a.gen_ramp_down[j];
        m = m < r ? m : r;
        return m < 0.f ? 0.f : m;
    }
    case OS_GEN_P_DELTA: return go ? 0.f : rec[R.unit_p + a.n_hidden + j] - crow[2 * a.n_load + j];
    case OS_TS_PROTECTION_ENGAGED: return go ? 0.f : (float)tspr[j];
    default: return 0.f;          // dispatch, storage power, curtailment, detachment: features unused
    }
}

// One instance: advance the overflow counters (once per step stamp), write the vector, compute the reward.
// lane / nlanes: the lanes of the warp that own the instance (host build: 0 / 1).  The reward's partial sums are returned through
// part[4] (gen_p sum, load_p sum, L2RPN score sum, max marginal cost) for the caller to reduce over the lanes.
OBS_HD inline void obs_instance(const ObsArgs &a, int inst, int lane, int nlanes, double part[4]) {
    const ObsRec R(a);
    const int32_t *hin = a.host + (size_t)inst * a.host_stride;
    const int stamp = hin[a.n_line + a.n_sub + 1], flags = hin[a.n_line + a.n_sub + 2];
    const bool go = (flags & OBS_F_DONE) != 0;
    const int sc = a.scen[inst];
    int row = a.t[inst] > 0 ? a.t[inst] - 1 : a.n_rows - 1;                // the row the last step solved
    const int gr = (flags & OBS_F_RESET_COUNTERS) ? -1 : a.go_row[inst];
    if (go && gr >= 0) row = gr;                                           // a finished episode keeps the date it ended on
    const float *rec = a.out + (size_t)inst * a.n_out;
    int32_t *tsov = a.ts_over + (size_t)inst * a.n_line, *tspr = a.ts_prot + (size_t)inst * a.n_line;
    const bool advance = a.stamp[inst] != stamp;
    if (advance || (flags & OBS_F_RESET_COUNTERS)) {
        for (int l = lane; l < a.n_line; l += nlanes) {
            int o = (flags & OBS_F_RESET_COUNTERS) ? 0 : tsov[l], p = (flags & OBS_F_RESET_COUNTERS) ? 0 : tspr[l];
            if (advance && !go) {
                const float flow = rec[R.a_or + l];
                o = flow > a.th_lim[l] ? o + 1 : 0;
                p = flow > obs_mul(a.th_lim[l], a.soft_thr) ? p + 1 : 0;
            }
            tsov[l] = o; tspr[l] = p;
        }
    }
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
    if (lane == 0) a.go_row[inst] = go ? row : -1;
    float *dst = a.obs + (size_t)inst * a.n_obs;
    for (int s = 0; s < a.n_seg; ++s) {
        const int src = a.seg[3 * s], off = a.seg[3 * s + 1], len = a.seg[3 * s + 2];
        for (int j = lane; j < len; j += nlanes) dst[off + j] = obs_value(a, R, inst, src, j, go, row, sc, rec, hin, tsov, tspr);
    }
    part[0] = part[1] = part[2] = 0.0; part[3] = -1e300;
    if (a.reward_kind == OBS_REWARD_NONE || go) return;
    for (int g = lane; g < a.n_gen; g += nlanes) {
        const float p = rec[R.unit_p + a.n_hidden + g];
        part[0] += (double)p;
        if (p > 0.f && (double)a.gen_cost[g] > part[3]) part[3] = (double)a.gen_cost[g];
    }
    const float *crow = a.chron + ((size_t)sc * a.n_rows + row) * (size_t)(2 * a.n_load + 2 * a.n_gen);
    for (int k = lane; k < a.n_load; k += nlanes) part[1] += (double)crow[k];
    if (a.reward_kind == OBS_REWARD_L2RPN)
        for (int l = lane; l < a.n_line; l += nlanes) {
            float x = rec[R.a_or + l];
            x = x < 0.f ? -x : x;
            x = x / (a.th_lim[l] + 0.1f);
            x = x < 1.f ? x : 1.f;
            const float s = 1.f - obs_mul(x, x);
            part[2] += (double)(s > 0.f ? s : 0.f);
        }
}

// reward of one instance from its reduced partial sums (RedispReward.__call__ / L2RPNReward.__call__)
OBS_HD inline float obs_reward(const ObsArgs &a, int inst, const double part[4]) {
    const int32_t *hin = a.host + (size_t)inst * a.host_stride;
    const int flags = hin[a.n_line + a.n_sub + 2];
    if (a.reward_kind == OBS_REWARD_L2RPN) return (flags & OBS_F_DONE) ? 0.f : (float)part[2];
    if (flags & OBS_F_DONE) return (float)a.reward_min;                  // game over = has_error
    if (flags & (OBS_F_ILLEGAL | OBS_F_AMBIGUOUS)) return (float)a.reward_illegal;   // reward_illegal_ambiguous
    const double mc = part[3] > -1e299 ? part[3] : 0.0;
    const double regret = (part[0] - part[1]) * a.dts_hours * mc;       // losses (MWh) x marginal cost; no redispatch, no storage
    return (float)((a.max_regret - regret) / part[1]);
}

#if defined(__CUDACC__)
// one warp per instance, 4 warps per CTA
__global__ void __launch_bounds__(128) pf_kernel_observe(ObsArgs a) {
    const int inst = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (inst >= a.batch) return;
    double part[4];
    obs_instance(a, inst, lane, 32, part);
    if (a.reward_kind == OBS_REWARD_NONE || !a.reward) { if (lane == 0) a.stamp[inst] = a.host[(size_t)inst * a.host_stride + a.n_line + a.n_sub + 1]; return; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        part[0] += __shfl_xor_sync(0xffffffffu, part[0], o);
        part[1] += __shfl_xor_sync(0xffffffffu, part[1], o);
        part[2] += __shfl_xor_sync(0xffffffffu, part[2], o);
        const double m = __shfl_xor_sync(0xffffffffu, part[3], o);
        part[3] = m > part[3] ? m : part[3];
    }
    if (lane == 0) {
        a.reward[inst] = obs_reward(a, inst, part);
        a.stamp[inst] = a.host[(size_t)inst * a.host_stride + a.n_line + a.n_sub + 1];
    }
}
#endif

}  // namespace b200pf

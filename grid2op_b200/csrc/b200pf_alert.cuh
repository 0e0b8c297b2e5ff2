// b200pf_alert.cuh — grid2op's line alerts (l2rpn_idf_2023) for a whole batch on the device: the environment's alert state, the
// AlertReward, and their reset.
//
// What the bodies restate, per instance (grid2op 1.12.5):
//   alert_update_instance   BaseEnv._update_alert_properties (grid2op/Environment/baseEnv.py:3295-3335), run for every live
//                           instance on an ordinary step (the attack of the step is known, the solve does not read the state);
//   alert_reward_instance   AlertReward._update_state + __call__ (grid2op/Reward/alertReward.py), which also writes the
//                           environment's _was_alert_used_after_attack (read by the observation in update_after_reward);
//   alert_reset_instance    BaseEnv._reset_alert (baseEnv.py:1677-1685) + AlertReward.reset.
// The state is per instance and per alertable line, in caller-owned (library) buffers; the step's attacked lines are the
// opponent's outputs of the same step (one line per instance, or one per area).  The bodies are __host__ __device__: the
// environment's post / reset launches call them, a host build (tests/emu/alert_emu.cpp) runs the same source.  The reward's
// fp64 arithmetic is rounded explicitly (no FMA contraction), so both builds are bit-identical.
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define ALERT_HD __host__ __device__
#else
#define ALERT_HD
#endif

namespace b200pf {

enum { ALERT_MAX_LINES = 64 };

struct AlertArgs {
    int n;                                   // dim_alerts (0: alerts not bound)
    const int32_t *lines;                    // [n] alertable line ids, in grid2op's order
    int window, ring;                        // ALERT_TIME_WINDOW, AlertReward's ring rows (window + 2)
    int reward;                              // AlertReward on: the reward and was_alert_used_after_attack are computed
    // AlertReward's float32 constants, widened: min / max with and without blackout, (max - min) with blackout and
    // (min - max) without blackout, both subtracted in float32 as the reference does
    double min_blackout, range_blackout, max_no_blackout, diff_no_blackout;
    // step inputs
    const uint8_t *raise;                    // [batch][n] raise_alert of the step (NULL: no alert)
    const int32_t *attack; int attack_stride;// [batch][attack_stride] the opponent's attacked lines of the step, -1: none (NULL: none)
    // environment state [batch][n] (total: [batch])
    uint8_t *last_alert, *already;           // _last_alert, _is_already_attacked
    int32_t *tsl_alert, *duration, *tsl_attack, *under_alert, *was_used, *total;
    // AlertReward state
    uint8_t *ts_attack, *launched;           // [batch][ring][n]
    uint8_t *current;                        // [batch][n] _lines_currently_attacked
    int32_t *cur_id;                         // [batch] _current_id
    double *reward_out;                      // [batch]
};

ALERT_HD inline double alert_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

ALERT_HD inline double alert_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// alertable line k attacked by the step's attack of instance i; *any: the step has an attack at all (lines_attacked is not None)
ALERT_HD inline bool alert_attacked(const AlertArgs &al, int i, int k, bool *any) {
    if (!al.attack) { *any = false; return false; }
    const int32_t *at = al.attack + (size_t)i * al.attack_stride;
    bool hit = false, a = false;
    for (int j = 0; j < al.attack_stride; ++j) {
        a |= at[j] >= 0;
        hit |= at[j] == al.lines[k];
    }
    *any = a;
    return hit;
}

// BaseEnv._update_alert_properties of a live instance on an ordinary step
ALERT_HD inline void alert_update_instance(const AlertArgs &al, int i) {
    const int n = al.n;
    const size_t o = (size_t)i * n;
    const uint8_t *raise = al.raise ? al.raise + o : nullptr;
    int added = 0;
    for (int k = 0; k < n; ++k) {
        const bool up = raise && raise[k] != 0;
        al.last_alert[o + k] = up ? 1 : 0;
        int32_t &t = al.tsl_alert[o + k];
        if (up) t = 0; else if (t != -1) t += 1;
        al.duration[o + k] = up ? al.duration[o + k] + 1 : 0;
        added += up ? 1 : 0;
        bool any;
        const bool hit = alert_attacked(al, i, k, &any);
        int32_t &ta = al.tsl_attack[o + k];
        if (any) {
            const bool first = hit && !al.already[o + k];
            if (first) ta = 0; else if (ta != -1) ta += 1;
            if (hit) al.already[o + k] = 1;
        } else {
            if (ta != -1) ta += 1;
            al.already[o + k] = 0;
        }
        if (ta == 0) al.under_alert[o + k] = up ? 1 : -1;
        if (ta > al.window) al.under_alert[o + k] = 0;
    }
    al.total[i] += added;
}

// AlertReward.__call__ for an instance that was live before the step (blackout: the step ended the episode with an error)
ALERT_HD inline void alert_reward_instance(const AlertArgs &al, int i, bool blackout) {
    const int n = al.n, R = al.ring;
    const size_t o = (size_t)i * n;
    uint8_t *ts = al.ts_attack + (size_t)i * R * n, *la = al.launched + (size_t)i * R * n, *cur = al.current + o;
    int32_t *used = al.was_used + o;
    // _update_state
    const int id = (al.cur_id[i] + 1) % R;
    al.cur_id[i] = id;
    bool any = false;
    for (int k = 0; k < n; ++k) alert_attacked(al, i, k, &any);
    for (int k = 0; k < n; ++k) {
        if (!any) { cur[k] = 0; ts[(size_t)id * n + k] = 0; }
        else {
            bool a;
            const bool hit = alert_attacked(al, i, k, &a);
            if (hit && !cur[k]) ts[(size_t)id * n + k] = 1;
            cur[k] = hit ? 1 : 0;
        }
        la[(size_t)id * n + k] = al.raise && al.raise[o + k] ? 1 : 0;
        used[k] = 0;
    }
    double res = 0.0;
    if (blackout) {
        // every line's first attack in the window (the window + 1 rows up to this step, oldest first)
        int n_att = 0, n_alert = 0;
        for (int k = 0; k < n; ++k)
            for (int d = -al.window; d <= 0; ++d) {
                const int r = ((id + d) % R + R) % R;
                if (ts[(size_t)r * n + k]) {
                    const bool up = la[(size_t)r * n + k] != 0;
                    used[k] = up ? 1 : -1;
                    ++n_att; n_alert += up ? 1 : 0;
                    break;
                }
            }
        if (n_att) res = alert_add(alert_mul((double)n_alert / (double)n_att, al.range_blackout), al.min_blackout);
    } else {
        // the attacks exactly `window` steps back: scored once, then forgotten
        const int r = ((id - al.window) % R + R) % R;
        int n_att = 0, n_alert = 0;
        for (int k = 0; k < n; ++k)
            if (ts[(size_t)r * n + k]) {
                const bool up = la[(size_t)r * n + k] != 0;
                used[k] = up ? -1 : 1;
                ++n_att; n_alert += up ? 1 : 0;
            }
        if (n_att) {
            res = alert_add(alert_mul(al.diff_no_blackout, (double)n_alert / (double)n_att), al.max_no_blackout);
            for (int k = 0; k < n; ++k) ts[(size_t)r * n + k] = 0;
        }
    }
    al.reward_out[i] = res;
}

// BaseEnv._reset_alert + AlertReward.reset
ALERT_HD inline void alert_reset_instance(const AlertArgs &al, int i) {
    const int n = al.n, R = al.ring;
    const size_t o = (size_t)i * n;
    for (int k = 0; k < n; ++k) {
        al.last_alert[o + k] = 0; al.already[o + k] = 0; al.tsl_alert[o + k] = -1; al.duration[o + k] = 0;
        al.tsl_attack[o + k] = -1; al.was_used[o + k] = 0; al.under_alert[o + k] = 0; al.current[o + k] = 0;
    }
    al.total[i] = 0;
    for (size_t j = (size_t)i * R * n; j < (size_t)(i + 1) * R * n; ++j) { al.ts_attack[j] = 0; al.launched[j] = 0; }
    al.cur_id[i] = 0;
    if (al.reward_out) al.reward_out[i] = 0.0;
}

// the observe layer's alert values of one instance (6 n + 1 int32, in the order of the attributes: active_alert,
// attack_under_alert, time_since_last_alert, alert_duration, total_number_of_alert, time_since_last_attack,
// was_alert_used_after_attack)
ALERT_HD inline void alert_obs_record(const AlertArgs &al, int i, int32_t *h) {
    const int n = al.n;
    const size_t o = (size_t)i * n;
    for (int k = 0; k < n; ++k) {
        h[k] = al.last_alert[o + k]; h[n + k] = al.under_alert[o + k]; h[2 * n + k] = al.tsl_alert[o + k];
        h[3 * n + k] = al.duration[o + k]; h[4 * n + 1 + k] = al.tsl_attack[o + k]; h[5 * n + 1 + k] = al.was_used[o + k];
    }
    h[4 * n] = al.total[i];
}

}  // namespace b200pf

// b200pf_alarm.cuh — grid2op's alarms (l2rpn_icaps_2021) for a whole batch on the device: the environment's attention budget, the
// AlarmReward, and their reset.
//
// What the bodies restate, per instance (grid2op 1.12.5):
//   alarm_register_instance  LinearAttentionBudget.register_action (grid2op/operator_attention/attention_budget.py:133), called
//                            in BaseEnv.step once the action's legality is known (baseEnv.py:3769-3775), with the step number
//                            nb_time_step already advanced;
//   alarm_reward_instance    AlarmReward.__call__ (grid2op/Reward/alarmReward.py:147) on a step that ended the episode with an
//                            error, which also sets the reward's is_alarm_used (the observation's was_alarm_used_after_game_over);
//   alarm_reset_instance     LinearAttentionBudget.reset (is_alarm_used is the reward object's, which no reset clears).
// AlarmReward scores only the successful alarms of the last best_time + window_size steps (an older one scores 0), so instead of
// _all_successful_alarms each instance keeps a ring of that many (step, zone mask) entries, indexed by step, and one flag "this
// episode had a successful alarm" for the reward's early return.
// The bodies are __host__ __device__: the environment's post / reset launches call them, a host build (tests/emu/alarm_emu.cpp)
// runs the same source.  The budget's float32 and the reward's float64 arithmetic are rounded explicitly (no contraction), so
// both builds are bit-identical.
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define ALARM_HD __host__ __device__
#else
#define ALARM_HD
#endif

namespace b200pf {

enum { ALARM_MAX_ZONES = 32, ALARM_MAX_RING = 1024 };

struct AlarmArgs {
    int n;                                   // dim_alarms (0: alarms not bound)
    const uint32_t *zone_mask;               // [n_line] zones of each line (bit z: zone z, in sorted zone-name order)
    int n_line;
    float max_budget, budget_per_ts, alarm_cost, init_budget;    // LinearAttentionBudget's float32 constants
    int best_time, window, ring;             // ALARM_BEST_TIME, ALARM_WINDOW_SIZE, ring = best_time + window
    int reward;                              // AlarmReward on: the reward and is_alarm_used are computed
    // step input
    const uint8_t *raise;                    // [batch][n] raise_alarm of the step
    // LinearAttentionBudget state
    float *budget;                           // [batch] _current_budget
    int32_t *time_last, *time_last_ok;       // [batch] _time_last_alarm_raised, _time_last_successful_alarm_raised
    int32_t *last, *last_ok;                 // [batch][n] _last_alarm_raised, _last_successful_alarm_raised
    int32_t *ring_step;                      // [batch][ring] step of the successful alarm in this slot (0: none)
    uint32_t *ring_mask;                     // [batch][ring] its zones
    uint8_t *any_ok;                         // [batch] the episode has had a successful alarm
    uint8_t *used;                           // [batch] AlarmReward.is_alarm_used (kept across resets)
    // per-step outputs (caller-owned)
    uint8_t *illegal;                        // [batch] env._is_alarm_illegal
    double *reward_out;                      // [batch]
};

ALARM_HD inline float alarm_fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

ALARM_HD inline float alarm_fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}

ALARM_HD inline double alarm_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

ALARM_HD inline double alarm_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

ALARM_HD inline int alarm_popc(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}

// LinearAttentionBudget.register_action of a live instance on an ordinary step (step: nb_time_step of the step, illegal_action:
// the agent's action was illegal, which records, charges and replenishes nothing)
ALARM_HD inline void alarm_register_instance(const AlarmArgs &al, int i, int step, bool illegal_action) {
    const int n = al.n;
    const size_t o = (size_t)i * n;
    al.illegal[i] = 0;
    if (illegal_action) return;
    uint32_t m = 0;
    for (int k = 0; k < n; ++k)
        if (al.raise[o + k]) m |= 1u << k;
    if (!m) {                                                 // min(max_budget, budget_per_ts + current), in float32
        const float b = alarm_fadd(al.budget_per_ts, al.budget[i]);
        al.budget[i] = b < al.max_budget ? b : al.max_budget;
        return;
    }
    al.time_last[i] = step;
    for (int k = 0; k < n; ++k)
        if (m >> k & 1u) al.last[o + k] = step;
    if (al.budget[i] >= al.alarm_cost) {                      // one charge, whatever the number of zones
        al.budget[i] = alarm_fsub(al.budget[i], al.alarm_cost);
        al.time_last_ok[i] = step;
        for (int k = 0; k < n; ++k)
            if (m >> k & 1u) al.last_ok[o + k] = step;
        const size_t r = (size_t)i * al.ring + (size_t)(step % al.ring);
        al.ring_step[r] = step; al.ring_mask[r] = m;
        al.any_ok[i] = 1;
    } else {
        al.illegal[i] = 1;                                    // NotEnoughAttentionBudget: the rest of the action still applies
    }
}

// AlarmReward.__call__ on the step `step` that ended the episode with an error (disc: the step's disc_lines [n_line], NULL when
// the protections are off, i.e. every entry -1)
ALARM_HD inline void alarm_reward_instance(const AlarmArgs &al, int i, int step, const int32_t *disc) {
    bool trip = false;
    uint32_t first = 0;                                       // zones of the lines tripped in the cascade's first round
    if (disc)
        for (int l = 0; l < al.n_line; ++l) {
            trip |= disc[l] != -1;
            if (disc[l] == 0) first |= al.zone_mask[l];
        }
    double best = -1.0;
    if (trip && al.any_ok[i]) {                               // (the two early returns leave is_alarm_used as it was)
        const int W = al.window, bt = al.best_time;
        const double w2 = (double)W * (double)W;
        for (int s = 0; s < al.ring; ++s) {
            const size_t r = (size_t)i * al.ring + s;
            const int sa = al.ring_step[r];
            const int dist = step - sa;
            if (sa <= 0 || dist < 0 || dist >= al.ring) continue;      // empty slot, or an alarm too old to score
            if (dist > bt + W || dist < bt - W) continue;
            const int d = dist - bt;
            const double t = alarm_div((double)(-((d - W) * (d + W))), w2);
            if (t == 0.0) continue;                           // at either end of the window: scores reward_min, "not used"
            const uint32_t m = al.ring_mask[r];
            const double mult = (alarm_popc(m) == 1 && (m & first)) ? 1.0 : 0.5;   // _mult_for_zone / mult_for_right_zone
            const double sc = alarm_mul(t, mult);
            if (sc > best) best = sc;
        }
        al.used[i] = best > -1.0 ? 1 : 0;
    }
    al.reward_out[i] = best;
}

// LinearAttentionBudget.reset (AlarmReward.reset keeps is_alarm_used)
ALARM_HD inline void alarm_reset_instance(const AlarmArgs &al, int i) {
    const int n = al.n;
    const size_t o = (size_t)i * n;
    al.budget[i] = al.init_budget;
    al.time_last[i] = -1; al.time_last_ok[i] = -1;
    for (int k = 0; k < n; ++k) { al.last[o + k] = -1; al.last_ok[o + k] = -1; }
    for (size_t r = (size_t)i * al.ring; r < (size_t)(i + 1) * al.ring; ++r) { al.ring_step[r] = 0; al.ring_mask[r] = 0; }
    al.any_ok[i] = 0; al.illegal[i] = 0;
    if (al.reward_out) al.reward_out[i] = 0.0;
}

// the observe layer's alarm values of one instance (n + 4 int32): is_alarm_illegal, time_since_last_alarm (current_step: the
// instance's nb_time_step), last_alarm[n], the budget's float32 bits, is_alarm_used
ALARM_HD inline void alarm_obs_record(const AlarmArgs &al, int i, int current_step, int32_t *h) {
    const int n = al.n;
    const size_t o = (size_t)i * n;
    const int32_t tok = al.time_last_ok[i];
    h[0] = al.illegal[i];
    h[1] = tok > 0 ? current_step - tok : -1;
    for (int k = 0; k < n; ++k) h[2 + k] = al.last_ok[o + k];
    union { float f; int32_t u; } b;
    b.f = al.budget[i];
    h[2 + n] = b.u;
    h[3 + n] = al.used[i];
}

}  // namespace b200pf

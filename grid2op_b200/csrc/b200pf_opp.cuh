// b200pf_opp.cuh — line-attack opponents of BatchedEnv for a whole batch on the device: grid2op's OpponentSpace with
// BaseActionBudget and a RandomLineOpponent, a WeightedRandomOpponent or a GeometricOpponent, restated per instance, with each
// instance's own numpy-legacy random stream (RandomState: MT19937 and its legacy draws).
//
// The body restates grid2op_b200/opponent.py (the numpy reference path) in the same order:
//   opp_decide_instance     OpponentSpace.attack and the opponent's attack / tell_attack_continues, on the line status and rho
//                           the previous step left;
//   opp_reset_instance      OpponentSpace.reset (the random stream is not reseeded: it continues);
//   opp_geo_reset_instance  the GeometricOpponent's part of it: a new attack schedule (sample_attack_times_and_durations);
//   opp_multi_reset_instance  the GeometricOpponentMultiArea's part: a new schedule per area, in area order.
// The GeometricOpponent's constants and schedules are an OppGeoArgs next to OppArgs (NULL for the other kinds); the
// GeometricOpponentMultiArea's, one GeometricOpponent per area with its own stream, are an OppMultiArgs.
// env_apply_instance (b200pf_env.cuh) calls the first before the agent's action and applies the attack after the environment's
// own outages; env_reset_instance calls the second.  The bodies are __host__ __device__: the CUDA launches run one thread per
// instance, a host build (tests/emu/opp_emu.cpp) runs the same source over the batch.  The fp64 arithmetic of the weighted draw is
// written with explicitly rounded operations (no contraction), so both builds round as numpy does.
#pragma once

#include <cmath>
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define OPP_HD __host__ __device__
#else
#define OPP_HD
#endif

namespace b200pf {

enum { OPP_NONE = 0, OPP_RANDOM_LINE = 1, OPP_WEIGHTED_RANDOM = 2, OPP_GEOMETRIC = 3, OPP_GEOMETRIC_MULTI = 4 };
enum { OPP_MT_N = 624, OPP_MAX_ATTACK = 64 };
// per-instance counters, int32 [batch][OPP_CTR]
enum { OPP_CTR_DURATION = 0, OPP_CTR_COOLDOWN = 1, OPP_CTR_LAST = 2, OPP_CTR_NEXT = 3, OPP_CTR = 4 };
static const int32_t OPP_NEXT_UNSET = INT32_MIN;    // WeightedRandomOpponent / GeometricOpponent._next_attack_time is None
// per-instance counters of the GeometricOpponent, int32 [batch][OPP_GEO_CTR]: attacks in the schedule, attacks consumed,
// OpponentSpace.previous_fails, schedules that did not fit the cap (their tail was drawn and dropped)
enum { OPP_GEO_N = 0, OPP_GEO_COUNTER = 1, OPP_GEO_FAILS = 2, OPP_GEO_OVERFLOW = 3, OPP_GEO_CTR = 4 };

// GeometricOpponent (kind OPP_GEOMETRIC): its constants and its schedule state, next to OppArgs (whose ctr[OPP_CTR_NEXT] is its
// _next_attack_time)
struct OppGeoArgs {
    const double *weights;                          // [n_attack] np.exp(b_beta * k), k = 0 .. n_attack - 1 (computed by numpy)
    double p_hazard, p_recovery;                    // p of the geometric waiting times / of the random part of the durations
    double logq_hazard, logq_recovery;              // log(1 - p) of both (the inversion's divisor, computed on the host)
    int recovery_min;                               // _recovery_minimum_duration
    int cap;                                        // schedule entries per instance
    const int32_t *emt;                             // [batch] _episode_max_time
    int32_t *wait, *dur;                            // [batch][cap] _attack_waiting_times, _attack_durations
    int32_t *gctr;                                  // [batch][OPP_GEO_CTR]
};

// GeometricOpponentMultiArea (kind OPP_GEOMETRIC_MULTI): per-area counters, int32 [batch][n_area][OPP_AREA_CTR].  The schedule
// length, attacks consumed and entries dropped at the cap sit where OPP_GEO_CTR has them, so both kinds share the schedule code; then
// the area's GeometricOpponent._next_attack_time (OPP_NEXT_UNSET: None), its _new_attack_time_counters entry and its
// _previous_attacks line (-1: None).
enum { OPP_AREA_N = 0, OPP_AREA_COUNTER = 1, OPP_AREA_NEXT = 2, OPP_AREA_OVERFLOW = 3, OPP_AREA_CLOCK = 4, OPP_AREA_PREV = 5,
       OPP_AREA_CTR = 6 };
static_assert((int)OPP_AREA_N == (int)OPP_GEO_N && (int)OPP_AREA_COUNTER == (int)OPP_GEO_COUNTER &&
              (int)OPP_AREA_OVERFLOW == (int)OPP_GEO_OVERFLOW, "the schedule code reads both layouts");
enum { OPP_MAX_AREA = 8 };

// The GeometricOpponentMultiArea: its areas (ranges of OppArgs.lines), their weight tables, the shared constants and every area's
// stream and schedule.  OppArgs keeps OpponentSpace's part (budget, duration, cooldown; ctr[OPP_CTR_LAST] is the first line of the
// landed attack, ctr[OPP_CTR_NEXT] stays OPP_NEXT_UNSET); previous_fails is here.
struct OppMultiArgs {
    int n_area;
    int area_off[OPP_MAX_AREA + 1];                 // area k's lines are OppArgs.lines[area_off[k] .. area_off[k + 1])
    const double *weights;                          // [n_attack] area k's np.exp(b_beta_k * r) at area_off[k] + r (computed by numpy)
    double p_hazard, p_recovery;                    // as OppGeoArgs (every area has the same)
    double logq_hazard, logq_recovery;
    int recovery_min;
    int cap;                                        // schedule entries per instance and area
    const int32_t *emt;                             // [batch] _episode_max_time
    uint32_t *mt; int32_t *mt_pos;                  // [batch][n_area][624], [batch][n_area]: each area's RandomState
    int32_t *wait, *dur;                            // [batch][n_area][cap]
    int32_t *actr;                                  // [batch][n_area][OPP_AREA_CTR]
    int32_t *fails;                                 // [batch] OpponentSpace.previous_fails
    int32_t *attack_lines;                          // [batch][n_area] per-step output, caller-owned: area k's line in the landed
                                                    // attack, -1 where the area put none in it
};

// one GeometricOpponent's stream and schedule: MT state [624] and position, waiting times and durations [cap], and counters laid out
// as OPP_GEO_CTR's schedule length, attacks consumed and dropped entries
struct OppGeoSched {
    uint32_t *mt; int32_t *pos;
    int32_t *wait, *dur;
    int32_t *gc;
};

struct OppArgs {
    int kind;                                       // OPP_NONE: no opponent bound
    int n_attack;                                   // attackable lines
    const int32_t *lines;                           // [n_attack] their line ids
    const double *rho_norm;                         // [n_attack] (weighted)
    int attack_period, attack_duration, attack_cooldown;
    float budget_per_ts, init_budget;
    // per-instance state
    double *budget;                                 // [batch] caller-owned; float32 value until the first charge (budget64)
    uint8_t *budget64;                              // [batch] the budget has become a float64 (numpy promotion)
    int32_t *ctr;                                   // [batch][OPP_CTR]
    uint32_t *mt; int32_t *mt_pos;                  // [batch][624], [batch]: MT19937 state as RandomState.get_state() gives it
    // per-step outputs, caller-owned [batch]
    int32_t *attack_line, *attack_dur;
    // the previous step's rho [batch][n_line] (read by the weighted opponent)
    const float *rho;
};

// ---- numpy legacy RandomState draws --------------------------------------------------------------------------------------
OPP_HD inline uint32_t opp_next_u32(uint32_t *mt, int32_t *pos) {
    if (*pos >= OPP_MT_N) {                                   // the twist (mt19937_gen)
        int k = 0;
        for (; k < OPP_MT_N - 397; ++k) {
            const uint32_t y = (mt[k] & 0x80000000u) | (mt[k + 1] & 0x7fffffffu);
            mt[k] = mt[k + 397] ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
        }
        for (; k < OPP_MT_N - 1; ++k) {
            const uint32_t y = (mt[k] & 0x80000000u) | (mt[k + 1] & 0x7fffffffu);
            mt[k] = mt[k + (397 - OPP_MT_N)] ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
        }
        const uint32_t y = (mt[OPP_MT_N - 1] & 0x80000000u) | (mt[0] & 0x7fffffffu);
        mt[OPP_MT_N - 1] = mt[396] ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
        *pos = 0;
    }
    uint32_t y = mt[(*pos)++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// randint(n) / choice(n) without p, n <= 2**32: masked rejection on 32-bit words; n == 1 draws nothing
OPP_HD inline uint32_t opp_randint(uint32_t *mt, int32_t *pos, uint32_t n) {
    const uint32_t rng = n - 1u;
    if (rng == 0u) return 0u;
    uint32_t mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    uint32_t w;
    while ((w = opp_next_u32(mt, pos) & mask) > rng) {}
    return w;
}

OPP_HD inline double opp_dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
OPP_HD inline double opp_dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
OPP_HD inline double opp_ddiv(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// random_sample(): 53 bits from two words
OPP_HD inline double opp_random_sample(uint32_t *mt, int32_t *pos) {
    const uint32_t a = opp_next_u32(mt, pos) >> 5, b = opp_next_u32(mt, pos) >> 6;
    return opp_ddiv(opp_dadd(opp_dmul((double)a, 67108864.0), (double)b), 9007199254740992.0);
}

// ndarray.sum() of n float64 values: numpy's pairwise summation (one block below 128 values)
OPP_HD inline double opp_np_sum(const double *v, int n) {
    if (n < 8) {
        double s = 0.0;
        for (int k = 0; k < n; ++k) s = opp_dadd(s, v[k]);
        return s;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = v[j];
    int k = 8;
    for (; k < n - (n % 8); k += 8)
        for (int j = 0; j < 8; ++j) r[j] = opp_dadd(r[j], v[k + j]);
    double s = opp_dadd(opp_dadd(opp_dadd(r[0], r[1]), opp_dadd(r[2], r[3])), opp_dadd(opp_dadd(r[4], r[5]), opp_dadd(r[6], r[7])));
    for (; k < n; ++k) s = opp_dadd(s, v[k]);
    return s;
}

// choice(n, p=w / w.sum()) for w >= 0 with a positive sum: cdf = cumsum(p), cdf /= cdf[-1], searchsorted(cdf, random_sample(), "right")
OPP_HD inline int opp_choice_weighted(uint32_t *mt, int32_t *pos, const double *w, int n, double wsum) {
    double cdf[OPP_MAX_ATTACK];
    double c = 0.0;
    for (int k = 0; k < n; ++k) { c = opp_dadd(c, opp_ddiv(w[k], wsum)); cdf[k] = c; }
    const double last = cdf[n - 1];
    const double u = opp_random_sample(mt, pos);
    int idx = 0;
    for (int k = 0; k < n; ++k) idx += opp_ddiv(cdf[k], last) <= u ? 1 : 0;
    return idx;
}

// geometric(p) (numpy's legacy_random_geometric): for p >= 1/3 the search on one random_sample(), else the inversion
// ceil(log1p(-U) / log(1 - p)) with logq = log(1 - p).  log1p is CUDA's on the device (within 1 ulp) and libm's in a host build;
// the quotient is rounded up to an integer, so a last-bit difference changes the draw only when it lies within an ulp or two of an
// integer (DESIGN §7 f.1).  The search stops where numpy would loop forever (the running product underflowed: its sum cannot grow).
OPP_HD inline int64_t opp_geometric(uint32_t *mt, int32_t *pos, double p, double logq) {
    if (p >= 0.333333333333333333333333) {
        const double q = opp_dadd(1.0, -p);
        const double u = opp_random_sample(mt, pos);
        double sum = p, prod = p;
        int64_t x = 1;
        while (u > sum && prod > 0.0) { prod = opp_dmul(prod, q); sum = opp_dadd(sum, prod); ++x; }
        return x;
    }
    return (int64_t)ceil(opp_ddiv(log1p(-opp_random_sample(mt, pos)), logq));
}

// ---- GeometricOpponent ----------------------------------------------------------------------------------------------------
// sample_attack_times_and_durations on one stream and schedule: waiting times and durations until emt.  Entries past the cap are
// drawn (the stream stays grid2op's) but dropped and counted in OPP_GEO_OVERFLOW.
OPP_HD inline void opp_geo_draw_schedule(const OppGeoSched &s, int64_t emt, double p_hazard, double logq_hazard, double p_recovery,
                                         double logq_recovery, int recovery_min, int cap) {
    int64_t t = 0;
    int n = 0;
    while (t < emt) {
        const int64_t tw = opp_geometric(s.mt, s.pos, p_hazard, logq_hazard);
        t += tw;
        if (t < emt) {
            const int64_t td = (int64_t)recovery_min + opp_geometric(s.mt, s.pos, p_recovery, logq_recovery);
            if (n < cap) { s.wait[n] = (int32_t)tw; s.dur[n] = (int32_t)td; ++n; }
            else s.gc[OPP_GEO_OVERFLOW] += 1;
            t += td;
        }
    }
    s.gc[OPP_GEO_N] = n; s.gc[OPP_GEO_COUNTER] = 0;
}

// the GeometricOpponent's schedule of instance i, on its stream
OPP_HD inline void opp_geo_sample(const OppGeoArgs &g, int i, uint32_t *mt, int32_t *pos) {
    int32_t *gc = g.gctr + (size_t)i * OPP_GEO_CTR;
    const OppGeoSched s{mt, pos, g.wait + (size_t)i * g.cap, g.dur + (size_t)i * g.cap, gc};
    opp_geo_draw_schedule(s, g.emt[i], g.p_hazard, g.logq_hazard, g.p_recovery, g.logq_recovery, g.recovery_min, g.cap);
    gc[OPP_GEO_FAILS] = 0;
}

// GeometricOpponent.attack of one opponent: its stream and schedule s, its _next_attack_time *next, OpponentSpace's previous_fails,
// its lines [n_lines] and their weight table, the previous step's rho of the instance -> the attacked line (-1: none); *dur: its
// duration from the schedule
OPP_HD inline int opp_geo_attack_lines(const OppGeoSched &s, int32_t *next, bool fails, const int32_t *lines, int n_lines,
                                       const double *weights, const float *rho, const int8_t *tv, const int32_t *line_or_pos,
                                       const int32_t *line_ex_pos, int *dur) {
    const int c = s.gc[OPP_GEO_COUNTER], n = s.gc[OPP_GEO_N];
    if (c >= n) return -1;                                                             // no attack left in the schedule
    const int32_t *w = s.wait, *d = s.dur;
    // (int32 sums wrap as numpy's do; d[-1] of a failure before any attack is numpy's last entry)
    if (fails) *next = (int32_t)((uint32_t)w[c] + (uint32_t)d[c > 0 ? c - 1 : n - 1]);
    if (*next == OPP_NEXT_UNSET) *next = (int32_t)(1u + (uint32_t)w[c]);
    *dur = d[c];
    *next -= 1;
    if (*next > 0) return -1;
    s.gc[OPP_GEO_COUNTER] = c + 1;                                                     // the attack is consumed, whatever follows
    for (int k = 0; k < n_lines; ++k) {                                                // ~status.all(): one line out -> no attack
        const int l = lines[k];
        if (!(tv[line_or_pos[l]] > 0 && tv[line_ex_pos[l]] > 0)) return -1;
    }
    if (n_lines == 1) return lines[0];
    // Boltzmann weights on the rho ranks: rank k = lines with a lower rho, ties ranked by line order (a stable argsort)
    double wv[OPP_MAX_ATTACK];
    for (int k = 0; k < n_lines; ++k) {
        const float r = rho[lines[k]];
        int rank = 0;
        for (int j = 0; j < n_lines; ++j) {
            const float rj = rho[lines[j]];
            rank += (rj < r || (rj == r && j < k)) ? 1 : 0;
        }
        wv[k] = weights[rank];
    }
    const double sum = opp_np_sum(wv, n_lines);
    return lines[opp_choice_weighted(s.mt, s.pos, wv, n_lines, sum)];
}

// GeometricOpponent.attack for instance i -> the attacked line (-1: none); *dur: its duration from the schedule
OPP_HD inline int opp_geo_attack(const OppArgs &o, const OppGeoArgs &g, int i, const int8_t *tv, const int32_t *line_or_pos,
                                 const int32_t *line_ex_pos, int n_line, int32_t *ctr, int32_t *gc, int *dur) {
    const OppGeoSched s{o.mt + (size_t)i * OPP_MT_N, o.mt_pos + i, g.wait + (size_t)i * g.cap, g.dur + (size_t)i * g.cap, gc};
    return opp_geo_attack_lines(s, &ctr[OPP_CTR_NEXT], gc[OPP_GEO_FAILS] != 0, o.lines, o.n_attack, g.weights,
                                o.rho + (size_t)i * n_line, tv, line_or_pos, line_ex_pos, dur);
}

// OpponentSpace.attack's call of the geometric opponent with its checks: refused (and previous_fails set) when the opponent's duration
// exceeds attack_max_duration or duration * cost exceeds the budget b; previous_fails is cleared otherwise
OPP_HD inline int opp_geo_asked(const OppArgs &o, const OppGeoArgs &g, int i, const int8_t *tv, const int32_t *line_or_pos,
                                const int32_t *line_ex_pos, int n_line, int32_t *ctr, double b) {
    int32_t *gc = g.gctr + (size_t)i * OPP_GEO_CTR;
    int d = 0;
    int attack = opp_geo_attack(o, g, i, tv, line_or_pos, line_ex_pos, n_line, ctr, gc, &d);
    const int duration = attack >= 0 ? d : o.attack_duration;                          // None -> attack_max_duration
    bool fails = false;
    if (duration > o.attack_duration) { attack = -1; fails = true; }
    if ((attack >= 0 ? (double)duration : 0.0) > b) { attack = -1; fails = true; }     // duration * cost > budget
    gc[OPP_GEO_FAILS] = fails ? 1 : 0;
    if (attack >= 0) { ctr[OPP_CTR_DURATION] = duration; ctr[OPP_CTR_COOLDOWN] += o.attack_cooldown; }
    return attack;
}

// ---- GeometricOpponentMultiArea -------------------------------------------------------------------------------------------
OPP_HD inline OppGeoSched opp_area_sched(const OppMultiArgs &m, int i, int k) {
    const size_t ka = (size_t)i * m.n_area + k;
    return OppGeoSched{m.mt + ka * OPP_MT_N, m.mt_pos + ka, m.wait + ka * m.cap, m.dur + ka * m.cap, m.actr + ka * OPP_AREA_CTR};
}

// GeometricOpponentMultiArea.attack for instance i, in area order: every area's counter ticks down (clamped at -1); an area at -1 asks
// its GeometricOpponent (with OpponentSpace's previous_fails), remembers what it returns and, for an attack, counts its duration; an
// area still counting tells its opponent the attack continues and repeats its remembered line.  out[k]: area k's line in the
// combined attack (-1: none) -> the number of lines in it (its cost)
OPP_HD inline int opp_multi_attack(const OppArgs &o, const OppMultiArgs &m, int i, const int8_t *tv, const int32_t *line_or_pos,
                                   const int32_t *line_ex_pos, int n_line, int32_t *out) {
    const bool fails = m.fails[i] != 0;
    const float *rho = o.rho + (size_t)i * n_line;
    int n = 0;
    for (int k = 0; k < m.n_area; ++k) {
        const OppGeoSched s = opp_area_sched(m, i, k);
        int32_t *ac = s.gc;
        ac[OPP_AREA_CLOCK] = ac[OPP_AREA_CLOCK] > 0 ? ac[OPP_AREA_CLOCK] - 1 : -1;
        int line;
        if (ac[OPP_AREA_CLOCK] == -1) {
            const int off = m.area_off[k];
            int d = 0;
            line = opp_geo_attack_lines(s, &ac[OPP_AREA_NEXT], fails, o.lines + off, m.area_off[k + 1] - off, m.weights + off, rho, tv,
                                        line_or_pos, line_ex_pos, &d);
            if (line >= 0) ac[OPP_AREA_CLOCK] = d;
            ac[OPP_AREA_PREV] = line;
        } else {
            ac[OPP_AREA_NEXT] = OPP_NEXT_UNSET;                                            // tell_attack_continues
            line = ac[OPP_AREA_PREV];
        }
        out[k] = line;
        n += line >= 0 ? 1 : 0;
    }
    return n;
}

// OpponentSpace.attack's call of the multi-area opponent, whose duration is always 1: the combined attack is refused whole (and
// previous_fails set) when 1 exceeds attack_max_duration or its line count exceeds the budget b.  The area counters and remembered
// lines stay as the call left them.  -> the first line of the landed attack (-1: none); *cost: its line count
OPP_HD inline int opp_multi_asked(const OppArgs &o, const OppMultiArgs &m, int i, const int8_t *tv, const int32_t *line_or_pos,
                                  const int32_t *line_ex_pos, int n_line, int32_t *ctr, double b, int *cost) {
    int32_t *out = m.attack_lines + (size_t)i * m.n_area;
    const int n = opp_multi_attack(o, m, i, tv, line_or_pos, line_ex_pos, n_line, out);
    bool landed = n > 0, fails = false;
    if (1 > o.attack_duration) { landed = false; fails = true; }
    if ((landed ? (double)n : 0.0) > b) { landed = false; fails = true; }                // duration * cost > budget
    m.fails[i] = fails ? 1 : 0;
    int first = -1;
    for (int k = 0; k < m.n_area; ++k) {
        if (!landed) out[k] = -1;
        else if (first < 0) first = out[k];
    }
    if (landed) { ctr[OPP_CTR_DURATION] = 1; ctr[OPP_CTR_COOLDOWN] += o.attack_cooldown; }
    *cost = landed ? n : 0;
    return first;
}

// OpponentSpace.reset's GeometricOpponentMultiArea.reset for instance i: every area counter to -1, then each area's
// GeometricOpponent.reset in area order (a new schedule from its continuing stream, _next_attack_time None); the remembered lines
// stay
OPP_HD inline void opp_multi_reset_instance(const OppMultiArgs &m, int i) {
    m.fails[i] = 0;
    for (int k = 0; k < m.n_area; ++k) m.actr[((size_t)i * m.n_area + k) * OPP_AREA_CTR + OPP_AREA_CLOCK] = -1;
    for (int k = 0; k < m.n_area; ++k) {
        const OppGeoSched s = opp_area_sched(m, i, k);
        opp_geo_draw_schedule(s, m.emt[i], m.p_hazard, m.logq_hazard, m.p_recovery, m.logq_recovery, m.recovery_min, m.cap);
        s.gc[OPP_AREA_NEXT] = OPP_NEXT_UNSET;
    }
}

// no multi-area attack for instance i this step
OPP_HD inline void opp_multi_none(const OppMultiArgs &m, int i) {
    for (int k = 0; k < m.n_area; ++k) m.attack_lines[(size_t)i * m.n_area + k] = -1;
}

// ---- the opponent ---------------------------------------------------------------------------------------------------------
// The opponent's choice among the attackable lines that are connected in ``tv`` (the topology the previous step left): -1 for none.
OPP_HD inline int opp_choose(const OppArgs &o, int i, const int8_t *tv, const int32_t *line_or_pos, const int32_t *line_ex_pos,
                             int n_line, int32_t *ctr) {
    uint32_t *mt = o.mt + (size_t)i * OPP_MT_N;
    int32_t *pos = o.mt_pos + i;
    int on[OPP_MAX_ATTACK];
    int n_on = 0;
    if (o.kind == OPP_WEIGHTED_RANDOM) {
        if (ctr[OPP_CTR_NEXT] == OPP_NEXT_UNSET) ctr[OPP_CTR_NEXT] = 1 + (int32_t)opp_randint(mt, pos, (uint32_t)o.attack_period);
        ctr[OPP_CTR_NEXT] -= 1;
        if (ctr[OPP_CTR_NEXT] > 0) return -1;
    }
    for (int k = 0; k < o.n_attack; ++k) {
        const int l = o.lines[k];
        if (tv[line_or_pos[l]] > 0 && tv[line_ex_pos[l]] > 0) on[n_on++] = k;
    }
    if (n_on == 0) return -1;
    if (o.kind == OPP_RANDOM_LINE) return o.lines[on[opp_randint(mt, pos, (uint32_t)n_on)]];
    double w[OPP_MAX_ATTACK];
    const float *rho = o.rho + (size_t)i * n_line;
    for (int k = 0; k < n_on; ++k) w[k] = opp_ddiv((double)rho[o.lines[on[k]]], o.rho_norm[on[k]]);
    const double s = opp_np_sum(w, n_on);
    if (!(s > 0.0)) return -1;
    return o.lines[on[opp_choice_weighted(mt, pos, w, n_on, s)]];
}

// OpponentSpace.attack for instance i (not finished, not a reset step) -> the attacked line (-1: none); *dur: its duration
OPP_HD inline int opp_decide_instance(const OppArgs &o, int i, const int8_t *tv, const int32_t *line_or_pos, const int32_t *line_ex_pos,
                                      int n_line, int *dur, const OppGeoArgs *g = nullptr, const OppMultiArgs *m = nullptr) {
    int32_t *ctr = o.ctr + (size_t)i * OPP_CTR;
    double b = o.budget[i];
    const bool b64 = o.budget64[i] != 0;
    b = b64 ? b + (double)o.budget_per_ts : (double)((float)b + o.budget_per_ts);      // budget += budget_per_timestep
    ctr[OPP_CTR_DURATION] = ctr[OPP_CTR_DURATION] > 1 ? ctr[OPP_CTR_DURATION] - 1 : 0;
    ctr[OPP_CTR_COOLDOWN] = ctr[OPP_CTR_COOLDOWN] > 1 ? ctr[OPP_CTR_COOLDOWN] - 1 : 0;
    int attack = -1, cost = 1;
    bool asked = false;
    // (the multi-area opponent's duration is 1 and its attack_cooldown at most 1, so it is asked on every step: grid2op's own
    // tell_attack_continues of it raises, and the host path refuses the configurations that would reach it)
    if (ctr[OPP_CTR_DURATION] > 0) attack = ctr[OPP_CTR_LAST];                           // the running attack continues
    else if (ctr[OPP_CTR_COOLDOWN] <= o.attack_cooldown) {
        asked = true;
        if (o.kind == OPP_GEOMETRIC_MULTI) {
            if (m) attack = opp_multi_asked(o, *m, i, tv, line_or_pos, line_ex_pos, n_line, ctr, b, &cost);
        } else if (o.kind == OPP_GEOMETRIC) {
            if (g) attack = opp_geo_asked(o, *g, i, tv, line_or_pos, line_ex_pos, n_line, ctr, b);
        } else {
            attack = opp_choose(o, i, tv, line_or_pos, line_ex_pos, n_line, ctr);
            // duration None -> attack_max_duration; the cost of one line is 1: refused when duration * cost > budget
            if (attack >= 0 && (double)o.attack_duration > b) attack = -1;
            if (attack >= 0) { ctr[OPP_CTR_DURATION] = o.attack_duration; ctr[OPP_CTR_COOLDOWN] += o.attack_cooldown; }
        }
    }
    if (!asked && o.kind != OPP_RANDOM_LINE) ctr[OPP_CTR_NEXT] = OPP_NEXT_UNSET;        // tell_attack_continues
    if (!asked && g) g->gctr[(size_t)i * OPP_GEO_CTR + OPP_GEO_FAILS] = 0;               // (OpponentSpace clears previous_fails)
    if (!asked && m) { m->fails[i] = 0; opp_multi_none(*m, i); attack = -1; }
    ctr[OPP_CTR_LAST] = attack;
    if (attack >= 0) { b = b - (double)cost; o.budget64[i] = 1; }                           // budget -= cost: float32 - int64 -> float64
    o.budget[i] = b;
    *dur = attack >= 0 ? ctr[OPP_CTR_DURATION] : 0;
    return attack;
}

// OpponentSpace.reset for instance i
OPP_HD inline void opp_reset_instance(const OppArgs &o, int i) {
    int32_t *ctr = o.ctr + (size_t)i * OPP_CTR;
    o.budget[i] = (double)o.init_budget; o.budget64[i] = 0;
    ctr[OPP_CTR_DURATION] = 0; ctr[OPP_CTR_COOLDOWN] = o.attack_cooldown; ctr[OPP_CTR_LAST] = -1; ctr[OPP_CTR_NEXT] = OPP_NEXT_UNSET;
}

// OpponentSpace.reset's GeometricOpponent.reset for instance i: a new schedule from the continuing stream
OPP_HD inline void opp_geo_reset_instance(const OppArgs &o, const OppGeoArgs &g, int i) {
    opp_geo_sample(g, i, o.mt + (size_t)i * OPP_MT_N, o.mt_pos + i);
}

}  // namespace b200pf

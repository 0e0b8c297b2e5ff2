// b200pf_env.cuh — BatchedEnv's environment bookkeeping for a whole batch on the device: the agent's action (legality, busbar
// writes, reconnections, line switching), the environment's forced outages, and what follows the power flow (trips, the
// isolated-busbar rule, cooldowns, game over, the observe layer's per-instance input record).
//
// Every body restates, per instance, the numpy code of grid2op_b200/batched_env.py in the same order:
//   env_apply_instance   BatchedEnv._apply_agent (or, with the vector action, _apply_actions: act_vec_instance), then
//                        _apply_environment (and the bus count of _bus_cap), with the opponent's decision before the agent's action
//                        and its attack after the outages when one is bound (b200pf_opp.cuh); both encodings share the legality
//                        rules of BatchedEnv._illegal (ActLegal);
//   env_post_instance    the rest of BatchedEnv.step behind the solve;
//   env_reset_instance   BatchedEnv.reset_instances (with the library's part, b200pf_series_reset_instances, and the opponent's).
// With line alerts bound (b200pf_alert.cuh), the post body updates the alert state and the AlertReward after the step's attack,
// and the reset body resets them; with alarms bound (b200pf_alarm.cuh), the post body registers the step's alarm once its
// legality is known and computes the AlarmReward, and the reset body resets the attention budget.
// The bodies are __host__ __device__: the CUDA launches run one thread per instance, a host build (tests/emu/env_emu.cpp,
// tests/emu/opp_emu.cpp) runs the same source over the batch.  Integer arithmetic, and the opponent's fp64 operations explicitly
// rounded: the two builds are bit-identical by construction.
#pragma once

#include <cstddef>
#include <cstdint>

#include "b200pf_alarm.cuh"
#include "b200pf_alert.cuh"
#include "b200pf_opp.cuh"

#if defined(__CUDACC__)
#define ENV_HD __host__ __device__
#else
#define ENV_HD
#endif

namespace b200pf {

// control words of one env step (device, copied to the host in the step's single wait)
enum { ENV_CTL_N_DIRTY = 0, ENV_CTL_CAP_MAX = 1, ENV_CTL_ERR = 2, ENV_CTL_N_COPY = 3, ENV_CTL_N_ILLEGAL = 4, ENV_CTL_WORDS = 8 };
enum { ENV_MAX_SLOT = 1024 };            // bus slots (n_sub * n_busbar) the device bus count handles

struct EnvArgs {
    int batch;
    int n_line, n_sub, dim_topo, n_topo_in, n_busbar, n_slot, max_sub, n_rows;
    // static tables (b200pf_env_bind)
    const int32_t *sub_pos;                         // [n_sub][max_sub] topology positions of each substation's elements, -1 padded
    const int32_t *line_or_pos, *line_ex_pos;       // [n_line]
    const int32_t *line_of_pos, *other_end_pos;     // [dim_topo]: line whose end sits there (-1: none), position of its other end
    const int32_t *elem_pos, *elem_sub; int n_elem; // every element of the record (bus count)
    int cd_line, cd_sub, cd_reco;                   // NB_TIMESTEP_COOLDOWN_LINE / _SUB, NB_TIMESTEP_RECONNECTION
    const uint8_t *maint, *haz;                     // [n_scen][n_rows][n_line] forced outages, or NULL
    const int32_t *maint_time, *maint_dur, *haz_dur;// [n_scen][n_rows][n_line], or NULL
    const int32_t *iso_cols, *iso_seg; int n_iso_seg, n_iso_cols;   // isolated-busbar rule: column segments (start offsets)
    const int8_t *topo0;                            // [batch][n_topo_in]
    const int32_t *t0, *scen;                       // [batch]
    // series state of the library
    int8_t *topo;                                   // [batch][n_topo_in] (d_series_topo)
    int32_t *t;                                     // [batch] chronics row of the next solve
    int32_t *lib_done, *pcount, *ts_over, *lib_disc;// protection state (cleared by a reset)
    int8_t *trip, *incdone;
    // per-instance state, caller-owned
    int8_t *last_bus;                               // [batch][dim_topo]
    int32_t *line_cd, *sub_cd;                      // [batch][n_line], [batch][n_sub]
    uint8_t *done, *is_illegal, *newly_done;        // [batch]
    int32_t *current_step, *status_out;             // [batch]
    // library scratch
    uint8_t *aff_l;                                 // [batch][n_line] lines the legal action touched
    int32_t *aff_s;                                 // [batch] substation the legal action touched (-1: none)
    int32_t *row_used;                              // [batch] row the step solves
    uint8_t *stale, *cap_dirty, *obs_reset;         // [batch]
    int32_t *nb_inst;                               // [batch] active buses per instance
    int32_t *copy_list; int8_t *copy_rows;          // compacted rows for the host's plan mirror
    int32_t *ctl;                                   // [ENV_CTL_WORDS]
    // step inputs
    const int32_t *sub_id; const int8_t *sub_bus; int sub_bus_stride, sub_bus_cols;
    const int32_t *line_id, *line_status;
    int from_reset, tight_cap, prot;
    const int32_t *status, *disc;                   // what the solve left
    int32_t *obs_in; int obs_stride; int stamp;     // observe layer input record (NULL: not bound)
    // reset inputs
    const uint8_t *reset_mask; const int32_t *reset_rows;
};

enum { ACT_MAX_AREA = 16 };            // RulesByArea areas the legality counts handle

// The agent's action rules and grid2op's native topology action (b200pf_act_bind).  The rules apply to both encodings: LookParam
// (MAX_SUB_CHANGED / MAX_LINE_STATUS_CHANGED over the whole grid; n_area = 0) or RulesByArea._lookparam_byarea (the same maxima per
// area: a substation counts in the areas of its mask bits, a line in those of its origin substation), and PreventReconnection.
// With vec = 1 the step's action is the four vectors below instead of EnvArgs' sub_id / line_id pair.
struct ActArgs {
    int max_sub, max_line;                          // MAX_SUB_CHANGED, MAX_LINE_STATUS_CHANGED
    int n_area;                                     // 0: LookParam over the whole grid
    const uint32_t *sub_area, *line_area;           // [n_sub], [n_line] area masks (n_area > 0)
    const int32_t *sub_of_pos;                      // [dim_topo] substation of each topology position
    int vec;                                        // this step's action is the vector action
    const int8_t *set_bus;                          // [batch][dim_topo] 0 leave, -1 disconnect (line ends), 1..n_busbar
    const uint8_t *change_bus;                      // [batch][dim_topo] 0 / 1 (two busbars per substation)
    const int8_t *set_status;                       // [batch][n_line] -1 / 0 / +1
    const uint8_t *change_status;                   // [batch][n_line] 0 / 1
    uint8_t *is_ambiguous;                          // [batch] caller-owned: the action was replaced by "do nothing" as ambiguous
    uint8_t *aff_sub;                               // [batch][n_sub] library scratch: substations the legal vector action touched
};

// The discrete action ids of a b200pf_env_step_ids step: ActArgs' four pointers are then the n rows of the bound action table
// (b200pf_act_table_bind) and instance i acts with row id[i].
struct ActIds {
    const int32_t *id;                              // [batch]
    int n;                                          // rows of the table
};

// the row of the four vectors instance i acts with (ids: NULL without an action table)
ENV_HD inline size_t act_row(const ActIds *ids, int i) { return ids ? (size_t)ids->id[i] : (size_t)i; }

#if defined(__CUDA_ARCH__)
#define ENV_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#define ENV_ATOMIC_MAX(p, v) atomicMax((p), (v))
#define ENV_ATOMIC_OR(p, v) atomicOr((p), (v))
#else
inline int32_t env_fetch_add(int32_t *p, int32_t v) { const int32_t o = *p; *p = o + v; return o; }
#define ENV_ATOMIC_ADD(p, v) env_fetch_add((p), (v))
#define ENV_ATOMIC_MAX(p, v) (*(p) = (*(p) > (v) ? *(p) : (v)))
#define ENV_ATOMIC_OR(p, v) (*(p) |= (v))
#endif

// Inputs the host path accepts: substation / line ids in [-1, n), busbars in [-1, n_busbar]; any line status (> 0 reconnects,
// < 0 disconnects, 0 leaves the line).
ENV_HD inline bool env_input_ok(const EnvArgs &a, int i) {
    if (a.sub_id) {
        const int s = a.sub_id[i];
        if (s < -1 || s >= a.n_sub) return false;
        const int8_t *bus = a.sub_bus + (size_t)i * a.sub_bus_stride;
        for (int k = 0; k < a.sub_bus_cols; ++k)
            if (bus[k] < -1 || bus[k] > a.n_busbar) return false;
    }
    if (a.line_id) {
        const int l = a.line_id[i];
        if (l < -1 || l >= a.n_line) return false;
    }
    return true;
}

// The vector action of instance i: busbars in [-1, n_busbar] with -1 on line ends only (detaching a load, generator or storage unit
// is not restated), change_bus only with two busbars per substation, line statuses in {-1, 0, 1}.  With an action table (ids), its
// id in [0, n): the table's rows were checked when it was bound.
ENV_HD inline bool act_input_ok(const EnvArgs &a, const ActArgs &r, int i, const ActIds *ids = nullptr) {
    if (ids) return ids->id[i] >= 0 && ids->id[i] < ids->n;
    const int8_t *sb = r.set_bus + (size_t)i * a.dim_topo;
    const uint8_t *cb = r.change_bus + (size_t)i * a.dim_topo;
    for (int p = 0; p < a.dim_topo; ++p) {
        if (sb[p] < -1 || sb[p] > a.n_busbar || (sb[p] == -1 && a.line_of_pos[p] < 0)) return false;
        if (cb[p] > 1 || (cb[p] && a.n_busbar != 2)) return false;
    }
    const int8_t *ss = r.set_status + (size_t)i * a.n_line;
    const uint8_t *cs = r.change_status + (size_t)i * a.n_line;
    for (int l = 0; l < a.n_line; ++l)
        if (ss[l] < -1 || ss[l] > 1 || cs[l] > 1) return false;
    return true;
}

// What an action's topological impact counts for the legality rules: lines and substations per area (one area without
// RulesByArea), and whether one of them is in cooldown (PreventReconnection).  Both encodings fill it, one element at a time.
struct ActLegal {
    int n_line[ACT_MAX_AREA], n_sub[ACT_MAX_AREA];
    bool cooldown;
};

ENV_HD inline void act_legal_init(ActLegal &c) {
    for (int k = 0; k < ACT_MAX_AREA; ++k) { c.n_line[k] = 0; c.n_sub[k] = 0; }
    c.cooldown = false;
}

ENV_HD inline void act_count(const ActArgs *r, const uint32_t *area, int id, int *n) {
    if (!r || !r->n_area) { n[0] += 1; return; }
    const uint32_t m = area[id];
    for (int k = 0; k < r->n_area; ++k) n[k] += (int)((m >> k) & 1u);
}

ENV_HD inline void act_impact_line(ActLegal &c, const EnvArgs &a, const ActArgs *r, int i, int l) {
    c.cooldown |= a.line_cd[(size_t)i * a.n_line + l] > 0;
    act_count(r, r ? r->line_area : nullptr, l, c.n_line);
}

ENV_HD inline void act_impact_sub(ActLegal &c, const EnvArgs &a, const ActArgs *r, int i, int s) {
    c.cooldown |= a.sub_cd[(size_t)i * a.n_sub + s] > 0;
    act_count(r, r ? r->sub_area : nullptr, s, c.n_sub);
}

// LookParam (or RulesByArea's counts) and PreventReconnection; without bound rules, DefaultRules with both maxima at 1
ENV_HD inline bool act_illegal(const ActLegal &c, const ActArgs *r) {
    const int max_line = r ? r->max_line : 1, max_sub = r ? r->max_sub : 1, na = r && r->n_area ? r->n_area : 1;
    bool bad = c.cooldown;
    for (int k = 0; k < na; ++k) bad |= c.n_line[k] > max_line || c.n_sub[k] > max_sub;
    return bad;
}

// _BackendAction's topology stage for one position: change_bus (connected elements toggle 1 <-> 2), then set_bus
ENV_HD inline int act_topo_value(int v, uint8_t change, int8_t set) {
    if (change && v > 0) v = 3 - v;
    return set != 0 ? set : v;
}

// grid2op's native topology action for instance i (BaseEnv.step, baseEnv.py:3706-3767): ambiguity, topological impact on the line
// status the previous step left, legality, and _BackendAction.__iadd__'s application (line status change then set, change_bus then
// set_bus, then the reconciliation of disconnected / reconnected line ends).  A disconnected end is one <= 0.  Writes is_ambiguous,
// is_illegal, the impacted lines (affl) and substations (aff_sub) of a legal action; -> the topology may have changed.
ENV_HD inline bool act_vec_instance(const EnvArgs &a, const ActArgs &r, int i, bool done, uint8_t *affl, const ActIds *ids = nullptr) {
    const int nl = a.n_line, ns = a.n_sub, nt = a.dim_topo;
    int8_t *tv = a.topo + (size_t)i * a.n_topo_in;
    int8_t *lb = a.last_bus + (size_t)i * nt;
    const size_t row = act_row(ids, i);
    const int8_t *sb = r.set_bus + row * nt;
    const uint8_t *cb = r.change_bus + row * nt;
    const int8_t *ss = r.set_status + row * nl;
    const uint8_t *cs = r.change_status + row * nl;
    uint8_t *affs = r.aff_sub + (size_t)i * ns;
    for (int s = 0; s < ns; ++s) affs[s] = 0;
    // 1. BaseAction._check_for_ambiguity, topology part (baseAction.py:3558-3565, :3670-3771)
    bool any = false, amb = false;
    for (int p = 0; p < nt; ++p) {
        amb |= sb[p] != 0 && cb[p];
        any |= sb[p] != 0 || cb[p];
    }
    for (int l = 0; l < nl; ++l) {
        const int so = sb[a.line_or_pos[l]], se = sb[a.line_ex_pos[l]];
        const bool ch = cb[a.line_or_pos[l]] || cb[a.line_ex_pos[l]];
        amb |= ss[l] != 0 && cs[l];
        amb |= (so == -1 && se > 0) || (se == -1 && so > 0);
        amb |= ss[l] == -1 && (so > 0 || se > 0 || ch);
        amb |= ss[l] == 1 && (so == -1 || se == -1 || ch);
        any |= ss[l] != 0 || cs[l];
    }
    amb = amb && !done;
    r.is_ambiguous[i] = amb ? 1 : 0;
    // 2. get_topological_impact (baseAction.py:1796-2022): the lines whose status the action sets, changes, or reaches through a
    // busbar of one end; the substations of the remaining bus changes (ends of those lines excluded when they reconnect a line or
    // the status action targets a disconnected line)
    ActLegal c;
    act_legal_init(c);
    for (int l = 0; l < nl; ++l) {
        const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
        const bool on = tv[po] > 0 && tv[pe] > 0, named = cs[l] || ss[l] != 0;
        const bool conn = (sb[po] > 0 || sb[pe] > 0) && !on, disc = (sb[po] < 0 || sb[pe] < 0) && on;
        affl[l] = (named || conn || disc) ? 1 : 0;
        if (affl[l]) act_impact_line(c, a, &r, i, l);
    }
    for (int p = 0; p < nt; ++p) {
        if (!(cb[p] || sb[p] != 0)) continue;
        const int l = a.line_of_pos[p];
        if (l >= 0) {                                         // an end of an impacted line that was out, or of one it disconnects
            const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
            const bool on = tv[po] > 0 && tv[pe] > 0;
            if (on ? (sb[po] < 0 || sb[pe] < 0) : affl[l] != 0) continue;
        }
        const int s = r.sub_of_pos[p];
        if (!affs[s]) { affs[s] = 1; act_impact_sub(c, a, &r, i, s); }
    }
    // 3. legality; an ambiguous, illegal or finished instance's action is "do nothing"
    const bool illegal = !amb && act_illegal(c, &r);
    const bool counted = illegal && !done;
    a.is_illegal[i] = counted ? 1 : 0;
    if (counted) ENV_ATOMIC_ADD(&a.ctl[ENV_CTL_N_ILLEGAL], 1);
    if (amb || illegal || done) {
        for (int l = 0; l < nl; ++l) affl[l] = 0;
        for (int s = 0; s < ns; ++s) affs[s] = 0;
        return false;
    }
    if (!any) return false;
    // 4. _BackendAction.__iadd__ (_backendAction.py:738-765, :810-919), with the busbars last registered (last_bus)
    for (int l = 0; l < nl; ++l) {
        const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
        int vo = tv[po], ve = tv[pe];
        if (cs[l]) {                                          // change_status
            if (vo > 0 || ve > 0) { vo = -1; ve = -1; }
            else { vo = lb[po]; ve = lb[pe]; }
        }
        if (ss[l] < 0) { vo = -1; ve = -1; }                  // set_status
        else if (ss[l] > 0) {
            if (vo <= 0) vo = lb[po];
            if (ve <= 0) ve = lb[pe];
        }
        const bool before_off = vo <= 0;                      // _status_or_before
        const bool disco = before_off || ve <= 0;
        vo = act_topo_value(vo, cb[po], sb[po]);
        ve = act_topo_value(ve, cb[pe], sb[pe]);
        if (before_off && (vo > 0 || ve > 0)) {               // _aux_iadd_reconcile_disco_reco: reconnected, the other end on its last busbar
            if (vo <= 0) vo = lb[po];
            if (ve <= 0) ve = lb[pe];
        } else if (disco || vo <= 0 || ve <= 0) { vo = -1; ve = -1; }
        tv[po] = (int8_t)vo; tv[pe] = (int8_t)ve;
    }
    for (int p = 0; p < nt; ++p)
        if (a.line_of_pos[p] < 0) tv[p] = (int8_t)act_topo_value(tv[p], cb[p], sb[p]);
    for (int p = 0; p < nt; ++p)                              // last_topo_registered.update_connected
        if (tv[p] > 0) lb[p] = tv[p];
    return true;
}

// active buses of one topology record (b200pf_grid_max_active_buses)
ENV_HD inline int env_count_buses(const EnvArgs &a, const int8_t *tv) {
    uint32_t bits[ENV_MAX_SLOT / 32];
    const int nw = (a.n_slot + 31) / 32;
    for (int w = 0; w < nw; ++w) bits[w] = 0u;
    for (int e = 0; e < a.n_elem; ++e) {
        const int b = tv[a.elem_pos[e]];
        if (b > 0 && b <= a.n_busbar) {
            const int s = a.elem_sub[e] + (b - 1) * a.n_sub;
            bits[s >> 5] |= 1u << (s & 31);
        }
    }
    int n = 0;
    for (int w = 0; w < nw; ++w) {
#if defined(__CUDA_ARCH__)
        n += __popc(bits[w]);
#else
        n += __builtin_popcount(bits[w]);
#endif
    }
    return n;
}

// BatchedEnv._apply_agent (or _apply_actions, ac->vec) followed by _apply_environment and the opponent's attack (o: NULL or no
// opponent bound), for instance i (g: the GeometricOpponent's part, m: the GeometricOpponentMultiArea's; NULL for the other kinds;
// ac: NULL or the bound action rules; ids: NULL or the ids into the action table of a b200pf_env_step_ids step)
ENV_HD inline void env_apply_instance(const EnvArgs &a, int i, const OppArgs *o = nullptr, const OppGeoArgs *g = nullptr,
                                      const OppMultiArgs *m = nullptr, const ActArgs *ac = nullptr, const ActIds *ids = nullptr) {
    const int nl = a.n_line;
    int8_t *tv = a.topo + (size_t)i * a.n_topo_in;
    int8_t *lb = a.last_bus + (size_t)i * a.dim_topo;
    uint8_t *affl = a.aff_l + (size_t)i * nl;
    for (int l = 0; l < nl; ++l) affl[l] = 0;
    a.aff_s[i] = -1;
    const bool done = a.done[i] != 0;
    bool dirty = false;
    // the opponent decides first, on the line status the previous step left (grid2op's current_obs); its attack lands last
    int opp_line = -1, opp_dur = 0;
    if (o && o->kind != OPP_NONE) {
        if (!done && !a.from_reset) opp_line = opp_decide_instance(*o, i, tv, a.line_or_pos, a.line_ex_pos, nl, &opp_dur, g, m);
        else if (m) opp_multi_none(*m, i);
        o->attack_line[i] = opp_line; o->attack_dur[i] = opp_dur;
    }
    if (ac && ac->is_ambiguous && (a.from_reset || !ac->vec)) ac->is_ambiguous[i] = 0;
    if (!a.from_reset && ac && ac->vec) {
        dirty = act_vec_instance(a, *ac, i, done, affl, ids);
    } else if (!a.from_reset) {
        bool has_sub = false, has_line = false;
        int sid = -1, lid = -1, lst = 0;
        const int8_t *bus = nullptr;
        if (a.sub_id) {
            sid = a.sub_id[i];
            bus = a.sub_bus + (size_t)i * a.sub_bus_stride;
            bool any = false;
            for (int k = 0; k < a.sub_bus_cols; ++k) any |= bus[k] != 0;
            has_sub = sid >= 0 && any;
        }
        if (a.line_id) {
            lid = a.line_id[i]; lst = a.line_status[i];
            has_line = lid >= 0 && lst != 0;
        }
        // a busbar > 0 for the end of a disconnected line reconnects that line (baseAction.py:1836-1860)
        // (each reconnecting entry counts as one line, as BatchedEnv._apply_agent counts them)
        ActLegal c;
        act_legal_init(c);
        int n_reco = 0;
        bool reco_is_line = false, m_not_reco = false, sub_impacted = has_sub;
        const int32_t *pos = has_sub ? a.sub_pos + (size_t)sid * a.max_sub : nullptr;
        if (has_sub) {
            for (int k = 0; k < a.max_sub; ++k) {
                const int p = pos[k], v = bus[k];
                if (p < 0 || v <= 0) continue;
                const int lp = a.line_of_pos[p];
                if (tv[p] <= 0 && lp >= 0) {
                    ++n_reco;
                    act_impact_line(c, a, ac, i, lp);
                    reco_is_line |= has_line && lp == lid;
                } else m_not_reco = true;
            }
            if (n_reco) sub_impacted = m_not_reco;
            if (sub_impacted) act_impact_sub(c, a, ac, i, sid);
        }
        if (has_line && !reco_is_line) act_impact_line(c, a, ac, i, lid);
        // the legality rules; finished instances ignore their action
        const bool illegal = act_illegal(c, ac);
        const bool counted = illegal && !done;
        a.is_illegal[i] = counted ? 1 : 0;
        if (counted) ENV_ATOMIC_ADD(&a.ctl[ENV_CTL_N_ILLEGAL], 1);
        const bool ok = !illegal && !done;
        if (has_sub && ok) {
            for (int k = 0; k < a.max_sub; ++k) {            // connected elements take the named busbar
                const int p = pos[k], v = bus[k];
                if (p >= 0 && v > 0 && tv[p] > 0) { tv[p] = (int8_t)v; lb[p] = (int8_t)v; }
            }
            if (n_reco) {                                     // reconnections, in the order of the numpy code
                for (int k = 0; k < a.max_sub; ++k) {
                    const int p = pos[k], v = bus[k];
                    if (p >= 0 && v > 0 && tv[p] <= 0 && a.line_of_pos[p] >= 0) { tv[p] = (int8_t)v; affl[a.line_of_pos[p]] = 2; }
                }
                for (int k = 0; k < a.max_sub; ++k) {
                    const int p = pos[k];
                    if (p >= 0 && bus[k] > 0 && a.line_of_pos[p] >= 0 && affl[a.line_of_pos[p]] == 2) lb[p] = bus[k];
                }
                for (int k = 0; k < a.max_sub; ++k) {
                    const int p = pos[k];
                    if (p >= 0 && bus[k] > 0 && a.line_of_pos[p] >= 0 && affl[a.line_of_pos[p]] == 2) {
                        const int po = a.other_end_pos[p];
                        tv[po] = lb[po];
                    }
                }
                for (int l = 0; l < nl; ++l) affl[l] = affl[l] ? 1 : 0;
            }
            if (sub_impacted) a.aff_s[i] = sid;
            dirty = true;
        }
        if (has_line && ok) {
            const int po = a.line_or_pos[lid], pe = a.line_ex_pos[lid];
            if (lst < 0) { tv[po] = -1; tv[pe] = -1; }
            else { tv[po] = lb[po]; tv[pe] = lb[pe]; }
            affl[lid] = 1;
            dirty = true;
        }
    }
    // maintenance / hazards of the row this instance is about to solve: those lines are out
    const int r = a.t[i];
    a.row_used[i] = r;
    if ((a.maint || a.haz) && !done) {
        const size_t base = ((size_t)a.scen[i] * a.n_rows + r) * nl;
        for (int l = 0; l < nl; ++l) {
            const bool forced = (a.maint && a.maint[base + l]) || (a.haz && a.haz[base + l]);
            if (!forced) continue;
            const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
            if (tv[po] > 0 || tv[pe] > 0) dirty = true;
            tv[po] = -1; tv[pe] = -1;
        }
    }
    if (opp_line >= 0) {                                      // the attack: its lines are out, their cooldown at least its duration
        int32_t *lc = a.line_cd + (size_t)i * nl;
        const int n_hit = m ? m->n_area : 1;
        for (int k = 0; k < n_hit; ++k) {
            const int l = m ? m->attack_lines[(size_t)i * m->n_area + k] : opp_line;
            if (l < 0) continue;
            if (lc[l] < opp_dur) lc[l] = opp_dur;
            const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
            if (tv[po] > 0 || tv[pe] > 0) dirty = true;
            tv[po] = -1; tv[pe] = -1;
        }
    }
    if (dirty) { a.cap_dirty[i] = 1; ENV_ATOMIC_ADD(&a.ctl[ENV_CTL_N_DIRTY], 1); }
    if (dirty || a.stale[i]) {                                // rows the host's plan mirror has not seen
        const int k = ENV_ATOMIC_ADD(&a.ctl[ENV_CTL_N_COPY], 1);
        a.copy_list[k] = i;
        int8_t *dst = a.copy_rows + (size_t)k * a.n_topo_in;
        for (int j = 0; j < a.n_topo_in; ++j) dst[j] = tv[j];
    }
    if (a.tight_cap) {                                        // _bus_cap: count the instances whose topology changed
        if (a.cap_dirty[i]) { a.nb_inst[i] = env_count_buses(a, tv); a.cap_dirty[i] = 0; }
        ENV_ATOMIC_MAX(&a.ctl[ENV_CTL_CAP_MAX], a.nb_inst[i]);
    }
}

// the rest of BatchedEnv.step behind the solve, for instance i (al: NULL or the line alerts, am: NULL or the alarms, ac: NULL or the
// bound action rules)
ENV_HD inline void env_post_instance(const EnvArgs &a, int i, const AlertArgs *al = nullptr, const AlarmArgs *am = nullptr,
                                     const ActArgs *ac = nullptr) {
    const int nl = a.n_line, ns = a.n_sub;
    int8_t *tv = a.topo + (size_t)i * a.n_topo_in;
    const bool live = a.done[i] == 0;
    const int32_t *disc = a.prot && a.disc ? a.disc + (size_t)i * nl : nullptr;
    if (disc && live) {                                       // _backend_action.update_state(disc_lines): tripped lines stay out
        bool any = false;
        for (int l = 0; l < nl; ++l)
            if (disc[l] >= 0) { tv[a.line_or_pos[l]] = -1; tv[a.line_ex_pos[l]] = -1; any = true; }
        if (any) a.stale[i] = 1;
    } else if (disc) {
        // A finished instance keeps its topology (the host path masks the trips with ~done).  The library may still have solved it
        // and tripped lines of it on the device (an episode the isolated-busbar rule ended is not finished for the library): put
        // those lines back on their busbars, which last_bus holds for every connected end.
        bool any = false;
        const int8_t *lb = a.last_bus + (size_t)i * a.dim_topo;
        for (int l = 0; l < nl; ++l)
            if (disc[l] >= 0) {
                const int po = a.line_or_pos[l], pe = a.line_ex_pos[l];
                tv[po] = lb[po]; tv[pe] = lb[pe]; any = true;
            }
        if (any) a.stale[i] = 1;
    }
    int st = a.status[i];
    for (int s = 0; s < a.n_iso_seg; ++s) {                   // _isolated_shunt_busbar, after this step's trips
        const int lo = a.iso_seg[s], hi = s + 1 < a.n_iso_seg ? a.iso_seg[s + 1] : a.n_iso_cols;
        int on1 = 0;
        for (int j = lo; j < hi; ++j) on1 += tv[a.iso_cols[j]] == 1;
        if (on1 == 0) { st = 2; break; }
    }
    a.status_out[i] = st;
    // cooldowns (baseEnv.py:3352-3393, :2566-2597), in the reference's order
    const size_t base = ((size_t)a.scen[i] * a.n_rows + a.row_used[i]) * nl;
    int32_t *lc = a.line_cd + (size_t)i * nl;
    const uint8_t *affl = a.aff_l + (size_t)i * nl;
    for (int l = 0; l < nl; ++l) {
        int c = lc[l];
        if (c > 0 && live) c -= 1;
        if (disc && disc[l] >= 0 && live) c = a.cd_reco;
        if (a.maint_time && live && a.maint_time[base + l] == 0) c = c > a.maint_dur[base + l] ? c : a.maint_dur[base + l];
        if (a.haz_dur && live) c = c > a.haz_dur[base + l] ? c : a.haz_dur[base + l];
        if (!a.from_reset && a.cd_line > 0 && affl[l] && c < a.cd_line) c = a.cd_line;
        lc[l] = c;
    }
    int32_t *sc = a.sub_cd + (size_t)i * ns;
    if (!a.from_reset && a.cd_sub > 0) {
        for (int s = 0; s < ns; ++s)
            if (sc[s] > 0 && live) sc[s] -= 1;
        if (a.aff_s[i] >= 0) sc[a.aff_s[i]] = a.cd_sub;
        if (ac && ac->vec)
            for (int s = 0; s < ns; ++s)
                if (ac->aff_sub[(size_t)i * ns + s]) sc[s] = a.cd_sub;
    }
    // an ambiguous action was "do nothing": not illegal, but rewarded as one and registering no alarm
    const bool ambiguous = ac && ac->is_ambiguous && ac->is_ambiguous[i];
    const bool newly = live && st != 0;
    a.newly_done[i] = newly ? 1 : 0;
    if (newly) a.done[i] = 1;
    if (a.from_reset) {
        a.is_illegal[i] = 0;
        if (live) { a.current_step[i] = 0; a.obs_reset[i] = 1; }
    } else if (live) a.current_step[i] += 1;
    const bool alerts = al && al->n;
    if (alerts) {                                             // an instance finished before the step keeps its alert state
        if (live && !a.from_reset) {
            alert_update_instance(*al, i);
            if (al->reward) alert_reward_instance(*al, i, newly);
            else al->reward_out[i] = 0.0;
        } else al->reward_out[i] = 0.0;
    }
    const bool alarms = am && am->n;
    if (alarms) {                                             // an instance finished before the step keeps its alarm state
        if (live && !a.from_reset) {
            alarm_register_instance(*am, i, a.current_step[i], a.is_illegal[i] != 0 || ambiguous);
            if (am->reward && newly) alarm_reward_instance(*am, i, a.current_step[i], disc);
            else am->reward_out[i] = 0.0;
        } else { am->illegal[i] = 0; am->reward_out[i] = 0.0; }
    }
    if (a.obs_in) {                                           // BatchedEnv.observe_inputs
        int32_t *h = a.obs_in + (size_t)i * a.obs_stride;
        for (int l = 0; l < nl; ++l) h[l] = lc[l];
        for (int s = 0; s < ns; ++s) h[nl + s] = sc[s];
        h[nl + ns] = a.current_step[i]; h[nl + ns + 1] = a.stamp;
        h[nl + ns + 2] = (a.is_illegal[i] ? 1 : 0) + (a.done[i] ? 2 : 0) + (a.obs_reset[i] ? 4 : 0) + (ambiguous ? 8 : 0);
        if (alerts) alert_obs_record(*al, i, h + nl + ns + 3);
        if (alarms) alarm_obs_record(*am, i, a.current_step[i], h + nl + ns + 3 + (alerts ? 6 * al->n + 1 : 0));
    }
}

// BatchedEnv.reset_instances for the instances of the mask (rows: next chronics row, default t0), opponent state included
ENV_HD inline void env_reset_instance(const EnvArgs &a, int i, const OppArgs *o = nullptr, const OppGeoArgs *g = nullptr,
                                      const OppMultiArgs *m = nullptr, const AlertArgs *al = nullptr, const AlarmArgs *am = nullptr,
                                      const ActArgs *ac = nullptr) {
    if (!a.reset_mask[i]) return;
    if (ac && ac->is_ambiguous) ac->is_ambiguous[i] = 0;
    if (al && al->n) alert_reset_instance(*al, i);
    if (am && am->n) alarm_reset_instance(*am, i);
    if (o && o->kind != OPP_NONE) opp_reset_instance(*o, i);
    if (o && g && o->kind == OPP_GEOMETRIC) opp_geo_reset_instance(*o, *g, i);
    if (o && m && o->kind == OPP_GEOMETRIC_MULTI) opp_multi_reset_instance(*m, i);
    const int nl = a.n_line;
    int8_t *tv = a.topo + (size_t)i * a.n_topo_in;
    const int8_t *t0v = a.topo0 + (size_t)i * a.n_topo_in;
    for (int j = 0; j < a.n_topo_in; ++j) tv[j] = t0v[j];
    int8_t *lb = a.last_bus + (size_t)i * a.dim_topo;
    for (int j = 0; j < a.dim_topo; ++j) lb[j] = t0v[j] > 0 ? t0v[j] : 1;
    for (int l = 0; l < nl; ++l) a.line_cd[(size_t)i * nl + l] = 0;
    for (int s = 0; s < a.n_sub; ++s) a.sub_cd[(size_t)i * a.n_sub + s] = 0;
    a.done[i] = 0; a.current_step[i] = 0; a.is_illegal[i] = 0; a.obs_reset[i] = 1;
    int r = a.reset_rows ? a.reset_rows[i] % a.n_rows : a.t0[i];
    if (r < 0) r += a.n_rows;
    a.t[i] = r;
    if (a.lib_done) a.lib_done[i] = 0;
    for (int l = 0; l < nl; ++l) {
        const size_t o = (size_t)i * nl + l;
        if (a.pcount) a.pcount[o] = 0;
        if (a.ts_over) a.ts_over[o] = 0;
        if (a.lib_disc) a.lib_disc[o] = -1;
        if (a.trip) a.trip[o] = 0;
        if (a.incdone) a.incdone[o] = 0;
    }
    a.cap_dirty[i] = 1; a.stale[i] = 1;
    if (a.obs_in) {                                           // what observe_inputs gives right after a reset (stamp kept)
        int32_t *h = a.obs_in + (size_t)i * a.obs_stride;
        for (int j = 0; j < nl + a.n_sub + 1; ++j) h[j] = 0;
        h[nl + a.n_sub + 2] = 4;
        if (al && al->n) alert_obs_record(*al, i, h + nl + a.n_sub + 3);
        if (am && am->n) alarm_obs_record(*am, i, 0, h + nl + a.n_sub + 3 + (al && al->n ? 6 * al->n + 1 : 0));
    }
}

// after an observe launch: the reset flags have been consumed (BatchedEnv.observe clears them)
ENV_HD inline void env_observed_instance(const EnvArgs &a, int i) {
    a.obs_reset[i] = 0;
    if (a.obs_in) a.obs_in[(size_t)i * a.obs_stride + a.n_line + a.n_sub + 2] &= ~4;
}

#if defined(__CUDACC__)
// (r.aff_sub is NULL when no action rules are bound; ids.id NULL without an action table)
__global__ void __launch_bounds__(128) pf_kernel_env_validate(EnvArgs a, ActArgs r, ActIds ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.batch && !(r.vec ? act_input_ok(a, r, i, ids.id ? &ids : nullptr) : env_input_ok(a, i))) atomicOr(&a.ctl[ENV_CTL_ERR], 1);
}

// one thread per instance; nothing is written when the validation flagged an input
__global__ void __launch_bounds__(128) pf_kernel_env_apply(EnvArgs a, OppArgs o, OppGeoArgs g, OppMultiArgs m, ActArgs r, ActIds ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.batch || *(volatile int32_t *)&a.ctl[ENV_CTL_ERR]) return;
    env_apply_instance(a, i, &o, o.kind == OPP_GEOMETRIC ? &g : nullptr, o.kind == OPP_GEOMETRIC_MULTI ? &m : nullptr,
                       r.aff_sub ? &r : nullptr, ids.id ? &ids : nullptr);
}

__global__ void __launch_bounds__(128) pf_kernel_env_post(EnvArgs a, AlertArgs al, AlarmArgs am, ActArgs r) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.batch) env_post_instance(a, i, al.n ? &al : nullptr, am.n ? &am : nullptr, r.aff_sub ? &r : nullptr);
}

__global__ void __launch_bounds__(128) pf_kernel_env_reset(EnvArgs a, OppArgs o, OppGeoArgs g, OppMultiArgs m, AlertArgs al, AlarmArgs am,
                                                           ActArgs r) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.batch)
        env_reset_instance(a, i, &o, o.kind == OPP_GEOMETRIC ? &g : nullptr, o.kind == OPP_GEOMETRIC_MULTI ? &m : nullptr, al.n ? &al : nullptr,
                           am.n ? &am : nullptr, r.aff_sub ? &r : nullptr);
}

__global__ void __launch_bounds__(128) pf_kernel_env_observed(EnvArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.batch) env_observed_instance(a, i);
}
#endif

}  // namespace b200pf

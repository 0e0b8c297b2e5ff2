// TEST INFRASTRUCTURE (never part of the product): host build of the alarm bodies (grid2op_b200/csrc/b200pf_alarm.cuh) inside the
// environment bodies (b200pf_env.cuh) with a GeometricOpponent, and of the observation layer's body with the alarm values in its
// input record (b200pf_obs.cuh), so that BatchedEnv's alarms on the device can be checked against the numpy path and grid2op
// without a GPU.
#include "../../grid2op_b200/csrc/b200pf_env.cuh"
#include "../../grid2op_b200/csrc/b200pf_obs.cuh"
#include "../../include/b200pf.h"

using namespace b200pf;

extern "C" int alarm_emu_args_size(void) { return (int)sizeof(AlarmArgs); }

// what: 2 post (with the alarms), 3 reset (with the opponent and the alarms); g: the GeometricOpponent or NULL
extern "C" int alarm_emu_run(const EnvArgs *a, const OppArgs *o, const OppGeoArgs *g, const AlarmArgs *am, int what) {
    for (int i = 0; i < a->batch; ++i) {
        switch (what) {
        case 2: env_post_instance(*a, i, nullptr, am); break;
        case 3: env_reset_instance(*a, i, o, g, nullptr, nullptr, am); break;
        default: return -1;
        }
    }
    return 0;
}

// AlarmReward of instance i on a game-over step (disc: the step's disc_lines [n_line])
extern "C" int alarm_emu_reward(const AlarmArgs *am, int i, int step, const int32_t *disc) {
    alarm_reward_instance(*am, i, step, disc);
    return 0;
}

// pf_kernel_observe with one lane, the input record as b200pf_obs_bind lays it out (sizes as tests/emu/obs_emu.cpp)
extern "C" int alarm_emu_observe(const b200pf_obs_desc *d, const int32_t *sizes, const int32_t *line_or_pos, const int32_t *line_ex_pos,
                                 int batch, const float *out, const float *rho, const int8_t *topo, const int32_t *t, const int32_t *scen,
                                 const float *chron, int n_rows, const float *th_lim, const int32_t *host_in, int32_t *ts_over,
                                 int32_t *ts_prot, int32_t *stamp, int32_t *go_row, float *obs, float *reward) {
    ObsArgs a{};
    a.batch = batch;
    a.n_line = sizes[0]; a.n_sub = sizes[1]; a.n_gen = sizes[2]; a.n_hidden = sizes[3]; a.n_load = sizes[4]; a.n_sto = sizes[5];
    a.n_shunt = sizes[6]; a.dim_topo = sizes[7]; a.n_topo_in = sizes[8]; a.n_out = sizes[9];
    a.line_or_pos = line_or_pos; a.line_ex_pos = line_ex_pos;
    a.out = out; a.rho = rho; a.topo = topo; a.t = t; a.scen = scen; a.chron = chron; a.n_rows = n_rows; a.th_lim = th_lim;
    a.calendar = d->calendar; a.max_step = d->max_step; a.delta_time = d->delta_time; a.maint_time = d->maint_time; a.maint_dur = d->maint_dur;
    a.gen_pmin = d->gen_pmin; a.gen_pmax = d->gen_pmax; a.gen_ramp_up = d->gen_ramp_up; a.gen_ramp_down = d->gen_ramp_down;
    a.gen_cost = d->gen_cost; a.gen_renewable = d->gen_renewable; a.redisp_available = d->redisp_available;
    a.sto_charge0 = d->sto_charge0; a.sto_loss_step = d->sto_loss_step; a.seg = d->seg; a.n_seg = d->n_seg; a.n_obs = d->n_obs;
    a.reward_kind = d->reward_kind; a.max_regret = d->max_regret; a.reward_min = d->reward_min; a.reward_illegal = d->reward_illegal;
    a.dts_hours = d->dts_hours; a.soft_thr = d->soft_thr;
    a.n_alert = d->n_alert; a.n_alarm = d->n_alarm;
    a.host = host_in;
    a.host_stride = a.n_line + a.n_sub + 3 + (d->n_alert ? 6 * d->n_alert + 1 : 0) + (d->n_alarm ? d->n_alarm + 4 : 0);
    a.ts_over = ts_over; a.ts_prot = ts_prot; a.stamp = stamp; a.go_row = go_row; a.obs = obs; a.reward = reward;
    for (int inst = 0; inst < batch; ++inst) {
        double part[4];
        obs_instance(a, inst, 0, 1, part);
        if (reward && a.reward_kind != OBS_REWARD_NONE) reward[inst] = obs_reward(a, inst, part);
        stamp[inst] = host_in[(size_t)inst * a.host_stride + a.n_line + a.n_sub + 1];
    }
    return 0;
}

// b200pf.cu — C-ABI of the batched GPU power-flow engine (see include/b200pf.h).
// Host side: owns the device copy of the static grid description, the staging buffers, one CUDA
// stream per handle, and picks the thread-group size / shared-memory budget per launch.
#include "b200pf_kernel.cuh"
#include "b200pf_small.cuh"
#include "b200pf_sparse.cuh"
#include "b200pf_block.cuh"
#include "b200pf_redo.cuh"
#include "b200pf_obs.cuh"
#include "b200pf_env.cuh"
#include "../../include/b200pf.h"

#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

using namespace b200pf;

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }

#define CU(call)                                                                                 \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess)                                                                  \
            return fail(B200PF_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));     \
    } while (0)

// device buffers of one layer of the device environment (observation, environment, opponent, alerts, alarms), freed together
struct DevBufs {
    std::vector<void *> p;
    void release() { for (void *q : p) cudaFree(q); p.clear(); }
};

// kernel family of a launch, as b200pf_plan_stats reports it
enum LaunchKind { KERN_NONE = 0, KERN_WARP_PIVOTING = 1, KERN_CTA_PIVOTING = 2, KERN_PLANNED_SPARSE = 3, KERN_PLANNED_BLOCK = 4 };

struct b200pf_handle {
    int device = 0;
    int max_batch = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t own_stream = nullptr;
    cudaStream_t chunk_stream[4] = {nullptr, nullptr, nullptr, nullptr};
    int chunk_next = 0;
    cudaStream_t group_stream[B200PF_MAX_GROUPS] = {};
    cudaEvent_t group_event[B200PF_MAX_GROUPS] = {};
    bool group_pending[B200PF_MAX_GROUPS] = {};
    int small_occ[2][33] = {};
    int group_flags = 0;                                    // bit 0: kernels store results straight into pinned host memory
    float *x_out = nullptr; int *x_status = nullptr; int *x_iters = nullptr; float *x_rho = nullptr;
    DevGrid g{};
    std::vector<void *> dev_allocs;
    int sm_count = 132;
    int max_smem_optin = 0;
    // staging (run_host)
    int8_t *d_topo = nullptr; double *d_inj = nullptr; float *d_out = nullptr; int *d_status = nullptr;
    int *d_iters = nullptr; double *d_busv = nullptr;
    int8_t *h_topo = nullptr; double *h_inj = nullptr; float *h_out = nullptr; int *h_status = nullptr;
    int *h_iters = nullptr; double *h_busv = nullptr;
    float *h_rows = nullptr; float *d_rows = nullptr;
    // series
    float *d_chron = nullptr; int *d_scen = nullptr; int *d_t = nullptr; double *d_static_inj = nullptr;
    float *d_thlim = nullptr; float *d_rho = nullptr; int8_t *d_series_topo = nullptr;
    int series_batch = 0, n_scen = 0, n_rows = 0;
    int *d_pcount = nullptr, *d_tsover = nullptr, *d_disc = nullptr, *d_done = nullptr;
    int prot = 0, next_reset = 0, max_pc = 2; float hard_thr = 2.0f, soft_thr = 1.0f;
    // planned sparse kernel: cache of topology plans (host blobs + their device copy)
    HostGrid hg;
    std::unordered_map<uint64_t, int> plan_index;           // hash of (topology row, outage) -> newest plan with that hash
    std::vector<int8_t> plan_keys;                          // topology row of every plan (verification)
    std::vector<int> plan_outage, plan_next;                // outage of every plan; next plan with the same hash
    std::vector<int> plan_off, plan_smem;
    std::vector<unsigned char> plan_blobs;                  // concatenated, every plan 16-byte aligned
    unsigned char *d_plan_blobs = nullptr; size_t d_plan_cap = 0, d_plan_used = 0;
    int *d_plan_off = nullptr; int d_plan_off_n = 0;
    int *d_inst_plan = nullptr, *h_inst_plan = nullptr;     // [max_batch]
    std::vector<int8_t> h_series_topo;                      // host mirror of the series topology (protections re-plan from it)
    std::vector<int> h_series_plan;
    int8_t *d_trip = nullptr, *d_incdone = nullptr; int *d_nflag = nullptr, *d_flaglist = nullptr, *d_casclist = nullptr;
    std::vector<int8_t> h_trip; std::vector<int> h_flaglist;
    int last_cascade_rounds = 0;
    int *d_series_plan = nullptr; int series_plan_state = 0; // 0 none, 1 per-instance plans, 2 all instances on one plan
    int series_plan_single = 0, series_plan_smem = 0;
    int plan_policy = 0;                                    // 0 auto, 1 never, 2 whenever a host copy of the topology exists
    int plan_max_smem = 0, plan_max_nb = 0, plan_max_nblkA = 0;
    int series_lay_nb = 0, series_lay_nblkA = 0;
    const void *sparse_occ_kern = nullptr; int sparse_occ_smem = -1, sparse_occ = 0;   // planned kernels: last occupancy query
    int sparse_cta_cap = 0;                                 // > 0: resident CTAs per SM of the planned kernel are capped (rest of the SM's memory = L1); < 0: never
    int sparse_minb = 32;                                   // tuning: one-warp CTAs per SM the small-workspace variant is compiled for (32 or 28)
    int plan_T = 32;                                        // threads per instance of the planned kernel (32, 64, 128)
    int blk = 1;                                            // 1: BLOCK plans + pf_kernel_block (default), 0: scalar plans + pf_kernel_sparse
    int blk_T = 4, blk_U = 2;                               // lanes per instance / operations per lane and row of the block kernel
    int blk_wpc = 4, blk_stage = 1, blk_uni = 1, blk_wpc_pinned = 0, blk_spec = 1;   // experiment knobs: warps per CTA, TMA staging of a shared plan
    unsigned char *d_stat = nullptr; PlanArgs::StatOff stat_off{}; bool stat_dirty = true;   // packed static arrays for staged launches
    int last_kernel = KERN_NONE;                            // LaunchKind of the last launch (b200pf_plan_stats)
    int64_t plans_built = 0, plan_cache_resets = 0, plan_lookups = 0, plan_hits = 0;
    bool series_dev_topo_ahead = false;                     // the warp kernel tripped lines in d_series_topo on the device: the host mirror / plans lag
    bool series_plans_stale = false;                        // the cache was reset under the series' plan ids: re-resolve before the next step
    int64_t launches = 0;
    int redo_enabled = 1;                                   // pivoting re-solve of what the planned kernel leaves as ST_DIV (B200PF_NO_REDO=1 turns it off)
    int dbg_div_mod = 0;                                    // test knob, see b200pf_set_debug
    int *series_flag = nullptr; int series_step_no = 0;    // completion flag of series steps
    // safety net, per launching stream (chunk / group launches of one handle run concurrently): the control word of its tail
    // launch (one stream's armed re-solve must not stand in for another's), and on the large grids the global-memory matrices
    // (two safety-net launches in flight must never share a CTA's matrix)
    struct RedoStream { RedoCtl *ctl = nullptr; unsigned char *mat = nullptr; size_t stride = 0; int ctas = 0; };
    std::unordered_map<cudaStream_t, RedoStream> redo_streams;
    bool on_side_stream = false;                            // a chunk / group launch is being issued (h->stream is swapped for it)
    cudaEvent_t inst_plan_ev = nullptr; bool inst_plan_pending = false;   // last H2D copy out of h_inst_plan
    int last_smem = 0, last_T = 0, last_grid = 0, last_block = 0;
    int last_cfg[8] = {-1, -1, -1, -1, -1, -1, -1, -1};    // template parameters of the last launch (b200pf_last_launch_config)
    // observation layer (b200pf_obs_bind / b200pf_observe)
    ObsArgs obs{}; int obs_batch = 0, obs_rows = 0;
    DevBufs obs_bufs;
    int32_t *h_obs_in = nullptr, *d_obs_in = nullptr;       // pinned host record of the per-instance inputs and its device copy
    cudaEvent_t obs_ev = nullptr; bool obs_ev_pending = false;
    int64_t obs_launches = 0, obs_h2d_bytes = 0, d2h_bytes = 0;
    // device environment state (b200pf_env_bind / b200pf_env_step)
    EnvArgs env{}; int env_batch = 0;
    DevBufs env_bufs;
    int32_t *h_env_ctl = nullptr;                           // pinned copy of the step's control words
    std::vector<int8_t> env_mirror;                         // host mirror of the device topology the plans are looked up from
    std::vector<int32_t> env_list; std::vector<int8_t> env_rows;
    std::vector<int8_t> env_topo0; std::vector<uint8_t> env_mask;   // host copies: reset topologies, the last reset mask
    int64_t env_steps = 0, env_h2d = 0, env_d2h = 0, env_waits = 0, env_illegal = 0, env_plan_refresh = 0;
    int env_last_cap = 0, env_last_dirty = 0;
    // line-attack opponent of the device environment (b200pf_opp_bind)
    OppArgs opp{}; int opp_batch = 0;
    DevBufs opp_bufs;
    OppGeoArgs opp_geo{}; bool opp_geo_bound = false;            // kind OPP_GEOMETRIC (b200pf_opp_geo_bind; its buffers in opp_bufs)
    OppMultiArgs opp_multi{}; bool opp_multi_bound = false;      // kind OPP_GEOMETRIC_MULTI (b200pf_opp_multi_bind; likewise)
    // line alerts of the device environment (b200pf_alert_bind)
    AlertArgs alert{}; int alert_batch = 0;
    DevBufs alert_bufs;
    // alarms of the device environment (b200pf_alarm_bind)
    AlarmArgs alarm{}; int alarm_batch = 0;
    DevBufs alarm_bufs;
    // the agent's action rules and vector-action buffers of the device environment (b200pf_act_bind)
    ActArgs act{}; int act_batch = 0;
    DevBufs act_bufs;
    // the discrete action table of the device environment (b200pf_act_table_bind): n_act rows in the layout of the vector buffers
    int n_act = 0;
    int8_t *tab_set_bus = nullptr, *tab_set_status = nullptr; uint8_t *tab_change_bus = nullptr, *tab_change_status = nullptr;
    DevBufs act_table_bufs;
};

// Host -> device copy of caller memory (pageable as a rule) that launches on ANY stream of the handle may read afterwards.  A plain
// cudaMemcpy may return before its DMA has finished and the handle's non-blocking streams are not ordered against the legacy
// stream; so the copy is issued on the handle's stream and the stream drained before returning.  Set-up calls only (never per step
// of the device-resident paths).
static int h2d_sync(b200pf_handle *h, void *dst, const void *src, size_t bytes) {
    if (!bytes) return 0;
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}
#define TRY(call) do { int rc__ = (call); if (rc__) return rc__; } while (0)
#define H2D(dst, src, bytes) TRY(h2d_sync(h, (dst), (src), (bytes)))

template <typename Tp>
static int upload(b200pf_handle *h, const Tp *src, size_t n, const Tp **dst) {
    Tp *d = nullptr;
    size_t bytes = (n ? n : 1) * sizeof(Tp);
    CU(cudaMalloc(&d, bytes));
    h->dev_allocs.push_back(d);
    if (n) H2D(d, src, n * sizeof(Tp));
    *dst = d;
    return 0;
}

static bool block_variant_exists(int T, int U);

extern "C" const char *b200pf_last_error(void) { return g_err.c_str(); }
extern "C" int b200pf_abi_version(void) { return B200PF_ABI_VERSION; }
extern "C" int b200pf_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

#if PB_CLOCK_ON
// Measurement build only (-DB200PF_PHASE_CLOCK): copies the block kernel's phase clock (b200pf_block.cuh, PC_SLOTS counters
// of the current device) to dst after a device synchronise, then clears it.  Not part of the ABI of include/b200pf.h.
extern "C" int b200pf_phase_clock_read(unsigned long long *dst, int n) {
    if (!dst || n < PC_SLOTS) return fail(B200PF_E_ARG, "phase clock: destination too small");
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpyFromSymbol(dst, pb_phase_clk, sizeof(unsigned long long) * PC_SLOTS));
    static const unsigned long long zeros[PC_SLOTS] = {};
    CU(cudaMemcpyToSymbol(pb_phase_clk, zeros, sizeof(zeros)));
    return PC_SLOTS;
}
#endif

extern "C" int b200pf_create(const b200pf_grid_desc *gd, int max_batch, int device, b200pf_handle **out) {
    if (!gd || !out || max_batch <= 0) return fail(B200PF_E_ARG, "null argument or max_batch <= 0");
    if (gd->abi_version != B200PF_ABI_VERSION) return fail(B200PF_E_ARG, "ABI version mismatch");
    if (gd->n_sub <= 0 || gd->n_busbar <= 0 || gd->n_line < 0) return fail(B200PF_E_ARG, "bad grid sizes");
    if ((long)gd->n_sub * gd->n_busbar > 30000) return fail(B200PF_E_ARG, "too many bus slots");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(B200PF_E_CUDA, "no CUDA device available: this engine has no CPU fallback");
    }
    if (device < 0 || device >= ndev) return fail(B200PF_E_ARG, "bad device index");
    CU(cudaSetDevice(device));
    b200pf_handle *h = new b200pf_handle();
    h->device = device;
    h->max_batch = max_batch;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    h->sm_count = prop.multiProcessorCount;
    h->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    CU(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    h->stream = h->own_stream;
    DevGrid &g = h->g;
    g.n_sub = gd->n_sub; g.n_busbar = gd->n_busbar; g.n_slot = gd->n_sub * gd->n_busbar;
    g.n_line = gd->n_line; g.n_gen = gd->n_gen; g.n_hidden = gd->n_hidden; g.n_unit = gd->n_gen + gd->n_hidden;
    g.n_load = gd->n_load; g.n_sto = gd->n_storage; g.n_shunt = gd->n_shunt; g.dim_topo = gd->dim_topo;
    g.n_topo_in = g.dim_topo + g.n_shunt + g.n_hidden;
    g.n_inj = g.n_gen + g.n_unit + 2 * g.n_load + g.n_sto + 2 * g.n_shunt;
    g.n_out = 10 * g.n_line + 4 * g.n_unit + 2 * g.n_load + g.n_sto + 3 * g.n_shunt;
    g.base_mva = gd->sn_mva;
    int rc = 0;
#define UP(field, src, n) if ((rc = upload(h, src, (size_t)(n), &g.field)) != 0) { b200pf_destroy(h); return rc; }
    UP(line_or_sub, gd->line_or_sub, g.n_line) UP(line_ex_sub, gd->line_ex_sub, g.n_line)
    UP(line_or_pos, gd->line_or_pos, g.n_line) UP(line_ex_pos, gd->line_ex_pos, g.n_line)
    UP(line_y, gd->line_y, 8 * g.n_line) UP(line_bdc, gd->line_bdc, g.n_line) UP(line_pshift, gd->line_pshift, g.n_line)
    UP(line_or_vn, gd->line_or_vn, g.n_line) UP(line_ex_vn, gd->line_ex_vn, g.n_line)
    UP(unit_sub, gd->unit_sub, g.n_unit) UP(unit_pos, gd->unit_pos, g.n_unit) UP(unit_is_ref, gd->unit_is_ref, g.n_unit)
    UP(unit_qmin, gd->unit_qmin, g.n_unit) UP(unit_qmax, gd->unit_qmax, g.n_unit) UP(unit_vn, gd->unit_vn, g.n_unit)
    UP(load_sub, gd->load_sub, g.n_load) UP(load_pos, gd->load_pos, g.n_load) UP(load_vn, gd->load_vn, g.n_load)
    UP(sto_sub, gd->storage_sub, g.n_sto) UP(sto_pos, gd->storage_pos, g.n_sto) UP(sto_vn, gd->storage_vn, g.n_sto)
    UP(sto_q, gd->storage_q, g.n_sto)
    UP(sh_sub, gd->shunt_sub, g.n_shunt) UP(sh_vn, gd->shunt_vn, g.n_shunt) UP(sh_vratio, gd->shunt_vratio, g.n_shunt)
    {   // substation order (bandwidth reduction) and its inverse
        std::vector<int> rank(g.n_sub), order(g.n_sub);
        std::vector<char> seen(g.n_sub, 0);
        bool ok = gd->sub_rank != nullptr;
        for (int s = 0; ok && s < g.n_sub; ++s) {
            const int r = gd->sub_rank[s];
            if (r < 0 || r >= g.n_sub || seen[r]) ok = false; else seen[r] = 1;
        }
        for (int s = 0; s < g.n_sub; ++s) rank[s] = ok ? gd->sub_rank[s] : s;
        for (int s = 0; s < g.n_sub; ++s) order[rank[s]] = s;
        UP(sub_rank, rank.data(), rank.size()) UP(sub_order, order.data(), order.size())
    }
    // static incidence lists: line ends per substation, in line order (deterministic summation order)
    {
        std::vector<int> ptr(g.n_sub + 1, 0), ends(2 * (size_t)g.n_line);
        for (int l = 0; l < g.n_line; ++l) {
            if (gd->line_or_sub[l] < 0 || gd->line_or_sub[l] >= g.n_sub || gd->line_ex_sub[l] < 0 || gd->line_ex_sub[l] >= g.n_sub) {
                b200pf_destroy(h);
                return fail(B200PF_E_ARG, "line substation id out of range");
            }
            ptr[gd->line_or_sub[l] + 1]++; ptr[gd->line_ex_sub[l] + 1]++;
        }
        for (int s = 0; s < g.n_sub; ++s) ptr[s + 1] += ptr[s];
        std::vector<int> fill(ptr.begin(), ptr.end() - 1);
        for (int l = 0; l < g.n_line; ++l) {
            ends[fill[gd->line_or_sub[l]]++] = 2 * l;
            ends[fill[gd->line_ex_sub[l]]++] = 2 * l + 1;
        }
        UP(sub_end_ptr, ptr.data(), ptr.size()) UP(sub_end, ends.data(), ends.size())
    }
#undef UP
    size_t B = (size_t)max_batch;
    auto dmal = [&](void **p, size_t bytes) -> int { CU(cudaMalloc(p, bytes ? bytes : 1)); h->dev_allocs.push_back(*p); return 0; };
    if ((rc = dmal((void **)&h->d_topo, B * g.n_topo_in)) || (rc = dmal((void **)&h->d_inj, B * g.n_inj * 8)) ||
        (rc = dmal((void **)&h->d_out, B * g.n_out * 4)) || (rc = dmal((void **)&h->d_status, B * 4)) ||
        (rc = dmal((void **)&h->d_iters, B * 4)) || (rc = dmal((void **)&h->d_busv, B * 2 * g.n_slot * 8))) {
        b200pf_destroy(h);
        return rc;
    }
    if (cudaMallocHost(&h->h_topo, B * g.n_topo_in + 1) != cudaSuccess || cudaMallocHost(&h->h_inj, B * g.n_inj * 8 + 8) != cudaSuccess ||
        cudaMallocHost(&h->h_out, B * g.n_out * 4 + 4) != cudaSuccess || cudaMallocHost(&h->h_status, B * 4) != cudaSuccess ||
        cudaMallocHost(&h->h_iters, B * 4) != cudaSuccess || cudaMallocHost(&h->h_busv, B * 2 * g.n_slot * 8 + 8) != cudaSuccess) {
        b200pf_destroy(h);
        return fail(B200PF_E_CUDA, "pinned host allocation failed");
    }
    {
        const size_t ncol = 2 * (size_t)g.n_load + 2 * (size_t)g.n_gen;
        if ((rc = dmal((void **)&h->d_rows, B * ncol * 4)) || (rc = dmal((void **)&h->d_static_inj, (size_t)g.n_inj * 8)) ||
            (rc = dmal((void **)&h->d_thlim, (size_t)g.n_line * 4)) || (rc = dmal((void **)&h->d_rho, B * g.n_line * 4))) { b200pf_destroy(h); return rc; }
        if (cudaMallocHost(&h->h_rows, B * ncol * 4 + 4) != cudaSuccess) { b200pf_destroy(h); return fail(B200PF_E_CUDA, "pinned host allocation failed"); }
    }
    {   // host copy of the grid for the plan builder; per-instance plan ids
        HostGrid &hg = h->hg;
        hg.n_sub = g.n_sub; hg.n_busbar = g.n_busbar; hg.n_slot = g.n_slot; hg.n_line = g.n_line; hg.n_gen = g.n_gen; hg.n_hidden = g.n_hidden;
        hg.n_unit = g.n_unit; hg.n_load = g.n_load; hg.n_sto = g.n_sto; hg.n_shunt = g.n_shunt; hg.dim_topo = g.dim_topo;
        hg.n_topo_in = g.n_topo_in; hg.base_mva = g.base_mva;
#define CP(dst, src, n) hg.dst.assign(gd->src, gd->src + (size_t)(n))
        CP(line_or_sub, line_or_sub, g.n_line); CP(line_ex_sub, line_ex_sub, g.n_line); CP(line_or_pos, line_or_pos, g.n_line);
        CP(line_ex_pos, line_ex_pos, g.n_line); CP(line_y, line_y, 8 * g.n_line); CP(line_bdc, line_bdc, g.n_line);
        CP(line_pshift, line_pshift, g.n_line); CP(unit_sub, unit_sub, g.n_unit); CP(unit_pos, unit_pos, g.n_unit);
        CP(unit_is_ref, unit_is_ref, g.n_unit); CP(unit_qmin, unit_qmin, g.n_unit); CP(unit_qmax, unit_qmax, g.n_unit);
        CP(load_sub, load_sub, g.n_load); CP(load_pos, load_pos, g.n_load); CP(sto_sub, storage_sub, g.n_sto);
        CP(sto_pos, storage_pos, g.n_sto); CP(sh_sub, shunt_sub, g.n_shunt);
#undef CP
        if ((rc = dmal((void **)&h->d_inst_plan, B * 4))) { b200pf_destroy(h); return rc; }
        if (cudaMallocHost(&h->h_inst_plan, B * 4 + 4) != cudaSuccess) { b200pf_destroy(h); return fail(B200PF_E_CUDA, "pinned host allocation failed"); }
        const char *pol = getenv("B200PF_PLAN_POLICY");
        if (pol && pol[0] >= '0' && pol[0] <= '2') h->plan_policy = pol[0] - '0';
        // one warp per instance, two for the large grids — and for the mid-size ones when the batch cannot fill the SMs anyway
        // (36 substations: batch 1024 21.4 vs 19.9 M env.step/s with 64 threads, batch 8192 26 vs 35 M/s)
        h->plan_T = g.n_line > 64 ? 64 : ((g.n_line > 32 && max_batch <= 2048) ? 64 : 32);
        const char *mb = getenv("B200PF_SPARSE_MINB");
        if (mb && atoi(mb) == 28) h->sparse_minb = 28;
        const char *capv = getenv("B200PF_SPARSE_CTAS");        // tuning: cap of resident CTAs per SM (planned kernel)
        if (capv) h->sparse_cta_cap = atoi(capv);
        // block kernel: lanes per instance x operations per lane and row (B200PF_BLOCK=0: scalar planned kernel)
        // 8 lanes x 1 operation on the 5 / 14-substation grids; on the 36 / 118-substation grids the scalar planned kernel is the
        // default (scripts/sweep_block.py compares the variants)
        h->blk_T = g.n_line <= 32 ? 8 : (g.n_line <= 64 ? 32 : 64);
        h->blk_U = 1;
        h->blk = g.n_line <= 32 ? 1 : 0;
        const char *bk = getenv("B200PF_BLOCK"), *bt = getenv("B200PF_BLOCK_T"), *bu = getenv("B200PF_BLOCK_U");
        if (bk && bk[0] == '0') h->blk = 0;
        if (bk && bk[0] == '1') h->blk = 1;
        if (bt && bu && block_variant_exists(atoi(bt), atoi(bu))) { h->blk_T = atoi(bt); h->blk_U = atoi(bu); }
        const char *bsp = getenv("B200PF_BLOCK_SPEC");
        if (bsp && bsp[0] == '0') h->blk_spec = 0;
        const char *bun = getenv("B200PF_BLOCK_UNI");
        if (bun && bun[0] == '0') h->blk_uni = 0;
        const char *bw = getenv("B200PF_BLOCK_WPC"), *bs = getenv("B200PF_BLOCK_STAGE");
        if (bw && (atoi(bw) == 1 || atoi(bw) == 2 || atoi(bw) == 4)) { h->blk_wpc = atoi(bw); h->blk_wpc_pinned = 1; }
        if (bs && (bs[0] == '0' || bs[0] == '1')) h->blk_stage = bs[0] - '0';
        const char *nr = getenv("B200PF_NO_REDO");              // measurement only: planned kernel without its safety net
        if (nr && nr[0] == '1') h->redo_enabled = 0;
        const char *var = getenv("B200PF_SPARSE_T");            // tuning: threads per instance of the planned kernel
        if (var) { const int t = atoi(var); if (t == 32 || t == 64 || t == 128) h->plan_T = t; }
    }
    *out = h;
    return 0;
}

extern "C" int b200pf_destroy(b200pf_handle *h) {
    if (!h) return 0;
    cudaSetDevice(h->device);
    if (h->own_stream) cudaStreamSynchronize(h->own_stream);
    for (void *p : h->dev_allocs) cudaFree(p);
    if (h->d_plan_blobs) cudaFree(h->d_plan_blobs);
    if (h->d_plan_off) cudaFree(h->d_plan_off);
    for (auto &kv : h->redo_streams) { if (kv.second.ctl) cudaFree(kv.second.ctl); if (kv.second.mat) cudaFree(kv.second.mat); }
    void *pinned[] = {h->h_topo, h->h_inj, h->h_out, h->h_status, h->h_iters, h->h_busv, h->h_rows, h->h_inst_plan};
    for (void *p : pinned) if (p) cudaFreeHost(p);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    for (auto &cs : h->chunk_stream) if (cs) cudaStreamDestroy(cs);
    for (auto &cs : h->group_stream) if (cs) { cudaStreamSynchronize(cs); cudaStreamDestroy(cs); }
    for (auto &ev : h->group_event) if (ev) cudaEventDestroy(ev);
    if (h->inst_plan_ev) cudaEventDestroy(h->inst_plan_ev);
    h->obs_bufs.release();
    if (h->h_obs_in) cudaFreeHost(h->h_obs_in);
    if (h->obs_ev) cudaEventDestroy(h->obs_ev);
    h->env_bufs.release();
    if (h->h_env_ctl) cudaFreeHost(h->h_env_ctl);
    h->opp_bufs.release();
    h->alert_bufs.release();
    h->alarm_bufs.release();
    h->act_bufs.release();
    h->act_table_bufs.release();
    delete h;
    return 0;
}

extern "C" int b200pf_sizes(const b200pf_handle *h, int *n_topo_in, int *n_inj, int *n_out, int *n_slot) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (n_topo_in) *n_topo_in = h->g.n_topo_in;
    if (n_inj) *n_inj = h->g.n_inj;
    if (n_out) *n_out = h->g.n_out;
    if (n_slot) *n_slot = h->g.n_slot;
    return 0;
}

// Active buses (bus slots with at least one connected element; the count the on-device-topology kernels arrive at, b200pf_kernel.cuh
// step 1) of n topology records: the tight nb_cap of a launch.  Pure host function of the grid description (no device, no handle).
extern "C" int b200pf_grid_max_active_buses(const b200pf_grid_desc *gd, int n, const int8_t *topo, int32_t *per_instance, int32_t *max_out) {
    if (!gd || !max_out || (n > 0 && !topo)) return fail(B200PF_E_ARG, "null pointer");
    if (gd->abi_version != B200PF_ABI_VERSION) return fail(B200PF_E_ARG, "grid description: ABI version mismatch");
    const int nbb = gd->n_busbar, n_unit = gd->n_hidden + gd->n_gen;
    const size_t nt = (size_t)gd->dim_topo + gd->n_shunt + gd->n_hidden;
    if (nbb < 1 || nbb > 8) return fail(B200PF_E_ARG, "1 to 8 busbars per substation");
    // (position in the record, substation) of every element
    std::vector<int> pos, sub;
    auto add = [&](const int32_t *p, const int32_t *s, int cnt, int base) {
        for (int k = 0; k < cnt; ++k) { pos.push_back(p ? p[k] : base + k); sub.push_back(s[k]); }
    };
    add(gd->line_or_pos, gd->line_or_sub, gd->n_line, 0); add(gd->line_ex_pos, gd->line_ex_sub, gd->n_line, 0);
    add(gd->unit_pos, gd->unit_sub, n_unit, 0); add(gd->load_pos, gd->load_sub, gd->n_load, 0);
    add(gd->storage_pos, gd->storage_sub, gd->n_storage, 0); add(nullptr, gd->shunt_sub, gd->n_shunt, gd->dim_topo);
    for (size_t e = 0; e < pos.size(); ++e)
        if (pos[e] < 0 || (size_t)pos[e] >= nt || sub[e] < 0 || sub[e] >= gd->n_sub) return fail(B200PF_E_ARG, "grid description: position / substation out of range");
    std::vector<uint8_t> bars(gd->n_sub);        // bit b-1: busbar b of the substation carries a connected element
    int best = 0;
    const size_t ne = pos.size();
    for (int r = 0; r < n; ++r) {
        const int8_t *tv = topo + (size_t)r * nt;
        std::fill(bars.begin(), bars.end(), (uint8_t)0);
        for (size_t e = 0; e < ne; ++e) {
            const int b = tv[pos[e]];
            if (b > 0 && b <= nbb) bars[sub[e]] |= (uint8_t)(1u << (b - 1));
        }
        int cnt = 0;
        for (int s2 = 0; s2 < gd->n_sub; ++s2) cnt += __builtin_popcount(bars[s2]);
        if (per_instance) per_instance[r] = cnt;
        if (cnt > best) best = cnt;
    }
    *max_out = best;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// launch configuration
// ------------------------------------------------------------------------------------------------
// Raises a kernel's dynamic shared-memory limit to at least `bytes`.  The attribute belongs to the function, not to a handle
// (launches from the device and every other handle see it too), so it is only ever raised: a larger limit never hurts, and
// lowering it would break another handle's launch of a larger workspace.  The record of what was set is per device and
// kernel and shared by all handles: setting the attribute on every launch kept the GPU waiting for the host between steps.
static int raise_smem_limit(const b200pf_handle *h, const void *kern, int bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, int> done;   // (device, kernel) -> largest limit set
    std::lock_guard<std::mutex> lock(mu);
    int &cur = done[{h->device, kern}];
    if (bytes > cur) {
        CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        cur = bytes;
    }
    return 0;
}

// Grid of a persistent launch over `work` items (instances, or CTAs' worth of them) with `resident` CTAs on the device at
// once, sized so that every CTA gets the same number of items (no ragged last wave): rounds = ceil(work / resident),
// grid = ceil(work / rounds)
static int balanced_grid(int work, int resident) {
    const int rounds = (work + resident - 1) / resident;
    const int grid = rounds > 0 ? (work + rounds - 1) / rounds : 1;
    return grid < 1 ? 1 : grid;
}

// Bookkeeping of the launch just issued (b200pf_launch_count, b200pf_plan_stats, b200pf_last_launch_info), with its
// template parameters in the order of b200pf_last_launch_config (missing ones: -1).  Returns the launch error, if any.
static int launched(b200pf_handle *h, LaunchKind kind, int smem, int T, int grid, int block, std::initializer_list<int> cfg = {}) {
    CU(cudaGetLastError());
    h->launches++;
    h->last_kernel = kind; h->last_smem = smem; h->last_T = T; h->last_grid = grid; h->last_block = block;
    int k = 0;
    for (int v : cfg) h->last_cfg[k++] = v;
    for (; k < 8; ++k) h->last_cfg[k] = -1;
    return 0;
}

// threads per instance of the pivoting kernels for a Newton system of dimension d: the big systems are latency bound -> many
// warps per instance
static int pivot_threads(size_t d) { return d <= 64 ? 32 : (d <= 128 ? 128 : (d <= 256 ? 256 : 512)); }

// The warp-per-instance kernel (b200pf_small.cuh) takes a launch when every element class fits one warp and at most `cap`
// <= 17 buses are active (a Newton system of <= 32 unknowns)
static bool warp_kernel_fits(const DevGrid &g, int cap) {
    return g.n_slot <= 32 && g.n_line <= 32 && g.n_unit <= 32 && g.n_load <= 32 && g.n_sto <= 32 && g.n_shunt <= 32 && cap <= 17;
}

template <int T>
static int launch_t(b200pf_handle *h, const RunArgs &a) {
    const DevGrid &g = h->g;
    WsLayout L = ws_layout(a.nb_cap, g.n_slot, g.n_line, g.n_inj, (size_t)a.mat_bytes);
    const int smem = (int)L.total;
    if (L.total > (size_t)h->max_smem_optin)
        return fail(B200PF_E_CAPACITY, "workspace does not fit in shared memory");
    auto kern = pf_kernel<T, float>;
    int rc = raise_smem_limit(h, (const void *)kern, smem);
    if (rc) return rc;
    int occ = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, T, (size_t)smem));
    if (occ < 1) occ = 1;
    const int grid = balanced_grid(a.batch, h->sm_count * occ);
    kern<<<grid, T, (size_t)smem, h->stream>>>(g, a, smem);
    return launched(h, KERN_CTA_PIVOTING, smem, T, grid, T);
}

// Sizing policy.  nb_cap (bus arrays) = the caller's bound or every slot.  The matrix region gets
// what the worst case of nb_cap buses needs, clipped to what is left on chip; the kernel checks the
// ACTUAL system size of each instance against it (B200PF_ST_TOO_LARGE), so e.g. the 118-substation
// grid (236 slots) runs as long as its Newton system (191 unknowns + splits) fits.
static int launch_small(b200pf_handle *h, RunArgs a, int cap) {
    a.nb_cap = cap;
    SmallLayout L = small_layout(cap);
    a.mat_bytes = L.total - L.off_mat;
    auto kern = a.prot ? pf_kernel_small<true> : pf_kernel_small<false>;
    int &occ = h->small_occ[a.prot ? 1 : 0][cap];          // launch configuration cached per (variant, capacity)
    if (occ == 0) {
        int rc = raise_smem_limit(h, (const void *)kern, L.total);
        if (rc) return rc;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 32, (size_t)L.total));
        if (occ < 1) occ = 1;
    }
    const int grid = balanced_grid(a.batch, h->sm_count * occ);
    kern<<<grid, 32, L.total, h->stream>>>(h->g, a, L);
    return launched(h, KERN_WARP_PIVOTING, L.total, 32, grid, 32);
}

// ------------------------------------------------------------------------------------------------
// topology plans of the sparse kernel (b200pf_plan.hpp): cache keyed by the topology bytes
// ------------------------------------------------------------------------------------------------
static const int PLAN_MAX = 32768;          // plans kept per handle
static const size_t PLAN_MAX_BYTES = size_t(1) << 30;   // ... and their total size (host copy + device copy each)
static const int PLAN_BUILD_BUDGET = 512;   // new plans one call may build in automatic mode before it falls back

struct PlanSel {
    const int *d_inst_plan;   // device, per instance of the launch; nullptr = every instance uses plan `single`
    int single;
    int smem;                 // per-instance workspace bytes the launch must provide
    int lay_nb = 0, lay_nblkA = 0;   // block kernel: layout strides of the launch (one plan: its sizes; several: the handle's maxima)
};

// plan builder of the handle's kernel family (scalar stream laid out for plan_T threads, or block stream for blk_T x blk_U)
static PlanBuilder make_builder(const b200pf_handle *h, bool optimize_layout = false, int seed = 0) {
    PlanBuilder pb(h->hg, h->plan_T, optimize_layout && !h->blk, seed);
    if (h->blk) pb.block_mode(h->blk_T, h->blk_U);
    return pb;
}
static inline int blk_G(const b200pf_handle *h) { return (h->blk && h->blk_T < 32) ? 32 / h->blk_T : 1; }

// workspace bytes + layout strides of a launch: one plan -> that plan's; several -> the maxima over the cached plans
static void sel_layout(const b200pf_handle *h, PlanSel *sel, bool single) {
    const DevGrid &g = h->g;
    if (single) {
        const PlanHeader *H = reinterpret_cast<const PlanHeader *>(h->plan_blobs.data() + h->plan_off[sel->single]);
        sel->smem = h->plan_smem[sel->single]; sel->lay_nb = H->nb; sel->lay_nblkA = H->nblkA;
    } else if (h->blk) {
        sel->lay_nb = h->plan_max_nb; sel->lay_nblkA = h->plan_max_nblkA;
        sel->smem = plan_block_smem_bytes(h->plan_max_nb, g.n_line, h->plan_max_nblkA, 2 * g.n_load + 2 * g.n_gen, g.n_shunt);
        if (sel->smem < h->plan_max_smem) sel->smem = h->plan_max_smem;
    } else sel->smem = h->plan_max_smem;
}

// 64-bit hash of a topology row (8 bytes at a time)
static inline uint64_t topo_hash(const int8_t *tv, size_t n) {
    uint64_t hsh = 0x9E3779B97F4A7C15ull ^ (uint64_t)n;
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, tv + i, 8);
        hsh = (hsh ^ w) * 0xFF51AFD7ED558CCDull;
        hsh ^= hsh >> 29;
    }
    uint64_t w = 0;
    if (i < n) memcpy(&w, tv + i, n - i);
    hsh = (hsh ^ w) * 0xC4CEB9FE1A85EC53ull;
    hsh ^= hsh >> 32;
    return hsh;
}

static inline uint64_t plan_key(uint64_t row_hash, int outage) { return row_hash ^ ((uint64_t)(outage + 1) * 0x9E3779B97F4A7C15ull); }

// cached plan of (topology row, outage), or -1
static int plan_find(const b200pf_handle *h, const int8_t *tv, uint64_t row_hash, int outage) {
    const size_t nt = (size_t)h->g.n_topo_in;
    auto it = h->plan_index.find(plan_key(row_hash, outage));
    if (it == h->plan_index.end()) return -1;
    for (int id = it->second; id >= 0; id = h->plan_next[id])
        if (h->plan_outage[id] == outage && memcmp(h->plan_keys.data() + (size_t)id * nt, tv, nt) == 0) return id;
    return -1;
}

// appends a freshly built plan to the cache; -1 when it cannot be used (does not fit the format / the shared memory)
static int plan_insert(b200pf_handle *h, const int8_t *tv, uint64_t row_hash, int outage, const std::vector<unsigned char> &blob) {
    const size_t nt = (size_t)h->g.n_topo_in;
    const PlanHeader *H = reinterpret_cast<const PlanHeader *>(blob.data());
    if ((int)h->plan_off.size() >= PLAN_MAX || h->plan_blobs.size() + blob.size() > PLAN_MAX_BYTES || !PlanBuilder::fits(*H) ||
        (long)H->smem_bytes * blk_G(h) > (long)h->max_smem_optin)
        return -1;      // the caller falls back to the pivoting kernels
    const uint64_t key = plan_key(row_hash, outage);
    auto it = h->plan_index.find(key);
    const int id = (int)h->plan_off.size();
    h->plan_off.push_back((int)h->plan_blobs.size());
    h->plan_smem.push_back(H->smem_bytes);
    h->plan_blobs.insert(h->plan_blobs.end(), blob.begin(), blob.end());
    while (h->plan_blobs.size() % 16) h->plan_blobs.push_back(0);
    h->plan_keys.insert(h->plan_keys.end(), tv, tv + nt);
    h->plan_outage.push_back(outage);
    h->plan_next.push_back(it != h->plan_index.end() ? it->second : -1);
    h->plan_index[key] = id;
    if (H->smem_bytes > h->plan_max_smem) h->plan_max_smem = H->smem_bytes;
    if (H->nb > h->plan_max_nb) h->plan_max_nb = H->nb;
    if (H->nblkA > h->plan_max_nblkA) h->plan_max_nblkA = H->nblkA;
    h->plans_built++;
    return id;
}

// device copy of the plans built since the last call.  The copies are issued on the launching stream and the stream is
// drained before returning: the sources are pageable host vectors (a plain cudaMemcpy may return before its DMA has
// finished, and the handle's non-blocking streams are not ordered against the legacy stream), and a plan must be visible
// to every stream of the handle.  Building a plan is a rare event (a new topology), the wait is noise next to it.
static int plans_sync_device(b200pf_handle *h, cudaStream_t st) {
    if (h->d_plan_used == h->plan_blobs.size() && h->d_plan_off_n == (int)h->plan_off.size()) return 0;
    if (h->plan_blobs.size() > h->d_plan_cap) {
        CU(cudaDeviceSynchronize());                       // launches in flight may still read the old buffer
        if (h->d_plan_blobs) CU(cudaFree(h->d_plan_blobs));
        h->d_plan_blobs = nullptr; h->d_plan_used = 0;
        size_t cap = h->plan_blobs.size() * 2;
        if (cap < (size_t(1) << 20)) cap = size_t(1) << 20;
        CU(cudaMalloc(&h->d_plan_blobs, cap));
        h->d_plan_cap = cap;
    }
    if (!h->d_plan_off) CU(cudaMalloc(&h->d_plan_off, (size_t)PLAN_MAX * 4));
    CU(cudaMemcpyAsync(h->d_plan_blobs + h->d_plan_used, h->plan_blobs.data() + h->d_plan_used, h->plan_blobs.size() - h->d_plan_used,
                       cudaMemcpyHostToDevice, st));
    h->d_plan_used = h->plan_blobs.size();
    CU(cudaMemcpyAsync(h->d_plan_off + h->d_plan_off_n, h->plan_off.data() + h->d_plan_off_n,
                       (h->plan_off.size() - (size_t)h->d_plan_off_n) * 4, cudaMemcpyHostToDevice, st));
    h->d_plan_off_n = (int)h->plan_off.size();
    CU(cudaStreamSynchronize(st));
    return 0;
}

// Drops every cached plan (host + device copy).  Plan ids handed out before are void afterwards: the series mode re-resolves
// its ids before its next step (series_plans_stale).  Launches in flight may still read the device copy -> device-wide sync.
static int plan_cache_clear(b200pf_handle *h) {
    CU(cudaDeviceSynchronize());
    h->plan_index.clear(); h->plan_keys.clear(); h->plan_outage.clear(); h->plan_next.clear();
    h->plan_off.clear(); h->plan_smem.clear(); h->plan_blobs.clear();
    h->d_plan_used = 0; h->d_plan_off_n = 0; h->plan_max_smem = 0; h->plan_max_nb = 0; h->plan_max_nblkA = 0;
    h->plan_cache_resets++;
    if (h->series_plan_state) h->series_plans_stale = true;
    return 0;
}

// Plans of the instances [0, n_src) whose topology rows are at host_topo (times n1_lines outages each in contingency
// mode); ids go to h_inst_plan[first ...] and, unless all are equal, to d_inst_plan[first ...] on stream st.
// Returns 1 = use the sparse kernel with *sel, 0 = fall back to the pivoting kernels, < 0 error.
static int plan_select(b200pf_handle *h, const int8_t *host_topo, int n_src, int n1_lines, int first, cudaStream_t st, PlanSel *sel) {
    if (h->plan_policy == 1 || !host_topo) return 0;
    const DevGrid &g = h->g;
    const size_t nt = (size_t)g.n_topo_in;
    const int per = n1_lines > 0 ? n1_lines : 1;
    if (h->inst_plan_pending) { CU(cudaEventSynchronize(h->inst_plan_ev)); h->inst_plan_pending = false; }
    int *ids = h->h_inst_plan + first;
    // pass 1: cached plans; the misses of this call are collected (once each) ...
    struct Miss { const int8_t *tv; uint64_t rh; int outage; int id; };
    std::vector<Miss> miss;
    std::unordered_map<uint64_t, std::vector<int>> miss_index;
    for (int attempt = 0; attempt < 2; ++attempt) {
        miss.clear(); miss_index.clear();
        for (int s = 0; s < n_src; ++s) {
            const int8_t *tv = host_topo + (size_t)s * nt;
            if (s > 0 && memcmp(tv, tv - nt, nt) == 0) {
                for (int l = 0; l < per; ++l) ids[(size_t)s * per + l] = ids[(size_t)(s - 1) * per + l];
                continue;
            }
            const uint64_t rh = topo_hash(tv, nt);
            for (int l = 0; l < per; ++l) {
                const int outage = n1_lines > 0 ? l : -1;
                int id = plan_find(h, tv, rh, outage);
                if (attempt == 0) { h->plan_lookups++; if (id >= 0) h->plan_hits++; }
                if (id < 0) {
                    std::vector<int> &cand = miss_index[plan_key(rh, outage)];
                    int m = -1;
                    for (int c : cand) if (miss[c].outage == outage && memcmp(miss[c].tv, tv, nt) == 0) { m = c; break; }
                    if (m < 0) { m = (int)miss.size(); miss.push_back({tv, rh, outage, -1}); cand.push_back(m); }
                    id = -2 - m;                      // placeholder, resolved below
                }
                ids[(size_t)s * per + l] = id;
            }
        }
        // the cache is a plain append-only store: when this call's new plans would overflow it, start over with an empty one
        // (agents that walk through ever new topologies — BASELINE configs[2] — fill any cache)
        const size_t avg = h->plan_off.empty() ? (size_t)64 * 1024 : h->plan_blobs.size() / h->plan_off.size() + 1;
        const bool overflow = h->plan_off.size() + miss.size() > (size_t)PLAN_MAX || h->plan_blobs.size() + miss.size() * avg > PLAN_MAX_BYTES;
        if (!overflow || attempt == 1 || h->plan_off.empty()) break;
        int rc = plan_cache_clear(h);
        if (rc) return rc;
    }
    // ... built in parallel on the host threads (the builder is pure), inserted in order
    if (!miss.empty()) {
        // automatic mode: planning pays when plans are re-used.  A call that would have to plan more than an eighth of its
        // instances from scratch (agents walking through ever new topologies) runs on the pivoting kernels, which discover the
        // topology on the device (scripts/bench_config3.py: 36 substations, batch 1024, one random substation change per
        // instance and step)
        if (h->plan_policy == 0 && ((int)miss.size() > PLAN_BUILD_BUDGET || (n_src >= 64 && miss.size() * 8 > (size_t)n_src * per))) return 0;
        std::vector<std::vector<unsigned char>> blobs(miss.size());
        // a handful of new plans of a batched launch: they will be re-used by many solves (rollouts, N-1 sweeps) -> searched
        // elimination order + bank-conflict-optimised layout (not for single environments: there the build time of a new
        // topology is part of the step latency; not for bulk builds)
        const bool searched = miss.size() <= 32 && (size_t)n_src * per >= 256;
        const int n_seeds = h->g.n_slot <= 128 ? 12 : 4;
        const PlanBuilder pb = make_builder(h);
        auto build_one = [&](size_t m) {
            blobs[m] = searched ? build_plan_searched(h->hg, h->plan_T, miss[m].tv, miss[m].outage, n_seeds, h->blk ? h->blk_T : 0, h->blk_U)
                                : pb.build(miss[m].tv, miss[m].outage);
        };
        unsigned nthr = std::thread::hardware_concurrency();
        if (nthr > 64) nthr = 64;
        {   // containers: a cgroup CPU quota below the visible CPUs (the GPU boxes: 128 visible, quota 16) — more threads only thrash
            static int quota = -1;
            if (quota < 0) {
                quota = 0;
                if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
                    char q[32] = {0}; long per = 0;
                    if (fscanf(f, "%31s %ld", q, &per) == 2 && q[0] != 'm' && per > 0) quota = (int)((atol(q) + per - 1) / per);
                    fclose(f);
                }
            }
            if (quota > 0 && (unsigned)quota < nthr) nthr = (unsigned)quota;
        }
        {   // (a cgroup CPU quota smaller than the visible CPUs: B200PF_PLAN_THREADS caps the builder threads)
            const char *pt = getenv("B200PF_PLAN_THREADS");
            if (pt && atoi(pt) > 0 && (unsigned)atoi(pt) < nthr) nthr = (unsigned)atoi(pt);
        }
        if (nthr < 1) nthr = 1;
        if ((size_t)nthr > miss.size() / 4 + 1) nthr = (unsigned)(miss.size() / 4 + 1);
        if (nthr <= 1) {
            for (size_t m = 0; m < miss.size(); ++m) build_one(m);
        } else {
            std::vector<std::thread> pool;
            for (unsigned t = 0; t < nthr; ++t)
                pool.emplace_back([&, t]() { for (size_t m = t; m < miss.size(); m += nthr) build_one(m); });
            for (auto &th : pool) th.join();
        }
        for (size_t m = 0; m < miss.size(); ++m) {
            miss[m].id = plan_insert(h, miss[m].tv, miss[m].rh, miss[m].outage, blobs[m]);
            if (miss[m].id < 0) { int rc = plans_sync_device(h, st); return rc ? rc : 0; }
        }
        const size_t n = (size_t)n_src * per;
        for (size_t k = 0; k < n; ++k) if (ids[k] <= -2) ids[k] = miss[(size_t)(-2 - ids[k])].id;
    }
    int rc = plans_sync_device(h, st);
    if (rc) return rc;
    const size_t n = (size_t)n_src * per;
    bool single = true;
    for (size_t k = 1; k < n && single; ++k) single = ids[k] == ids[0];
    sel->single = ids[0]; sel->d_inst_plan = nullptr;
    sel_layout(h, sel, single);
    if (!single) {
        CU(cudaMemcpyAsync(h->d_inst_plan + first, ids, n * 4, cudaMemcpyHostToDevice, st));
        if (!h->inst_plan_ev) CU(cudaEventCreateWithFlags(&h->inst_plan_ev, cudaEventDisableTiming));
        CU(cudaEventRecord(h->inst_plan_ev, st));          // the next call waits for this copy before it reuses h_inst_plan
        h->inst_plan_pending = true;
        sel->d_inst_plan = h->d_inst_plan + first;
    }
    return 1;
}

// Resident CTAs per SM of a planned kernel (scalar or block) with `smem` bytes of dynamic shared memory per CTA, in
// h->sparse_occ.  One entry per handle, re-queried when the kernel or the workspace changes: the carveout set here changes
// what the next query returns.  `smem_limit` is the kernel's dynamic shared-memory limit; auto_cap lets a large workspace cap
// the resident CTAs by itself.
static int planned_occupancy(b200pf_handle *h, const void *kern, int block, int smem, int smem_limit, bool auto_cap) {
    if (h->sparse_occ_kern == kern && h->sparse_occ_smem == smem) return 0;
    int rc = raise_smem_limit(h, kern, smem_limit);
    if (rc) return rc;
    int occ = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, block, (size_t)smem));
    if (occ < 1) occ = 1;
    int cap = h->sparse_cta_cap;
    if (cap == 0 && auto_cap && smem >= 16 * 1024) cap = (164 * 1024) / (smem + 1024);   // large workspaces (118 substations): leave ~90 KB of L1 (measured +10%)
    if (cap > 0 && occ > cap) {
        // fewer resident instances, more L1: the plan arrays (operation stream, positions, line data) are re-read by
        // every instance and every Newton iteration; what shared memory does not take is L1 for them
        occ = cap;
        int pct = (int)(((size_t)occ * (size_t)(smem + 1024) * 100 + (size_t)h->max_smem_optin - 1) / (size_t)h->max_smem_optin);
        if (pct > 100) pct = 100;
        CU(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    }
    h->sparse_occ = occ; h->sparse_occ_kern = kern; h->sparse_occ_smem = smem;
    return 0;
}

template <int T, int MINB, bool PROT = false>
static int launch_sparse_t(b200pf_handle *h, const RunArgs &a, const PlanSel &sel, const RedoDesc &rd) {
    auto kern = pf_kernel_sparse<T, MINB, PROT>;
    const int smem = sel.smem;
    int rc = planned_occupancy(h, (const void *)kern, T, smem, h->max_smem_optin, true);
    if (rc) return rc;
    PlanArgs pa{};
    pa.blobs = h->d_plan_blobs;
    pa.plan_off = h->d_plan_off + (sel.d_inst_plan ? 0 : sel.single);
    pa.inst_plan = sel.d_inst_plan;
    pa.lay_nb = 0; pa.lay_nblkA = 0;
    const int grid = balanced_grid(a.batch, h->sm_count * h->sparse_occ);
    kern<<<grid, T, (size_t)smem, h->stream>>>(h->g, a, pa, rd);
    return launched(h, KERN_PLANNED_SPARSE, smem, T, grid, T, {T, -1, MINB, PROT ? 1 : 0});
}

// Threads per instance (fixed per handle: the plans' operation streams are laid out for it) and register budget of the
// planned kernel: one warp per instance for the 5/14/36-substation grids, with as many one-warp CTAs per SM as the
// workspace allows (up to the hardware's 32); two warps per instance for the large grids (118 substations, ~22 KB of
// workspace per instance limit an SM to ~10 instances: the second warp doubles the warps in flight).
static int launch_block(b200pf_handle *h, const RunArgs &a, const PlanSel &sel, const RedoDesc &rd);
static int launch_sparse(b200pf_handle *h, const RunArgs &a, const PlanSel &sel, const RedoDesc &rd) {
    if (h->blk) return launch_block(h, a, sel, rd);
    const int per_sm = h->max_smem_optin / (sel.smem + 1024);
    if (a.prot) {     // protections: one launch per cascade round, see series_step_planned_prot
        if (h->plan_T == 128) return launch_sparse_t<128, 4, true>(h, a, sel, rd);
        if (h->plan_T == 64) return launch_sparse_t<64, 10, true>(h, a, sel, rd);
        return launch_sparse_t<32, 16, true>(h, a, sel, rd);
    }
    if (h->plan_T == 128) return launch_sparse_t<128, 4>(h, a, sel, rd);
    if (h->plan_T == 64) return launch_sparse_t<64, 10>(h, a, sel, rd);
    if (per_sm >= 32 && h->sparse_minb == 28) return launch_sparse_t<32, 28>(h, a, sel, rd);   // 73 registers, 4144 resident warps
    if (per_sm >= 32) return launch_sparse_t<32, 32>(h, a, sel, rd);
    if (per_sm >= 24) return launch_sparse_t<32, 24>(h, a, sel, rd);
    if (per_sm >= 16) return launch_sparse_t<32, 16>(h, a, sel, rd);
    return launch_sparse_t<32, 8>(h, a, sel, rd);
}

// Sizing of the generic pivoting kernel for nb_cap active buses: threads per instance, matrix bytes (see the policy above
// launch_small).  jt = bytes of a Jacobian entry.  Returns 0, or an error when not even a clipped matrix fits.
static int generic_config(b200pf_handle *h, int cap, int jt, int *T_out, size_t *want_out) {
    const DevGrid &g = h->g;
    const size_t fixed = ws_fixed_bytes(cap, g.n_slot, g.n_line, g.n_inj);
    size_t want = ws_mat_worst(cap, jt);
    int T = pivot_threads(2 * (size_t)cap);
    if (fixed + want > (size_t)h->max_smem_optin) {
        // does not fit with the worst case: clipped matrix (the kernel checks the ACTUAL system of every instance against it)
        if (fixed + 1024 > (size_t)h->max_smem_optin) return fail(B200PF_E_CAPACITY, "grid too large for the on-chip workspace");
        size_t avail = ((size_t)h->max_smem_optin - fixed) & ~size_t(15);
        if (want > avail) want = avail;
        size_t dmax = 1;
        while ((dmax + 1) * (dmax + 3) * jt <= want) ++dmax;
        T = dmax <= 128 ? 128 : (dmax <= 256 ? 256 : 512);
    }
    *T_out = T; *want_out = want;
    return 0;
}

// Safety net of a planned launch (b200pf_redo.cuh): the configuration of the pivoting re-solve the planned kernel tail-launches
// when one of its instances ends as ST_DIV (RedoDesc).  fp64 Jacobian whenever the actual systems fit the workspace with it
// (5 / 14 / 36 substations), in global memory otherwise (118 substations).
static int redo_config(b200pf_handle *h, const RunArgs &a, int nb_cap_req, RedoDesc *rd) {
    *rd = RedoDesc{};
    if (!h->redo_enabled || a.is_dc || !a.topo) return 0;     // (the DC solve is a product with the plan's inverse: nothing to pivot)
    const DevGrid &g = h->g;
    int cap = nb_cap_req;
    if (cap <= 0 || cap > g.n_slot) cap = g.n_slot;
    b200pf_handle::RedoStream &rs = h->redo_streams[h->stream];
    if (!rs.ctl) {
        CU(cudaMalloc(&rs.ctl, sizeof(RedoCtl)));
        CU(cudaMemsetAsync(rs.ctl, 0, sizeof(RedoCtl), h->stream));
    }
    // always an fp64 Jacobian with partial pivoting, like the reference's solver.  Where the worst-case system (every bus slot
    // active) fits the shared-memory workspace it lives there; on the large grids (118 substations: 472 x 474 x 8 B) every
    // CTA of the launch gets a matrix in global memory instead
    int T = 32;
    size_t want = 0;
    const size_t fixed = ws_fixed_bytes(cap, g.n_slot, g.n_line, g.n_inj);
    const size_t worst = ws_mat_worst(cap, 8);
    int max_ctas = h->sm_count * 8;
    if (fixed + worst > (size_t)h->max_smem_optin) {
        // (the handle's main stream gets one matrix per SM; the chunk / group streams a smaller set each: the path is rare)
        max_ctas = h->on_side_stream ? 32 : h->sm_count;
        if (!rs.mat || rs.stride < worst || rs.ctas < max_ctas) {
            CU(cudaStreamSynchronize(h->stream));
            if (rs.mat) CU(cudaFree(rs.mat));
            rs.mat = nullptr;
            CU(cudaMalloc(&rs.mat, worst * (size_t)max_ctas));
            rs.stride = worst; rs.ctas = max_ctas;
        }
        rd->mat = rs.mat; rd->mat_stride = rs.stride;
        want = worst;
        T = pivot_threads(2 * (size_t)cap);
    } else {
        int rc = generic_config(h, cap, 8, &T, &want);
        if (rc) return rc;
    }
    rd->T = T; rd->nb_cap = cap; rd->mat_bytes = (int)want; rd->ctl = rs.ctl;
    rd->grid = (a.batch + 31) / 32;
    if (rd->grid > max_ctas) rd->grid = max_ctas;
    if (rd->grid < 1) rd->grid = 1;
    // (matrix in global memory: the shared-memory workspace only holds the bus arrays)
    WsLayout L = ws_layout(cap, g.n_slot, g.n_line, g.n_inj, rd->mat ? (size_t)16 : want);
    if (L.total > (size_t)h->max_smem_optin) return fail(B200PF_E_CAPACITY, "workspace does not fit in shared memory");
    rd->smem = (int)L.total;
    const void *kern;
    switch (T) {
        case 32: kern = (const void *)pf_kernel_redo<32, double>; break;
        case 128: kern = (const void *)pf_kernel_redo<128, double>; break;
        case 256: kern = (const void *)pf_kernel_redo<256, double>; break;
        default: kern = (const void *)pf_kernel_redo<512, double>; break;
    }
    int rc = raise_smem_limit(h, kern, rd->smem);
    if (rc) return rc;
    rd->on = 1;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// block-planned kernel (b200pf_block.cuh)
// ------------------------------------------------------------------------------------------------
// One device blob with the static arrays a staged block launch reads (D2D copies of the handle's own arrays; rebuilt when the
// static injections / thermal limits change).  Every section 16-byte aligned (bulk copy + vector loads).
static int stat_sync(b200pf_handle *h) {
    if (h->d_stat && !h->stat_dirty) return 0;
    const DevGrid &g = h->g;
    PlanArgs::StatOff &o = h->stat_off;
    size_t off = 0;
    auto sec = [&](int *field, size_t bytes) { *field = (int)off; off += (bytes + 15) & ~size_t(15); };
    sec(&o.line_y, (size_t)g.n_line * 64); sec(&o.line_bdc, (size_t)g.n_line * 8); sec(&o.line_pshift, (size_t)g.n_line * 8);
    sec(&o.line_or_vn, (size_t)g.n_line * 4); sec(&o.line_ex_vn, (size_t)g.n_line * 4); sec(&o.unit_is_ref, (size_t)g.n_unit * 4);
    sec(&o.unit_qmin, (size_t)g.n_unit * 8); sec(&o.unit_qmax, (size_t)g.n_unit * 8); sec(&o.unit_vn, (size_t)g.n_unit * 4);
    sec(&o.load_vn, (size_t)g.n_load * 4); sec(&o.sto_vn, (size_t)g.n_sto * 4); sec(&o.sto_q, (size_t)g.n_sto * 8);
    sec(&o.sh_vn, (size_t)g.n_shunt * 4); sec(&o.sh_vratio, (size_t)g.n_shunt * 8); sec(&o.static_inj, (size_t)g.n_inj * 8);
    sec(&o.th_lim, (size_t)g.n_line * 4);
    o.total = (int)off;
    if (!h->d_stat) { CU(cudaMalloc(&h->d_stat, off)); h->dev_allocs.push_back(h->d_stat); CU(cudaMemsetAsync(h->d_stat, 0, off, h->stream)); }
    cudaStream_t st = h->stream;
#define CPY(field, src, bytes) if ((bytes) > 0) CU(cudaMemcpyAsync(h->d_stat + o.field, (src), (bytes), cudaMemcpyDeviceToDevice, st));
    CPY(line_y, g.line_y, (size_t)g.n_line * 64) CPY(line_bdc, g.line_bdc, (size_t)g.n_line * 8) CPY(line_pshift, g.line_pshift, (size_t)g.n_line * 8)
    CPY(line_or_vn, g.line_or_vn, (size_t)g.n_line * 4) CPY(line_ex_vn, g.line_ex_vn, (size_t)g.n_line * 4) CPY(unit_is_ref, g.unit_is_ref, (size_t)g.n_unit * 4)
    CPY(unit_qmin, g.unit_qmin, (size_t)g.n_unit * 8) CPY(unit_qmax, g.unit_qmax, (size_t)g.n_unit * 8) CPY(unit_vn, g.unit_vn, (size_t)g.n_unit * 4)
    CPY(load_vn, g.load_vn, (size_t)g.n_load * 4) CPY(sto_vn, g.sto_vn, (size_t)g.n_sto * 4) CPY(sto_q, g.sto_q, (size_t)g.n_sto * 8)
    CPY(sh_vn, g.sh_vn, (size_t)g.n_shunt * 4) CPY(sh_vratio, g.sh_vratio, (size_t)g.n_shunt * 8)
    CPY(static_inj, h->d_static_inj, (size_t)g.n_inj * 8) CPY(th_lim, h->d_thlim, (size_t)g.n_line * 4)
#undef CPY
    CU(cudaStreamSynchronize(st));      // rare (first launch, new static injections / limits); every stream of the handle reads the blob afterwards
    h->stat_dirty = false;
    return 0;
}

template <int T, int U, int MINB, bool PROT, int WPC = 1, bool STAGE = false, bool UNI = false, int MODE = 0>
static int launch_block_t(b200pf_handle *h, const RunArgs &a, const PlanSel &sel, const RedoDesc &rd) {
    constexpr int G = T < 32 ? 32 / T : 1;
    constexpr int BLOCK = (T < 32 ? 32 : T) * WPC;
    auto kern = pf_kernel_block<T, U, MINB, PROT, WPC, STAGE, UNI, MODE>;
    const int ws = sel.smem * G;                         // workspace of one warp / CTA
    int plan_bytes = 0, row_ahead = 0;
    const unsigned char *plan_src = nullptr;
    if (STAGE) {
        // (the kernel starts the plan's bulk copy from its address and, for a solvable plan, loads the chronics rows meanwhile)
        const PlanHeader *H = reinterpret_cast<const PlanHeader *>(h->plan_blobs.data() + h->plan_off[sel.single]);
        plan_bytes = H->total_bytes;
        plan_src = h->d_plan_blobs + h->plan_off[sel.single];
        row_ahead = H->status == PLAN_ST_OK;        // (one plan: sel.lay_nb / lay_nblkA are its sizes, sel_layout)
    }
    if (STAGE) { int rc = stat_sync(h); if (rc) return rc; }
    const int smem = ws * WPC + plan_bytes + (STAGE ? h->stat_off.total : 0);
    // (the staged variant owns a few bytes of static shared memory: dynamic + static must stay within the opt-in limit)
    int rc = planned_occupancy(h, (const void *)kern, BLOCK, smem, h->max_smem_optin - 256, G == 1);
    if (rc) return rc;
    PlanArgs pa{};
    pa.blobs = h->d_plan_blobs;
    pa.plan_off = h->d_plan_off + (sel.d_inst_plan ? 0 : sel.single);
    pa.inst_plan = sel.d_inst_plan;
    pa.lay_nb = sel.lay_nb; pa.lay_nblkA = sel.lay_nblkA;
    pa.stat = STAGE ? h->d_stat : nullptr; pa.so = h->stat_off;
    const int n_cta_work = ((a.batch + G - 1) / G + WPC - 1) / WPC;
    const int grid = balanced_grid(n_cta_work, h->sm_count * h->sparse_occ);
    kern<<<grid, BLOCK, (size_t)smem, h->stream>>>(h->g, a, pa, ws, plan_bytes, plan_src, row_ahead, rd);
    return launched(h, KERN_PLANNED_BLOCK, smem, T, grid, BLOCK, {T, U, MINB, PROT ? 1 : 0, WPC, STAGE ? 1 : 0, UNI ? 1 : 0, MODE});
}

// compiled (lanes, operations per lane and row) variants; U > 1 and 2 lanes per instance were slower in variant sweeps
// (scripts/sweep_block.py), so they are not built
#define B200PF_BLOCK_VARIANTS(X) X(4, 1) X(4, 2) X(8, 1) X(16, 1) X(32, 1) X(64, 1)
static bool block_variant_exists(int T, int U) {
#define X(t, u) if (T == t && U == u) return true;
    B200PF_BLOCK_VARIANTS(X)
#undef X
    return false;
}

static int launch_block(b200pf_handle *h, const RunArgs &a, const PlanSel &sel, const RedoDesc &rd) {
    const int T = h->blk_T, U = h->blk_U;
    // Shared-plan launches of the default (8 x 1) variant: CTAs of WPC warps that fetch the plan ONCE into shared memory with a bulk
    // asynchronous copy (TMA) and run in lockstep (DESIGN.md 4.2).  Knobs to compare: B200PF_BLOCK_STAGE=0 (plan through L1), B200PF_BLOCK_WPC=1/2/4, B200PF_BLOCK_UNI=0.
    if (!a.prot && T == 8 && U == 1 && !sel.d_inst_plan && h->blk_stage && a.batch % 4 == 0 &&
        reinterpret_cast<const PlanHeader *>(h->plan_blobs.data() + h->plan_off[sel.single])->total_bytes <= 32 * 1024) {
        if (h->blk_uni) {
            // warps per CTA: 2 up to 32 k instances (finer SM balance: 167 vs 158 M/s at batch 16 384), 4 beyond (197 vs 189 M/s at
            // 65 536: one staged copy serves more instances); B200PF_BLOCK_WPC pins it
            const int wpc = h->blk_wpc_pinned ? h->blk_wpc : (a.batch <= 32768 ? 2 : 4);
            if (wpc == 1) return launch_block_t<8, 1, 16, false, 1, true, true>(h, a, sel, rd);
            // the stepping paths (AC, inputs = chronics rows) run the variant specialised for exactly that
            const bool ac_rows = !a.is_dc && a.series && h->blk_spec;
            if (wpc == 2) return ac_rows ? launch_block_t<8, 1, 8, false, 2, true, true, 1>(h, a, sel, rd) : launch_block_t<8, 1, 8, false, 2, true, true>(h, a, sel, rd);
            return ac_rows ? launch_block_t<8, 1, 4, false, 4, true, true, 1>(h, a, sel, rd) : launch_block_t<8, 1, 4, false, 4, true, true>(h, a, sel, rd);
        }
        return launch_block_t<8, 1, 4, false, 4, true, false>(h, a, sel, rd);
    }
    if (!a.prot && T == 8 && U == 1 && h->blk_wpc == 4 && h->blk_wpc_pinned && !h->blk_stage) return launch_block_t<8, 1, 4, false, 4, false, false>(h, a, sel, rd);
    if (!a.prot && T == 8 && U == 1) {
        // lockstep warps (one plan for the whole launch, whole warps): full-mask barriers / votes instead of per-instance collectives
        const bool uni = h->blk_uni && !sel.d_inst_plan && a.batch % 4 == 0;
        // register budget: 16 warps x 128 registers per SM
        if (uni) return launch_block_t<8, 1, 16, false, 1, false, true>(h, a, sel, rd);
        return launch_block_t<8, 1, 16, false>(h, a, sel, rd);
    }
    if (a.prot) {
#define X(t, u) if (T == t && U == u) return launch_block_t<t, u, (t <= 32 ? 8 : 4), true>(h, a, sel, rd);
        B200PF_BLOCK_VARIANTS(X)
#undef X
    } else {
#define X(t, u) if (T == t && U == u) return launch_block_t<t, u, (t <= 32 ? 8 : 4), false>(h, a, sel, rd);
        B200PF_BLOCK_VARIANTS(X)
#undef X
    }
    return fail(B200PF_E_ARG, "no block kernel variant for this (lanes, operations per lane) pair");
}

static int launch(b200pf_handle *h, RunArgs a, int nb_cap_req, const PlanSel *sel = nullptr) {
    if (sel) {
        RedoDesc rd;
        int rc = redo_config(h, a, nb_cap_req, &rd);
        return rc ? rc : launch_sparse(h, a, *sel, rd);
    }
    const DevGrid &g = h->g;
    int cap = nb_cap_req;
    if (cap <= 0 || cap > g.n_slot) cap = g.n_slot;
    // (no bound from the caller is every slot: a grid of at most 17 bus slots takes the warp kernel without one)
    if (warp_kernel_fits(g, cap)) return launch_small(h, a, cap);
    if (a.prot) return fail(B200PF_E_STATE, "device-side protections need the warp-per-instance kernel (<= 32 lines / bus slots, nb_cap <= 17)");
    int T = 32;
    size_t want = 0;
    int rc = generic_config(h, cap, 4, &T, &want);
    if (rc) return rc;
    a.nb_cap = cap;
    a.mat_bytes = (int)want;
    switch (T) {
        case 32: return launch_t<32>(h, a);
        case 128: return launch_t<128>(h, a);
        case 256: return launch_t<256>(h, a);
        default: return launch_t<512>(h, a);
    }
}

static int series_plans(b200pf_handle *h, const int8_t *topo);
static RunArgs base_args(const b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva) {
    RunArgs a{};
    a.batch = batch; a.is_dc = is_dc; a.max_iter = max_iter;
    a.tol_pu = tol_mva / h->g.base_mva;
    a.dbg_div_mod = h->dbg_div_mod;
    return a;
}

extern "C" int b200pf_run_device(b200pf_handle *h, int batch, const int8_t *d_topo, const double *d_inj, int is_dc,
                                 int max_iter, double tol_mva, int nb_cap, float *d_out, int32_t *d_status,
                                 int32_t *d_iters, double *d_busv) {
    if (!h || !d_topo || !d_inj || !d_out || !d_status || !d_iters) return fail(B200PF_E_ARG, "null pointer");
    if (batch <= 0) return fail(B200PF_E_ARG, "batch <= 0");
    CU(cudaSetDevice(h->device));
    RunArgs a = base_args(h, batch, is_dc, max_iter, tol_mva);
    a.topo = d_topo; a.inj = d_inj; a.out = d_out; a.status = d_status; a.iters = d_iters; a.busv = d_busv;
    return launch(h, a, nb_cap);
}

// kernel launch for the records staged in d_topo / d_inj (host copy of the topology: h_topo)
static int run_staged_device(b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva, int nb_cap, bool want_busv) {
    RunArgs a = base_args(h, batch, is_dc, max_iter, tol_mva);
    a.topo = h->d_topo; a.inj = h->d_inj; a.out = h->d_out; a.status = h->d_status; a.iters = h->d_iters;
    a.busv = want_busv ? h->d_busv : nullptr;
    PlanSel sel;
    const int use = plan_select(h, h->h_topo, batch, 0, 0, h->stream, &sel);
    if (use < 0) return use;
    return launch(h, a, nb_cap, use ? &sel : nullptr);
}

extern "C" int b200pf_run_device_topo(b200pf_handle *h, int batch, const int8_t *host_topo, const int8_t *d_topo, const double *d_inj,
                                      int is_dc, int max_iter, double tol_mva, int nb_cap, float *d_out, int32_t *d_status,
                                      int32_t *d_iters, double *d_busv) {
    if (!h || !host_topo || !d_topo || !d_inj || !d_out || !d_status || !d_iters) return fail(B200PF_E_ARG, "null pointer");
    if (batch <= 0 || batch > h->max_batch) return fail(B200PF_E_ARG, "batch out of range (max_batch)");
    CU(cudaSetDevice(h->device));
    RunArgs a = base_args(h, batch, is_dc, max_iter, tol_mva);
    a.topo = d_topo; a.inj = d_inj; a.out = d_out; a.status = d_status; a.iters = d_iters; a.busv = d_busv;
    PlanSel sel;
    const int use = plan_select(h, host_topo, batch, 0, 0, h->stream, &sel);
    if (use < 0) return use;
    return launch(h, a, nb_cap, use ? &sel : nullptr);
}

extern "C" int b200pf_run_host(b200pf_handle *h, int batch, const int8_t *topo, const double *inj, int is_dc,
                               int max_iter, double tol_mva, int nb_cap, float *out, int32_t *status,
                               int32_t *iters, double *busv) {
    if (!h || !topo || !inj || !out || !status || !iters) return fail(B200PF_E_ARG, "null pointer");
    if (batch <= 0 || batch > h->max_batch) return fail(B200PF_E_ARG, "batch out of range (max_batch)");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const size_t B = (size_t)batch;
    memcpy(h->h_topo, topo, B * g.n_topo_in);
    memcpy(h->h_inj, inj, B * g.n_inj * 8);
    CU(cudaMemcpyAsync(h->d_topo, h->h_topo, B * g.n_topo_in, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_inj, h->h_inj, B * g.n_inj * 8, cudaMemcpyHostToDevice, h->stream));
    int rc = run_staged_device(h, batch, is_dc, max_iter, tol_mva, nb_cap, busv != nullptr);
    if (rc) return rc;
    CU(cudaMemcpyAsync(h->h_out, h->d_out, B * g.n_out * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_status, h->d_status, B * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_iters, h->d_iters, B * 4, cudaMemcpyDeviceToHost, h->stream));
    if (busv) CU(cudaMemcpyAsync(h->h_busv, h->d_busv, B * 2 * g.n_slot * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    memcpy(out, h->h_out, B * g.n_out * 4);
    memcpy(status, h->h_status, B * 4);
    memcpy(iters, h->h_iters, B * 4);
    if (busv) memcpy(busv, h->h_busv, B * 2 * g.n_slot * 8);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// time-series stepping
// ------------------------------------------------------------------------------------------------
extern "C" int b200pf_series_bind(b200pf_handle *h, const float *chron_host, int n_scen, int n_rows, const int32_t *scen,
                                  const int32_t *t0, int batch, const double *static_inj, const float *thermal_limit_a) {
    if (!h || !chron_host || !scen || !t0 || !static_inj || !thermal_limit_a) return fail(B200PF_E_ARG, "null pointer");
    if (batch <= 0 || batch > h->max_batch || n_scen <= 0 || n_rows <= 0) return fail(B200PF_E_ARG, "bad sizes");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    for (int i = 0; i < batch; ++i)
        if (scen[i] < 0 || scen[i] >= n_scen || t0[i] < 0 || t0[i] >= n_rows) return fail(B200PF_E_ARG, "scenario / row index out of range");
    const size_t ncol = 2 * (size_t)g.n_load + 2 * (size_t)g.n_gen;
    if (h->series_batch) {      // re-bind: the previous series' buffers go back first
        CU(cudaStreamSynchronize(h->stream));
        void *old[] = {h->d_chron, h->d_scen, h->d_t, h->d_series_topo, h->d_pcount, h->d_tsover, h->d_disc, h->d_done, h->d_series_plan, h->d_trip,
                       h->d_incdone, h->d_nflag, h->d_flaglist, h->d_casclist};
        for (void *p : old) {
            if (!p) continue;
            for (size_t q = 0; q < h->dev_allocs.size(); ++q) if (h->dev_allocs[q] == p) { h->dev_allocs.erase(h->dev_allocs.begin() + q); break; }
            cudaFree(p);
        }
        h->series_batch = 0; h->series_plan_state = 0; h->series_dev_topo_ahead = false;
    }
    auto dmal = [&](void **p, size_t bytes) -> int { CU(cudaMalloc(p, bytes ? bytes : 1)); h->dev_allocs.push_back(*p); return 0; };
    int rc;
    if ((rc = dmal((void **)&h->d_chron, (size_t)n_scen * n_rows * ncol * 4)) || (rc = dmal((void **)&h->d_scen, (size_t)batch * 4)) ||
        (rc = dmal((void **)&h->d_t, (size_t)batch * 4)) ||
        (rc = dmal((void **)&h->d_series_topo, (size_t)batch * g.n_topo_in)) ||
        (rc = dmal((void **)&h->d_pcount, (size_t)batch * g.n_line * 4)) || (rc = dmal((void **)&h->d_tsover, (size_t)batch * g.n_line * 4)) ||
        (rc = dmal((void **)&h->d_disc, (size_t)batch * g.n_line * 4)) || (rc = dmal((void **)&h->d_done, (size_t)batch * 4)))
        return rc;
    CU(cudaMemsetAsync(h->d_pcount, 0, (size_t)batch * g.n_line * 4, h->stream)); CU(cudaMemsetAsync(h->d_tsover, 0, (size_t)batch * g.n_line * 4, h->stream));
    CU(cudaMemsetAsync(h->d_disc, 0xff, (size_t)batch * g.n_line * 4, h->stream)); CU(cudaMemsetAsync(h->d_done, 0, (size_t)batch * 4, h->stream));
    H2D(h->d_chron, chron_host, (size_t)n_scen * n_rows * ncol * 4);
    H2D(h->d_scen, scen, (size_t)batch * 4);
    H2D(h->d_t, t0, (size_t)batch * 4);
    H2D(h->d_static_inj, static_inj, (size_t)g.n_inj * 8);
    H2D(h->d_thlim, thermal_limit_a, (size_t)g.n_line * 4);
    h->stat_dirty = true;
    CU(cudaMemsetAsync(h->d_series_topo, 1, (size_t)batch * g.n_topo_in, h->stream));
    h->series_batch = batch; h->n_scen = n_scen; h->n_rows = n_rows;
    if ((rc = dmal((void **)&h->d_series_plan, (size_t)batch * 4)) || (rc = dmal((void **)&h->d_trip, (size_t)batch * g.n_line + 4)) ||
        (rc = dmal((void **)&h->d_incdone, (size_t)batch * g.n_line + 4)) || (rc = dmal((void **)&h->d_nflag, 16)) ||
        (rc = dmal((void **)&h->d_flaglist, (size_t)batch * 4)) || (rc = dmal((void **)&h->d_casclist, (size_t)batch * 4))) return rc;
    CU(cudaMemsetAsync(h->d_trip, 0, (size_t)batch * g.n_line + 4, h->stream)); CU(cudaMemsetAsync(h->d_incdone, 0, (size_t)batch * g.n_line + 4, h->stream));
    {
        std::vector<int8_t> ones((size_t)batch * g.n_topo_in, 1);
        return series_plans(h, ones.data());
    }
}

// plans of the device-resident series topology (it only changes through b200pf_series_set_topo, or through the
// protections, which keep the pivoting kernels)
static int series_plans(b200pf_handle *h, const int8_t *topo) {
    h->series_plan_state = 0;
    h->series_plans_stale = false;
    PlanSel sel;
    CU(cudaStreamSynchronize(h->stream));
    const int use = plan_select(h, topo, h->series_batch, 0, 0, h->stream, &sel);
    if (use < 0) return use;
    if (!use) return 0;
    h->series_plan_single = sel.single; h->series_plan_smem = sel.smem; h->series_lay_nb = sel.lay_nb; h->series_lay_nblkA = sel.lay_nblkA;
    h->h_series_topo.assign(topo, topo + (size_t)h->series_batch * h->g.n_topo_in);
    h->h_series_plan.assign(h->h_inst_plan, h->h_inst_plan + h->series_batch);
    if (sel.d_inst_plan) {
        CU(cudaMemcpyAsync(h->d_series_plan, h->d_inst_plan, (size_t)h->series_batch * 4, cudaMemcpyDeviceToDevice, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        h->series_plan_state = 1;
    } else h->series_plan_state = 2;
    return 0;
}

extern "C" int b200pf_series_set_topo(b200pf_handle *h, const int8_t *topo) {
    if (!h || !topo) return fail(B200PF_E_ARG, "null pointer");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    CU(cudaSetDevice(h->device));
    H2D(h->d_series_topo, topo, (size_t)h->series_batch * h->g.n_topo_in);
    h->series_dev_topo_ahead = false;
    return series_plans(h, topo);
}

// One series step with protections on the planned kernel.  The kernel REPORTS the lines that must trip (a tripped line is a
// new topology, i.e. a new plan); the host takes them out of its mirror of the topology, looks the plan up (or builds it),
// and launches the next cascade round for the flagged instances only — the loop of Backend.next_grid_state
// (reference backend.py:1466-1521) with the power flows of a round batched.  Synchronous: one 4-byte read-back per round.
static int series_step_planned_prot(b200pf_handle *h, RunArgs a) {
    const DevGrid &g = h->g;
    const int B = h->series_batch, nl = g.n_line;
    const size_t nt = (size_t)g.n_topo_in;
    if (h->series_plan_state == 2) {      // make the per-instance plan array explicit
        CU(cudaMemcpyAsync(h->d_series_plan, h->h_series_plan.data(), (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
        h->series_plan_state = 1;
    }
    a.trip = h->d_trip; a.incdone = h->d_incdone; a.n_flag = h->d_nflag; a.flag_list = h->d_flaglist;
    h->h_trip.resize((size_t)B * nl); h->h_flaglist.resize(B);
    int n = B;
    const int *list = nullptr;
    for (int casc = 0;; ++casc) {
        if (casc > 2 * nl + 2) return fail(B200PF_E_STATE, "cascade did not terminate");
        CU(cudaMemsetAsync(h->d_nflag, 0, 4, h->stream));
        a.casc = casc; a.inst_list = list; a.batch = n;
        PlanSel sel;
        sel.single = 0; sel.d_inst_plan = h->d_series_plan;
        sel_layout(h, &sel, false);
        int rc = launch(h, a, 0, &sel);      // (the re-solve applies the protection rules to what it solves)
        if (rc) return rc;
        int nflag = 0;
        CU(cudaMemcpyAsync(&nflag, h->d_nflag, 4, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        h->last_cascade_rounds = casc + 1;
        if (nflag <= 0) break;
        CU(cudaMemcpyAsync(h->h_flaglist.data(), h->d_flaglist, (size_t)nflag * 4, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaMemcpyAsync(h->h_trip.data(), h->d_trip, (size_t)B * nl, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        for (int k = 0; k < nflag; ++k) {
            const int inst = h->h_flaglist[k];
            if (inst < 0 || inst >= B) return fail(B200PF_E_STATE, "bad instance in the cascade list");
            int8_t *row = h->h_series_topo.data() + (size_t)inst * nt;
            apply_trips(h->hg, row, h->h_trip.data() + (size_t)inst * nl);
            const uint64_t rh = topo_hash(row, nt);
            int id = plan_find(h, row, rh, -1);
            if (id < 0) {
                id = plan_insert(h, row, rh, -1, make_builder(h).build(row, -1));
                if (id < 0) return fail(B200PF_E_CAPACITY, "no plan for the topology after a line trip");
            }
            h->h_series_plan[inst] = id;
            CU(cudaMemcpyAsync(h->d_series_topo + (size_t)inst * nt, row, nt, cudaMemcpyHostToDevice, h->stream));
        }
        if ((rc = plans_sync_device(h, h->stream))) return rc;
        CU(cudaMemcpyAsync(h->d_series_plan, h->h_series_plan.data(), (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
        CU(cudaMemsetAsync(h->d_trip, 0, (size_t)B * nl, h->stream));
        CU(cudaMemcpyAsync(h->d_casclist, h->h_flaglist.data(), (size_t)nflag * 4, cudaMemcpyHostToDevice, h->stream));
        n = nflag; list = h->d_casclist;
    }
    return 0;
}

static int series_step_impl(b200pf_handle *h, int is_dc, int max_iter, double tol_mva, int nb_cap);

extern "C" int b200pf_series_step(b200pf_handle *h, int is_dc, int max_iter, double tol_mva, int nb_cap) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    CU(cudaSetDevice(h->device));
    if (h->series_flag) h->series_step_no++;
    int rc = series_step_impl(h, is_dc, max_iter, tol_mva, nb_cap);
    if (rc) return rc;
    if (h->series_flag) {
        pf_kernel_flag<<<1, 1, 0, h->stream>>>(h->series_flag, h->series_step_no);
        CU(cudaGetLastError());
    }
    return 0;
}

extern "C" int b200pf_series_bind_flag(b200pf_handle *h, int32_t *d_flag) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    CU(cudaSetDevice(h->device));
    h->series_flag = d_flag; h->series_step_no = 0;
    return 0;
}

static int series_step_impl(b200pf_handle *h, int is_dc, int max_iter, double tol_mva, int nb_cap) {
    RunArgs a = base_args(h, h->series_batch, is_dc, max_iter, tol_mva);
    a.topo = h->d_series_topo; a.inj = nullptr; a.out = h->x_out ? h->x_out : h->d_out; a.status = h->x_status ? h->x_status : h->d_status;
    a.iters = h->x_iters ? h->x_iters : h->d_iters; a.busv = nullptr;
    a.series = 1; a.chron = h->d_chron; a.n_scen = h->n_scen; a.n_rows = h->n_rows; a.scen = h->d_scen; a.t = h->d_t;
    a.static_inj = h->d_static_inj; a.th_lim = h->d_thlim; a.rho = h->x_rho ? h->x_rho : h->d_rho;
    if (h->prot) {
        a.prot = 1; a.from_reset = h->next_reset; a.max_pc = h->max_pc; a.hard_thr = h->hard_thr; a.soft_thr = h->soft_thr;
        a.pcount = h->d_pcount; a.ts_over = h->d_tsover; a.disc = h->d_disc; a.done = h->d_done;
    }
    h->next_reset = 0;
    // the warp kernel runs the series' protections only under a bound from the caller (nb_cap > 0), although launch() reads
    // nb_cap <= 0 as every slot and so takes the warp kernel without one on a grid of at most 17 bus slots
    const bool small_ok = nb_cap > 0 && warp_kernel_fits(h->g, nb_cap);
    if (h->series_dev_topo_ahead && h->plan_policy != 1) {
        // protections ran on the device (warp kernel: trips written into d_series_topo); whoever uses plans next — protections
        // switched off, policy switched to the planned kernel — must see those outages: refresh the host mirror and the plans
        const bool warp_again = h->prot && small_ok && h->plan_policy != 2 && !is_dc;
        if (!warp_again) {
            std::vector<int8_t> cur((size_t)h->series_batch * h->g.n_topo_in);
            CU(cudaStreamSynchronize(h->stream));
            CU(cudaMemcpy(cur.data(), h->d_series_topo, cur.size(), cudaMemcpyDeviceToHost));
            int rc = series_plans(h, cur.data());
            if (rc) return rc;
            h->series_dev_topo_ahead = false;
        }
    }
    if (h->series_plans_stale) {
        h->series_plans_stale = false;
        std::vector<int8_t> keep(h->h_series_topo);
        int rc = series_plans(h, keep.data());
        if (rc) return rc;
    }
    // protections: the warp kernel cascades entirely on the device (no host in the loop) and is preferred where it applies;
    // everything else runs the planned kernel with the host re-planning the instances whose lines trip
    if (h->prot && h->series_plan_state && h->plan_policy != 1 && (h->plan_policy == 2 || !small_ok) && !is_dc)
        return series_step_planned_prot(h, a);
    if (h->series_plan_state && !h->prot && h->plan_policy != 1) {
        PlanSel sel;
        sel.single = h->series_plan_single; sel.smem = h->series_plan_smem; sel.lay_nb = h->series_lay_nb; sel.lay_nblkA = h->series_lay_nblkA;
        sel.d_inst_plan = h->series_plan_state == 1 ? h->d_series_plan : nullptr;
        return launch(h, a, nb_cap, &sel);
    }
    if (h->prot) h->series_dev_topo_ahead = true;          // (device-side cascade of the warp kernel)
    return launch(h, a, nb_cap);
}

extern "C" int b200pf_series_reset_instances(b200pf_handle *h, int n, const int32_t *idx, const int32_t *t_new, const int8_t *topo_rows) {
    if (!h || (n > 0 && !idx)) return fail(B200PF_E_ARG, "null pointer");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    if (n <= 0) return 0;
    if (n > h->series_batch) return fail(B200PF_E_ARG, "more instances than the series holds");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const size_t nt = (size_t)g.n_topo_in;
    for (int k = 0; k < n; ++k) {
        if (idx[k] < 0 || idx[k] >= h->series_batch) return fail(B200PF_E_ARG, "instance index out of range");
        if (t_new && (t_new[k] < 0 || t_new[k] >= h->n_rows)) return fail(B200PF_E_ARG, "row index out of range");
    }
    CU(cudaStreamSynchronize(h->stream));
    // d_casclist / d_flaglist: scratch of batch ints each (idle between steps)
    H2D(h->d_casclist, idx, (size_t)n * 4);
    if (t_new) H2D(h->d_flaglist, t_new, (size_t)n * 4);
    pf_kernel_series_reset<<<n, 64, 0, h->stream>>>(n, h->d_casclist, t_new ? h->d_flaglist : nullptr, g.n_line, h->d_t, h->d_done, h->d_pcount,
                                                     h->d_tsover, h->d_disc, h->d_trip, h->d_incdone);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(h->stream));
    if (topo_rows) {
        // the instances' topology: device copy, host mirror, plans
        std::vector<int8_t> all;
        if (h->series_dev_topo_ahead || h->h_series_topo.size() != (size_t)h->series_batch * nt) {
            all.resize((size_t)h->series_batch * nt);
            CU(cudaMemcpy(all.data(), h->d_series_topo, all.size(), cudaMemcpyDeviceToHost));
        } else all = h->h_series_topo;
        for (int k = 0; k < n; ++k) {
            memcpy(all.data() + (size_t)idx[k] * nt, topo_rows + (size_t)k * nt, nt);
            // (stream-ordered; the stream is drained once, at the start of series_plans below)
            CU(cudaMemcpyAsync(h->d_series_topo + (size_t)idx[k] * nt, topo_rows + (size_t)k * nt, nt, cudaMemcpyHostToDevice, h->stream));
        }
        h->series_dev_topo_ahead = false;
        return series_plans(h, all.data());
    }
    return 0;
}

extern "C" int b200pf_series_protections(b200pf_handle *h, int enabled, float hard_thr, float soft_thr, int max_allowed) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    h->prot = enabled ? 1 : 0; h->hard_thr = hard_thr; h->soft_thr = soft_thr; h->max_pc = max_allowed;
    return 0;
}

extern "C" int b200pf_series_next_is_reset(b200pf_handle *h) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    h->next_reset = 1;
    return 0;
}

extern "C" int b200pf_series_fetch_state(b200pf_handle *h, int32_t *pc, int32_t *tso, int32_t *disc, int32_t *done) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    const size_t B = (size_t)h->series_batch, nl = (size_t)h->g.n_line;
    h->d2h_bytes += (int64_t)(((pc != nullptr) + (tso != nullptr) + (disc != nullptr)) * B * nl * 4 + (done != nullptr) * B * 4);
    if (pc) CU(cudaMemcpy(pc, h->d_pcount, B * nl * 4, cudaMemcpyDeviceToHost));
    if (tso) CU(cudaMemcpy(tso, h->d_tsover, B * nl * 4, cudaMemcpyDeviceToHost));
    if (disc) CU(cudaMemcpy(disc, h->d_disc, B * nl * 4, cudaMemcpyDeviceToHost));
    if (done) CU(cudaMemcpy(done, h->d_done, B * 4, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int b200pf_series_results(b200pf_handle *h, float **d_out, int32_t **d_status, int32_t **d_iters, float **d_rho, int32_t **d_t) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (d_out) *d_out = h->x_out ? h->x_out : h->d_out;
    if (d_status) *d_status = h->x_status ? h->x_status : h->d_status;
    if (d_iters) *d_iters = h->x_iters ? h->x_iters : h->d_iters;
    if (d_rho) *d_rho = h->x_rho ? h->x_rho : h->d_rho;
    if (d_t) *d_t = h->d_t;
    return 0;
}

extern "C" int b200pf_series_fetch(b200pf_handle *h, float *out, int32_t *status, int32_t *iters, float *rho) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    CU(cudaSetDevice(h->device));
    const size_t B = (size_t)h->series_batch;
    const DevGrid &g = h->g;
    CU(cudaStreamSynchronize(h->stream));
    h->d2h_bytes += (int64_t)((out != nullptr) * B * g.n_out * 4 + ((status != nullptr) + (iters != nullptr)) * B * 4 + (rho != nullptr) * B * g.n_line * 4);
    if (out) CU(cudaMemcpy(out, h->x_out ? h->x_out : h->d_out, B * g.n_out * 4, cudaMemcpyDeviceToHost));
    if (status) CU(cudaMemcpy(status, h->x_status ? h->x_status : h->d_status, B * 4, cudaMemcpyDeviceToHost));
    if (iters) CU(cudaMemcpy(iters, h->x_iters ? h->x_iters : h->d_iters, B * 4, cudaMemcpyDeviceToHost));
    if (rho) CU(cudaMemcpy(rho, h->x_rho ? h->x_rho : h->d_rho, B * g.n_line * 4, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int b200pf_staging(b200pf_handle *h, int8_t **topo, double **inj, float **out, int32_t **status, int32_t **iters,
                              double **busv) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (topo) *topo = h->h_topo;
    if (inj) *inj = h->h_inj;
    if (out) *out = h->h_out;
    if (status) *status = h->h_status;
    if (iters) *iters = h->h_iters;
    if (busv) *busv = h->h_busv;
    return 0;
}

extern "C" int b200pf_run_staged(b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva, int nb_cap, int want_busv) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (batch <= 0 || batch > h->max_batch) return fail(B200PF_E_ARG, "batch out of range (max_batch)");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const size_t B = (size_t)batch;
    CU(cudaMemcpyAsync(h->d_topo, h->h_topo, B * g.n_topo_in, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_inj, h->h_inj, B * g.n_inj * 8, cudaMemcpyHostToDevice, h->stream));
    int rc = run_staged_device(h, batch, is_dc, max_iter, tol_mva, nb_cap, want_busv != 0);
    if (rc) return rc;
    CU(cudaMemcpyAsync(h->h_out, h->d_out, B * g.n_out * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_status, h->d_status, B * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_iters, h->d_iters, B * 4, cudaMemcpyDeviceToHost, h->stream));
    if (want_busv) CU(cudaMemcpyAsync(h->h_busv, h->d_busv, B * 2 * g.n_slot * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int b200pf_set_thermal_limit(b200pf_handle *h, const float *thermal_limit_a) {
    if (!h || !thermal_limit_a) return fail(B200PF_E_ARG, "null pointer");
    CU(cudaSetDevice(h->device));
    H2D(h->d_thlim, thermal_limit_a, (size_t)h->g.n_line * 4);
    h->stat_dirty = true;
    return 0;
}

extern "C" int b200pf_n1_host(b200pf_handle *h, int batch, const int8_t *topo, const double *inj, int max_iter, double tol_mva,
                              int nb_cap, float *rho, int32_t *status) {
    if (!h || !topo || !inj || !rho || !status) return fail(B200PF_E_ARG, "null pointer");
    const DevGrid &g = h->g;
    if (batch <= 0 || (long)batch * g.n_line > h->max_batch) return fail(B200PF_E_ARG, "batch * n_line exceeds max_batch");
    CU(cudaSetDevice(h->device));
    const size_t B = (size_t)batch, N = B * g.n_line;
    CU(cudaMemcpyAsync(h->d_topo, topo, B * g.n_topo_in, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_inj, inj, B * g.n_inj * 8, cudaMemcpyHostToDevice, h->stream));
    RunArgs a = base_args(h, (int)N, 0, max_iter, tol_mva);
    a.topo = h->d_topo; a.inj = h->d_inj; a.out = nullptr; a.status = h->d_status; a.iters = h->d_iters; a.busv = nullptr;
    a.n1_lines = g.n_line; a.th_lim = h->d_thlim; a.rho = h->d_rho;
    PlanSel sel;
    const int use = plan_select(h, topo, batch, g.n_line, 0, h->stream, &sel);
    if (use < 0) return use;
    int rc = launch(h, a, nb_cap, use ? &sel : nullptr);
    if (rc) return rc;
    CU(cudaMemcpyAsync(rho, h->d_rho, N * g.n_line * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(status, h->d_status, N * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int b200pf_set_static_inj(b200pf_handle *h, const double *static_inj) {
    if (!h || !static_inj) return fail(B200PF_E_ARG, "null pointer");
    CU(cudaSetDevice(h->device));
    H2D(h->d_static_inj, static_inj, (size_t)h->g.n_inj * 8);
    h->stat_dirty = true;
    return 0;
}

extern "C" int b200pf_rows_staging(b200pf_handle *h, float **rows) {
    if (!h || !rows) return fail(B200PF_E_ARG, "null pointer");
    *rows = h->h_rows;
    return 0;
}

extern "C" int b200pf_run_rows_staged(b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva, int nb_cap) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (batch <= 0 || batch > h->max_batch) return fail(B200PF_E_ARG, "batch out of range (max_batch)");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const size_t B = (size_t)batch, ncol = 2 * (size_t)g.n_load + 2 * (size_t)g.n_gen;
    CU(cudaMemcpyAsync(h->d_topo, h->h_topo, B * g.n_topo_in, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_rows, h->h_rows, B * ncol * 4, cudaMemcpyHostToDevice, h->stream));
    RunArgs a = base_args(h, batch, is_dc, max_iter, tol_mva);
    a.topo = h->d_topo; a.inj = nullptr; a.out = h->d_out; a.status = h->d_status; a.iters = h->d_iters; a.busv = nullptr;
    a.series = 1; a.rows = h->d_rows; a.static_inj = h->d_static_inj;
    PlanSel sel;
    const int use = plan_select(h, h->h_topo, batch, 0, 0, h->stream, &sel);
    if (use < 0) return use;
    int rc = launch(h, a, nb_cap, use ? &sel : nullptr);
    if (rc) return rc;
    CU(cudaMemcpyAsync(h->h_out, h->d_out, B * g.n_out * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_status, h->d_status, B * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_iters, h->d_iters, B * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int b200pf_pinned_alloc(size_t bytes, void **ptr) {
    if (!ptr) return fail(B200PF_E_ARG, "null pointer");
    CU(cudaMallocHost(ptr, bytes ? bytes : 1));
    return 0;
}
extern "C" int b200pf_pinned_free(void *ptr) {
    if (ptr) CU(cudaFreeHost(ptr));
    return 0;
}

static int rows_chunk_launch_impl(b200pf_handle *h, int first, int count, const float *src_rows, int is_dc, int max_iter,
                                  double tol_mva, int nb_cap, int group = -1);

extern "C" int b200pf_rows_chunk_launch(b200pf_handle *h, int first, int count, int is_dc, int max_iter, double tol_mva, int nb_cap) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    const size_t ncol = 2 * (size_t)h->g.n_load + 2 * (size_t)h->g.n_gen;
    return rows_chunk_launch_impl(h, first, count, h->h_rows + (size_t)(first < 0 ? 0 : first) * ncol, is_dc, max_iter, tol_mva, nb_cap);
}

extern "C" int b200pf_rows_chunk_launch_from(b200pf_handle *h, int first, int count, const float *pinned_rows, int is_dc,
                                             int max_iter, double tol_mva, int nb_cap) {
    if (!h || !pinned_rows) return fail(B200PF_E_ARG, "null pointer");
    return rows_chunk_launch_impl(h, first, count, pinned_rows, is_dc, max_iter, tol_mva, nb_cap);
}

static int rows_chunk_launch_impl(b200pf_handle *h, int first, int count, const float *src_rows, int is_dc, int max_iter,
                                  double tol_mva, int nb_cap, int group) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (first < 0 || count <= 0 || first + count > h->max_batch) return fail(B200PF_E_ARG, "chunk out of range (max_batch)");
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    cudaStream_t st;
    if (group >= 0) {
        if (!h->group_stream[group]) {
            CU(cudaStreamCreateWithFlags(&h->group_stream[group], cudaStreamNonBlocking));
            CU(cudaEventCreateWithFlags(&h->group_event[group], cudaEventDisableTiming));
        }
        st = h->group_stream[group];
    } else {
        const int ci = h->chunk_next++ & 3;
        if (!h->chunk_stream[ci]) CU(cudaStreamCreateWithFlags(&h->chunk_stream[ci], cudaStreamNonBlocking));
        st = h->chunk_stream[ci];
    }
    const size_t F = (size_t)first, C = (size_t)count, ncol = 2 * (size_t)g.n_load + 2 * (size_t)g.n_gen;
    PlanSel sel;
    const int use = plan_select(h, h->h_topo + F * g.n_topo_in, count, 0, first, st, &sel);
    if (use < 0) return use;
    RunArgs a = base_args(h, count, is_dc, max_iter, tol_mva);
    a.topo = h->d_topo + F * g.n_topo_in; a.inj = nullptr; a.out = h->d_out + F * g.n_out; a.status = h->d_status + F;
    a.iters = h->d_iters + F; a.busv = nullptr; a.series = 1; a.rows = h->d_rows + F * ncol; a.static_inj = h->d_static_inj;
    // group flags: bit 1 = the kernel reads its inputs straight from the pinned host buffers (a few hundred bytes per
    // instance, read once: no H2D calls at all; the planned kernel does not read the topology records), bit 2 = status /
    // iteration counts stored by the kernel straight into pinned host memory (8 bytes per instance), bit 0 = everything is
    const bool zc_in = group >= 0 && (h->group_flags & 2);
    if (zc_in) {
        a.rows = src_rows;
        a.topo = h->h_topo + F * g.n_topo_in;
    } else {
        // planned kernel: no topology record crosses PCIe; the (rare) pivoting re-solve reads it from the pinned staging buffer
        if (use) a.topo = h->h_topo + F * g.n_topo_in;
        if (!use) CU(cudaMemcpyAsync(h->d_topo + F * g.n_topo_in, h->h_topo + F * g.n_topo_in, C * g.n_topo_in, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(h->d_rows + F * ncol, src_rows, C * ncol * 4, cudaMemcpyHostToDevice, st));
    }
    const bool direct = group >= 0 && (h->group_flags & 1);
    const bool direct_st = direct || (group >= 0 && (h->group_flags & 4));
    if (direct) a.out = h->h_out + F * g.n_out;   // pinned host memory is device-addressable (unified addressing): posted PCIe writes
    if (direct_st) { a.status = h->h_status + F; a.iters = h->h_iters + F; }
    cudaStream_t keep = h->stream;
    h->stream = st; h->on_side_stream = true;
    int rc = launch(h, a, nb_cap, use ? &sel : nullptr);
    h->stream = keep; h->on_side_stream = false;
    if (rc) return rc;
    if (!direct) CU(cudaMemcpyAsync(h->h_out + F * g.n_out, h->d_out + F * g.n_out, C * g.n_out * 4, cudaMemcpyDeviceToHost, st));
    if (!direct_st) {
        CU(cudaMemcpyAsync(h->h_status + F, h->d_status + F, C * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(h->h_iters + F, h->d_iters + F, C * 4, cudaMemcpyDeviceToHost, st));
    }
    if (group >= 0) { CU(cudaEventRecord(h->group_event[group], st)); h->group_pending[group] = true; }
    return 0;
}

extern "C" int b200pf_rows_group_launch(b200pf_handle *h, int group, int first, int count, const float *pinned_rows, int is_dc,
                                        int max_iter, double tol_mva, int nb_cap) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (group < 0 || group >= B200PF_MAX_GROUPS) return fail(B200PF_E_ARG, "group out of range");
    if (h->group_pending[group]) return fail(B200PF_E_ARG, "group still in flight: call b200pf_rows_group_wait first");
    const size_t ncol = 2 * (size_t)h->g.n_load + 2 * (size_t)h->g.n_gen;
    const float *src = pinned_rows ? pinned_rows : h->h_rows + (size_t)(first < 0 ? 0 : first) * ncol;
    return rows_chunk_launch_impl(h, first, count, src, is_dc, max_iter, tol_mva, nb_cap, group);
}

extern "C" int b200pf_rows_group_config(b200pf_handle *h, int flags) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    for (bool p : h->group_pending) if (p) return fail(B200PF_E_STATE, "groups in flight");
    h->group_flags = flags;
    return 0;
}

extern "C" int b200pf_rows_group_wait(b200pf_handle *h, int group) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (group < 0 || group >= B200PF_MAX_GROUPS) return fail(B200PF_E_ARG, "group out of range");
    if (!h->group_pending[group]) return 0;
    CU(cudaEventSynchronize(h->group_event[group]));
    h->group_pending[group] = false;
    return 0;
}

extern "C" int b200pf_rows_chunk_wait(b200pf_handle *h) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    CU(cudaSetDevice(h->device));
    for (auto &cs : h->chunk_stream) if (cs) CU(cudaStreamSynchronize(cs));
    return 0;
}

extern "C" int b200pf_series_bind_outputs(b200pf_handle *h, float *d_out, int32_t *d_status, int32_t *d_iters, float *d_rho) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    h->x_out = d_out; h->x_status = d_status; h->x_iters = d_iters; h->x_rho = d_rho;
    return 0;
}

extern "C" int b200pf_set_stream(b200pf_handle *h, uint64_t stream) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    h->stream = stream ? (cudaStream_t)(uintptr_t)stream : h->own_stream;
    return 0;
}

extern "C" int b200pf_set_kernel_policy(b200pf_handle *h, int policy) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (policy < 0 || policy > 2) return fail(B200PF_E_ARG, "policy must be 0 (auto), 1 (pivoting kernels only) or 2 (planned sparse kernel)");
    h->plan_policy = policy;
    return 0;
}

extern "C" int b200pf_plan_stats(const b200pf_handle *h, int64_t *n_plans, int64_t *plan_bytes, int *last_kernel) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (n_plans) *n_plans = (int64_t)h->plan_off.size();
    if (plan_bytes) *plan_bytes = (int64_t)h->plan_blobs.size();
    if (last_kernel) *last_kernel = h->last_kernel;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// multi-GPU result collection without a collective launch: peer-mapped device memory (CUDA IPC over NVLink)
// ------------------------------------------------------------------------------------------------
extern "C" int b200pf_device_alloc(size_t bytes, void **d_ptr) {
    if (!d_ptr) return fail(B200PF_E_ARG, "null pointer");
    CU(cudaMalloc(d_ptr, bytes ? bytes : 1));
    CU(cudaMemset(*d_ptr, 0, bytes ? bytes : 1));
    CU(cudaDeviceSynchronize());      // (the legacy stream is not ordered against the handles' non-blocking streams)
    return 0;
}
extern "C" int b200pf_device_free(void *d_ptr) {
    if (d_ptr) CU(cudaFree(d_ptr));
    return 0;
}
extern "C" int b200pf_device_read(const void *d_src, void *host_dst, size_t bytes) {
    if (!d_src || !host_dst) return fail(B200PF_E_ARG, "null pointer");
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(host_dst, d_src, bytes, cudaMemcpyDeviceToHost));
    return 0;
}
extern "C" int b200pf_ipc_export(const void *d_ptr, unsigned char *handle64) {
    if (!d_ptr || !handle64) return fail(B200PF_E_ARG, "null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t hd;
    CU(cudaIpcGetMemHandle(&hd, const_cast<void *>(d_ptr)));
    memcpy(handle64, &hd, 64);
    return 0;
}
extern "C" int b200pf_ipc_open(const unsigned char *handle64, void **d_ptr) {
    if (!d_ptr || !handle64) return fail(B200PF_E_ARG, "null pointer");
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, 64);
    CU(cudaIpcOpenMemHandle(d_ptr, hd, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}
extern "C" int b200pf_ipc_close(void *d_ptr) {
    if (d_ptr) CU(cudaIpcCloseMemHandle(d_ptr));
    return 0;
}

extern "C" int b200pf_set_debug(b200pf_handle *h, int planned_div_mod, int redo_enabled) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    h->dbg_div_mod = planned_div_mod > 0 ? planned_div_mod : 0;
    h->redo_enabled = redo_enabled ? 1 : 0;
    return 0;
}

// the planned kernels count their tail launches in the control words: waits for the device, then reads them
extern "C" int64_t b200pf_redo_launch_count(const b200pf_handle *h) {
    if (!h || cudaSetDevice(h->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return 0;
    int64_t n = 0;
    for (const auto &kv : h->redo_streams) {
        RedoCtl c{};
        if (!kv.second.ctl) continue;
        if (cudaMemcpy(&c, kv.second.ctl, sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
        n += c.launches;
    }
    return n;
}

extern "C" int b200pf_plan_counters(const b200pf_handle *h, int64_t *out4) {
    if (!h || !out4) return fail(B200PF_E_ARG, "null pointer");
    out4[0] = h->plan_lookups; out4[1] = h->plan_hits; out4[2] = h->plans_built; out4[3] = h->plan_cache_resets;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// host code shared by the layers of the device environment (observation, environment, opponent, alerts, alarms)
// ------------------------------------------------------------------------------------------------
// Start of a layer's bind: drain the stream, mark the layer unbound (*batch = 0), then free its buffers.  Every bind sets its
// *batch again last, after everything else succeeded: a bind that fails half way (an allocation, a copy, an event) leaves its
// layer unbound, never bound over freed memory.
static int unbind(b200pf_handle *h, int *batch, DevBufs &bufs) {
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    *batch = 0;
    bufs.release();
    return 0;
}

// One device buffer of a layer, owned by `bufs`: `bytes` uploaded from the host `src`, or with `src` NULL set to the byte `fill`
// on h->stream.  `src` NULL and `fill` < 0 is an absent optional table: NULL (the kernels read it as absent), nothing allocated.
// A zero-byte request allocates 1 byte.
template <typename Tp>
static int dev_alloc(b200pf_handle *h, DevBufs &bufs, Tp *&dst, size_t bytes, const void *src, int fill = -1) {
    dst = nullptr;
    if (!src && fill < 0) return 0;
    void *p = nullptr;
    CU(cudaMalloc(&p, bytes ? bytes : 1));
    bufs.p.push_back(p);
    dst = (Tp *)p;
    if (src) H2D(p, src, bytes);
    else CU(cudaMemsetAsync(p, fill, bytes ? bytes : 1, h->stream));
    return 0;
}

// One per-instance state array of a layer: its device buffer and its bytes.  A layer's table follows the argument order of its
// get / set entry points.
struct StateBuf { void *dev; size_t bytes; };

// b200pf_*_get_state: drain the stream, then a blocking copy of every array the caller asked for (non-NULL destination)
template <size_t N>
static int state_get(b200pf_handle *h, const std::array<StateBuf, N> &t, void *const (&dst)[N]) {
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    for (size_t k = 0; k < N; ++k)
        if (dst[k]) { CU(cudaMemcpy(dst[k], t[k].dev, t[k].bytes, cudaMemcpyDeviceToHost)); h->env_d2h += (int64_t)t[k].bytes; }
    return 0;
}

// b200pf_*_set_state, once the caller has validated every array it was given (so that a rejected call changes nothing): every
// non-NULL source through h2d_sync, then one stream sync
template <size_t N>
static int state_set(b200pf_handle *h, const std::array<StateBuf, N> &t, const void *const (&src)[N]) {
    CU(cudaSetDevice(h->device));
    for (size_t k = 0; k < N; ++k)
        if (src[k]) { H2D(t[k].dev, src[k], t[k].bytes); h->env_h2d += (int64_t)t[k].bytes; }
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// observation layer: grid2op observation vectors + rewards of the bound series, assembled on the device (b200pf_obs.cuh)
// ------------------------------------------------------------------------------------------------
// the observation layer is bound to the current series (b200pf_obs_bind)
static bool obs_bound(const b200pf_handle *h) { return h->obs_batch && h->obs_batch == h->series_batch && h->obs_rows == h->n_rows; }

// ints per instance of the observe input record: the observation layer's, or the record without alerts and alarms when it is unbound
static int obs_stride(const b200pf_handle *h) { return obs_bound(h) ? h->obs.host_stride : h->g.n_line + h->g.n_sub + 3; }

// the observe launch: the bound tables over the series' current results and the input record, writing d_obs / d_reward
static ObsArgs obs_args(const b200pf_handle *h, float *d_obs, float *d_reward) {
    const DevGrid &g = h->g;
    ObsArgs a = h->obs;
    a.batch = h->obs_batch;
    a.n_line = g.n_line; a.n_sub = g.n_sub; a.n_gen = g.n_gen; a.n_hidden = g.n_hidden; a.n_load = g.n_load; a.n_sto = g.n_sto;
    a.n_shunt = g.n_shunt; a.dim_topo = g.dim_topo; a.n_topo_in = g.n_topo_in; a.n_out = g.n_out;
    a.line_or_pos = g.line_or_pos; a.line_ex_pos = g.line_ex_pos;
    a.out = h->x_out ? h->x_out : h->d_out; a.rho = h->x_rho ? h->x_rho : h->d_rho; a.topo = h->d_series_topo;
    a.t = h->d_t; a.scen = h->d_scen; a.chron = h->d_chron; a.n_rows = h->n_rows; a.th_lim = h->d_thlim;
    a.host = h->d_obs_in; a.obs = d_obs; a.reward = d_reward;
    return a;
}

extern "C" int b200pf_obs_bind(b200pf_handle *h, const b200pf_obs_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    if (d->n_seg < 0 || d->n_obs < 0 || (d->n_seg && !d->seg) || !d->calendar || !d->max_step) return fail(B200PF_E_ARG, "bad observation spec");
    const DevGrid &g = h->g;
    if (g.n_gen && (!d->gen_pmin || !d->gen_pmax || !d->gen_ramp_up || !d->gen_ramp_down || !d->gen_cost || !d->gen_renewable))
        return fail(B200PF_E_ARG, "generator tables missing");
    if (g.n_sto && (!d->sto_charge0 || !d->sto_loss_step)) return fail(B200PF_E_ARG, "storage tables missing");
    if (d->reward_kind < B200PF_REWARD_NONE || d->reward_kind > B200PF_REWARD_L2RPN) return fail(B200PF_E_ARG, "unknown reward kind");
    if (d->n_alert < 0 || d->n_alert > ALERT_MAX_LINES) return fail(B200PF_E_ARG, "n_alert out of range");
    if (d->n_alarm < 0 || d->n_alarm > ALARM_MAX_ZONES) return fail(B200PF_E_ARG, "n_alarm out of range");
    for (int s = 0; s < d->n_seg; ++s)
        if (d->seg[3 * s] < 0 || d->seg[3 * s] >= OS_N_SOURCES || d->seg[3 * s + 1] < 0 || d->seg[3 * s + 2] < 0 ||
            d->seg[3 * s + 1] + d->seg[3 * s + 2] > d->n_obs) return fail(B200PF_E_ARG, "observation segment out of range");
    TRY(unbind(h, &h->obs_batch, h->obs_bufs));
    if (h->h_obs_in) { cudaFreeHost(h->h_obs_in); h->h_obs_in = nullptr; }
    if (!h->obs_ev) CU(cudaEventCreateWithFlags(&h->obs_ev, cudaEventDisableTiming));
    h->obs_ev_pending = false;
    const size_t B = (size_t)h->series_batch, R = (size_t)h->n_scen * h->n_rows, nl = (size_t)g.n_line, ng = (size_t)g.n_gen;
    DevBufs &o = h->obs_bufs;
    ObsArgs a{};
    TRY(dev_alloc(h, o, a.seg, (size_t)d->n_seg * 12, d->seg));
    TRY(dev_alloc(h, o, a.calendar, R * 24, d->calendar));
    TRY(dev_alloc(h, o, a.max_step, (size_t)h->n_scen * 4, d->max_step));
    TRY(dev_alloc(h, o, a.maint_time, R * nl * 4, d->maint_time));
    TRY(dev_alloc(h, o, a.maint_dur, R * nl * 4, d->maint_dur));
    TRY(dev_alloc(h, o, a.gen_pmin, ng * 4, d->gen_pmin));
    TRY(dev_alloc(h, o, a.gen_pmax, ng * 4, d->gen_pmax));
    TRY(dev_alloc(h, o, a.gen_ramp_up, ng * 4, d->gen_ramp_up));
    TRY(dev_alloc(h, o, a.gen_ramp_down, ng * 4, d->gen_ramp_down));
    TRY(dev_alloc(h, o, a.gen_cost, ng * 4, d->gen_cost));
    TRY(dev_alloc(h, o, a.gen_renewable, ng, d->gen_renewable));
    TRY(dev_alloc(h, o, a.sto_charge0, (size_t)g.n_sto * 4, d->sto_charge0));
    TRY(dev_alloc(h, o, a.sto_loss_step, (size_t)g.n_sto * 4, d->sto_loss_step));
    TRY(dev_alloc(h, o, a.ts_over, B * nl * 4, nullptr, 0));
    TRY(dev_alloc(h, o, a.ts_prot, B * nl * 4, nullptr, 0));
    TRY(dev_alloc(h, o, a.stamp, B * 4, nullptr, 0xff));
    TRY(dev_alloc(h, o, a.go_row, B * 4, nullptr, 0xff));
    a.n_seg = d->n_seg; a.n_obs = d->n_obs; a.delta_time = d->delta_time; a.redisp_available = d->redisp_available;
    a.reward_kind = d->reward_kind; a.max_regret = d->max_regret; a.reward_min = d->reward_min; a.reward_illegal = d->reward_illegal;
    a.dts_hours = d->dts_hours; a.soft_thr = d->soft_thr;
    a.n_alert = d->n_alert; a.n_alarm = d->n_alarm;
    a.host_stride = g.n_line + g.n_sub + 3 + (d->n_alert ? 6 * d->n_alert + 1 : 0) + (d->n_alarm ? d->n_alarm + 4 : 0);
    if (cudaMallocHost(&h->h_obs_in, B * a.host_stride * 4) != cudaSuccess) return fail(B200PF_E_CUDA, "pinned host allocation failed");
    TRY(dev_alloc(h, o, h->d_obs_in, B * a.host_stride * 4, nullptr, 0));
    CU(cudaStreamSynchronize(h->stream));
    h->obs = a; h->obs_rows = h->n_rows; h->obs_batch = h->series_batch;
    return 0;
}

extern "C" int b200pf_observe(b200pf_handle *h, const int32_t *host_in, float *d_obs, float *d_reward) {
    if (!h || !host_in || !d_obs) return fail(B200PF_E_ARG, "null pointer");
    if (!obs_bound(h)) return fail(B200PF_E_STATE, "observation not bound to the current series (b200pf_obs_bind)");
    CU(cudaSetDevice(h->device));
    const ObsArgs a = obs_args(h, d_obs, d_reward);
    const size_t in_bytes = (size_t)a.batch * a.host_stride * 4;
    if (h->obs_ev_pending) CU(cudaEventSynchronize(h->obs_ev));        // the previous copy out of the pinned record has left
    memcpy(h->h_obs_in, host_in, in_bytes);
    CU(cudaMemcpyAsync(h->d_obs_in, h->h_obs_in, in_bytes, cudaMemcpyHostToDevice, h->stream));
    CU(cudaEventRecord(h->obs_ev, h->stream));
    h->obs_ev_pending = true;
    pf_kernel_observe<<<(a.batch + 3) / 4, 128, 0, h->stream>>>(a);
    CU(cudaGetLastError());
    h->obs_launches++; h->obs_h2d_bytes += (int64_t)in_bytes;
    return 0;
}

extern "C" int b200pf_obs_stats(const b200pf_handle *h, int64_t *out4) {
    if (!h || !out4) return fail(B200PF_E_ARG, "null pointer");
    out4[0] = h->obs_launches; out4[1] = h->obs_h2d_bytes; out4[2] = h->d2h_bytes;
    out4[3] = (int64_t)h->obs_batch * ((int64_t)h->obs.n_obs * 4 + (h->obs.reward_kind ? 4 : 0));
    return 0;
}

extern "C" int b200pf_sync(b200pf_handle *h) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" uint64_t b200pf_stream(b200pf_handle *h) { return h ? (uint64_t)(uintptr_t)h->stream : 0; }
extern "C" int64_t b200pf_launch_count(const b200pf_handle *h) { return h ? h->launches : 0; }
extern "C" int b200pf_last_launch_info(const b200pf_handle *h, int *smem_bytes, int *threads_per_instance, int *grid_blocks,
                                       int *block_threads) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (smem_bytes) *smem_bytes = h->last_smem;
    if (threads_per_instance) *threads_per_instance = h->last_T;
    if (grid_blocks) *grid_blocks = h->last_grid;
    if (block_threads) *block_threads = h->last_block;
    return 0;
}
extern "C" int b200pf_last_launch_config(const b200pf_handle *h, int *cfg8) {
    if (!h || !cfg8) return fail(B200PF_E_ARG, "null pointer");
    for (int k = 0; k < 8; ++k) cfg8[k] = h->last_cfg[k];
    return 0;
}

// ------------------------------------------------------------------------------------------------
// device environment state: BatchedEnv's bookkeeping on the device (b200pf_env.cuh)
// ------------------------------------------------------------------------------------------------
static bool env_bound(const b200pf_handle *h) { return h->env_batch && h->env_batch == h->series_batch && h->env.topo == h->d_series_topo; }

// a layer bound for `batch` instances (the opponent, the alerts, the alarms) belongs to the current environment
static bool layer_bound(const b200pf_handle *h, int batch) { return env_bound(h) && batch == h->env_batch; }

extern "C" int b200pf_env_bind(b200pf_handle *h, const b200pf_env_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    const DevGrid &g = h->g;
    if (d->max_sub <= 0 || !d->sub_pos || !d->line_of_pos || !d->other_end_pos || !d->topo0 || !d->t0 || (d->n_iso_seg && !d->iso_seg) ||
        (d->n_iso_cols && !d->iso_cols) || d->n_iso_seg < 0 || d->n_iso_cols < 0 || (!d->maint) != (!d->maint_time) || (d->maint && !d->maint_dur) ||
        (!d->haz) != (!d->haz_dur))
        return fail(B200PF_E_ARG, "bad environment tables");
    if (!d->last_bus || !d->line_cd || !d->sub_cd || !d->done || !d->is_illegal || !d->newly_done || !d->current_step || !d->status)
        return fail(B200PF_E_ARG, "state buffers missing");
    if (g.n_slot > ENV_MAX_SLOT) return fail(B200PF_E_CAPACITY, "more bus slots than the device bus count handles");
    for (int k = 0; k < g.n_sub * d->max_sub; ++k) if (d->sub_pos[k] < -1 || d->sub_pos[k] >= g.dim_topo) return fail(B200PF_E_ARG, "sub_pos out of range");
    for (int k = 0; k < g.dim_topo; ++k)
        if (d->line_of_pos[k] < -1 || d->line_of_pos[k] >= g.n_line || d->other_end_pos[k] < -1 || d->other_end_pos[k] >= g.dim_topo)
            return fail(B200PF_E_ARG, "line_of_pos / other_end_pos out of range");
    for (int k = 0; k < d->n_iso_cols; ++k) if (d->iso_cols[k] < 0 || d->iso_cols[k] >= g.n_topo_in) return fail(B200PF_E_ARG, "iso_cols out of range");
    for (int k = 0; k < d->n_iso_seg; ++k) if (d->iso_seg[k] < 0 || d->iso_seg[k] > d->n_iso_cols) return fail(B200PF_E_ARG, "iso_seg out of range");
    const int B = h->series_batch;
    for (int i = 0; i < B; ++i) if (d->t0[i] < 0 || d->t0[i] >= h->n_rows) return fail(B200PF_E_ARG, "t0 out of range");
    TRY(unbind(h, &h->env_batch, h->env_bufs));
    if (!h->h_env_ctl && cudaMallocHost(&h->h_env_ctl, ENV_CTL_WORDS * 4) != cudaSuccess) return fail(B200PF_E_CUDA, "pinned host allocation failed");
    std::vector<int32_t> epos, esub;           // every element of the record and its substation (b200pf_grid_max_active_buses)
    const HostGrid &hg = h->hg;
    for (int k = 0; k < hg.n_line; ++k) { epos.push_back(hg.line_or_pos[k]); esub.push_back(hg.line_or_sub[k]); }
    for (int k = 0; k < hg.n_line; ++k) { epos.push_back(hg.line_ex_pos[k]); esub.push_back(hg.line_ex_sub[k]); }
    for (int k = 0; k < hg.n_unit; ++k) { epos.push_back(hg.unit_pos[k]); esub.push_back(hg.unit_sub[k]); }
    for (int k = 0; k < hg.n_load; ++k) { epos.push_back(hg.load_pos[k]); esub.push_back(hg.load_sub[k]); }
    for (int k = 0; k < hg.n_sto; ++k) { epos.push_back(hg.sto_pos[k]); esub.push_back(hg.sto_sub[k]); }
    for (int k = 0; k < hg.n_shunt; ++k) { epos.push_back(hg.dim_topo + k); esub.push_back(hg.sh_sub[k]); }
    const size_t R = (size_t)h->n_scen * h->n_rows * g.n_line, nl = (size_t)g.n_line, nt = (size_t)g.n_topo_in, Bs = (size_t)B;
    DevBufs &o = h->env_bufs;
    EnvArgs a{};
    TRY(dev_alloc(h, o, a.sub_pos, (size_t)g.n_sub * d->max_sub * 4, d->sub_pos));
    TRY(dev_alloc(h, o, a.line_of_pos, (size_t)g.dim_topo * 4, d->line_of_pos));
    TRY(dev_alloc(h, o, a.other_end_pos, (size_t)g.dim_topo * 4, d->other_end_pos));
    TRY(dev_alloc(h, o, a.elem_pos, epos.size() * 4, epos.data()));
    TRY(dev_alloc(h, o, a.elem_sub, esub.size() * 4, esub.data()));
    TRY(dev_alloc(h, o, a.maint, R, d->maint));
    TRY(dev_alloc(h, o, a.haz, R, d->haz));
    TRY(dev_alloc(h, o, a.maint_time, R * 4, d->maint_time));
    TRY(dev_alloc(h, o, a.maint_dur, R * 4, d->maint_dur));
    TRY(dev_alloc(h, o, a.haz_dur, R * 4, d->haz_dur));
    TRY(dev_alloc(h, o, a.iso_cols, (size_t)d->n_iso_cols * 4, d->iso_cols));
    TRY(dev_alloc(h, o, a.iso_seg, (size_t)d->n_iso_seg * 4, d->iso_seg));
    TRY(dev_alloc(h, o, a.topo0, Bs * nt, d->topo0));
    TRY(dev_alloc(h, o, a.t0, Bs * 4, d->t0));
    TRY(dev_alloc(h, o, a.aff_l, Bs * nl, nullptr, 0));
    TRY(dev_alloc(h, o, a.aff_s, Bs * 4, nullptr, 0xff));
    TRY(dev_alloc(h, o, a.row_used, Bs * 4, nullptr, 0));
    TRY(dev_alloc(h, o, a.stale, Bs, nullptr, 0));
    TRY(dev_alloc(h, o, a.cap_dirty, Bs, nullptr, 1));
    TRY(dev_alloc(h, o, a.obs_reset, Bs, nullptr, 1));
    TRY(dev_alloc(h, o, a.nb_inst, Bs * 4, nullptr, 0));
    TRY(dev_alloc(h, o, a.copy_list, Bs * 4, nullptr, 0));
    TRY(dev_alloc(h, o, a.copy_rows, Bs * nt, nullptr, 0));
    TRY(dev_alloc(h, o, a.ctl, ENV_CTL_WORDS * 4, nullptr, 0));
    a.batch = B;
    a.n_line = g.n_line; a.n_sub = g.n_sub; a.dim_topo = g.dim_topo; a.n_topo_in = g.n_topo_in; a.n_busbar = g.n_busbar; a.n_slot = g.n_slot;
    a.max_sub = d->max_sub; a.n_rows = h->n_rows;
    a.line_or_pos = g.line_or_pos; a.line_ex_pos = g.line_ex_pos; a.n_elem = (int)epos.size();
    a.cd_line = d->cd_line; a.cd_sub = d->cd_sub; a.cd_reco = d->cd_reco;
    a.n_iso_seg = d->n_iso_seg; a.n_iso_cols = d->n_iso_cols; a.scen = h->d_scen;
    a.topo = h->d_series_topo; a.t = h->d_t;
    a.lib_done = h->d_done; a.pcount = h->d_pcount; a.ts_over = h->d_tsover; a.lib_disc = h->d_disc; a.trip = h->d_trip; a.incdone = h->d_incdone;
    a.last_bus = d->last_bus; a.line_cd = d->line_cd; a.sub_cd = d->sub_cd; a.done = d->done; a.is_illegal = d->is_illegal;
    a.newly_done = d->newly_done; a.current_step = d->current_step; a.status_out = d->status;
    // the stale flags start set: the first step that refreshes the plans copies every row into the mirror
    CU(cudaMemsetAsync(a.stale, 1, Bs, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->env = a;
    h->env_mirror.assign(Bs * nt, 0);
    h->env_topo0.assign(d->topo0, d->topo0 + Bs * nt);
    h->env_batch = B;
    return 0;
}

static inline unsigned env_grid(int n) { return (unsigned)((n + 127) / 128); }

// What the env launches run besides the EnvArgs: the bound opponent (kind OPP_NONE: none), the line alerts (n = 0: none; they read
// the attacked lines the opponent of the same launches writes), the alarms (n = 0: none) and the observe input record (NULL when
// the observation layer is not bound to this series).  An error when a GeometricOpponent lacks its schedules, a multi-area one its
// areas, or when the observation layer's alert or alarm values do not match the bound alerts or alarms.
struct EnvLayers { OppArgs opp; AlertArgs al; AlarmArgs am; ActArgs act; int32_t *obs_rec; int obs_stride; };
static int env_layers(const b200pf_handle *h, EnvLayers *l) {
    if (h->opp_batch && h->opp.kind == OPP_GEOMETRIC && !h->opp_geo_bound)
        return fail(B200PF_E_STATE, "GeometricOpponent bound without its schedules (b200pf_opp_geo_bind)");
    if (h->opp_batch && h->opp.kind == OPP_GEOMETRIC_MULTI && !h->opp_multi_bound)
        return fail(B200PF_E_STATE, "GeometricOpponentMultiArea bound without its areas (b200pf_opp_multi_bind)");
    l->opp = OppArgs{};
    if (layer_bound(h, h->opp_batch)) {
        l->opp = h->opp;
        l->opp.rho = h->x_rho ? h->x_rho : h->d_rho;                  // what the previous step wrote
    }
    l->al = AlertArgs{};
    if (layer_bound(h, h->alert_batch)) {
        l->al = h->alert;
        if (l->opp.kind == OPP_GEOMETRIC_MULTI && h->opp_multi_bound) { l->al.attack = h->opp_multi.attack_lines; l->al.attack_stride = h->opp_multi.n_area; }
        else if (l->opp.kind != OPP_NONE) { l->al.attack = l->opp.attack_line; l->al.attack_stride = 1; }
    }
    l->am = layer_bound(h, h->alarm_batch) ? h->alarm : AlarmArgs{};
    l->act = layer_bound(h, h->act_batch) ? h->act : ActArgs{};      // (aff_sub NULL: no rules bound, DefaultRules at 1 / 1)
    const bool obs = obs_bound(h);
    l->obs_rec = obs ? h->d_obs_in : nullptr;
    l->obs_stride = obs_stride(h);
    if (obs && h->obs.n_alert != l->al.n)
        return fail(B200PF_E_STATE, "the observation layer and the line alerts disagree on dim_alerts (b200pf_obs_bind / b200pf_alert_bind)");
    if (obs && h->obs.n_alarm != l->am.n)
        return fail(B200PF_E_STATE, "the observation layer and the alarms disagree on dim_alarms (b200pf_obs_bind / b200pf_alarm_bind)");
    return 0;
}

// Where env_step takes the agent's action from: the sub_id / line_id pair (b200pf_env_step), the vector buffers of b200pf_act_bind
// (b200pf_env_step_act), or the rows of the bound action table picked by one id per instance (b200pf_env_step_ids)
enum ActMode { ACT_LEGACY = 0, ACT_VECTORS = 1, ACT_IDS = 2 };

static int env_step(b200pf_handle *h, const int32_t *d_sub_id, const int8_t *d_sub_bus, int sub_bus_stride, int sub_bus_cols,
                    const int32_t *d_line_id, const int32_t *d_line_status, ActMode mode, const int32_t *d_action_id, int from_reset,
                    int is_dc, int max_iter, double tol_mva, int tight_cap, int stamp) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    if ((!d_sub_id) != (!d_sub_bus) || (!d_line_id) != (!d_line_status)) return fail(B200PF_E_ARG, "ids without values");
    if (d_sub_id && (sub_bus_cols < h->env.max_sub || sub_bus_stride < sub_bus_cols)) return fail(B200PF_E_ARG, "sub_bus narrower than the largest substation");
    if (mode != ACT_LEGACY && !layer_bound(h, h->act_batch)) return fail(B200PF_E_STATE, "no action buffers bound to the current environment (b200pf_act_bind)");
    if (mode == ACT_IDS && !h->n_act) return fail(B200PF_E_STATE, "no action table bound (b200pf_act_table_bind)");
    if (mode == ACT_IDS && !d_action_id) return fail(B200PF_E_ARG, "null action ids");
    EnvLayers l;
    TRY(env_layers(h, &l));
    l.act.vec = mode != ACT_LEGACY && !from_reset ? 1 : 0;
    ActIds ids{};
    if (mode == ACT_IDS) {
        l.act.set_bus = h->tab_set_bus; l.act.change_bus = h->tab_change_bus;
        l.act.set_status = h->tab_set_status; l.act.change_status = h->tab_change_status;
        if (!from_reset) { ids.id = d_action_id; ids.n = h->n_act; }
    }
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const int B = h->env_batch;
    const size_t nt = (size_t)g.n_topo_in;
    EnvArgs a = h->env;
    a.sub_id = from_reset ? nullptr : d_sub_id; a.sub_bus = from_reset ? nullptr : d_sub_bus;
    a.sub_bus_stride = sub_bus_stride; a.sub_bus_cols = sub_bus_cols;
    a.line_id = from_reset ? nullptr : d_line_id; a.line_status = from_reset ? nullptr : d_line_status;
    a.from_reset = from_reset ? 1 : 0; a.tight_cap = tight_cap ? 1 : 0; a.prot = h->prot;
    // 1. validation + apply (the apply kernel writes nothing when an input was rejected)
    CU(cudaMemsetAsync(a.ctl, 0, ENV_CTL_WORDS * 4, h->stream));
    if (a.sub_id || a.line_id || l.act.vec) {
        pf_kernel_env_validate<<<env_grid(B), 128, 0, h->stream>>>(a, l.act, ids);
        CU(cudaGetLastError());
    }
    pf_kernel_env_apply<<<env_grid(B), 128, 0, h->stream>>>(a, l.opp, h->opp_geo, h->opp_multi, l.act, ids);
    CU(cudaGetLastError());
    // 2. the step's one host wait: dirty count, bus cap, input error
    CU(cudaMemcpyAsync(h->h_env_ctl, a.ctl, ENV_CTL_WORDS * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->env_d2h += ENV_CTL_WORDS * 4; h->env_waits++;
    const int32_t *c = h->h_env_ctl;
    if (c[ENV_CTL_ERR])
        return fail(B200PF_E_ARG, ids.id ? "action id outside [0, n) of the bound action table"
                                : l.act.vec ? "vector action out of range (busbar outside [-1, n_busbar], -1 on an element other than a line end, "
                                              "change_bus without two busbars, line status outside {-1, 0, 1}, or a flag other than 0 / 1)"
                                            : "action out of range (substation / line id outside [-1, n), busbar outside [-1, n_busbar])");
    h->env_illegal += c[ENV_CTL_N_ILLEGAL];
    int nb_cap = 0;
    if (tight_cap) {
        nb_cap = c[ENV_CTL_CAP_MAX];
        if (nb_cap > 17) nb_cap = (nb_cap + 7) / 8 * 8;
        if (nb_cap > g.n_slot) nb_cap = g.n_slot;
    }
    h->env_last_cap = nb_cap; h->env_last_dirty = c[ENV_CTL_N_DIRTY];
    // 3.-4. a changed topology: patch the mirror with the compacted rows, then the plans of the full mirror (as series_set_topo)
    if (c[ENV_CTL_N_DIRTY] > 0) {
        const int n = c[ENV_CTL_N_COPY];
        if (n < 0 || n > B) return fail(B200PF_E_STATE, "bad row count");
        if (n) {
            h->env_list.resize(n); h->env_rows.resize((size_t)n * nt);
            CU(cudaMemcpyAsync(h->env_list.data(), a.copy_list, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
            CU(cudaMemcpyAsync(h->env_rows.data(), a.copy_rows, (size_t)n * nt, cudaMemcpyDeviceToHost, h->stream));
            CU(cudaMemsetAsync(a.stale, 0, (size_t)B, h->stream));
            CU(cudaStreamSynchronize(h->stream));
            h->env_d2h += (int64_t)n * (4 + (int64_t)nt); h->env_waits++;
            for (int k = 0; k < n; ++k) {
                const int i = h->env_list[k];
                if (i < 0 || i >= B) return fail(B200PF_E_STATE, "bad instance in the row list");
                memcpy(h->env_mirror.data() + (size_t)i * nt, h->env_rows.data() + (size_t)k * nt, nt);
            }
        }
        int rc = series_plans(h, h->env_mirror.data());
        if (rc) return rc;
        h->series_dev_topo_ahead = false;
        h->env_plan_refresh++;
    }
    // 5. the series step (kernel selection, protections, cascades and safety net unchanged)
    h->next_reset = from_reset ? 1 : 0;
    int rc = b200pf_series_step(h, is_dc, max_iter, tol_mva, nb_cap);
    if (rc) return rc;
    // 6. trips, isolated busbars, cooldowns, game over, the observe layer's input record
    a.status = h->x_status ? h->x_status : h->d_status;
    a.disc = h->prot ? h->d_disc : nullptr;
    a.obs_in = l.obs_rec; a.obs_stride = l.obs_stride; a.stamp = stamp;
    pf_kernel_env_post<<<env_grid(B), 128, 0, h->stream>>>(a, l.al, l.am, l.act);
    CU(cudaGetLastError());
    h->env_steps++;
    return 0;
}

extern "C" int b200pf_env_step(b200pf_handle *h, const int32_t *d_sub_id, const int8_t *d_sub_bus, int sub_bus_stride, int sub_bus_cols,
                               const int32_t *d_line_id, const int32_t *d_line_status, int from_reset, int is_dc, int max_iter,
                               double tol_mva, int tight_cap, int stamp) {
    return env_step(h, d_sub_id, d_sub_bus, sub_bus_stride, sub_bus_cols, d_line_id, d_line_status, ACT_LEGACY, nullptr, from_reset, is_dc,
                    max_iter, tol_mva, tight_cap, stamp);
}

extern "C" int b200pf_env_step_act(b200pf_handle *h, int from_reset, int is_dc, int max_iter, double tol_mva, int tight_cap, int stamp) {
    return env_step(h, nullptr, nullptr, 0, 0, nullptr, nullptr, ACT_VECTORS, nullptr, from_reset, is_dc, max_iter, tol_mva, tight_cap, stamp);
}

extern "C" int b200pf_env_step_ids(b200pf_handle *h, const int32_t *d_action_id, int from_reset, int is_dc, int max_iter, double tol_mva,
                                   int tight_cap, int stamp) {
    return env_step(h, nullptr, nullptr, 0, 0, nullptr, nullptr, ACT_IDS, d_action_id, from_reset, is_dc, max_iter, tol_mva, tight_cap, stamp);
}

extern "C" int b200pf_act_table_bind(b200pf_handle *h, const b200pf_act_table_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!layer_bound(h, h->act_batch)) return fail(B200PF_E_STATE, "no action rules bound to the current environment (b200pf_act_bind)");
    if (d->n_act <= 0 || !d->set_bus || !d->change_bus || !d->set_status || !d->change_status) return fail(B200PF_E_ARG, "empty action table");
    const HostGrid &hg = h->hg;
    // every row under the rules of a vector action (act_input_ok, run here on the host), before anything is bound
    std::vector<int32_t> line_of_pos(hg.dim_topo, -1);
    for (int k = 0; k < hg.n_line; ++k) line_of_pos[hg.line_or_pos[k]] = k, line_of_pos[hg.line_ex_pos[k]] = k;
    EnvArgs e{};
    e.n_line = hg.n_line; e.dim_topo = hg.dim_topo; e.n_busbar = hg.n_busbar; e.line_of_pos = line_of_pos.data();
    ActArgs r{};
    r.set_bus = d->set_bus; r.change_bus = d->change_bus; r.set_status = d->set_status; r.change_status = d->change_status;
    for (int i = 0; i < d->n_act; ++i)
        if (!act_input_ok(e, r, i)) return fail(B200PF_E_ARG, "action table row " + std::to_string(i) + " out of range (busbar outside [-1, n_busbar], "
                                                                "-1 on an element other than a line end, change_bus without two busbars, line status outside {-1, 0, 1}, or a flag other than 0 / 1)");
    TRY(unbind(h, &h->n_act, h->act_table_bufs));
    const size_t n = (size_t)d->n_act, nt = (size_t)hg.dim_topo, nl = (size_t)hg.n_line;
    DevBufs &o = h->act_table_bufs;
    TRY(dev_alloc(h, o, h->tab_set_bus, n * nt, d->set_bus));
    TRY(dev_alloc(h, o, h->tab_change_bus, n * nt, d->change_bus));
    TRY(dev_alloc(h, o, h->tab_set_status, n * nl, d->set_status));
    TRY(dev_alloc(h, o, h->tab_change_status, n * nl, d->change_status));
    CU(cudaStreamSynchronize(h->stream));
    h->n_act = d->n_act;
    return 0;
}

extern "C" int b200pf_act_bind(b200pf_handle *h, const b200pf_act_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    const HostGrid &hg = h->hg;
    if (d->max_sub_changed < 0 || d->max_line_status_changed < 0 || d->n_area < 0 || d->n_area > ACT_MAX_AREA ||
        (d->n_area && (!d->sub_area || !d->line_area)))
        return fail(B200PF_E_ARG, "bad action rules");
    if (!d->set_bus || !d->change_bus || !d->set_status || !d->change_status || !d->is_ambiguous) return fail(B200PF_E_ARG, "action buffers missing");
    if (d->n_area) {
        const uint32_t areas = d->n_area == 32 ? 0xffffffffu : (1u << d->n_area) - 1u;
        for (int s = 0; s < hg.n_sub; ++s) if (d->sub_area[s] & ~areas) return fail(B200PF_E_ARG, "a substation in an area past n_area");
        for (int l = 0; l < hg.n_line; ++l) if (d->line_area[l] & ~areas) return fail(B200PF_E_ARG, "a line in an area past n_area");
    }
    TRY(unbind(h, &h->act_batch, h->act_bufs));
    // the substation of every topology position (the shunts sit past dim_topo)
    std::vector<int32_t> sub_of_pos(hg.dim_topo, 0);
    for (int k = 0; k < hg.n_line; ++k) { sub_of_pos[hg.line_or_pos[k]] = hg.line_or_sub[k]; sub_of_pos[hg.line_ex_pos[k]] = hg.line_ex_sub[k]; }
    for (int k = 0; k < hg.n_unit; ++k) if (hg.unit_pos[k] >= 0 && hg.unit_pos[k] < hg.dim_topo) sub_of_pos[hg.unit_pos[k]] = hg.unit_sub[k];
    for (int k = 0; k < hg.n_load; ++k) sub_of_pos[hg.load_pos[k]] = hg.load_sub[k];
    for (int k = 0; k < hg.n_sto; ++k) sub_of_pos[hg.sto_pos[k]] = hg.sto_sub[k];
    const size_t B = (size_t)h->env_batch;
    ActArgs r{};
    r.max_sub = d->max_sub_changed; r.max_line = d->max_line_status_changed; r.n_area = d->n_area;
    DevBufs &o = h->act_bufs;
    TRY(dev_alloc(h, o, r.sub_of_pos, sub_of_pos.size() * 4, sub_of_pos.data()));
    if (d->n_area) {
        TRY(dev_alloc(h, o, r.sub_area, (size_t)hg.n_sub * 4, d->sub_area));
        TRY(dev_alloc(h, o, r.line_area, (size_t)hg.n_line * 4, d->line_area));
    }
    TRY(dev_alloc(h, o, r.aff_sub, B * (size_t)hg.n_sub, nullptr, 0));
    r.set_bus = d->set_bus; r.change_bus = d->change_bus; r.set_status = d->set_status; r.change_status = d->change_status;
    r.is_ambiguous = d->is_ambiguous;
    CU(cudaMemsetAsync(r.is_ambiguous, 0, B, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->act = r; h->act_batch = (int)B;
    return 0;
}

extern "C" int b200pf_env_reset(b200pf_handle *h, const uint8_t *d_mask, const int32_t *d_rows) {
    if (!h || !d_mask) return fail(B200PF_E_ARG, "null pointer");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    EnvLayers l;
    TRY(env_layers(h, &l));
    CU(cudaSetDevice(h->device));
    const DevGrid &g = h->g;
    const int B = h->env_batch;
    const size_t nt = (size_t)g.n_topo_in;
    EnvArgs a = h->env;
    a.reset_mask = d_mask; a.reset_rows = d_rows;
    a.obs_in = l.obs_rec; a.obs_stride = l.obs_stride;
    pf_kernel_env_reset<<<env_grid(B), 128, 0, h->stream>>>(a, l.opp, h->opp_geo, h->opp_multi, l.al, l.am, l.act);
    CU(cudaGetLastError());
    // the plans of the reset rows, looked up now and over the same topology as b200pf_series_reset_instances does for the host
    // path, so that both paths make the same plan lookups in the same calls (which plans a call builds, their ids, and the kernel
    // it chooses depend on the new topologies of each call)
    h->env_mask.resize(B);
    CU(cudaMemcpyAsync(h->env_mask.data(), d_mask, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->env_d2h += B; h->env_waits++;
    std::vector<int8_t> all;
    bool any = false;
    for (int i = 0; i < B; ++i) any |= h->env_mask[i] != 0;
    if (!any) return 0;
    if (h->series_dev_topo_ahead || h->h_series_topo.size() != (size_t)B * nt) {
        all.resize((size_t)B * nt);
        CU(cudaMemcpy(all.data(), h->d_series_topo, all.size(), cudaMemcpyDeviceToHost));
        h->env_d2h += (int64_t)all.size();
    } else all = h->h_series_topo;
    for (int i = 0; i < B; ++i)
        if (h->env_mask[i]) memcpy(all.data() + (size_t)i * nt, h->env_topo0.data() + (size_t)i * nt, nt);
    h->series_dev_topo_ahead = false;
    return series_plans(h, all.data());
}

extern "C" int b200pf_env_get_state(b200pf_handle *h, int8_t *topo, int32_t *t, int32_t *nb_inst, uint8_t *cap_dirty, uint8_t *obs_reset) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    const size_t B = (size_t)h->env_batch, nt = (size_t)h->g.n_topo_in;
    const std::array<StateBuf, 5> tab = {{{h->d_series_topo, B * nt}, {h->d_t, B * 4}, {h->env.nb_inst, B * 4}, {h->env.cap_dirty, B},
                                          {h->env.obs_reset, B}}};
    return state_get(h, tab, {topo, t, nb_inst, cap_dirty, obs_reset});
}

extern "C" int b200pf_env_set_state(b200pf_handle *h, const int8_t *topo, const int32_t *nb_inst, const uint8_t *cap_dirty, const uint8_t *obs_reset,
                                    const int32_t *obs_in) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    CU(cudaSetDevice(h->device));
    const size_t B = (size_t)h->env_batch, nt = (size_t)h->g.n_topo_in;
    const bool obs = obs_bound(h);
    // a new topology leaves no row stale: the flags are cleared on the stream ahead of the copies (state_set's closing sync
    // covers it), the host mirror is patched once the topology is on the device
    if (topo) CU(cudaMemsetAsync(h->env.stale, 0, B, h->stream));
    if (obs_in && obs && h->obs_ev_pending) CU(cudaEventSynchronize(h->obs_ev));    // (b200pf_observe's copy into the same record has left)
    const std::array<StateBuf, 5> tab = {{{h->d_series_topo, B * nt}, {h->env.nb_inst, B * 4}, {h->env.cap_dirty, B}, {h->env.obs_reset, B},
                                          {h->d_obs_in, B * (size_t)obs_stride(h) * 4}}};
    TRY(state_set(h, tab, {topo, nb_inst, cap_dirty, obs_reset, obs ? obs_in : nullptr}));
    if (topo) h->env_mirror.assign(topo, topo + B * nt);
    return 0;
}

extern "C" int b200pf_env_pointers(b200pf_handle *h, int8_t **d_topo, int32_t **d_t, int32_t **d_disc) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!h->series_batch) return fail(B200PF_E_STATE, "series not bound");
    if (d_topo) *d_topo = h->d_series_topo;
    if (d_t) *d_t = h->d_t;
    if (d_disc) *d_disc = h->d_disc;
    return 0;
}

extern "C" int b200pf_observe_device(b200pf_handle *h, float *d_obs, float *d_reward) {
    if (!h || !d_obs) return fail(B200PF_E_ARG, "null pointer");
    if (!obs_bound(h)) return fail(B200PF_E_STATE, "observation not bound to the current series (b200pf_obs_bind)");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    CU(cudaSetDevice(h->device));
    const ObsArgs a = obs_args(h, d_obs, d_reward);
    pf_kernel_observe<<<(a.batch + 3) / 4, 128, 0, h->stream>>>(a);
    CU(cudaGetLastError());
    EnvArgs e = h->env;                  // the reset flags have been consumed
    e.obs_in = h->d_obs_in; e.obs_stride = a.host_stride;
    pf_kernel_env_observed<<<env_grid(e.batch), 128, 0, h->stream>>>(e);
    CU(cudaGetLastError());
    h->obs_launches++;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// line-attack opponent of the device environment (b200pf_opp.cuh)
// ------------------------------------------------------------------------------------------------
// the checks of the opponent's random states and schedule counters, shared by its binds and its set_state entry points: n MT19937
// positions; n blocks of schedule counters, `stride` ints each (OPP_GEO_CTR, or OPP_AREA_CTR per area: the same leading counters)
static int mt_pos_check(const int32_t *mt_pos, size_t n) {
    for (size_t k = 0; mt_pos && k < n; ++k)
        if (mt_pos[k] < 0 || mt_pos[k] > OPP_MT_N) return fail(B200PF_E_ARG, "random state position out of range");
    return 0;
}
static int sched_ctr_check(const int32_t *ctr, size_t n, int stride, int cap) {
    for (size_t k = 0; ctr && k < n; ++k) {
        const int32_t *c = ctr + k * stride;
        if (c[OPP_GEO_N] < 0 || c[OPP_GEO_N] > cap || c[OPP_GEO_COUNTER] < 0) return fail(B200PF_E_ARG, "schedule counters out of range");
    }
    return 0;
}

extern "C" int b200pf_opp_bind(b200pf_handle *h, const b200pf_opp_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    const DevGrid &g = h->g;
    if ((d->kind != OPP_RANDOM_LINE && d->kind != OPP_WEIGHTED_RANDOM && d->kind != OPP_GEOMETRIC && d->kind != OPP_GEOMETRIC_MULTI) ||
        d->n_attack < 1 ||
        d->n_attack > OPP_MAX_ATTACK || !d->lines ||
        (d->kind == OPP_WEIGHTED_RANDOM && (!d->rho_norm || d->attack_period < 1)) || d->attack_duration < 0 || d->attack_cooldown < 0 ||
        !d->mt || !d->mt_pos || !d->attack_line || !d->attack_dur || !d->budget)
        return fail(B200PF_E_ARG, "bad opponent description");
    for (int k = 0; k < d->n_attack; ++k) if (d->lines[k] < 0 || d->lines[k] >= g.n_line) return fail(B200PF_E_ARG, "attacked line out of range");
    const int B = h->env_batch;
    TRY(mt_pos_check(d->mt_pos, (size_t)B));
    TRY(unbind(h, &h->opp_batch, h->opp_bufs));
    h->opp_geo = OppGeoArgs{}; h->opp_geo_bound = false;
    h->opp_multi = OppMultiArgs{}; h->opp_multi_bound = false;
    OppArgs o{};
    o.kind = d->kind; o.n_attack = d->n_attack;
    o.attack_period = d->attack_period; o.attack_duration = d->attack_duration; o.attack_cooldown = d->attack_cooldown;
    o.budget_per_ts = d->budget_per_ts; o.init_budget = d->init_budget;
    o.budget = d->budget; o.attack_line = d->attack_line; o.attack_dur = d->attack_dur;
    // every instance starts from OpponentSpace.reset()
    std::vector<double> bud((size_t)B, (double)d->init_budget);
    std::vector<int32_t> ctr((size_t)B * OPP_CTR);
    for (int i = 0; i < B; ++i) {
        ctr[(size_t)i * OPP_CTR + OPP_CTR_DURATION] = 0; ctr[(size_t)i * OPP_CTR + OPP_CTR_COOLDOWN] = d->attack_cooldown;
        ctr[(size_t)i * OPP_CTR + OPP_CTR_LAST] = -1; ctr[(size_t)i * OPP_CTR + OPP_CTR_NEXT] = OPP_NEXT_UNSET;
    }
    DevBufs &ob = h->opp_bufs;
    TRY(dev_alloc(h, ob, o.lines, (size_t)d->n_attack * 4, d->lines));
    TRY(dev_alloc(h, ob, o.rho_norm, (size_t)d->n_attack * 8, d->rho_norm, 0));    // (read by kind OPP_WEIGHTED_RANDOM only)
    TRY(dev_alloc(h, ob, o.budget64, (size_t)B, nullptr, 0));
    TRY(dev_alloc(h, ob, o.ctr, ctr.size() * 4, ctr.data()));
    TRY(dev_alloc(h, ob, o.mt, (size_t)B * OPP_MT_N * 4, d->mt));
    TRY(dev_alloc(h, ob, o.mt_pos, (size_t)B * 4, d->mt_pos));
    H2D(o.budget, bud.data(), (size_t)B * 8);
    CU(cudaStreamSynchronize(h->stream));
    h->opp = o; h->opp_batch = B;
    return 0;
}

// the opponent's per-instance state, in the argument order of b200pf_opp_get_state / _set_state
static std::array<StateBuf, 5> opp_state(const b200pf_handle *h) {
    const OppArgs &o = h->opp;
    const size_t B = (size_t)h->opp_batch;
    return {{{o.budget, B * 8}, {o.budget64, B}, {o.ctr, B * OPP_CTR * 4}, {o.mt, B * OPP_MT_N * 4}, {o.mt_pos, B * 4}}};
}

extern "C" int b200pf_opp_get_state(b200pf_handle *h, double *budget, uint8_t *budget64, int32_t *ctr, uint32_t *mt, int32_t *mt_pos) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->opp_batch)) return fail(B200PF_E_STATE, "no opponent bound to the current environment (b200pf_opp_bind)");
    return state_get(h, opp_state(h), {budget, budget64, ctr, mt, mt_pos});
}

extern "C" int b200pf_opp_set_state(b200pf_handle *h, const double *budget, const uint8_t *budget64, const int32_t *ctr, const uint32_t *mt,
                                    const int32_t *mt_pos) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->opp_batch)) return fail(B200PF_E_STATE, "no opponent bound to the current environment (b200pf_opp_bind)");
    TRY(mt_pos_check(mt_pos, (size_t)h->opp_batch));
    return state_set(h, opp_state(h), {budget, budget64, ctr, mt, mt_pos});
}

extern "C" int b200pf_opp_geo_bind(b200pf_handle *h, const b200pf_opp_geo_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!layer_bound(h, h->opp_batch) || h->opp.kind != OPP_GEOMETRIC) return fail(B200PF_E_STATE, "no GeometricOpponent bound (b200pf_opp_bind, kind 3)");
    if (!d->weights || !d->episode_max_time || !d->wait || !d->dur || !d->gctr || d->cap < 1 || d->recovery_min < 0 ||
        !(d->p_hazard > 0.0 && d->p_hazard <= 1.0) || !(d->p_recovery > 0.0 && d->p_recovery <= 1.0))
        return fail(B200PF_E_ARG, "bad GeometricOpponent description");
    const int B = h->opp_batch;
    TRY(sched_ctr_check(d->gctr, (size_t)B, OPP_GEO_CTR, d->cap));
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    const size_t n_sched = (size_t)B * (size_t)d->cap * 4;
    DevBufs &ob = h->opp_bufs;
    OppGeoArgs g{};
    TRY(dev_alloc(h, ob, g.weights, (size_t)h->opp.n_attack * 8, d->weights));
    TRY(dev_alloc(h, ob, g.emt, (size_t)B * 4, d->episode_max_time));
    TRY(dev_alloc(h, ob, g.wait, n_sched, d->wait));
    TRY(dev_alloc(h, ob, g.dur, n_sched, d->dur));
    TRY(dev_alloc(h, ob, g.gctr, (size_t)B * OPP_GEO_CTR * 4, d->gctr));
    CU(cudaStreamSynchronize(h->stream));
    g.p_hazard = d->p_hazard; g.p_recovery = d->p_recovery;
    g.logq_hazard = d->logq_hazard; g.logq_recovery = d->logq_recovery; g.recovery_min = d->recovery_min; g.cap = d->cap;
    h->opp_geo = g; h->opp_geo_bound = true;
    return 0;
}

static bool opp_geo_ready(const b200pf_handle *h) { return layer_bound(h, h->opp_batch) && h->opp.kind == OPP_GEOMETRIC && h->opp_geo_bound; }

// the GeometricOpponent's per-instance state, in the argument order of b200pf_opp_geo_get_state / _set_state
static std::array<StateBuf, 3> opp_geo_state(const b200pf_handle *h) {
    const OppGeoArgs &g = h->opp_geo;
    const size_t B = (size_t)h->opp_batch, n_sched = B * (size_t)g.cap * 4;
    return {{{g.wait, n_sched}, {g.dur, n_sched}, {g.gctr, B * OPP_GEO_CTR * 4}}};
}

extern "C" int b200pf_opp_geo_get_state(b200pf_handle *h, int32_t *wait, int32_t *dur, int32_t *gctr) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!opp_geo_ready(h)) return fail(B200PF_E_STATE, "no GeometricOpponent bound (b200pf_opp_geo_bind)");
    return state_get(h, opp_geo_state(h), {wait, dur, gctr});
}

extern "C" int b200pf_opp_geo_set_state(b200pf_handle *h, const int32_t *wait, const int32_t *dur, const int32_t *gctr) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!opp_geo_ready(h)) return fail(B200PF_E_STATE, "no GeometricOpponent bound (b200pf_opp_geo_bind)");
    TRY(sched_ctr_check(gctr, (size_t)h->opp_batch, OPP_GEO_CTR, h->opp_geo.cap));
    return state_set(h, opp_geo_state(h), {wait, dur, gctr});
}

extern "C" int b200pf_opp_multi_bind(b200pf_handle *h, const b200pf_opp_multi_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!layer_bound(h, h->opp_batch) || h->opp.kind != OPP_GEOMETRIC_MULTI)
        return fail(B200PF_E_STATE, "no GeometricOpponentMultiArea bound (b200pf_opp_bind, kind 4)");
    if (d->n_area < 1 || d->n_area > OPP_MAX_AREA || !d->area_off || !d->weights || !d->episode_max_time || !d->mt || !d->mt_pos ||
        !d->wait || !d->dur || !d->actr || !d->fails || !d->attack_lines || d->cap < 1 || d->recovery_min < 0 ||
        !(d->p_hazard > 0.0 && d->p_hazard <= 1.0) || !(d->p_recovery > 0.0 && d->p_recovery <= 1.0))
        return fail(B200PF_E_ARG, "bad GeometricOpponentMultiArea description");
    if (d->area_off[0] != 0 || d->area_off[d->n_area] != h->opp.n_attack) return fail(B200PF_E_ARG, "areas do not cover the attacked lines");
    for (int k = 0; k < d->n_area; ++k)
        if (d->area_off[k + 1] <= d->area_off[k]) return fail(B200PF_E_ARG, "empty area");
    const int B = h->opp_batch;
    const size_t ba = (size_t)B * d->n_area, n_sched = ba * (size_t)d->cap * 4;
    TRY(mt_pos_check(d->mt_pos, ba));
    TRY(sched_ctr_check(d->actr, ba, OPP_AREA_CTR, d->cap));
    OppMultiArgs m{};
    m.n_area = d->n_area;
    for (int k = 0; k <= d->n_area; ++k) m.area_off[k] = d->area_off[k];
    m.p_hazard = d->p_hazard; m.p_recovery = d->p_recovery; m.logq_hazard = d->logq_hazard; m.logq_recovery = d->logq_recovery;
    m.recovery_min = d->recovery_min; m.cap = d->cap; m.attack_lines = d->attack_lines;
    CU(cudaSetDevice(h->device));
    CU(cudaStreamSynchronize(h->stream));
    DevBufs &ob = h->opp_bufs;
    TRY(dev_alloc(h, ob, m.weights, (size_t)h->opp.n_attack * 8, d->weights));
    TRY(dev_alloc(h, ob, m.emt, (size_t)B * 4, d->episode_max_time));
    TRY(dev_alloc(h, ob, m.mt, ba * OPP_MT_N * 4, d->mt));
    TRY(dev_alloc(h, ob, m.mt_pos, ba * 4, d->mt_pos));
    TRY(dev_alloc(h, ob, m.wait, n_sched, d->wait));
    TRY(dev_alloc(h, ob, m.dur, n_sched, d->dur));
    TRY(dev_alloc(h, ob, m.actr, ba * OPP_AREA_CTR * 4, d->actr));
    TRY(dev_alloc(h, ob, m.fails, (size_t)B * 4, d->fails));
    CU(cudaStreamSynchronize(h->stream));
    h->opp_multi = m; h->opp_multi_bound = true;
    return 0;
}

static bool opp_multi_ready(const b200pf_handle *h) { return layer_bound(h, h->opp_batch) && h->opp.kind == OPP_GEOMETRIC_MULTI && h->opp_multi_bound; }

// the GeometricOpponentMultiArea's per-instance state, in the argument order of b200pf_opp_multi_get_state / _set_state: MT
// words, MT positions, waiting times, durations, counters of every area, previous_fails
static std::array<StateBuf, 6> opp_multi_state(const b200pf_handle *h) {
    const OppMultiArgs &m = h->opp_multi;
    const size_t B = (size_t)h->opp_batch, ba = B * (size_t)m.n_area, n_sched = ba * (size_t)m.cap * 4;
    return {{{m.mt, ba * OPP_MT_N * 4}, {m.mt_pos, ba * 4}, {m.wait, n_sched}, {m.dur, n_sched}, {m.actr, ba * OPP_AREA_CTR * 4}, {m.fails, B * 4}}};
}

extern "C" int b200pf_opp_multi_get_state(b200pf_handle *h, uint32_t *mt, int32_t *mt_pos, int32_t *wait, int32_t *dur, int32_t *actr,
                                          int32_t *fails) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!opp_multi_ready(h)) return fail(B200PF_E_STATE, "no GeometricOpponentMultiArea bound (b200pf_opp_multi_bind)");
    return state_get(h, opp_multi_state(h), {mt, mt_pos, wait, dur, actr, fails});
}

extern "C" int b200pf_opp_multi_set_state(b200pf_handle *h, const uint32_t *mt, const int32_t *mt_pos, const int32_t *wait, const int32_t *dur,
                                          const int32_t *actr, const int32_t *fails) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!opp_multi_ready(h)) return fail(B200PF_E_STATE, "no GeometricOpponentMultiArea bound (b200pf_opp_multi_bind)");
    const size_t ba = (size_t)h->opp_batch * h->opp_multi.n_area;
    TRY(mt_pos_check(mt_pos, ba));
    TRY(sched_ctr_check(actr, ba, OPP_AREA_CTR, h->opp_multi.cap));
    return state_set(h, opp_multi_state(h), {mt, mt_pos, wait, dur, actr, fails});
}

// ------------------------------------------------------------------------------------------------
// line alerts and alarms of the device environment (b200pf_alert.cuh, b200pf_alarm.cuh)
// ------------------------------------------------------------------------------------------------
extern "C" int b200pf_alert_bind(b200pf_handle *h, const b200pf_alert_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    if (d->n_alert < 1 || d->n_alert > ALERT_MAX_LINES || !d->lines || d->window < 1 || !d->raise_alert || !d->reward_out)
        return fail(B200PF_E_ARG, "bad alert description");
    for (int k = 0; k < d->n_alert; ++k) {
        if (d->lines[k] < 0 || d->lines[k] >= h->g.n_line) return fail(B200PF_E_ARG, "alertable line out of range");
        for (int j = 0; j < k; ++j) if (d->lines[j] == d->lines[k]) return fail(B200PF_E_ARG, "alertable line listed twice");
    }
    TRY(unbind(h, &h->alert_batch, h->alert_bufs));
    const size_t B = (size_t)h->env_batch;
    AlertArgs al{};
    al.n = d->n_alert; al.window = d->window; al.ring = d->window + 2; al.reward = d->reward ? 1 : 0;
    al.min_blackout = (double)d->reward_min_blackout;
    al.range_blackout = (double)(d->reward_max_blackout - d->reward_min_blackout);           // float32, as AlertReward
    al.max_no_blackout = (double)d->reward_max_no_blackout;
    al.diff_no_blackout = (double)(d->reward_min_no_blackout - d->reward_max_no_blackout);    // float32, as AlertReward
    al.raise = d->raise_alert; al.reward_out = d->reward_out;
    const size_t bn = B * (size_t)al.n, br = bn * (size_t)al.ring;
    DevBufs &ob = h->alert_bufs;
    TRY(dev_alloc(h, ob, al.lines, (size_t)al.n * 4, d->lines));
    // every instance starts from _reset_alert + AlertReward.reset: zeros, and -1 for the two "time since" counters
    TRY(dev_alloc(h, ob, al.last_alert, bn, nullptr, 0));
    TRY(dev_alloc(h, ob, al.already, bn, nullptr, 0));
    TRY(dev_alloc(h, ob, al.tsl_alert, bn * 4, nullptr, 0xff));
    TRY(dev_alloc(h, ob, al.duration, bn * 4, nullptr, 0));
    TRY(dev_alloc(h, ob, al.tsl_attack, bn * 4, nullptr, 0xff));
    TRY(dev_alloc(h, ob, al.under_alert, bn * 4, nullptr, 0));
    TRY(dev_alloc(h, ob, al.was_used, bn * 4, nullptr, 0));
    TRY(dev_alloc(h, ob, al.total, B * 4, nullptr, 0));
    TRY(dev_alloc(h, ob, al.ts_attack, br, nullptr, 0));
    TRY(dev_alloc(h, ob, al.launched, br, nullptr, 0));
    TRY(dev_alloc(h, ob, al.current, bn, nullptr, 0));
    TRY(dev_alloc(h, ob, al.cur_id, B * 4, nullptr, 0));
    CU(cudaMemsetAsync(al.reward_out, 0, B * 8, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->alert = al; h->alert_batch = (int)B;
    return 0;
}

// the alerts' per-instance state, in the argument order of b200pf_alert_get_state / _set_state
static std::array<StateBuf, 12> alert_state(const b200pf_handle *h) {
    const AlertArgs &al = h->alert;
    const size_t B = (size_t)h->alert_batch, bn = B * (size_t)al.n, br = bn * (size_t)al.ring;
    return {{{al.last_alert, bn}, {al.already, bn}, {al.tsl_alert, bn * 4}, {al.duration, bn * 4}, {al.tsl_attack, bn * 4},
             {al.under_alert, bn * 4}, {al.was_used, bn * 4}, {al.total, B * 4}, {al.ts_attack, br}, {al.launched, br}, {al.current, bn},
             {al.cur_id, B * 4}}};
}

extern "C" int b200pf_alert_get_state(b200pf_handle *h, uint8_t *last_alert, uint8_t *already, int32_t *tsl_alert, int32_t *duration,
                                      int32_t *tsl_attack, int32_t *under_alert, int32_t *was_used, int32_t *total, uint8_t *ts_attack,
                                      uint8_t *launched, uint8_t *current, int32_t *cur_id) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->alert_batch)) return fail(B200PF_E_STATE, "no line alerts bound to the current environment (b200pf_alert_bind)");
    return state_get(h, alert_state(h), {last_alert, already, tsl_alert, duration, tsl_attack, under_alert, was_used, total, ts_attack,
                                         launched, current, cur_id});
}

extern "C" int b200pf_alert_set_state(b200pf_handle *h, const uint8_t *last_alert, const uint8_t *already, const int32_t *tsl_alert,
                                      const int32_t *duration, const int32_t *tsl_attack, const int32_t *under_alert, const int32_t *was_used,
                                      const int32_t *total, const uint8_t *ts_attack, const uint8_t *launched, const uint8_t *current,
                                      const int32_t *cur_id) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->alert_batch)) return fail(B200PF_E_STATE, "no line alerts bound to the current environment (b200pf_alert_bind)");
    const size_t B = (size_t)h->alert_batch;
    if (cur_id) for (size_t i = 0; i < B; ++i) if (cur_id[i] < 0 || cur_id[i] >= h->alert.ring) return fail(B200PF_E_ARG, "ring index out of range");
    return state_set(h, alert_state(h), {last_alert, already, tsl_alert, duration, tsl_attack, under_alert, was_used, total, ts_attack,
                                         launched, current, cur_id});
}

extern "C" int b200pf_alarm_bind(b200pf_handle *h, const b200pf_alarm_desc *d) {
    if (!h || !d) return fail(B200PF_E_ARG, "null pointer");
    if (!env_bound(h)) return fail(B200PF_E_STATE, "environment not bound to the current series (b200pf_env_bind)");
    if (d->n_zone < 1 || d->n_zone > ALARM_MAX_ZONES || !d->zone_mask || d->best_time < 1 || d->window_size < 1 ||
        d->best_time > ALARM_MAX_RING - d->window_size || !d->raise_alarm || !d->reward_out || !d->is_alarm_illegal)
        return fail(B200PF_E_ARG, "bad alarm description");
    const uint32_t zones = d->n_zone == 32 ? 0xffffffffu : (1u << d->n_zone) - 1u;
    for (int l = 0; l < h->g.n_line; ++l)
        if (!d->zone_mask[l] || (d->zone_mask[l] & ~zones)) return fail(B200PF_E_ARG, "a line in no zone, or in a zone past n_zone");
    TRY(unbind(h, &h->alarm_batch, h->alarm_bufs));
    const size_t B = (size_t)h->env_batch;
    AlarmArgs am{};
    am.n = d->n_zone; am.n_line = h->g.n_line;
    am.max_budget = d->max_budget; am.budget_per_ts = d->budget_per_ts; am.alarm_cost = d->alarm_cost; am.init_budget = d->init_budget;
    am.best_time = d->best_time; am.window = d->window_size; am.ring = d->best_time + d->window_size; am.reward = d->reward ? 1 : 0;
    am.raise = d->raise_alarm; am.reward_out = d->reward_out; am.illegal = d->is_alarm_illegal;
    const size_t bn = B * (size_t)am.n * 4, br = B * (size_t)am.ring * 4;
    DevBufs &ob = h->alarm_bufs;
    TRY(dev_alloc(h, ob, am.zone_mask, (size_t)am.n_line * 4, d->zone_mask));
    // every instance starts from LinearAttentionBudget.reset: the initial budget, -1 for the times and zones, an empty ring
    const std::vector<float> b0(B, d->init_budget);
    TRY(dev_alloc(h, ob, am.budget, B * 4, b0.data()));
    TRY(dev_alloc(h, ob, am.time_last, B * 4, nullptr, 0xff));
    TRY(dev_alloc(h, ob, am.time_last_ok, B * 4, nullptr, 0xff));
    TRY(dev_alloc(h, ob, am.last, bn, nullptr, 0xff));
    TRY(dev_alloc(h, ob, am.last_ok, bn, nullptr, 0xff));
    TRY(dev_alloc(h, ob, am.ring_step, br, nullptr, 0));
    TRY(dev_alloc(h, ob, am.ring_mask, br, nullptr, 0));
    TRY(dev_alloc(h, ob, am.any_ok, B, nullptr, 0));
    TRY(dev_alloc(h, ob, am.used, B, nullptr, 0));
    CU(cudaMemsetAsync(am.illegal, 0, B, h->stream));
    CU(cudaMemsetAsync(am.reward_out, 0, B * 8, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->alarm = am; h->alarm_batch = (int)B;
    return 0;
}

// the alarms' per-instance state, in the argument order of b200pf_alarm_get_state / _set_state (the last one, is_alarm_illegal,
// is the caller's buffer)
static std::array<StateBuf, 10> alarm_state(const b200pf_handle *h) {
    const AlarmArgs &am = h->alarm;
    const size_t B = (size_t)h->alarm_batch, bn = B * (size_t)am.n * 4, br = B * (size_t)am.ring * 4;
    return {{{am.budget, B * 4}, {am.time_last, B * 4}, {am.time_last_ok, B * 4}, {am.last, bn}, {am.last_ok, bn}, {am.ring_step, br},
             {am.ring_mask, br}, {am.any_ok, B}, {am.used, B}, {am.illegal, B}}};
}

extern "C" int b200pf_alarm_get_state(b200pf_handle *h, float *budget, int32_t *time_last, int32_t *time_last_ok, int32_t *last,
                                      int32_t *last_ok, int32_t *ring_step, uint32_t *ring_mask, uint8_t *any_ok, uint8_t *used,
                                      uint8_t *illegal) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->alarm_batch)) return fail(B200PF_E_STATE, "no alarms bound to the current environment (b200pf_alarm_bind)");
    return state_get(h, alarm_state(h), {budget, time_last, time_last_ok, last, last_ok, ring_step, ring_mask, any_ok, used, illegal});
}

extern "C" int b200pf_alarm_set_state(b200pf_handle *h, const float *budget, const int32_t *time_last, const int32_t *time_last_ok,
                                      const int32_t *last, const int32_t *last_ok, const int32_t *ring_step, const uint32_t *ring_mask,
                                      const uint8_t *any_ok, const uint8_t *used, const uint8_t *illegal) {
    if (!h) return fail(B200PF_E_ARG, "null handle");
    if (!layer_bound(h, h->alarm_batch)) return fail(B200PF_E_STATE, "no alarms bound to the current environment (b200pf_alarm_bind)");
    return state_set(h, alarm_state(h), {budget, time_last, time_last_ok, last, last_ok, ring_step, ring_mask, any_ok, used, illegal});
}

extern "C" int b200pf_env_stats(const b200pf_handle *h, int64_t *out8) {
    if (!h || !out8) return fail(B200PF_E_ARG, "null pointer");
    out8[0] = h->env_steps; out8[1] = h->env_h2d; out8[2] = h->env_d2h; out8[3] = h->env_waits;
    out8[4] = h->env_illegal; out8[5] = h->env_last_cap; out8[6] = h->env_last_dirty; out8[7] = h->env_plan_refresh;
    return 0;
}

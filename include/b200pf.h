/*
 * b200pf.h — C ABI of the batched GPU power-flow engine (libb200pf.so).
 *
 * This is the drop-in boundary for ONE path of Grid2Op: what
 * grid2op.Backend.PandaPowerBackend delegates to pandapower in
 *   runpf()                     reference grid2op/Backend/pandaPowerBackend.py:1220-1255
 *     -> pp.runpp(init="dc", max_iteration=10, check_connectivity=False)   pPB:1097-1105
 *     -> pp.rundcpp(check_connectivity=True)                               pPB:1090
 *   _fetch_data_pf_converged()  pPB:1122-1218 (+ _gens_info :1526, _loads_info :1549,
 *                               _storages_info :1621, shunt_info :1596)
 * for a *batch* of independent grid instances that share one static grid description.
 *
 * Plain C: pointers and sizes only, no torch types.  Every function returns 0 on success or a
 * negative B200PF_E_* code; b200pf_last_error() gives the message.  A handle is not thread safe;
 * different handles are independent (one CUDA stream each).  No CPU fallback exists: with no
 * CUDA device b200pf_create() fails with B200PF_E_CUDA.
 * Ordering: every call that takes HOST data which later launches read (grid description, series bind / set_topo /
 * reset_instances, static injections, thermal limits) copies it on the handle's stream and returns when the copy has
 * arrived (the caller may reuse its buffer at once, and launches on any stream of the handle — chunk and group launches
 * run on internal streams — see the data); nothing is issued on the legacy default stream.
 *
 * Data layout (all row-major, instance-major so that one warp/CTA reads one contiguous record):
 *   topo   int8  [batch][n_topo_in]   n_topo_in = dim_topo + n_shunt + n_hidden
 *            [0, dim_topo)            local busbar of every element, grid2op topo_vect order,
 *                                     -1 = disconnected, 1..n_busbar        (pPB:1489-1524)
 *            [dim_topo, +n_shunt)     local busbar of every shunt (-1 = off) (pPB:1609-1611)
 *            [.., +n_hidden)          local busbar of every hidden reference unit (ext_grid kept
 *                                     next to the generator the reference creates, pPB:394-453)
 *   inj    f64   [batch][n_inj]       n_inj = n_gen + n_unit + 2 n_load + n_storage + 2 n_shunt
 *            gen_p[n_gen] MW | unit_vm[n_unit] p.u. (hidden units first) | load_p | load_q |
 *            storage_p | shunt_p | shunt_q        (what pPB:926-969 writes into its tables)
 *   out    f32   [batch][n_out]       n_out = 10 n_line + 4 n_unit + 2 n_load + n_storage + 3 n_shunt
 *            p_or q_or v_or a_or theta_or p_ex q_ex v_ex a_ex theta_ex   (each n_line)
 *            unit_p unit_q unit_v unit_theta (each n_unit, hidden units first)
 *            load_v load_theta (n_load) | storage_v (n_storage) | shunt_p shunt_q shunt_v (n_shunt)
 *            units: MW, MVAr, kV, A, degrees — the float32 values PandaPowerBackend returns.
 *   status int32 [batch]              B200PF_ST_*
 *   iters  int32 [batch]              Newton iterations used (0 in DC mode)
 *   busv   f64   [batch][2*n_slot]    optional: |V| p.u. then angle rad per bus slot
 *                                     (slot = sub + (busbar-1)*n_sub, NaN when unused)
 */
#ifndef B200PF_H
#define B200PF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PF_ABI_VERSION 2

enum {
    B200PF_OK = 0,
    B200PF_E_ARG = -1,      /* bad argument */
    B200PF_E_CUDA = -2,     /* CUDA runtime error / no device */
    B200PF_E_CAPACITY = -3, /* grid does not fit the on-chip budget of this build */
    B200PF_E_STATE = -4     /* call sequence error */
};

/* per-instance solver status (what runpf() turns into (bool, exception), pPB:1248-1255) */
enum {
    B200PF_ST_CONVERGED = 0,
    B200PF_ST_DIVERGED = 1,   /* Newton did not reach the tolerance / singular matrix / NaN */
    B200PF_ST_UNSUPPLIED = 2, /* an in-service bus is not connected to a reference bus */
    B200PF_ST_NO_REF = 3,     /* no reference unit in service */
    B200PF_ST_TOO_LARGE = 4,  /* more active buses than the launch was sized for (nb_cap) */
    B200PF_ST_DONE = 5        /* series mode with protections: the instance diverged at an earlier step */
};

/* Static grid description (host pointers, copied at create).  Element order = the reference's
 * (lines then trafos = "lines"; pPB:481-483).  Sub ids are substation indices 0..n_sub-1. */
typedef struct b200pf_grid_desc {
    int32_t abi_version; /* B200PF_ABI_VERSION */
    int32_t n_sub, n_busbar;
    int32_t n_line, n_gen, n_hidden, n_load, n_storage, n_shunt, dim_topo;
    double sn_mva;
    /* lines (n_line) */
    const int32_t *line_or_sub, *line_ex_sub, *line_or_pos, *line_ex_pos;
    const double *line_y;     /* [n_line][8]: yff.re yff.im yft.re yft.im ytf.re ytf.im ytt.re ytt.im (p.u.) */
    const double *line_bdc;   /* [n_line] 1/(x*ratio) */
    const double *line_pshift;/* [n_line] DC phase-shift injection  b*(-shift_rad) */
    const float *line_or_vn, *line_ex_vn; /* kV (float32 like pPB:796-801) */
    /* units (n_unit = n_hidden + n_gen; hidden reference units first, like the ppc gen table) */
    const int32_t *unit_sub;  /* [n_unit] */
    const int32_t *unit_pos;  /* [n_unit] topo_vect position; hidden unit h: dim_topo + n_shunt + h */
    const int32_t *unit_is_ref; /* [n_unit] ext_grid or gen.slack */
    const double *unit_qmin, *unit_qmax; /* [n_unit] MVAr (reactive sharing, PYPOWER pfsoln) */
    const float *unit_vn;     /* [n_unit] kV */
    /* loads / storages / shunts */
    const int32_t *load_sub, *load_pos;        const float *load_vn;
    const int32_t *storage_sub, *storage_pos;  const float *storage_vn;  const double *storage_q;
    const int32_t *shunt_sub;                  const float *shunt_vn;    const double *shunt_vratio; /* (vn_bus/vn_shunt)^2*step */
    /* [n_sub] position of every substation in a bandwidth-reducing order of the substation graph (e.g.
     * reverse Cuthill-McKee; identity is valid): the CTA-per-instance kernel numbers buses in this order so
     * that the Jacobian is banded and solves it with a band-limited LU.  NULL = identity. */
    const int32_t *sub_rank;
} b200pf_grid_desc;

typedef struct b200pf_handle b200pf_handle;

const char *b200pf_last_error(void);
int b200pf_abi_version(void);
int b200pf_device_count(void);

/* create / destroy.  max_batch sizes the device and pinned staging buffers. */
int b200pf_create(const b200pf_grid_desc *grid, int max_batch, int device, b200pf_handle **out);
int b200pf_destroy(b200pf_handle *h);

/* Active buses (bus slots with at least one connected element) of n topology records int8 [n][n_topo_in]: per_instance (may be
 * NULL) int32 [n], *max_out their maximum = the tight nb_cap of a launch on these records (the bound the callers of the reference's
 * backend never need because pandapower re-derives the bus set per call, pPB:1097-1105 -> pandapower pd2ppc).  Pure host function
 * of the grid description: no device, no handle. */
int b200pf_grid_max_active_buses(const b200pf_grid_desc *grid, int n, const int8_t *topo, int32_t *per_instance, int32_t *max_out);

/* sizes derived from the grid description */
int b200pf_sizes(const b200pf_handle *h, int *n_topo_in, int *n_inj, int *n_out, int *n_slot);

/* One batched power flow from HOST buffers: H2D copies, kernel, D2H copies, synchronised on return.
 * busv may be NULL.  nb_cap = upper bound of active buses per instance the launch is sized for
 * (<= 0: all n_sub*n_busbar slots, or the largest size that fits on chip).
 * tol_mva: 1e-8 reproduces pandapower's default tolerance_mva; max_iter 10 = pPB:124. */
int b200pf_run_host(b200pf_handle *h, int batch, const int8_t *topo, const double *inj, int is_dc,
                    int max_iter, double tol_mva, int nb_cap, float *out, int32_t *status,
                    int32_t *iters, double *busv);

/* Same with DEVICE pointers, asynchronous on the handle's stream (b200pf_sync to wait). */
int b200pf_run_device(b200pf_handle *h, int batch, const int8_t *d_topo, const double *d_inj,
                      int is_dc, int max_iter, double tol_mva, int nb_cap, float *d_out,
                      int32_t *d_status, int32_t *d_iters, double *d_busv);

/* b200pf_run_device plus a HOST copy of the same topology records: with it the engine can use the planned sparse kernel
 * (its topology plans are looked up / built on the host) for inputs that already live in device memory, e.g. injections
 * written by another kernel or a torch model.  The per-instance plan ids travel on the handle's stream before the launch. */
int b200pf_run_device_topo(b200pf_handle *h, int batch, const int8_t *host_topo, const int8_t *d_topo, const double *d_inj,
                           int is_dc, int max_iter, double tol_mva, int nb_cap, float *d_out, int32_t *d_status,
                           int32_t *d_iters, double *d_busv);

/* Batched time-series stepping (the DoNothing subset of BaseEnv.step, reference
 * grid2op/Environment/baseEnv.py:3778-3872 with NO_OVERFLOW_DISCONNECTION): the chronics
 * (grid2op/Chronics/gridStateFromFile.py:749-808 rows: load_p, load_q, prod_p, prod_v[kV] in
 * BACKEND element order) live in HBM as float32 [n_scen][n_rows][2 n_load + 2 n_gen]; instance i
 * replays scenario scen[i] from row t0[i], wrapping around.  Every call advances all instances by
 * one row, solves, and writes out/status/iters plus rho = a_or / thermal_limit (f32 [batch][n_line]).
 * topo is device state owned by the handle (set with b200pf_series_set_topo). */
int b200pf_series_bind(b200pf_handle *h, const float *chron_host, int n_scen, int n_rows,
                       const int32_t *scen, const int32_t *t0, int batch,
                       const double *static_inj /* [n_inj] defaults for storage / shunt / hidden vm */,
                       const float *thermal_limit_a /* [n_line] */);
int b200pf_series_set_topo(b200pf_handle *h, const int8_t *topo /* [batch][n_topo_in] host */);
int b200pf_series_step(b200pf_handle *h, int is_dc, int max_iter, double tol_mva, int nb_cap);
/* Protections / cascading failure inside the series step (reference Backend.next_grid_state,
 * grid2op/Backend/backend.py:1433-1521, and the counters of BaseEnv._aux_register_env_converged,
 * grid2op/Environment/baseEnv.py:3361-3370): lines whose flow exceeds hard_thr * limit, or that stayed above
 * soft_thr * limit for more than max_allowed consecutive steps, are disconnected and the flow is re-solved
 * until no line trips; the outages persist in the device topology; an instance whose flow diverges is
 * "done" (B200PF_ST_DONE from then on).  enabled = 0 restores NO_OVERFLOW_DISCONNECTION.
 * Two implementations: grids that fit the warp-per-instance kernel (<= 32 lines / bus slots) cascade entirely on the
 * device, inside one launch; all other grids (and every grid under kernel policy 2) run the planned kernel, which reports
 * the lines that trip — a tripped line is a new topology, i.e. a new plan — and the library re-plans those instances on
 * the host and launches the next cascade round for them (b200pf_series_step is then synchronous: one 4-byte read-back
 * per round). */
int b200pf_series_protections(b200pf_handle *h, int enabled, float hard_thr, float soft_thr, int max_allowed);
/* the NEXT series step is an environment reset step: no soft-overflow counting (backend.py:1488-1490) */
int b200pf_series_next_is_reset(b200pf_handle *h);
/* host copies of the protection state after the last step (any pointer may be NULL):
 * counters / timestep_overflow / disc_lines int32 [batch][n_line], done int32 [batch] */
int b200pf_series_fetch_state(b200pf_handle *h, int32_t *protection_counter, int32_t *timestep_overflow,
                              int32_t *disc_lines, int32_t *done);
/* device pointers of the resident results of the last series step (valid until destroy) */
int b200pf_series_results(b200pf_handle *h, float **d_out, int32_t **d_status, int32_t **d_iters,
                          float **d_rho, int32_t **d_t);
/* copy results of the last series step to host buffers (any pointer may be NULL) */
int b200pf_series_fetch(b200pf_handle *h, float *out, int32_t *status, int32_t *iters, float *rho);

/* Pinned host staging buffers owned by the handle (sized for max_batch): a caller that fills topo /
 * inj in place and reads out / status / iters in place avoids one host copy in each direction. */
int b200pf_staging(b200pf_handle *h, int8_t **topo, double **inj, float **out, int32_t **status,
                   int32_t **iters, double **busv);
/* b200pf_run_host on the staging buffers (H2D, kernel, D2H, synchronised on return) */
int b200pf_run_staged(b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva, int nb_cap,
                      int want_busv);
/* let the series results land in caller-owned DEVICE buffers (e.g. torch tensors); NULL keeps the
 * handle's own buffer for that array */
int b200pf_series_bind_outputs(b200pf_handle *h, float *d_out, int32_t *d_status, int32_t *d_iters,
                               float *d_rho);
/* N-1 contingency sweep (the reference's pattern: copy_public(); _disconnect_line(i); runpf();
 * get_relative_flow() for every line i - examples/backend_dependant_code/_obs_with_n1.py:111-125, and
 * obs.simulate, grid2op/Observation/baseObservation.py:3365): batch base states x n_line single-line
 * outages = batch*n_line independent AC power flows in ONE launch sharing the base records.
 *   rho    f32   [batch][n_line outages][n_line]   a_or / thermal_limit (NaN rows where the flow diverged)
 *   status int32 [batch][n_line]
 * Host pointers; thermal limits from b200pf_set_thermal_limit.  batch*n_line must be <= max_batch. */
int b200pf_set_thermal_limit(b200pf_handle *h, const float *thermal_limit_a /* [n_line] */);
int b200pf_n1_host(b200pf_handle *h, int batch, const int8_t *topo, const double *inj, int max_iter,
                   double tol_mva, int nb_cap, float *rho, int32_t *status);
/* "rows" entry point: like b200pf_run_staged but the injections of this step come as the float32
 * chronics ROW of every instance (load_p, load_q, prod_p, prod_v[kV]; 2 n_load + 2 n_gen values, backend
 * element order) written by the caller into the pinned rows staging buffer (b200pf_rows_staging);
 * storage / shunt / hidden-unit values come from static_inj (b200pf_set_static_inj).  Less than half
 * the host->device bytes of the f64 record, and no host-side float64 packing. */
int b200pf_set_static_inj(b200pf_handle *h, const double *static_inj /* [n_inj] */);
int b200pf_rows_staging(b200pf_handle *h, float **rows);
int b200pf_run_rows_staged(b200pf_handle *h, int batch, int is_dc, int max_iter, double tol_mva, int nb_cap);
/* Pipelined variant of b200pf_run_rows_staged: the caller fills the pinned rows / topo staging buffers chunk by
 * chunk and launches every chunk as soon as it is ready (asynchronous: H2D, kernel, D2H of that chunk on one of
 * a few internal streams), so host-side preparation of chunk c+1 overlaps the device work of chunk c;
 * b200pf_rows_chunk_wait returns when every launched chunk has landed in the pinned out/status/iters buffers. */
int b200pf_rows_chunk_launch(b200pf_handle *h, int first, int count, int is_dc, int max_iter, double tol_mva, int nb_cap);
int b200pf_rows_chunk_wait(b200pf_handle *h);
/* same, but the rows of the chunk are read from caller-provided PINNED host memory (b200pf_pinned_alloc) instead of
 * the rows staging buffer: lets a driver pre-collate the time series once (rows of all instances for step k
 * contiguous) and feed every step without touching the data on the host. */
int b200pf_rows_chunk_launch_from(b200pf_handle *h, int first, int count, const float *pinned_rows, int is_dc,
                                  int max_iter, double tol_mva, int nb_cap);
/* Group-pipelined stepping (asynchronous vectorised environments): the batch is cut into up to B200PF_MAX_GROUPS
 * groups of instances [first, first+count); each group owns a stream and an event.  launch enqueues H2D (topology
 * records from the pinned staging buffer, rows from pinned_rows or, when NULL, from the pinned rows staging buffer)
 * -> fused kernel -> D2H into the pinned out/status/iters staging buffers and returns at once; wait blocks until that
 * group's results have landed.  While the caller consumes group g (the agent of reference
 * grid2op/Environment/baseEnv.py:3778 `step` acting on its observations) the other groups are in flight, so PCIe
 * transfers of one group overlap the kernels of the others.  A group must be waited for before it is launched again. */
#define B200PF_MAX_GROUPS 16
int b200pf_rows_group_launch(b200pf_handle *h, int group, int first, int count, const float *pinned_rows, int is_dc,
                             int max_iter, double tol_mva, int nb_cap);
int b200pf_rows_group_wait(b200pf_handle *h, int group);
/* flags bit 0 (B200PF_GROUP_DIRECT_OUT): the kernel stores result records / status / iters straight into the pinned
 * staging buffers (device-addressable host memory, posted PCIe writes that overlap the solve of the other instances)
 * instead of a copy-engine D2H after the kernel.  Only while no group is in flight. */
#define B200PF_GROUP_DIRECT_OUT 1
/* flags bit 1 (B200PF_GROUP_ZEROCOPY_IN): the kernel reads the chronics rows (and, for the pivoting kernels, the topology
 * records) of its instances straight from the pinned host buffers — a few hundred bytes per instance, read once — instead
 * of two copy-engine H2D transfers per launch; bit 2 (B200PF_GROUP_DIRECT_STATUS): status / iteration counts (8 bytes per
 * instance) are stored by the kernel straight into the pinned staging buffers, the result records still travel by the copy
 * engine.  Both cut the number of driver calls per group launch (7 -> 3), which bounds the host-side stepping rate. */
#define B200PF_GROUP_ZEROCOPY_IN 2
#define B200PF_GROUP_DIRECT_STATUS 4
int b200pf_rows_group_config(b200pf_handle *h, int flags);
int b200pf_pinned_alloc(size_t bytes, void **ptr);
int b200pf_pinned_free(void *ptr);
/* run all work of this handle on the caller's stream (cudaStream_t as integer; 0 = the handle's own) */
int b200pf_set_stream(b200pf_handle *h, uint64_t stream);

/* Kernel selection.  The engine owns three kernels for the same path (reference pPB:1090 / 1097-1105):
 *   - the PLANNED SPARSE kernel (csrc/b200pf_sparse.cuh): everything that depends on the topology only (bus fusion, bus
 *     types, connectivity check, elimination order, filled Jacobian pattern, factorisation schedule, factorised DC matrix)
 *     is computed once per distinct topology vector on the host and cached ("plan"); the device runs the numeric part.
 *     Needs a host copy of the topology (every entry point except b200pf_run_device has one) and no device-side
 *     protections;
 *   - the warp-per-instance and CTA-per-instance kernels with on-device topology discovery and partial pivoting.
 * policy 0 (default): planned kernel whenever it applies, unless one call would have to build more than a few hundred
 * new plans; 1: pivoting kernels only; 2: planned kernel whenever it applies.  Env B200PF_PLAN_POLICY presets it. */
int b200pf_set_kernel_policy(b200pf_handle *h, int policy);
/* number of cached plans, their bytes, and the kernel of the last launch (1 warp/pivoting, 2 CTA/pivoting, 3 planned sparse) */
int b200pf_plan_stats(const b200pf_handle *h, int64_t *n_plans, int64_t *plan_bytes, int *last_kernel);
/* out4 = { topology rows looked up in the plan cache, of which found, plans built, cache resets (the cache is append-only and
 * starts over when it is full: 32768 plans / 1 GiB) } since b200pf_create.  New plans of one call are built in parallel on the
 * host threads (env B200PF_PLAN_THREADS caps them). */
int b200pf_plan_counters(const b200pf_handle *h, int64_t *out4);

/* Multi-GPU result collection (SURVEY 8(e): instances shard across GPUs, the step results go to the agent's rank).  Instead
 * of one collective launch per 60-microsecond step, the agent's rank allocates the result buffer with b200pf_device_alloc
 * and exports it (CUDA IPC); every other rank (one process per GPU) opens the handle — the buffer is then peer-mapped over
 * NVLink — and binds a slice of it as its `rho` output (b200pf_series_bind_outputs): the kernel's own result stores land in
 * the agent's HBM, fused with the solve, no extra launch.  Completion is signalled by whatever orders the streams (a tiny
 * NCCL all-reduce every K steps in bench.py).  handle64: 64 bytes (cudaIpcMemHandle_t). */
/* env.reset() of single instances of a bound series (reference Environment.reset, environment.py; BaseEnv counters
 * baseEnv.py:3352-3393): done flag, protection counters, overflow counters and disc_lines back to a fresh episode; t_new (may be
 * NULL): the chronics row the instance's next solve uses; topo_rows (may be NULL): int8 [n][n_topo_in], its topology. */
int b200pf_series_reset_instances(b200pf_handle *h, int n, const int32_t *idx, const int32_t *t_new, const int8_t *topo_rows);
/* b200pf_series_bind_flag: after every b200pf_series_step the device stores the number of steps done so far to *d_flag (behind
 * all the step's kernels, system-wide visible) — d_flag may point into the agent rank's buffer, next to the results: the agent
 * learns that a rank's step k has fully arrived by reading a 4-byte word, no collective involved.  NULL unbinds. */
int b200pf_series_bind_flag(b200pf_handle *h, int32_t *d_flag);
int b200pf_device_alloc(size_t bytes, void **d_ptr);
int b200pf_device_free(void *d_ptr);
int b200pf_device_read(const void *d_src, void *host_dst, size_t bytes);   /* synchronous D2H copy (checks) */
int b200pf_ipc_export(const void *d_ptr, unsigned char *handle64);
int b200pf_ipc_open(const unsigned char *handle64, void **d_ptr);
int b200pf_ipc_close(void *d_ptr);

/* Safety net of the planned kernel.  The planned kernel eliminates without pivoting on an fp32 Jacobian; the reference's
 * solver (pp.runpp, pPB:1097-1105) pivots in fp64, and a failed power flow is a game over (pPB:1241-1255,
 * grid2op/Environment/baseEnv.py:3523-3524).  A planned launch that leaves an instance as DIVERGED therefore launches, from
 * the device, on the same stream and inside the same C-ABI call, a re-solve with partial pivoting (fp64 Jacobian where the
 * workspace allows) of every such instance; a status only leaves the library after that.  b200pf_set_debug is a TEST knob:
 * planned_div_mod > 0 makes the planned kernel give up on every instance with (index % planned_div_mod == 0), which
 * exercises the re-solve path; redo_enabled = 0 switches the safety net off (measurements).  Env B200PF_NO_REDO=1 presets
 * the latter.  b200pf_redo_launch_count: safety-net launches so far (they are not part of b200pf_launch_count); it waits
 * for the device, so read it after a fetch, not between the launches of a step. */
int b200pf_set_debug(b200pf_handle *h, int planned_div_mod, int redo_enabled);
int64_t b200pf_redo_launch_count(const b200pf_handle *h);

/* Observation layer: grid2op observation vectors (obs.to_vect(), every attribute as float32) and rewards for the whole bound
 * series, assembled on the device from what a series step leaves there (result records, rho, device topology, chronics row
 * index) — no device-to-host copy of the result records.  b200pf_obs_bind copies the static tables below (host pointers) and
 * clears the overflow counters the layer keeps (timestep_overflow / timestep_protection_engaged, reference
 * grid2op/Environment/baseEnv.py:3361-3370, counted whether the protections are on or not); a re-bound series needs a new
 * b200pf_obs_bind.  The attribute sources of `seg` are enum ObsSrc of csrc/b200pf_obs.cuh (grid2op_b200/observation.py builds them
 * from attribute names).
 * b200pf_observe enqueues, on the handle's stream and behind the last series step, one H2D copy of the per-instance host inputs
 * (from a pinned buffer of the handle) and one launch (a warp per instance) writing obs f32 [batch][n_obs] and reward f32 [batch]
 * into caller-owned DEVICE buffers (torch tensors, like b200pf_series_bind_outputs; reward may be NULL).  host_in: int32
 * [batch][n_line + n_sub + 3] = time_before_cooldown_line | time_before_cooldown_sub | current_step | stamp | flags — 4 (n_line +
 * n_sub + 3) bytes per instance.  The counters advance once per distinct stamp (the caller's step number): observe after every
 * step.  flags: B200PF_OBS_ILLEGAL (the step's action was replaced by "do nothing"), B200PF_OBS_DONE (the instance is game over:
 * the game-over observation of BaseObservation.set_game_over, baseObservation.py:1551, and reward_min), B200PF_OBS_RESET (the
 * instance was reset: its counters restart from 0).  With line alerts (n_alert > 0, b200pf_alert_bind) the record of an instance
 * continues with 6 n_alert + 1 int32: active_alert | attack_under_alert | time_since_last_alert | alert_duration |
 * total_number_of_alert | time_since_last_attack | was_alert_used_after_attack, and the alert attributes of `seg` read them.
 * With alarms (n_alarm > 0, b200pf_alarm_bind) it continues with n_alarm + 4 int32: is_alarm_illegal | time_since_last_alarm |
 * last_alarm[n_alarm] | the attention budget's float32 bits | AlarmReward.is_alarm_used, and the five alarm attributes read them. */
enum { B200PF_REWARD_NONE = 0, B200PF_REWARD_REDISP = 1, B200PF_REWARD_L2RPN = 2 };
enum { B200PF_OBS_ILLEGAL = 1, B200PF_OBS_DONE = 2, B200PF_OBS_RESET = 4 };
typedef struct b200pf_obs_desc {
    int32_t n_seg, n_obs;
    const int32_t *seg;                 /* [n_seg][3]: attribute source, offset in the vector, length */
    const int32_t *calendar;            /* [n_scen][n_rows][6] year month day hour minute weekday(Monday = 0) of every row */
    const int32_t *max_step;            /* [n_scen] */
    float delta_time;                   /* minutes */
    const int32_t *maint_time, *maint_dur; /* [n_scen][n_rows][n_line] or NULL: time_next_maintenance / duration_next_maintenance */
    const float *gen_pmin, *gen_pmax, *gen_ramp_up, *gen_ramp_down, *gen_cost;  /* [n_gen] (prods_charac.csv) */
    const int8_t *gen_renewable;        /* [n_gen] */
    int32_t redisp_available;
    const float *sto_charge0, *sto_loss_step;  /* [n_storage] MWh: charge after the reset step, loss withdrawn per step */
    int32_t reward_kind;                /* B200PF_REWARD_* */
    double max_regret, reward_min, reward_illegal, dts_hours;   /* RedispReward constants; step length in hours */
    float soft_thr;                     /* SOFT_OVERFLOW_THRESHOLD (timestep_protection_engaged) */
    int32_t n_alert;                    /* dim_alerts: alert values in the host record (0: none, the record as without alerts) */
    int32_t n_alarm;                    /* dim_alarms: alarm values in the host record (0: none, the record as without alarms) */
} b200pf_obs_desc;
int b200pf_obs_bind(b200pf_handle *h, const b200pf_obs_desc *desc);
int b200pf_observe(b200pf_handle *h, const int32_t *host_in, float *d_obs, float *d_reward);
/* out4 = { observe launches, bytes of their host inputs copied H2D, bytes this handle copied device-to-host since create (series
 * fetch / fetch_state), bytes one observe launch writes } */
int b200pf_obs_stats(const b200pf_handle *h, int64_t *out4);

/* Device environment state: BatchedEnv's bookkeeping for the bound series on the device (csrc/b200pf_env.cuh), so that an agent
 * steps with device tensors and the host touches no per-instance data.  b200pf_env_bind copies the static tables below (host
 * pointers) and keeps the per-instance state pointers: caller-owned DEVICE buffers (torch tensors, like
 * b200pf_series_bind_outputs), which the kernels read and write in place.  Booleans are one byte (0 / 1).  A re-bound series
 * needs a new b200pf_env_bind.
 * b200pf_env_step, on the handle's stream: (1) one launch restating BatchedEnv._apply_agent + _apply_environment for every
 * instance (DefaultRules legality, busbar writes, reconnections, line switching, maintenance / hazards of the row the solve uses,
 * active-bus recount of the changed instances for the bus cap when tight_cap); (2) ONE host wait for a few control words;
 * (3) when some topology changed (or a device reset happened since the last plan refresh): the changed rows, and the rows a trip or
 * a reset changed since, are copied back to patch the host mirror of the device topology, and (4) the plans of the whole mirror are
 * looked up exactly as b200pf_series_set_topo does; (5) the series step; (6) one launch for the rest of BatchedEnv.step: trips,
 * the isolated-busbar status override, cooldowns, done / newly_done, current_step and the observe layer's input record (stamp =
 * the caller's step number).  Actions: sub_id int32 [batch] (-1: none) with sub_bus int8 [batch][>= max_sub] (row stride
 * sub_bus_stride bytes, sub_bus_cols columns), line_id int32 [batch] (-1: none) with line_status int32 [batch] (+1 / -1); either
 * pair may be NULL.  A substation / line id outside [-1, n) or a busbar outside [-1, n_busbar] fails the call with B200PF_E_ARG
 * before anything is written; any line status is accepted (> 0 reconnects, < 0 disconnects, 0 leaves the line, as the host path).
 * b200pf_env_reset: env.reset() of the instances whose mask byte is 1 (topology and last busbars from topo0, cooldowns, done,
 * current_step, is_illegal and the library's protection state cleared, next row rows[i] mod n_rows or t0[i] when rows is NULL),
 * on the device.  The observe input record of those instances becomes what BatchedEnv.observe_inputs gives right after a reset.  The
 * call then waits for the mask (batch bytes) and looks the plans of the reset rows up in the same call, over the same topology, as
 * b200pf_series_reset_instances does for the host path, so that both paths build the same plans in the same calls.
 * b200pf_env_get_state / b200pf_env_set_state: hand the state over to the host path and back (device topology, chronics row,
 * active buses per instance, the instances waiting for a bus recount, the observe layer's reset flags; any pointer may be NULL;
 * set_state's obs_in: the observe input record, int32 [batch][n_line + n_sub + 3], used when the observation layer is bound).
 * b200pf_env_pointers: device topology, row index and disc_lines of
 * the series (for zero-copy views).  b200pf_observe_device: b200pf_observe on the input record the last b200pf_env_step (or
 * b200pf_env_reset) wrote, without a host copy; the reset flags it reported are cleared afterwards.
 * b200pf_env_stats out8 = { env steps, bytes the env calls copied host-to-device, device-to-host, host waits of the env steps,
 * illegal actions counted, bus cap of the last step, topology-changed instances of the last step, plan refreshes }. */
typedef struct b200pf_env_desc {
    int32_t max_sub;                    /* elements of the largest substation */
    const int32_t *sub_pos;             /* [n_sub][max_sub] topology positions of each substation's elements, -1 padded */
    const int32_t *line_of_pos, *other_end_pos;  /* [dim_topo] line whose end sits there (-1: none), position of its other end */
    int32_t cd_line, cd_sub, cd_reco;   /* NB_TIMESTEP_COOLDOWN_LINE, NB_TIMESTEP_COOLDOWN_SUB, NB_TIMESTEP_RECONNECTION */
    const uint8_t *maint, *haz;         /* [n_scen][n_rows][n_line] forced outages, or NULL */
    const int32_t *maint_time, *maint_dur;  /* [n_scen][n_rows][n_line] (with maint) */
    const int32_t *haz_dur;             /* [n_scen][n_rows][n_line] (with haz) */
    int32_t n_iso_seg, n_iso_cols;      /* isolated-busbar rule: busbar 1 of these column segments must keep an element */
    const int32_t *iso_seg, *iso_cols;  /* segment start offsets [n_iso_seg], topology columns [n_iso_cols] */
    const int8_t *topo0;                /* [batch][n_topo_in] topology of a reset */
    const int32_t *t0;                  /* [batch] row of a reset */
    /* per-instance state: caller-owned device buffers */
    int8_t *last_bus;                   /* [batch][dim_topo] */
    int32_t *line_cd, *sub_cd;          /* [batch][n_line], [batch][n_sub] */
    uint8_t *done, *is_illegal, *newly_done;  /* [batch] */
    int32_t *current_step, *status;     /* [batch]; status: the step's status with the isolated-busbar override */
} b200pf_env_desc;
int b200pf_env_bind(b200pf_handle *h, const b200pf_env_desc *desc);
int b200pf_env_step(b200pf_handle *h, const int32_t *d_sub_id, const int8_t *d_sub_bus, int sub_bus_stride, int sub_bus_cols,
                    const int32_t *d_line_id, const int32_t *d_line_status, int from_reset, int is_dc, int max_iter, double tol_mva,
                    int tight_cap, int stamp);
int b200pf_env_reset(b200pf_handle *h, const uint8_t *d_mask, const int32_t *d_rows);
int b200pf_env_get_state(b200pf_handle *h, int8_t *topo, int32_t *t, int32_t *nb_inst, uint8_t *cap_dirty, uint8_t *obs_reset);
int b200pf_env_set_state(b200pf_handle *h, const int8_t *topo, const int32_t *nb_inst, const uint8_t *cap_dirty, const uint8_t *obs_reset,
                         const int32_t *obs_in);
int b200pf_env_pointers(b200pf_handle *h, int8_t **d_topo, int32_t **d_t, int32_t **d_disc);
int b200pf_observe_device(b200pf_handle *h, float *d_obs, float *d_reward);
int b200pf_env_stats(const b200pf_handle *h, int64_t *out8);

/* The agent's action rules and grid2op's native topology action for the device environment (csrc/b200pf_env.cuh, ActArgs).
 * b200pf_act_bind needs a bound environment (b200pf_env_bind).  It copies the rules (host tables) and keeps the action buffers:
 * caller-owned DEVICE buffers the caller writes before each b200pf_env_step_act, like the alerts' raise buffer.  Once bound, the rules
 * apply to b200pf_env_step too: LookParam with max_sub_changed / max_line_status_changed over the whole grid (n_area = 0), or
 * RulesByArea's per-area counts (sub_area / line_area: bit k set for a substation / line of area k, a line in the area of its
 * origin substation; at most 16 areas), and PreventReconnection.  Without a bind, DefaultRules with both maxima at 1.
 * b200pf_env_step_act is b200pf_env_step with the step's action taken from these buffers: set_bus int8 [batch][dim_topo] (0 leave,
 * -1 disconnect a line end, 1..n_busbar), change_bus uint8 [batch][dim_topo] (0 / 1, two busbars per substation only), set_status
 * int8 [batch][n_line] (-1 / 0 / +1), change_status uint8 [batch][n_line] (0 / 1).  Per live instance, in BaseEnv.step's order:
 * BaseAction's topology ambiguity (an ambiguous action becomes "do nothing", is_ambiguous[i] = 1, is_illegal[i] = 0), the
 * topological impact on the line status the previous step left, the rules above, and _BackendAction's application (line status
 * change, then set, change_bus, then set_bus, then the reconnection / disconnection of line ends, last registered busbars from
 * last_bus).  Every impacted line and substation gets its cooldown.  An entry out of range fails the call with B200PF_E_ARG before
 * anything is written.  is_ambiguous uint8 [batch]: written by every step (0 on b200pf_env_step) and cleared by b200pf_env_reset;
 * the observe record's flags word then carries B200PF_OBS_AMBIGUOUS (RedispReward pays reward_illegal for it), and an ambiguous
 * action registers no alarm.  Host waits and bytes moved per step are those of b200pf_env_step. */
enum { B200PF_OBS_AMBIGUOUS = 8 };
typedef struct b200pf_act_desc {
    int32_t max_sub_changed, max_line_status_changed;   /* MAX_SUB_CHANGED, MAX_LINE_STATUS_CHANGED */
    int32_t n_area;                     /* RulesByArea areas, 0: none */
    const uint32_t *sub_area;           /* [n_sub] area mask of each substation (n_area > 0) */
    const uint32_t *line_area;          /* [n_line] area mask of each line (n_area > 0) */
    /* caller-owned device buffers */
    const int8_t *set_bus;              /* [batch][dim_topo] */
    const uint8_t *change_bus;          /* [batch][dim_topo] */
    const int8_t *set_status;           /* [batch][n_line] */
    const uint8_t *change_status;       /* [batch][n_line] */
    uint8_t *is_ambiguous;              /* [batch] */
} b200pf_act_desc;
int b200pf_act_bind(b200pf_handle *h, const b200pf_act_desc *desc);
int b200pf_env_step_act(b200pf_handle *h, int from_reset, int is_dc, int max_iter, double tol_mva, int tight_cap, int stamp);

/* A discrete action table for the device environment: n_act rows of grid2op's native topology action (IdToAct's list, say), each
 * instance acting with one row picked by its id.  b200pf_act_table_bind needs b200pf_act_bind (the rules, is_ambiguous and the
 * library's scratch come from there).  It checks every row with the rules of b200pf_env_step_act's vectors and fails with
 * B200PF_E_ARG, binding nothing, when one is out of range; else it copies the four HOST arrays (the layout of b200pf_act_desc's
 * buffers with n_act rows instead of batch) to device memory the library owns.  A new bind replaces the table.
 * b200pf_env_step_ids is b200pf_env_step_act with instance i taking row d_action_id[i] (DEVICE int32 [batch]) of the table.  An id
 * outside [0, n_act) fails the call with B200PF_E_ARG before anything is written.  Launches, host waits and bytes moved per step
 * are those of b200pf_env_step_act; no action data is copied. */
typedef struct b200pf_act_table_desc {
    int32_t n_act;                      /* rows */
    const int8_t *set_bus;              /* [n_act][dim_topo] */
    const uint8_t *change_bus;          /* [n_act][dim_topo] */
    const int8_t *set_status;           /* [n_act][n_line] */
    const uint8_t *change_status;       /* [n_act][n_line] */
} b200pf_act_table_desc;
int b200pf_act_table_bind(b200pf_handle *h, const b200pf_act_table_desc *desc);
int b200pf_env_step_ids(b200pf_handle *h, const int32_t *d_action_id, int from_reset, int is_dc, int max_iter, double tol_mva, int tight_cap,
                        int stamp);

/* Line-attack opponent of the device environment (csrc/b200pf_opp.cuh): grid2op's OpponentSpace with BaseActionBudget and a
 * RandomLineOpponent (kind 1) or a WeightedRandomOpponent (kind 2), attacking one line at a time with set_line_status -1, each
 * instance with its own numpy-legacy random stream (RandomState: MT19937 state of 624 words and a position, as get_state() gives
 * them).  b200pf_opp_bind needs a bound environment (b200pf_env_bind); it copies the constants and the initial random states, and
 * sets every instance to OpponentSpace.reset()'s state.  From then on the apply launch of b200pf_env_step runs the opponent of every
 * live instance before the agent's action, on the line status and rho the previous step left, and takes the attacked line out after
 * the environment's outages, with its line cooldown raised to the attack's duration; a reset step and a finished instance attack
 * nothing and draw nothing.  b200pf_env_reset resets the opponent of the reset instances (the random stream continues).  After
 * each b200pf_env_step the caller-owned device buffers hold: attack_line int32 [batch] (-1: none), attack_dur int32 [batch] (0: none)
 * and budget float64 [batch] (the opponent's budget, which is also its state).  b200pf_opp_get_state / b200pf_opp_set_state: the
 * opponent state to the host and back (any pointer may be NULL): budget float64 [batch], budget64 uint8 [batch] (the budget has been
 * charged since the last reset: grid2op then holds it as a float64, before as a float32), ctr int32 [batch][4] (current attack
 * duration, current attack cooldown, last attacked line or -1, steps to the weighted opponent's next attack or INT32_MIN for
 * none), mt uint32 [batch][624] and mt_pos int32 [batch].  Unbound (b200pf_opp_bind never called), nothing of the above runs. */
typedef struct b200pf_opp_desc {
    int32_t kind;                       /* 1: RandomLineOpponent, 2: WeightedRandomOpponent, 3: GeometricOpponent,
                                           4: GeometricOpponentMultiArea */
    int32_t n_attack;                   /* attackable lines, 1..64 */
    const int32_t *lines;               /* [n_attack] their line ids */
    const double *rho_norm;             /* [n_attack] rho normalisation (kind 2) */
    int32_t attack_period;              /* kind 2: an attack is drawn uniformly within this many steps */
    int32_t attack_duration, attack_cooldown;
    float budget_per_ts, init_budget;
    const uint32_t *mt;                 /* [batch][624] initial MT19937 states */
    const int32_t *mt_pos;              /* [batch] their positions (0..624) */
    /* caller-owned device buffers [batch] */
    int32_t *attack_line, *attack_dur;
    double *budget;
} b200pf_opp_desc;
int b200pf_opp_bind(b200pf_handle *h, const b200pf_opp_desc *desc);
int b200pf_opp_get_state(b200pf_handle *h, double *budget, uint8_t *budget64, int32_t *ctr, uint32_t *mt, int32_t *mt_pos);
int b200pf_opp_set_state(b200pf_handle *h, const double *budget, const uint8_t *budget64, const int32_t *ctr, const uint32_t *mt,
                         const int32_t *mt_pos);

/* GeometricOpponent (kind 3): b200pf_opp_bind with kind 3 (rho_norm and attack_period unused), then b200pf_opp_geo_bind with its
 * constants and every instance's first schedule; b200pf_env_step refuses to step a kind-3 opponent without it.  Each instance keeps
 * an attack schedule (waiting times and durations int32 [cap], drawn by GeometricOpponent.sample_attack_times_and_durations with
 * RandomState.geometric on the instance's stream) and four int32 counters: schedule length, attacks consumed, OpponentSpace's
 * previous_fails, and schedule entries dropped because they did not fit the cap (0 unless cap is too small).  ctr[3] of
 * b200pf_opp_get_state is the opponent's _next_attack_time (INT32_MIN for None).  b200pf_env_reset draws a new schedule for each
 * reset instance on the device.  The apply launch reads the rho the previous step left, as for kind 2. */
typedef struct b200pf_opp_geo_desc {
    const double *weights;              /* [n_attack] np.exp(b_beta * k), k = 0 .. n_attack - 1 */
    double p_hazard, p_recovery;        /* attack hazard rate, recovery rate */
    double logq_hazard, logq_recovery;  /* log(1 - p) of both */
    int32_t recovery_min;               /* minimum attack duration in steps */
    int32_t cap;                        /* schedule entries per instance, >= 1 */
    const int32_t *episode_max_time;    /* [batch] */
    const int32_t *wait, *dur;          /* [batch][cap] the initial schedules */
    const int32_t *gctr;                /* [batch][4] their counters */
} b200pf_opp_geo_desc;
int b200pf_opp_geo_bind(b200pf_handle *h, const b200pf_opp_geo_desc *desc);
int b200pf_opp_geo_get_state(b200pf_handle *h, int32_t *wait, int32_t *dur, int32_t *gctr);
int b200pf_opp_geo_set_state(b200pf_handle *h, const int32_t *wait, const int32_t *dur, const int32_t *gctr);

/* GeometricOpponentMultiArea (kind 4): b200pf_opp_bind with kind 4 and the lines of every area one after the other (rho_norm and
 * attack_period unused; mt is the multi-area opponent's own stream, which only seeds the areas and is not drawn from again), then
 * b200pf_opp_multi_bind; b200pf_env_step and b200pf_env_reset refuse a kind-4 opponent without it.  Each area is a GeometricOpponent
 * with its own stream (mt uint32 [batch][n_area][624], mt_pos int32 [batch][n_area]), its own schedule (wait / dur int32
 * [batch][n_area][cap]) and six int32 counters (actr [batch][n_area][6]: schedule length, attacks consumed, _next_attack_time or
 * INT32_MIN for None, schedule entries dropped at the cap, _new_attack_time_counters, _previous_attacks line or -1); fails int32
 * [batch] is OpponentSpace's previous_fails.  Every step asks every live instance (the opponent's duration is always 1); the
 * combined attack costs one per line and is refused whole.  attack_lines (device, caller-owned, int32 [batch][n_area]) receives
 * each step's attacked line per area (-1: none); b200pf_opp_bind's attack_line receives the first of them (-1: none) and attack_dur
 * 1 or 0.  b200pf_env_reset draws every reset instance's area schedules on the device, in area order. */
typedef struct b200pf_opp_multi_desc {
    int32_t n_area;                     /* 1..8 */
    const int32_t *area_off;            /* [n_area + 1] area k's lines are lines[area_off[k] .. area_off[k + 1]), none empty */
    const double *weights;              /* [n_attack] area k's np.exp(b_beta_k * r) at area_off[k] + r */
    double p_hazard, p_recovery;        /* attack hazard rate, recovery rate */
    double logq_hazard, logq_recovery;  /* log(1 - p) of both */
    int32_t recovery_min;               /* minimum attack duration in steps */
    int32_t cap;                        /* schedule entries per instance and area, >= 1 */
    const int32_t *episode_max_time;    /* [batch] */
    const uint32_t *mt;                 /* [batch][n_area][624] the areas' initial streams */
    const int32_t *mt_pos;              /* [batch][n_area] */
    const int32_t *wait, *dur;          /* [batch][n_area][cap] the initial schedules */
    const int32_t *actr;                /* [batch][n_area][6] their counters */
    const int32_t *fails;               /* [batch] previous_fails */
    int32_t *attack_lines;              /* device [batch][n_area] per-step output */
} b200pf_opp_multi_desc;
int b200pf_opp_multi_bind(b200pf_handle *h, const b200pf_opp_multi_desc *desc);
int b200pf_opp_multi_get_state(b200pf_handle *h, uint32_t *mt, int32_t *mt_pos, int32_t *wait, int32_t *dur, int32_t *actr, int32_t *fails);
int b200pf_opp_multi_set_state(b200pf_handle *h, const uint32_t *mt, const int32_t *mt_pos, const int32_t *wait, const int32_t *dur,
                               const int32_t *actr, const int32_t *fails);

/* Line alerts of the device environment (grid2op's alerts of l2rpn_idf_2023, csrc/b200pf_alert.cuh), after b200pf_env_bind.
 * b200pf_alert_bind copies the alertable lines (host, n_alert <= 64, in grid2op's order) and the constants, allocates the
 * per-instance state in the library and sets every instance to BaseEnv._reset_alert + AlertReward.reset.  From then on the post
 * launch of b200pf_env_step updates, for every instance live before the step and not on a reset step, the environment's alert
 * state (BaseEnv._update_alert_properties, with the attacked lines of the opponent bound by b200pf_opp_bind / _multi_bind, none
 * without an opponent) and, when `reward`, the AlertReward into reward_out (float64 [batch], caller-owned device buffer; 0 for
 * the other instances).  raise_alert: caller-owned DEVICE uint8 [batch][n_alert] the caller fills before each step (0 / 1).
 * b200pf_env_reset resets the alert state of the reset instances.  With the observation layer bound with the same n_alert, the
 * post and reset launches write the alert values into the observe input record.  get_state / set_state copy the whole state
 * between the device and host arrays (any pointer may be NULL): last_alert / already uint8 [batch][n], tsl_alert / duration /
 * tsl_attack / under_alert / was_used int32 [batch][n], total / cur_id int32 [batch], ts_attack / launched uint8
 * [batch][window + 2][n], current uint8 [batch][n] (AlertReward._ts_attack, _alert_launched, _lines_currently_attacked). */
typedef struct b200pf_alert_desc {
    int32_t n_alert;                    /* dim_alerts, 1..64 */
    const int32_t *lines;               /* [n_alert] alertable line ids */
    int32_t window;                     /* ALERT_TIME_WINDOW, >= 1 */
    int32_t reward;                     /* compute AlertReward (and was_alert_used_after_attack) */
    float reward_min_no_blackout, reward_min_blackout, reward_max_no_blackout, reward_max_blackout;
    const uint8_t *raise_alert;         /* device [batch][n_alert] step input */
    double *reward_out;                 /* device [batch] per-step output */
} b200pf_alert_desc;
int b200pf_alert_bind(b200pf_handle *h, const b200pf_alert_desc *desc);
int b200pf_alert_get_state(b200pf_handle *h, uint8_t *last_alert, uint8_t *already, int32_t *tsl_alert, int32_t *duration,
                           int32_t *tsl_attack, int32_t *under_alert, int32_t *was_used, int32_t *total, uint8_t *ts_attack,
                           uint8_t *launched, uint8_t *current, int32_t *cur_id);
int b200pf_alert_set_state(b200pf_handle *h, const uint8_t *last_alert, const uint8_t *already, const int32_t *tsl_alert,
                           const int32_t *duration, const int32_t *tsl_attack, const int32_t *under_alert, const int32_t *was_used,
                           const int32_t *total, const uint8_t *ts_attack, const uint8_t *launched, const uint8_t *current,
                           const int32_t *cur_id);

/* Alarms of the device environment (grid2op's alarms of l2rpn_icaps_2021, csrc/b200pf_alarm.cuh), after b200pf_env_bind.
 * b200pf_alarm_bind copies the zones of every line (host uint32 [n_line], bit z: zone z of the sorted zone names; every line in
 * at least one zone) and the constants, allocates the per-instance state in the library and sets every instance to
 * LinearAttentionBudget.reset.  From then on the post launch of b200pf_env_step, for every instance live before the step and not
 * on a reset step, registers the step's alarm (LinearAttentionBudget.register_action, after the legality of the action) into
 * is_alarm_illegal (uint8 [batch], caller-owned device buffer; 0 for the other instances) and, when `reward`, computes the
 * AlarmReward into reward_out (float64 [batch], caller-owned device buffer; non-zero only on the step that ends an episode with
 * an error, with the step's disc_lines when the protections are on).  raise_alarm: caller-owned DEVICE uint8 [batch][n_zone] the
 * caller fills before each step (0 / 1).  b200pf_env_reset resets the attention budget of the reset instances and keeps the
 * reward's is_alarm_used.  With the observation layer bound with the same n_alarm, the post and reset launches write the alarm
 * values into the observe input record.  get_state / set_state copy the whole state between the device and host arrays (any
 * pointer may be NULL): budget float32 [batch]; time_last / time_last_ok int32 [batch]; last / last_ok int32 [batch][n_zone];
 * ring_step int32 / ring_mask uint32 [batch][best_time + window_size] (the successful alarms of the last steps, slot step %
 * ring, step 0: empty); any_ok / used / illegal uint8 [batch] (a successful alarm this episode, is_alarm_used, the caller's
 * is_alarm_illegal). */
typedef struct b200pf_alarm_desc {
    int32_t n_zone;                     /* dim_alarms, 1..32 */
    const uint32_t *zone_mask;          /* [n_line] zones of each line */
    float max_budget, budget_per_ts, alarm_cost, init_budget;   /* LinearAttentionBudget */
    int32_t best_time, window_size;     /* ALARM_BEST_TIME, ALARM_WINDOW_SIZE: >= 1, their sum <= 1024 */
    int32_t reward;                     /* compute AlarmReward (and is_alarm_used) */
    const uint8_t *raise_alarm;         /* device [batch][n_zone] step input */
    double *reward_out;                 /* device [batch] per-step output */
    uint8_t *is_alarm_illegal;          /* device [batch] per-step output */
} b200pf_alarm_desc;
int b200pf_alarm_bind(b200pf_handle *h, const b200pf_alarm_desc *desc);
int b200pf_alarm_get_state(b200pf_handle *h, float *budget, int32_t *time_last, int32_t *time_last_ok, int32_t *last, int32_t *last_ok,
                           int32_t *ring_step, uint32_t *ring_mask, uint8_t *any_ok, uint8_t *used, uint8_t *illegal);
int b200pf_alarm_set_state(b200pf_handle *h, const float *budget, const int32_t *time_last, const int32_t *time_last_ok,
                           const int32_t *last, const int32_t *last_ok, const int32_t *ring_step, const uint32_t *ring_mask,
                           const uint8_t *any_ok, const uint8_t *used, const uint8_t *illegal);

int b200pf_sync(b200pf_handle *h);
/* cudaStream_t of the handle as an integer (for event timing by the caller) */
uint64_t b200pf_stream(b200pf_handle *h);
/* number of kernels launched by this handle so far */
int64_t b200pf_launch_count(const b200pf_handle *h);
/* dynamic shared memory bytes and threads-per-instance the last launch used (diagnostics) */
int b200pf_last_launch_info(const b200pf_handle *h, int *smem_bytes, int *threads_per_instance,
                            int *grid_blocks, int *block_threads);
/* template parameters of the kernel the last launch ran (diagnostics; tests read which dispatch branch was taken), 8 ints:
 * block kernel (pf_kernel_block): T (lanes per instance), U (operations per lane and row), MINB (resident CTAs the register
 * budget is compiled for), PROT, WPC (warps per CTA), STAGE (shared plan copied into shared memory), UNI (lockstep warps),
 * MODE (1: AC solve fed by chronics rows); scalar planned kernel (pf_kernel_sparse): T, -1, MINB, PROT, -1, -1, -1, -1;
 * pivoting kernels: all -1.  With b200pf_last_launch_info, the launch ran ceil(batch / (grid_blocks * block_threads /
 * threads_per_instance)) waves: rounds of its persistent CTAs. */
int b200pf_last_launch_config(const b200pf_handle *h, int *cfg8);

#ifdef __cplusplus
}
#endif
#endif /* B200PF_H */

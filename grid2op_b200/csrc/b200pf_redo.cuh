// b200pf_redo.cuh — the safety net of the planned kernels.
//
// The planned kernels (b200pf_sparse.cuh, b200pf_block.cuh) eliminate WITHOUT pivoting, on an fp32 Jacobian.  The reference's
// solver (pandapower's newtonpf behind pp.runpp, grid2op/Backend/pandaPowerBackend.py:1097-1105) factorises with partial
// pivoting in fp64.  Whatever the planned kernel ends as ST_DIV — breakdown of the factorisation (non-finite update), a stalled
// iteration, or a genuine divergence — is therefore solved AGAIN here with the pivoting kernel (pf_kernel's solve_instance,
// fp64 Jacobian where the workspace allows it) before the status leaves the library, so that `runpf -> (False, exc)`
// (pPB:1241-1255) is only ever reported for states the pivoting solver gives up on as well.
//
// The planned kernel launches it itself, as a tail launch, the first time one of its instances ends as ST_DIV (redo_arm,
// b200pf_sparse.cuh): it runs once the planned grid has completed, on the same stream, no host round trip, and a planned
// launch without such an instance costs nothing here.  Every CTA scans the status words of 32 instances (one coalesced
// load) and re-solves those that read ST_DIV.
#pragma once
#include "b200pf_sparse.cuh"

namespace b200pf {

// Protections of one instance after a re-solve (planned kernel with PROT: the rules of Backend.next_grid_state,
// reference backend.py:1466-1521, counters baseEnv.py:3361-3370 — same arithmetic as the PROT block of solve_sparse).
// Line status comes from the topology record (the planned kernel takes it from its plan).
template <int T>
__device__ void redo_prot_round(const DevGrid &g, const RunArgs &a, int inst, int tid) {
    const int nl = g.n_line;
    const size_t base_l = (size_t)inst * nl;
    const int8_t *tv = a.topo + (size_t)inst * g.n_topo_in;
    const float *out = a.out + (size_t)inst * g.n_out;
    int any_trip = 0;
    for (int l = tid; l < nl; l += T) {
        const bool on = tv[g.line_or_pos[l]] > 0 && tv[g.line_ex_pos[l]] > 0;
        const float aor = out[3 * nl + l], lim = a.th_lim[l];
        int inc = a.casc > 0 ? (int)a.incdone[base_l + l] : 0;
        int pc = a.pcount[base_l + l] + inc;
        bool to_disc = on && (aor > __fmul_rn(a.hard_thr, lim));
        if (!a.from_reset && on && (aor > __fmul_rn(a.soft_thr, lim)) && !inc) { pc += 1; inc = 1; }
        if (on && pc > a.max_pc) to_disc = true;
        a.incdone[base_l + l] = (int8_t)inc;
        if (a.casc == 0) a.disc[base_l + l] = -1;
        if (to_disc) { a.trip[base_l + l] = 1; a.disc[base_l + l] = a.casc; any_trip = 1; }
    }
    any_trip = (T == 32) ? __any_sync(0xffffffffu, any_trip) : __syncthreads_or(any_trip);
    if (any_trip) {
        if (tid == 0) { const int slot = atomicAdd(a.n_flag, 1); a.flag_list[slot] = inst; }
    } else {
        for (int l = tid; l < nl; l += T) {
            const float aor = out[3 * nl + l], lim = a.th_lim[l];
            int *pcp = a.pcount + base_l, *tsp = a.ts_over + base_l;
            pcp[l] = (!a.from_reset && aor > __fmul_rn(a.soft_thr, lim)) ? pcp[l] + 1 : 0;
            tsp[l] = (!a.from_reset && aor > lim) ? tsp[l] + 1 : 0;
            a.incdone[base_l + l] = 0;
        }
    }
    gsync<T>();
}

template <int T, typename JT>
__global__ void __launch_bounds__(T, (T == 32) ? 8 : 1)
pf_kernel_redo(const DevGrid g, const RunArgs a, RedoCtl *ctl) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x;
    // no CTA of the planned grid that launched this one runs any more: the next planned launch on this stream may arm again
    if (blockIdx.x == 0 && tid == 0) ctl->armed = 0;
    for (int first = blockIdx.x * 32; first < a.batch; first += gridDim.x * 32) {
        // every warp of the CTA computes the same mask (the status words are only written at the very end of a
        // re-solve, behind group barriers that all warps pass)
        const int k = first + (tid & 31);
        const int st = k < a.batch ? a.status[a.inst_list ? a.inst_list[k] : k] : ST_OK;
        unsigned m = __ballot_sync(0xffffffffu, st == ST_DIV);
        while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const int inst = a.inst_list ? a.inst_list[first + b] : first + b;
            solve_instance<T, JT>(g, a, inst, smem, tid);
            if (a.prot) {
                gsync<T>();
                const int ok = a.status[inst] == ST_OK;
                if (ok) {
                    if (tid == 0) a.done[inst] = 0;       // the planned kernel had declared the instance game over
                    redo_prot_round<T>(g, a, inst, tid);
                }
            }
            gsync<T>();
        }
    }
}

// env.reset() of single instances of a bound series: counters, flags and the row pointer back to a fresh episode
__global__ void pf_kernel_series_reset(int n, const int *idx, const int *t_new, int n_line, int *t, int *done, int *pcount, int *ts_over, int *disc,
                                       int8_t *trip, int8_t *incdone) {
    const int k = blockIdx.x;
    if (k >= n) return;
    const int inst = idx[k];
    if (threadIdx.x == 0) { done[inst] = 0; if (t_new) t[inst] = t_new[k]; }
    for (int l = threadIdx.x; l < n_line; l += blockDim.x) {
        const size_t o = (size_t)inst * n_line + l;
        pcount[o] = 0; ts_over[o] = 0; disc[o] = -1; trip[o] = 0; incdone[o] = 0;
    }
}

// completion flag of a series step (multi-GPU result collection without a collective): one thread publishes the step number,
// system-wide (the flag may sit in the agent rank's HBM, next to the results the step stored there).  Stream order puts it
// behind the step's kernels, the safety net they tail-launched included.
__global__ void pf_kernel_flag(int *flag, int value) {
    __threadfence_system();
    *reinterpret_cast<volatile int *>(flag) = value;
}

}  // namespace b200pf

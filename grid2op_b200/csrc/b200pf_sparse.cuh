// b200pf_sparse.cuh — the PLANNED SPARSE kernel: one warp (T = 32) or one CTA (T > 32) per grid instance,
// driven by the topology plan of b200pf_plan.hpp.
//
// Compared with pf_kernel_small / pf_kernel (which discover the topology of every instance on the device and
// solve dense systems with partial pivoting) this kernel does no topology work and no dense algebra at all:
//   inputs -> per-bus sums (plan lists) -> DC start = one product with the plan's fp64 inverse of Bdc -> Newton { branch currents (lane = line), S(V) and |F|inf in fp64 (lane = bus), Jacobian values
//   scattered to their packed positions (fp32, shared memory), LU = the plan's passes of independent
//   A[ij] -= A[ik] A[kj] / A[kk] operations (lane = operation; elimination and both triangular solves),
//   fp64 state update } -> result record.
// Work per instance drops from O(d^3) to O(nnz of the filled Jacobian) and the per-instance workspace from a
// dense matrix to a few KB, so the 36- and 118-substation grids keep many instances resident per SM.
// Same arithmetic plan as the other kernels (fp64 state / mismatch / flows, fp32 Jacobian and solve, the fp64
// residual decides convergence with pandapower's criterion), same result record, same status classes.
// Elimination is WITHOUT pivoting on the (theta_i, |V|_i)-interleaved minimum-degree order: a breakdown shows
// up as a non-finite update and ends as ST_DIV.  ST_DIV is never final here: the first such instance makes this kernel
// tail-launch pf_kernel_redo (b200pf_redo.cuh), which re-solves every such instance with partial pivoting.
//
// The body is written as a sequence of PHASES separated by group barriers, every piece of state that crosses a
// phase lives in the (shared-memory) workspace.  With B200PF_EMULATE the same source compiles as plain host
// C++ where a phase is a loop over the lanes: tests/ use that build to debug the plan + numerics without a GPU
// (test infrastructure only — the product never executes it).
#pragma once
#include "b200pf_plan.hpp"

#ifdef B200PF_EMULATE
#include <math.h>
#include <stdint.h>
#include <cstddef>
namespace b200pf {
struct double2 { double x, y; };
struct uint2 { unsigned x, y; };
struct float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline double2 make_double2(double x, double y) { double2 r; r.x = x; r.y = y; return r; }
}
#define PF_DEV static inline
#define PF_PHASE for (int tid = 0; tid < T; ++tid)
#define PF_SYNC() ((void)0)
#define PF_ANY(x) (x)
#define PF_FDIV(a, b) ((float)(a) / (float)(b))
#define PF_FMUL(a, b) ((float)(a) * (float)(b))
#define PF_RCP(x) (1.0f / (x))
#define PF_SINCOS(x, s, c) do { *(s) = sin(x); *(c) = cos(x); } while (0)
#define PF_QNANF() (__builtin_nanf(""))
#define PF_QNAN() (__builtin_nan(""))
#define PF_LDCS(p) (*(p))
#else
#include "b200pf_kernel.cuh"
#define PF_DEV __device__ __forceinline__
#define PF_PHASE
#define PF_SYNC() sp_sync<T>()
#define PF_ANY(x) sp_any<T>(x)
#define PF_FDIV(a, b) __fdiv_rn((a), (b))
#define PF_FMUL(a, b) __fmul_rn((a), (b))
#define PF_RCP(x) sp_rcp(x)
#define PF_SINCOS(x, s, c) sincos((x), (s), (c))
#define PF_QNANF() __int_as_float(0x7fc00000)
#define PF_QNAN() __longlong_as_double(0x7ff8000000000000LL)
#define PF_LDCS(p) __ldcs(p)      // streaming load: read once per instance, must not evict the re-used plan arrays from L1
#endif

namespace b200pf {

#ifdef B200PF_EMULATE
// the slices of DevGrid / RunArgs the emulation build needs (same field names)
struct DevGrid {
    int n_sub, n_busbar, n_slot, n_line, n_gen, n_hidden, n_unit, n_load, n_sto, n_shunt, dim_topo;
    int n_topo_in, n_inj, n_out;
    double base_mva;
    const double *line_y, *line_bdc, *line_pshift;
    const float *line_or_vn, *line_ex_vn;
    const int *unit_is_ref;
    const double *unit_qmin, *unit_qmax;
    const float *unit_vn, *load_vn, *sto_vn, *sh_vn;
    const double *sto_q, *sh_vratio;
};
struct RunArgs {
    int batch;
    const double *inj;
    int is_dc, max_iter;
    double tol_pu;
    float *out;
    int *status, *iters;
    double *busv;
    int series;
    const float *chron;
    int n1_lines;
    const float *rows;
    int n_scen, n_rows;
    const int *scen;
    int *t;
    const double *static_inj;
    const float *th_lim;
    float *rho;
    int prot, from_reset, max_pc;
    float hard_thr, soft_thr;
    int *pcount, *ts_over, *disc, *done;
    int casc;
    const int *inst_list;
    int8_t *trip, *incdone;
    int *n_flag, *flag_list;
    int redo, dbg_div_mod;
    unsigned char *redo_mat; size_t redo_mat_stride;
};
enum { ST_OK = 0, ST_DIV = 1, ST_UNSUP = 2, ST_NOREF = 3, ST_LARGE = 4, ST_DONE = 5 };
enum { BT_PQ = 1, BT_PV = 2, BT_REF = 3 };
#else
template <int T> __device__ __forceinline__ void sp_sync() { if (T == 32) __syncwarp(); else __syncthreads(); }
template <int T> __device__ __forceinline__ int sp_any(int p) { return (T == 32) ? __any_sync(0xffffffffu, p) : __syncthreads_or(p); }
__device__ __forceinline__ float sp_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#endif

struct PlanArgs {
    const unsigned char *blobs;   // all plans of this launch, concatenated (each 16-byte aligned)
    const int *plan_off;          // [n_plan] byte offset of every plan
    const int *inst_plan;         // [batch] plan of every instance, or nullptr = plan 0 for all
    // block kernel: the instances interleaved in one warp must agree on the workspace layout whatever their plans are ->
    // array strides of the LAUNCH (maxima over its plans): buses, value blocks
    int lay_nb, lay_nblkA;
    // block kernel, staged launches: the static grid arrays the solve reads (line admittances, nominal voltages, unit limits, the
    // static injections, the thermal limits), packed into one blob that is staged next to the plan; nullptr: DevGrid's own
    // pointers (through L1 / L2 — cold after every L2 flush: ~15 dependent misses per warp in a one-wave launch)
    const unsigned char *stat;
    struct StatOff { int line_y, line_bdc, line_pshift, line_or_vn, line_ex_vn, unit_is_ref, unit_qmin, unit_qmax, unit_vn, load_vn, sto_vn, sto_q,
                         sh_vn, sh_vratio, static_inj, th_lim, total; } so;
};

// Safety net of the planned kernels (b200pf_redo.cuh).  The first instance of a planned launch that ends as ST_DIV makes
// the kernel itself launch the pivoting re-solve, as a tail launch of its grid: it starts once the planned grid has completed,
// and stream order counts the planned launch as complete only once the re-solve is.  A launch without such an instance
// launches nothing.
struct RedoCtl {              // one per stream of a handle, in device memory
    int armed;                // 1: this stream's running planned launch has queued its re-solve (pf_kernel_redo clears it)
    int launches;             // re-solves launched so far
};
struct RedoDesc {
    int on;                   // 0: no safety net behind this launch (B200PF_NO_REDO, b200pf_set_debug, DC solves)
    int T, grid, smem;        // pf_kernel_redo<T, double>: threads per instance, CTAs, dynamic shared memory
    int nb_cap, mat_bytes;    // the re-solve's RunArgs: the planned launch's, with redo = 1 and these
    unsigned char *mat; size_t mat_stride;      // -> RunArgs::redo_mat / redo_mat_stride
    RedoCtl *ctl;
};

#ifdef B200PF_EMULATE
#define PF_REDO_ARM(g, a, rd) ((void)(rd))
#else
template <int T, typename JT> __global__ void pf_kernel_redo(const DevGrid g, const RunArgs a, RedoCtl *ctl);
// Called by one lane of every instance a planned kernel ends as ST_DIV: the first one of the launch tail-launches the re-solve
// for the whole launch (pf_kernel_redo scans every status word of the launch).
__device__ __forceinline__ void redo_arm(const DevGrid &g, const RunArgs &a, const RedoDesc &rd) {
    if (!rd.on || atomicCAS(&rd.ctl->armed, 0, 1) != 0) return;
    RunArgs r = a;
    r.redo = 1; r.nb_cap = rd.nb_cap; r.mat_bytes = rd.mat_bytes; r.redo_mat = rd.mat; r.redo_mat_stride = rd.mat_stride;
    // (one launch site: the parameter block is written once, whichever of the four variants runs)
    void (*kern)(const DevGrid, const RunArgs, RedoCtl *);
    switch (rd.T) {
        case 32: kern = pf_kernel_redo<32, double>; break;
        case 128: kern = pf_kernel_redo<128, double>; break;
        case 256: kern = pf_kernel_redo<256, double>; break;
        default: kern = pf_kernel_redo<512, double>; break;
    }
    kern<<<rd.grid, rd.T, rd.smem, cudaStreamTailLaunch>>>(g, r, rd.ctl);
    atomicAdd(&rd.ctl->launches, 1);
}
#define PF_REDO_ARM(g, a, rd) redo_arm((g), (a), (rd))
#endif

template <int T>
PF_DEV void sparse_fail(const DevGrid &g, const RunArgs &a, int inst, int status, int iters, int tid0, const RedoDesc &rd) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
    PF_PHASE {
        if (tid == 0) {
            a.status[inst] = status; a.iters[inst] = iters; if (a.prot && a.done) a.done[inst] = 1;
            if (status == ST_DIV) PF_REDO_ARM(g, a, rd);
        }
        if (a.prot && a.disc && status == ST_DONE) for (int k = tid; k < g.n_line; k += T) a.disc[(size_t)inst * g.n_line + k] = -1;
        if (out) for (int k = tid; k < g.n_out; k += T) out[k] = PF_QNANF();
        if (a.busv) for (int k = tid; k < 2 * g.n_slot; k += T) a.busv[(size_t)inst * 2 * g.n_slot + k] = PF_QNAN();
        if (a.rho) for (int k = tid; k < g.n_line; k += T) a.rho[(size_t)inst * g.n_line + k] = PF_QNANF();
    }
    PF_SYNC();
    (void)tid0;
}

template <int T, bool PROT>
PF_DEV void solve_sparse(const DevGrid &g, const RunArgs &a, const PlanArgs &pa, int inst, unsigned char *sm, int tid0,
                         const RedoDesc &rd = RedoDesc()) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
    const int src = a.n1_lines > 0 ? inst / a.n1_lines : inst;          // record the inputs come from
    const unsigned char *blob = pa.blobs + pa.plan_off[pa.inst_plan ? pa.inst_plan[inst] : 0];
    const PlanHeader &H = *reinterpret_cast<const PlanHeader *>(blob);
    // series bookkeeping first (an instance advances its row even when its topology cannot be solved)
    int trow = 0, sc = 0;
    if (a.series && !a.rows) {
        sc = a.scen[src]; trow = a.t[src];
        PF_SYNC();
        if (PROT && a.casc > 0) trow = trow == 0 ? a.n_rows - 1 : trow - 1;       // later cascade rounds re-solve the SAME row
        PF_PHASE { if (tid == 0 && a.n1_lines <= 0 && !(PROT && a.casc > 0)) a.t[inst] = (trow + 1 >= a.n_rows) ? 0 : trow + 1; }
    }
    if (PROT && a.done[inst] && a.casc == 0) { sparse_fail<T>(g, a, inst, ST_DONE, 0, tid0, rd); return; }
    if (H.status != PLAN_ST_OK) { sparse_fail<T>(g, a, inst, H.status, 0, tid0, rd); return; }
    if (a.dbg_div_mod > 0 && inst % a.dbg_div_mod == 0) { sparse_fail<T>(g, a, inst, ST_DIV, 0, tid0, rd); return; }   // test knob (b200pf_set_debug)
    const int nb = H.nb, nl = g.n_line, nu = g.n_unit, nh = g.n_hidden, ng = g.n_gen, nld = g.n_load, nst = g.n_sto, nsh = g.n_shunt;
    const int d = H.d, nnzF = H.nnzF, nA = H.nA;
    const double base = g.base_mva;
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
#define U16(off) reinterpret_cast<const uint16_t *>(blob + H.off)
#define F64(off) reinterpret_cast<const double *>(blob + H.off)
    const uint16_t *p_colth = U16(o_colth), *p_colv = U16(o_colv), *p_dcidx = U16(o_dcidx);
    const uint16_t *p_brf = U16(o_brf), *p_brt = U16(o_brt);
    const uint16_t *adj_ptr = U16(o_adj_ptr), *adj = U16(o_adj), *shidx = U16(o_shidx);
    // ---- workspace ------------------------------------------------------------------------------------
    // A first: on the device it then sits at shared-memory offset 0 and the operation stream's byte offsets address it directly
    float *A = reinterpret_cast<float *>(sm);
    double *vm = reinterpret_cast<double *>(sm + (((size_t)(nA + 1) * 4 + 15) & ~(size_t)15)), *va = vm + nb, *psp = va + nb, *qsp = psp + nb,
           *Pc = qsp + nb, *Qc = Pc + nb, *gsh = Qc + nb, *bsh = gsh + nsh;     // gsh / bsh: per bus WITH a shunt (plan index shidx)
    double2 *V = reinterpret_cast<double2 *>(bsh + nsh);
    double2 *cur = V + nb;
    float *srow = reinterpret_cast<float *>(cur + 2 * nl);
    // ---- injections of this instance ----------------------------------------------------------------------
    const float *row = nullptr;
    const double *rec = nullptr, *si = a.static_inj;
    if (a.series) {
        // this step's row is staged in shared memory with one coalesced read (it may live in pinned HOST memory:
        // B200PF_GROUP_ZEROCOPY_IN), every later use is a shared-memory load
        const float *grow = a.rows ? a.rows + (size_t)src * (size_t)(2 * nld + 2 * ng)
                                   : a.chron + ((size_t)sc * a.n_rows + trow) * (size_t)(2 * nld + 2 * ng);
        PF_PHASE { for (int k = tid; k < 2 * nld + 2 * ng; k += T) srow[k] = grow[k]; }
        PF_SYNC();
        row = srow;
    } else rec = a.inj + (size_t)src * g.n_inj;
#define GEN_P(u) ((u) < nh ? 0.0 : (row ? (double)row[2 * nld + (u) - nh] : rec[(u) - nh]))
#define UNIT_VM(u) (row ? ((u) >= nh ? (double)PF_FDIV(row[2 * nld + ng + (u) - nh], g.unit_vn[u]) : si[ng + (u)]) : rec[ng + (u)])
#define LOAD_P(k) (row ? (double)row[k] : rec[ng + nu + (k)])
#define LOAD_Q(k) (row ? (double)row[nld + (k)] : rec[ng + nu + nld + (k)])
#define STO_P(k) (row ? si[ng + nu + 2 * nld + (k)] : rec[ng + nu + 2 * nld + (k)])
#define SH_P(k) (row ? si[ng + nu + 2 * nld + nst + (k)] : rec[ng + nu + 2 * nld + nst + (k)])
#define SH_Q(k) (row ? si[ng + nu + 2 * nld + nst + nsh + (k)] : rec[ng + nu + 2 * nld + nst + nsh + (k)])

    // ---- 1. per-bus sums in element order; right-hand side of the DC system (lane = bus) -----------------
    {
        const uint16_t *bu_ptr = U16(o_bu_ptr), *bu = U16(o_bu), *bl_ptr = U16(o_bl_ptr), *bl = U16(o_bl);
        const uint16_t *bs_ptr = U16(o_bs_ptr), *bs = U16(o_bs), *bh_ptr = U16(o_bh_ptr), *bh = U16(o_bh);
        const uint16_t *vmunit = U16(o_vmunit);
        const double *dcshift = F64(o_dcshift);
        PF_PHASE {
            for (int i = tid; i < nb; i += T) {
                double pg = 0.0, pd = 0.0, qd = 0.0, gs = 0.0, bsu = 0.0;
                for (int e = bu_ptr[i]; e < bu_ptr[i + 1]; ++e) { const int u = bu[e]; pg += GEN_P(u); }
                for (int e = bl_ptr[i]; e < bl_ptr[i + 1]; ++e) { const int k = bl[e]; pd += LOAD_P(k); qd += LOAD_Q(k); }
                for (int e = bs_ptr[i]; e < bs_ptr[i + 1]; ++e) { const int k = bs[e]; pd += STO_P(k); qd += g.sto_q[k]; }
                for (int e = bh_ptr[i]; e < bh_ptr[i + 1]; ++e) { const int k = bh[e]; gs += SH_P(k) * g.sh_vratio[k]; bsu -= SH_Q(k) * g.sh_vratio[k]; }
                const int vu = vmunit[i];
                vm[i] = vu != 0xFFFF ? UNIT_VM(vu) : 1.0;
                const double ps = (pg - pd) / base, gpu = gs / base;
                psp[i] = ps; qsp[i] = -qd / base;
                const int sx = shidx[i];
                if (sx != 0xFFFF) { gsh[sx] = gpu; bsh[sx] = bsu / base; }
                const int c = p_dcidx[i];
                if (c != 0xFFFF) Pc[c] = ps - gpu - dcshift[i];
            }
        }
        PF_SYNC();
    }
    // ---- 2. DC angles: theta = Bdc^-1 b with the plan's fp64 inverse (lane = row; Pc = right-hand side, Qc = result) ------
    {
        const double *inv = F64(o_dcinv);
        const int n1 = H.n1;
        PF_PHASE {
            for (int i = tid; i < n1; i += T) {
                double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;      // four independent chains: the loads of the inverse overlap
                const double *col = inv + i;
                int j = 0;
                for (; j + 3 < n1; j += 4) {
                    const double a0 = PF_LDCS(col + (size_t)j * n1), a1 = PF_LDCS(col + (size_t)(j + 1) * n1), a2 = PF_LDCS(col + (size_t)(j + 2) * n1),
                                 a3 = PF_LDCS(col + (size_t)(j + 3) * n1);
                    s0 += a0 * Pc[j]; s1 += a1 * Pc[j + 1]; s2 += a2 * Pc[j + 2]; s3 += a3 * Pc[j + 3];
                }
                for (; j < n1; ++j) s0 += PF_LDCS(col + (size_t)j * n1) * Pc[j];
                Qc[i] = (s0 + s1) + (s2 + s3);
            }
        }
        PF_SYNC();
    }
    {
        int bad = 0;
        PF_PHASE {
            for (int i = tid; i < nb; i += T) {
                const int c = p_dcidx[i];
                const double th = c != 0xFFFF ? Qc[c] : 0.0;
                va[i] = th;
                bad |= !(fabs(th) < 1e300);
                if (a.is_dc) V[i] = make_double2(th, vm[i]);
                else { double s, c2; PF_SINCOS(th, &s, &c2); V[i] = make_double2(vm[i] * c2, vm[i] * s); }
            }
        }
        bad = PF_ANY(bad);
        if (bad) { sparse_fail<T>(g, a, inst, ST_DIV, 0, tid0, rd); return; }
    }
    // ---- 3. Newton-Raphson ---------------------------------------------------------------------------------
    // Four phases per iteration: [lane = line: branch currents + off-diagonal Jacobian terms] [lane = bus: S(V), mismatch,
    // diagonal terms + right-hand side; vote] [operation stream] [lane = bus: state update; clear the dead values].
    // The Jacobian terms are computed before the convergence vote (same operands as the currents / mismatch: V, y, P, Q
    // are in registers) — wasted once, in the converged evaluation, instead of re-loading everything in two more phases.
    int iters = 0;
    if (!a.is_dc) {
        const uint16_t *dpos = U16(o_dpos), *jpos = U16(o_jpos), *rnd = U16(o_round), *zero = U16(o_zero), *late = U16(o_late);
        const double *ydiag = F64(o_ydiag);
        const uint2 *ops = reinterpret_cast<const uint2 *>(blob + H.o_ops);
        const int n_oprow = H.n_oprow, n_round = H.n_round, n_zero = H.n_zero, n_late = H.n_late;
        bool conv = false;
        PF_PHASE { for (int k = tid; k < n_zero; k += T) A[zero[k]] = 0.f; }      // entries the line lanes add into / pure fill
        PF_SYNC();
#define PF_OFFDIAG(l, Vf, Vt, y)                                                                                   \
        {                                                                                                          \
            const float ef = (float)(Vf).x, ff = (float)(Vf).y, et = (float)(Vt).x, ft = (float)(Vt).y;            \
            const uint16_t *jp = jpos + 8 * (l);                                                                   \
            {   /* rows of bus f, columns of bus t:  T = Vf conj(yft Vt) */                                        \
                const float yr = (float)(y)[2], yi = (float)(y)[3];                                                \
                const float ar = yr * et - yi * ft, ai = yr * ft + yi * et;                                        \
                const float tr = ef * ar + ff * ai, ti = ff * ar - ef * ai;                                        \
                A[jp[0]] += ti; A[jp[1]] += tr; A[jp[2]] -= tr; A[jp[3]] += ti;                                    \
            }                                                                                                      \
            {   /* rows of bus t, columns of bus f:  T = Vt conj(ytf Vf) */                                        \
                const float yr = (float)(y)[4], yi = (float)(y)[5];                                                \
                const float ar = yr * ef - yi * ff, ai = yr * ff + yi * ef;                                        \
                const float tr = et * ar + ft * ai, ti = ft * ar - et * ai;                                        \
                A[jp[4]] += ti; A[jp[5]] += tr; A[jp[6]] -= tr; A[jp[7]] += ti;                                    \
            }                                                                                                      \
        }
        for (int it = 0;; ++it) {
            PF_PHASE {                                         // lane = line: currents at both ends, off-diagonal terms (round 0)
                for (int l = tid; l < nl; l += T) {
                    const int f = p_brf[l];
                    if (f == 0xFFFF) continue;
                    const double2 Vf = V[f], Vt = V[p_brt[l]];
                    const double *y = g.line_y + (size_t)l * 8;
                    cur[2 * l] = make_double2(y[0] * Vf.x - y[1] * Vf.y + y[2] * Vt.x - y[3] * Vt.y,
                                              y[0] * Vf.y + y[1] * Vf.x + y[2] * Vt.y + y[3] * Vt.x);
                    cur[2 * l + 1] = make_double2(y[4] * Vf.x - y[5] * Vf.y + y[6] * Vt.x - y[7] * Vt.y,
                                                  y[4] * Vf.y + y[5] * Vf.x + y[6] * Vt.y + y[7] * Vt.x);
                    if (n_round <= 1 || rnd[l] == 0) PF_OFFDIAG(l, Vf, Vt, y)
                }
            }
            PF_SYNC();
            int viol = 0, wild = 0;
            PF_PHASE {                                         // lane = bus: S = V conj(I), mismatch, diagonal terms, right-hand side
                for (int i = tid; i < nb; i += T) {
                    const double2 Vi = V[i];
                    double ir = 0.0, ii = 0.0, gs = 0.0, bs = 0.0;
                    const int sx = shidx[i];
                    if (sx != 0xFFFF) { gs = gsh[sx]; bs = bsh[sx]; ir = gs * Vi.x - bs * Vi.y; ii = gs * Vi.y + bs * Vi.x; }
                    for (int e = adj_ptr[i]; e < adj_ptr[i + 1]; ++e) { const double2 c2 = cur[adj[e]]; ir += c2.x; ii += c2.y; }
                    const double P = Vi.x * ir + Vi.y * ii, Q = Vi.y * ir - Vi.x * ii;
                    Pc[i] = P; Qc[i] = Q;
                    const int cth = p_colth[i], cv = p_colv[i];          // (0xFFFF: reference bus / PV bus)
                    if (cth == 0xFFFF) continue;
                    const double dP = psp[i] - P;
                    { const double m1 = fabs(dP); viol |= !(m1 < a.tol_pu); wild |= !(m1 < 1e200); }
                    const float vi2 = (float)(Vi.x * Vi.x + Vi.y * Vi.y), Pf = (float)P, Qf = (float)Q;
                    const float gi = (float)(ydiag[2 * i] + gs), bi = (float)(ydiag[2 * i + 1] + bs);
                    const uint16_t *dp = dpos + 4 * i;
                    A[dp[0]] = -Qf - bi * vi2;
                    A[nnzF + cth] = (float)dP;
                    if (cv != 0xFFFF) {
                        const double dQ = qsp[i] - Q;
                        { const double m2 = fabs(dQ); viol |= !(m2 < a.tol_pu); wild |= !(m2 < 1e200); }
                        A[dp[1]] = Pf + gi * vi2; A[dp[2]] = Pf - gi * vi2; A[dp[3]] = Qf - bi * vi2;
                        A[nnzF + cv] = (float)dQ;
                    }
                }
            }
            viol = PF_ANY(viol);
            if (!viol) { conv = true; iters = it; break; }
            wild = PF_ANY(wild);
            if (it >= a.max_iter || wild) { iters = it; break; }
            for (int r = 1, q = 0; r < n_round; ++r) {         // parallel lines: later rounds, one barrier each (rare)
                PF_PHASE {
                    for (int k = q + tid; k < n_late && late[2 * k + 1] == r; k += T) {
                        const int l = late[2 * k];
                        const double2 Vf = V[p_brf[l]], Vt = V[p_brt[l]];
                        const double *y = g.line_y + (size_t)l * 8;
                        PF_OFFDIAG(l, Vf, Vt, y)
                    }
                }
                while (q < n_late && late[2 * q + 1] == r) ++q;
                PF_SYNC();
            }
            // numeric LU + triangular solves: the plan's operation stream, thread = slot of every row, rows prefetched
            // two ahead (the stream is static: its loads never wait for the arithmetic), group barrier where flagged
            {
#define PF_AT(off) (*reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(A) + (off)))
#ifdef B200PF_EMULATE
                for (int r = 0; r < n_oprow; ++r) {
                    for (int tid = 0; tid < T; ++tid) {
                        const uint2 op = ops[(size_t)r * T + tid];
                        const float lik = PF_AT(op.x >> 16), ukj = PF_AT(op.y & 0xffffu), piv = PF_AT((op.y >> 16) & 0xfffcu);
                        PF_AT(op.x & 0xffffu) -= lik * PF_RCP(piv) * ukj;
                    }
                }
#else
                // rows come in blocks of 4 (the plan pads the stream): the 4 loads of block b+1 are issued before block b runs.
                // One warp per instance: a warp barrier after every row (cheaper than testing the flag).
                const uint2 *op_t = ops + tid;
                uint2 q0 = op_t[0], q1 = op_t[T], q2 = op_t[2 * T], q3 = op_t[3 * T];      // (the stream ends with a guard block)
#define PF_EXEC(q)                                                                                                      \
                {                                                                                                       \
                    const float lik = PF_AT((q).x >> 16), ukj = PF_AT((q).y & 0xffffu), piv = PF_AT(((q).y >> 16) & 0xfffcu); \
                    PF_AT((q).x & 0xffffu) -= lik * PF_RCP(piv) * ukj;                                                  \
                    if (T == 32) __syncwarp(); else if ((q).y & 0x10000u) PF_SYNC();                                    \
                }
#pragma unroll 2
                for (int r = 0; r < n_oprow; r += 4) {
                    op_t += 4 * T;
                    const uint2 n0 = op_t[0], n1 = op_t[T], n2 = op_t[2 * T], n3 = op_t[3 * T];
                    PF_EXEC(q0) PF_EXEC(q1) PF_EXEC(q2) PF_EXEC(q3)
                    q0 = n0; q1 = n1; q2 = n2; q3 = n3;
                }
#undef PF_EXEC
#endif
#undef PF_AT
            }
            PF_PHASE {                                         // lane = bus: state update; the assembled / filled values are dead now
                for (int i = tid; i < nb; i += T) {
                    const int cth = p_colth[i], cv = p_colv[i];
                    double vmi = vm[i], vai = va[i];
                    const uint16_t *dp = dpos + 4 * i;                      // x_k = rhs_k / U_kk
                    const double dth = cth != 0xFFFF ? (double)(A[nnzF + cth] * PF_RCP(A[dp[0]])) : 0.0;
                    const double dvr = cv != 0xFFFF ? (double)(A[nnzF + cv] * PF_RCP(A[dp[3]])) : 0.0;
                    vai += dth;
                    const double vnew = vmi * (1.0 + dvr);
                    if (fabs(dth) < 0.25 && vnew > 0.0) {
                        // small angle step (every step but pathological ones): rotate (e, f) by dth with the Taylor series of
                        // sin / cos to x^13 / x^14 (remainder < 3e-18 for |x| < 0.25) instead of a full-range fp64 sincos
                        const double x2 = dth * dth;
                        const double sn = dth * (1.0 - x2 * (1.0 / 6.0) * (1.0 - x2 * (1.0 / 20.0) * (1.0 - x2 * (1.0 / 42.0) * (1.0 - x2 * (1.0 / 72.0) *
                                          (1.0 - x2 * (1.0 / 110.0) * (1.0 - x2 * (1.0 / 156.0)))))));
                        const double cs = 1.0 - x2 * 0.5 * (1.0 - x2 * (1.0 / 12.0) * (1.0 - x2 * (1.0 / 30.0) * (1.0 - x2 * (1.0 / 56.0) * (1.0 - x2 * (1.0 / 90.0) *
                                          (1.0 - x2 * (1.0 / 132.0) * (1.0 - x2 * (1.0 / 182.0)))))));
                        const double2 Vo = V[i];
                        const double sc = 1.0 + dvr;
                        V[i] = make_double2(sc * (Vo.x * cs - Vo.y * sn), sc * (Vo.x * sn + Vo.y * cs));
                        vm[i] = vnew; va[i] = vai;
                    } else {
                        vmi = vnew;
                        if (vmi < 0.0) { vmi = -vmi; vai += 3.14159265358979323846; }
                        vm[i] = vmi; va[i] = vai;
                        double s, c; PF_SINCOS(vai, &s, &c);
                        V[i] = make_double2(vmi * c, vmi * s);
                    }
                }
                // (the bus lanes above read only right-hand side and diagonal entries; the cleared set excludes them)
                for (int k = tid; k < n_zero; k += T) A[zero[k]] = 0.f;
            }
            PF_SYNC();
        }
#undef PF_OFFDIAG
        if (!conv) { sparse_fail<T>(g, a, inst, ST_DIV, iters, tid0, rd); return; }
    } else {
        // DC: line lanes compute flows from the angles, bus lanes sum them for the slack share
        PF_PHASE {
            for (int l = tid; l < nl; l += T) {
                const int f = p_brf[l];
                if (f == 0xFFFF) continue;
                const double pfl = g.line_bdc[l] * (V[f].x - V[p_brt[l]].x) + g.line_pshift[l];
                cur[2 * l] = make_double2(pfl, 0.0); cur[2 * l + 1] = make_double2(-pfl, 0.0);
            }
        }
        PF_SYNC();
        PF_PHASE {
            for (int i = tid; i < nb; i += T) {
                const int sx = shidx[i];
                double p = sx != 0xFFFF ? gsh[sx] : 0.0;
                for (int e = adj_ptr[i]; e < adj_ptr[i + 1]; ++e) p += cur[adj[e]].x;
                Pc[i] = p; Qc[i] = 0.0;
            }
        }
        PF_SYNC();
    }
    // ---- 4. results (same float32 rounding rules as the reference's read-back, pPB:1159-1183) ------------------
    PF_SYNC();
    if (!a.is_dc) {
        // pandapower reports Va = angle(V), i.e. angles in (-180, 180]; the Newton iteration accumulates them unwrapped
        PF_PHASE { for (int i = tid; i < nb; i += T) { const double x = va[i]; va[i] = x - 6.283185307179586477 * rint(x * 0.15915494309189533577); } }
        PF_SYNC();
    }
    const double RAD2DEG = 57.295779513082320877, SQRT3 = 1.7320508075688772935;
    {
        const uint16_t *unit_bus = U16(o_unit_bus), *load_bus = U16(o_load_bus), *sto_bus = U16(o_sto_bus), *sh_bus = U16(o_sh_bus);
        const uint16_t *bu_ptr = U16(o_bu_ptr), *bu = U16(o_bu), *bl_ptr = U16(o_bl_ptr), *bl = U16(o_bl);
        const uint16_t *bs_ptr = U16(o_bs_ptr), *bs = U16(o_bs), *p_cnt = U16(o_cnt), *p_nref = U16(o_nref), *p_slot = U16(o_slot);
        const double *qmins = F64(o_qmins), *qmaxs = F64(o_qmaxs);
        PF_PHASE {
            if (tid == 0) { a.status[inst] = ST_OK; a.iters[inst] = iters; }
            for (int l = tid; l < nl; l += T) {
                float r[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                const int f = p_brf[l];
                if (f != 0xFFFF) {
                    const int t = p_brt[l];
                    const double vmf = vm[f], vmt = vm[t];
                    double pf, qf, pt, qt, sf, st;
                    if (a.is_dc) { pf = cur[2 * l].x * base; pt = -pf; qf = 0.0; qt = 0.0; sf = fabs(pf); st = sf; }
                    else {
                        const double2 Aa = V[f], Bb = V[t], If = cur[2 * l], It = cur[2 * l + 1];
                        pf = (Aa.x * If.x + Aa.y * If.y) * base; qf = (Aa.y * If.x - Aa.x * If.y) * base;
                        pt = (Bb.x * It.x + Bb.y * It.y) * base; qt = (Bb.y * It.x - Bb.x * It.y) * base;
                        sf = sqrt(pf * pf + qf * qf); st = sqrt(pt * pt + qt * qt);
                    }
                    const float vnf = g.line_or_vn[l], vnt = g.line_ex_vn[l];
                    float a1 = (float)(sf / (SQRT3 * (vmf * (double)vnf)) * 1000.0), a2 = (float)(st / (SQRT3 * (vmt * (double)vnt)) * 1000.0);
                    if (!(fabsf(a1) <= 3.4e38f)) a1 = 0.f;
                    if (!(fabsf(a2) <= 3.4e38f)) a2 = 0.f;
                    r[0] = (float)pf; r[1] = (float)qf; r[2] = PF_FMUL((float)vmf, vnf); r[3] = a1; r[4] = (float)(va[f] * RAD2DEG);
                    r[5] = (float)pt; r[6] = (float)qt; r[7] = PF_FMUL((float)vmt, vnt); r[8] = a2; r[9] = (float)(va[t] * RAD2DEG);
                }
                if (out) for (int k = 0; k < 10; ++k) out[k * nl + l] = r[k];
                if (a.rho) a.rho[(size_t)inst * nl + l] = r[3] / a.th_lim[l];
            }
            if (out) {
                float *o = out + 10 * nl;
                for (int u = tid; u < nu; u += T) {
                    float p = 0.f, q = 0.f, v = 0.f, th = 0.f;
                    const int i = unit_bus[u];
                    if (i != 0xFFFF) {
                        double pd = 0.0, qd = 0.0, pnonref = 0.0;
                        for (int e = bl_ptr[i]; e < bl_ptr[i + 1]; ++e) { const int k = bl[e]; pd += LOAD_P(k); qd += LOAD_Q(k); }
                        for (int e = bs_ptr[i]; e < bs_ptr[i + 1]; ++e) { const int k = bs[e]; pd += STO_P(k); qd += g.sto_q[k]; }
                        for (int e = bu_ptr[i]; e < bu_ptr[i + 1]; ++e) { const int u2 = bu[e]; if (!g.unit_is_ref[u2]) pnonref += GEN_P(u2); }
                        double pu = GEN_P(u);
                        if (g.unit_is_ref[u]) pu = (Pc[i] * base + pd - pnonref) / (double)p_nref[i];     // slack share (pandapower pfsoln)
                        double qu = 0.0;
                        if (!a.is_dc) {
                            const double qtot = Qc[i] * base + qd, qmn = qmins[i], qmx = qmaxs[i];
                            const int cb = p_cnt[i];
                            if (cb <= 1 || qmn == qmx) qu = qtot / (double)cb;
                            else qu = g.unit_qmin[u] + (qtot - qmn) / (qmx - qmn + 2.220446049250313e-16) * (g.unit_qmax[u] - g.unit_qmin[u]);
                        }
                        p = (float)pu; q = (float)qu; v = PF_FMUL((float)vm[i], g.unit_vn[u]); th = (float)(va[i] * RAD2DEG);
                    }
                    o[u] = p; o[nu + u] = q; o[2 * nu + u] = v; o[3 * nu + u] = th;
                }
                o += 4 * nu;
                for (int k = tid; k < nld; k += T) {
                    const int i = load_bus[k];
                    o[k] = i != 0xFFFF ? PF_FMUL((float)vm[i], g.load_vn[k]) : 0.f;
                    o[nld + k] = i != 0xFFFF ? (float)(va[i] * RAD2DEG) : 0.f;
                }
                o += 2 * nld;
                for (int k = tid; k < nst; k += T) { const int i = sto_bus[k]; o[k] = i != 0xFFFF ? PF_FMUL((float)vm[i], g.sto_vn[k]) : 0.f; }
                o += nst;
                for (int k = tid; k < nsh; k += T) {
                    const int i = sh_bus[k];
                    float p = 0.f, q = 0.f, v = 0.f;
                    if (i != 0xFFFF) {
                        const double v2 = a.is_dc ? 1.0 : vm[i] * vm[i];
                        p = (float)(SH_P(k) * g.sh_vratio[k] * v2);
                        q = a.is_dc ? 0.f : (float)(SH_Q(k) * g.sh_vratio[k] * v2);
                        v = PF_FMUL((float)vm[i], g.sh_vn[k]);
                    }
                    o[k] = p; o[nsh + k] = q; o[2 * nsh + k] = v;
                }
            }
            if (a.busv) {
                double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
                for (int s = tid; s < 2 * g.n_slot; s += T) bv[s] = PF_QNAN();
            }
        }
        PF_SYNC();
        if (a.busv) {
            double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
            PF_PHASE { for (int i = tid; i < nb; i += T) { bv[p_slot[i]] = vm[i]; bv[g.n_slot + p_slot[i]] = va[i]; } }
            PF_SYNC();
        }
    }
    if (PROT) {
        // Cascading-failure round (reference Backend.next_grid_state, backend.py:1466-1521; counters baseEnv.py:3361-3370),
        // lane = line, same rules as pf_kernel_small: a line trips when its flow exceeds hard_thr * limit or stayed above
        // soft_thr * limit for more than max_pc steps.  A tripping line changes the topology, i.e. the plan: this launch
        // only REPORTS it (trip / flag_list); the host takes the lines out, re-plans the instance and launches the next
        // round for the flagged instances.  Without a trip the step is final: counters, disc, the next step's state.
        const size_t base_l = (size_t)inst * nl;
        int any_trip = 0;
        PF_PHASE {
            for (int l = tid; l < nl; l += T) {
                const bool on = p_brf[l] != 0xFFFF;
                const float aor = out[3 * nl + l], lim = a.th_lim[l];
                int inc = a.casc > 0 ? (int)a.incdone[base_l + l] : 0;
                int pc = a.pcount[base_l + l] + inc;
                bool to_disc = on && (aor > PF_FMUL(a.hard_thr, lim));
                if (!a.from_reset && on && (aor > PF_FMUL(a.soft_thr, lim)) && !inc) { pc += 1; inc = 1; }
                if (on && pc > a.max_pc) to_disc = true;
                a.incdone[base_l + l] = (int8_t)inc;
                if (a.casc == 0) a.disc[base_l + l] = -1;
                if (to_disc) { a.trip[base_l + l] = 1; a.disc[base_l + l] = a.casc; any_trip = 1; }
            }
        }
        any_trip = PF_ANY(any_trip);
        PF_PHASE {
            if (any_trip) {
                if (tid == 0) {
#ifdef B200PF_EMULATE
                    const int slot = (*a.n_flag)++;
#else
                    const int slot = atomicAdd(a.n_flag, 1);
#endif
                    a.flag_list[slot] = inst;
                }
            } else {
                for (int l = tid; l < nl; l += T) {
                    const float aor = out[3 * nl + l], lim = a.th_lim[l];
                    int *pcp = a.pcount + base_l, *tsp = a.ts_over + base_l;
                    pcp[l] = (!a.from_reset && aor > PF_FMUL(a.soft_thr, lim)) ? pcp[l] + 1 : 0;
                    tsp[l] = (!a.from_reset && aor > lim) ? tsp[l] + 1 : 0;
                    a.incdone[base_l + l] = 0;
                }
            }
        }
        PF_SYNC();
    }
    (void)d; (void)nA;
#undef U16
#undef F64
#undef GEN_P
#undef UNIT_VM
#undef LOAD_P
#undef LOAD_Q
#undef STO_P
#undef SH_P
#undef SH_Q
}

#ifndef B200PF_EMULATE
template <int T, int MINB, bool PROT>
__global__ void __launch_bounds__(T, MINB)
pf_kernel_sparse(const DevGrid g, const RunArgs a, const PlanArgs pa, const RedoDesc rd) {
    extern __shared__ __align__(16) unsigned char smem[];
    for (int k = blockIdx.x; k < a.batch; k += gridDim.x) {
        const int inst = (PROT && a.inst_list) ? a.inst_list[k] : k;
        solve_sparse<T, PROT>(g, a, pa, inst, smem, threadIdx.x, rd);
        sp_sync<T>();
    }
}
#endif

}  // namespace b200pf

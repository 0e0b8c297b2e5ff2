// b200pf_block.cuh — the BLOCK-PLANNED kernel: T lanes per grid instance, G = 32 / T instances per warp (T < 32), or one
// warp / CTA per instance (T >= 32, G = 1), driven by the BLOCK plan of b200pf_plan.hpp.
//
// What changes against the scalar planned kernel (b200pf_sparse.cuh), and why (Nsight Compute profiles):
// that kernel gives a 14-bus instance a whole warp — 20.5 of 32 lanes active on average — and spends its issue slots on
// 4 LDS + 1 STS + index unpacking per scalar multiply-subtract.
//   * Instances are interleaved inside a warp: lane = j * G + g is lane j of the instance g of its warp; element e of an
//     instance's workspace sits at e * G + g, so the 8 lanes of a quarter warp read 8 consecutive 16-byte words — every
//     vector access of the operation stream is bank-conflict free BY CONSTRUCTION, whatever the plan's indices are.
//     "lane = bus" / "lane = line" phases loop ceil(n / T) times with every lane busy; all lanes j of a warp fetch the same
//     plan words (one L1 wavefront).  The lanes of one instance synchronise among themselves only (__syncwarp(mask of the
//     instance)); instances of a warp that need different iteration counts, or use different plans, simply diverge.
//   * The Jacobian is stored and factorised as 2x2 blocks per bus pair (float4; a PV bus keeps the block shape with an
//     identity Q row and a zero |V| column): one block operation D -= A B is 3 x LDS.128 + 8 FMA + 1 x STS.128 and replaces
//     eight scalar operations of the old stream; pivot rows are normalised with the explicit 2x2 inverse (which pivots
//     inside the block), U operations per lane and row are loaded before any is stored (ILP inside a pass).
// Arithmetic plan unchanged: fp64 state / mismatch / flows, fp32 Jacobian and solve, the fp64 residual decides convergence
// with pandapower's criterion; same result record, same status classes.  ST_DIV is never final: the first such instance
// makes the kernel tail-launch pf_kernel_redo (b200pf_redo.cuh), which re-solves them with partial pivoting.
// With B200PF_EMULATE the same source compiles as plain host C++ (a phase = a loop over the lanes of ONE instance, the
// instances of a warp one after the other on the same interleaved workspace): tests/ use that build on machines without a GPU.
#pragma once
#include "b200pf_sparse.cuh"

namespace b200pf {

#ifdef B200PF_EMULATE
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
#define PB_SYNC() ((void)0)
#define PB_ANY(x) (x)
#define PB_LOOP
#define PB_UNROLL
#else
#define PB_UNROLL _Pragma("unroll")
#define PB_LOOP _Pragma("unroll 1")      // the lane loops run 1-3 times: unrolled copies only cost instruction-cache misses (ncu: no_inst 15 %)
// (also the per-bus element lists of the code that runs once per solve: 0-3 entries, and that code is fetched cold after an
// L2 flush; with the staged arrays known to be shared memory the compiler unrolls each of them 4x)
// UNI ("lockstep"): all instances of the warp share one plan and run the same control flow, so the whole warp
// synchronises with the plain full-mask primitives.  A per-lane mask (instances free to diverge) makes every barrier / vote a
// MATCH-based collective.
template <int T, int G, bool UNI> __device__ __forceinline__ void pb_sync(unsigned mask) {
    if (T < 32) { if (UNI) __syncwarp(); else __syncwarp(mask); } else if (T == 32) __syncwarp(); else __syncthreads();
}
template <int T, int G, bool UNI> __device__ __forceinline__ int pb_any(unsigned mask, int p) {
    if (T < 32) return UNI ? ((__ballot_sync(0xffffffffu, p) & mask) != 0u) : __any_sync(mask, p);
    return (T == 32) ? __any_sync(0xffffffffu, p) : __syncthreads_or(p);
}
#define PB_SYNC() pb_sync<T, G, UNI>(imask)
#define PB_ANY(x) pb_any<T, G, UNI>(imask, (x))
#endif

#if defined(B200PF_PHASE_CLOCK) && !defined(B200PF_EMULATE)
// Measurement build only (-DB200PF_PHASE_CLOCK, scripts/phase_clock.py); the production build compiles none of this.
// Lane 0 of every warp adds the SM cycles (clock64) spent between consecutive phase boundaries of solve_block to
// pb_phase_clk[phase] (summed over the Newton iterations, the warps and the launches until the host reads and clears it);
// pf_kernel_block adds every warp's cycle and globaltimer spans, from which the host converts cycles to time.
enum { PC_STAGE, PC_ROW, PC_SUMS, PC_DCINV, PC_DCANG, PC_BUSES, PC_STREAM, PC_UPDATE, PC_OUT, PC_N_PHASE,
       PC_SOLVES = PC_N_PHASE, PC_WARPS, PC_CYCLES, PC_NS, PC_SLOTS };
__device__ unsigned long long pb_phase_clk[PC_SLOTS];
#define PB_CLOCK_ON 1
#define PB_CLOCK(k)                                                                                                   \
    {                                                                                                                 \
        const long long t_ = clock64();                                                                               \
        if (clk_lane0) atomicAdd(&pb_phase_clk[k], (unsigned long long)(t_ - clk_last));                             \
        clk_last = t_;                                                                                                \
    }
#else
#define PB_CLOCK_ON 0
#define PB_CLOCK(k)
#endif

template <int T, int G, bool UNI = false>
PF_DEV void block_fail(const DevGrid &g, const RunArgs &a, int inst, int status, int iters, int tid0, unsigned imask) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
    PF_PHASE {
        if (tid == 0) { a.status[inst] = status; a.iters[inst] = iters; if (a.prot && a.done) a.done[inst] = 1; }
        if (a.prot && a.disc && status == ST_DONE) for (int k = tid; k < g.n_line; k += T) a.disc[(size_t)inst * g.n_line + k] = -1;
        if (out) for (int k = tid; k < g.n_out; k += T) out[k] = PF_QNANF();
        if (a.busv) for (int k = tid; k < 2 * g.n_slot; k += T) a.busv[(size_t)inst * 2 * g.n_slot + k] = PF_QNAN();
        if (a.rho) for (int k = tid; k < g.n_line; k += T) a.rho[(size_t)inst * g.n_line + k] = PF_QNANF();
    }
    PB_SYNC();
    (void)tid0; (void)imask;
}

// The chronics row an instance solves, from the kernel arguments alone (no plan needed): series entry point -> row a.t[src]
// of scenario a.scen[src], and a.t[inst] advances for the next step; rows entry point -> row src of a.rows.  nullptr: the
// instance reads an fp64 injection record instead (MODE 0 without a series).
template <int T, int G, bool PROT, bool UNI, int MODE>
PF_DEV const float *block_row(const DevGrid &g, const RunArgs &a, int inst, int tid0, unsigned imask) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
    const int src = a.n1_lines > 0 ? inst / a.n1_lines : inst;          // record the inputs come from
    int trow = 0, sc = 0;
    if (a.series && !a.rows) {
        sc = a.scen[src]; trow = a.t[src];
        PB_SYNC();
        if (PROT && a.casc > 0) trow = trow == 0 ? a.n_rows - 1 : trow - 1;       // later cascade rounds re-solve the SAME row
        PF_PHASE { if (tid == 0 && a.n1_lines <= 0 && !(PROT && a.casc > 0)) a.t[inst] = (trow + 1 >= a.n_rows) ? 0 : trow + 1; }
    }
    (void)tid0; (void)imask;
    if (!(MODE == 1 || a.series != 0)) return nullptr;
    const size_t n_row = (size_t)(2 * g.n_load + 2 * g.n_gen);
    return a.rows ? a.rows + (size_t)src * n_row : a.chron + ((size_t)sc * a.n_rows + trow) * n_row;
}

// the row into the instance's interleaved copy srow of the warp's workspace
template <int T, int G, bool UNI>
PF_DEV void block_row_copy(const float *grow, int n, float *srow, int gi, int tid0, unsigned imask) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
    PF_PHASE { for (int k = tid; k < n; k += T) srow[k * G + gi] = grow[k]; }
    PB_SYNC();
    (void)tid0; (void)imask;
}

// Byte offset of srow in a warp's workspace (the layout solve_block builds from the strides Lnb / LnblkA): value blocks, six
// bus arrays, the shunt pair, V, the branch currents, V in fp32, then the row.
template <int G>
PF_DEV size_t block_srow_off(int Lnb, int LnblkA, int nsh, int nl) {
    const size_t Lb = (size_t)Lnb * G, LA = (size_t)(LnblkA + 1) * G;
    return LA * 16 + (6 * Lb + 2 * (size_t)nsh * G) * 8 + (Lb + 2 * (size_t)nl * G) * 16 + Lb * 8;
}

// A bus's diagonal block, right-hand side and mismatch tests from its S = P + jQ (fp64) in the Newton evaluation: a PV bus
// keeps an identity Q row and no Q mismatch.  Arithmetic only, so that the two buses of a lane are independent chains.
struct PbBusRow { float4 D, R; int viol, wild; };
// (gi_, bi_: (float) of Y_ii + shunt)
PF_DEV PbBusRow pb_bus_row(double2 Vi, double P, double Q, double ps, double qs, float gi_, float bi_, bool pq, double tol) {
    PbBusRow r;
    const double dP = ps - P;
    { const double m1 = fabs(dP); r.viol = !(m1 < tol); r.wild = !(m1 < 1e200); }
    const float vi2 = (float)(Vi.x * Vi.x + Vi.y * Vi.y), Pf = (float)P, Qf = (float)Q;
    r.D = make_float4(-Qf - bi_ * vi2, 0.f, 0.f, 1.f); r.R = make_float4((float)dP, 0.f, 0.f, 0.f);
    if (pq) {
        const double dQ = qs - Q;
        { const double m2 = fabs(dQ); r.viol |= !(m2 < tol); r.wild |= !(m2 < 1e200); }
        r.D.y = Pf + gi_ * vi2; r.D.z = Pf - gi_ * vi2; r.D.w = Qf - bi_ * vi2;
        r.R.z = (float)dQ;
    }
    return r;
}

// State update of a bus from its solved step (dth, dvr = d|V| / |V|): V rotated by dth with the Taylor series of sin / cos
// (remainder < 3e-18 for |x| < 0.25) and scaled by 1 + dvr.  Arithmetic only; `small` false: the caller takes the sincos
// path (pb_update_slow) instead.
struct PbUpd { double2 V; double vm, va; bool small; };
PF_DEV PbUpd pb_update_small(double2 Vo, double vmi, double vai, double dth, double dvr) {
    PbUpd r;
    r.va = vai + dth;
    r.vm = vmi * (1.0 + dvr);
    r.small = fabs(dth) < 0.25 && r.vm > 0.0;
    const double x2 = dth * dth;
    const double sn = dth * (1.0 - x2 * (1.0 / 6.0) * (1.0 - x2 * (1.0 / 20.0) * (1.0 - x2 * (1.0 / 42.0) * (1.0 - x2 * (1.0 / 72.0) *
                      (1.0 - x2 * (1.0 / 110.0) * (1.0 - x2 * (1.0 / 156.0)))))));
    const double cs = 1.0 - x2 * 0.5 * (1.0 - x2 * (1.0 / 12.0) * (1.0 - x2 * (1.0 / 30.0) * (1.0 - x2 * (1.0 / 56.0) * (1.0 - x2 * (1.0 / 90.0) *
                      (1.0 - x2 * (1.0 / 132.0) * (1.0 - x2 * (1.0 / 182.0)))))));
    const double scl = 1.0 + dvr;
    r.V = make_double2(scl * (Vo.x * cs - Vo.y * sn), scl * (Vo.x * sn + Vo.y * cs));
    return r;
}
PF_DEV void pb_update_slow(PbUpd &r) {
    if (r.vm < 0.0) { r.vm = -r.vm; r.va += 3.14159265358979323846; }
    double s, c2; PF_SINCOS(r.va, &s, &c2);
    r.V = make_double2(r.vm * c2, r.vm * s);
}

// sm: workspace of the WARP (G instances, interleaved); gi: instance slot of this lane in the warp; tid0: lane of the instance
// MODE 1: AC solve fed by chronics rows (series / rows entry points) known at compile time — the DC branches and the fp64-record
// input paths drop out of the kernel (ncu: 13 % of the stall samples at batch 4096 were instruction-fetch stalls); 0: generic
// STAGE: the plan (and pa.stat) are the launch's copies in shared memory, and the kernel has already run block_row /
// block_row_copy for this instance (for its first instance group while the plan's bulk copy was in flight).
template <int T, int U, int G, bool PROT, bool UNI = false, int MODE = 0, bool STAGE = false>
PF_DEV void solve_block(const DevGrid &g, const RunArgs &a, const PlanArgs &pa, int inst, unsigned char *sm, int gi, int tid0, unsigned imask,
                        const RedoDesc &rd = RedoDesc()) {
#ifndef B200PF_EMULATE
    const int tid = tid0;
#endif
#if PB_CLOCK_ON
    const bool clk_lane0 = tid0 == 0 && gi == 0;
    long long clk_last = clock64();
#endif
    const int src = a.n1_lines > 0 ? inst / a.n1_lines : inst;          // record the inputs come from
    const unsigned char *blob = pa.blobs + pa.plan_off[pa.inst_plan ? pa.inst_plan[inst] : 0];
    const PlanHeader &H = *reinterpret_cast<const PlanHeader *>(blob);
    const float *grow = STAGE ? nullptr : block_row<T, G, PROT, UNI, MODE>(g, a, inst, tid0, imask);
    // fstat >= 0: the instance has failed with this status.  Free-running instances (UNI = false) leave at once; in lockstep
    // the lanes keep executing with the warp (their state is garbage from then on) and store the failure record at the end.
    int fstat = -1, fiters = 0;
#define PB_FAIL(st, its) { if (UNI) { if (fstat < 0) { fstat = (st); fiters = (its); } } else { block_fail<T, G, UNI>(g, a, inst, (st), (its), tid0, imask); return; } }
    if (PROT && a.done[inst] && a.casc == 0) { block_fail<T, G, UNI>(g, a, inst, ST_DONE, 0, tid0, imask); return; }
    if (H.status != PLAN_ST_OK) { block_fail<T, G, UNI>(g, a, inst, H.status, 0, tid0, imask); return; }      // (lockstep: one plan -> the whole warp leaves)
    if (a.dbg_div_mod > 0 && inst % a.dbg_div_mod == 0) PB_FAIL(ST_DIV, 0)   // test knob
    const int nb = H.nb, nl = g.n_line, nu = g.n_unit, nh = g.n_hidden, ng = g.n_gen, nld = g.n_load, nst = g.n_sto, nsh = g.n_shunt;
    const int nblk = H.nblk, nblkA = H.nblkA;
    const double base = g.base_mva, inv_base = 1.0 / base;
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
#define U16(off) reinterpret_cast<const uint16_t *>(blob + H.off)
#define F64(off) reinterpret_cast<const double *>(blob + H.off)
#define IX(i) ((i) * G + gi)
#define PB_STAT(name, type) const type *name##_ = STAGE ? reinterpret_cast<const type *>(pa.stat + pa.so.name) : g.name;
    PB_STAT(line_y, double) PB_STAT(line_bdc, double) PB_STAT(line_pshift, double) PB_STAT(line_or_vn, float) PB_STAT(line_ex_vn, float)
    PB_STAT(unit_is_ref, int) PB_STAT(unit_qmin, double) PB_STAT(unit_qmax, double) PB_STAT(unit_vn, float) PB_STAT(load_vn, float)
    PB_STAT(sto_vn, float) PB_STAT(sto_q, double) PB_STAT(sh_vn, float) PB_STAT(sh_vratio, double)
#undef PB_STAT
    const float *th_lim_ = STAGE ? reinterpret_cast<const float *>(pa.stat + pa.so.th_lim) : a.th_lim;
    const double *line_y = line_y_;
    const uint16_t *p_colth = U16(o_colth), *p_dcidx = U16(o_dcidx);
    const uint16_t *p_brf = U16(o_brf), *p_brt = U16(o_brt);
    const uint16_t *adj_ptr = U16(o_adj_ptr), *adj = U16(o_adj), *shidx = U16(o_shidx);
    // ---- workspace of the warp: every array holds G interleaved copies -------------------------------------------------
    // (strides = the launch's maxima pa.lay_*, not this plan's sizes: instances with different plans share the warp)
    const size_t Lb = (size_t)(pa.lay_nb > nb ? pa.lay_nb : nb) * G, LA = (size_t)((pa.lay_nblkA > nblkA ? pa.lay_nblkA : nblkA) + 1) * G;
    float4 *A4 = reinterpret_cast<float4 *>(sm);                         // [nblkA + 1] blocks; offset 0: the stream's byte offsets address it
    double *vm = reinterpret_cast<double *>(sm + LA * 16), *va = vm + Lb, *psp = va + Lb, *qsp = psp + Lb, *Pc = qsp + Lb, *Qc = Pc + Lb,
           *gsh = Qc + Lb, *bsh = gsh + (size_t)nsh * G;
    double2 *V = reinterpret_cast<double2 *>(bsh + (size_t)nsh * G);
    double2 *cur = V + Lb;
    float2 *Vf = reinterpret_cast<float2 *>(cur + (size_t)2 * nl * G);    // (float) of V, written with it
    float *srow = reinterpret_cast<float *>(Vf + Lb);
    // ---- injections of this instance ----------------------------------------------------------------------
    const bool has_row = MODE == 1 ? true : (a.series != 0);
    const bool is_dc = MODE == 1 ? false : (a.is_dc != 0);
    const double *rec = nullptr, *si = STAGE ? reinterpret_cast<const double *>(pa.stat + pa.so.static_inj) : a.static_inj;
    if (has_row) {
        if (!STAGE) block_row_copy<T, G, UNI>(grow, 2 * nld + 2 * ng, srow, gi, tid0, imask);
    } else rec = a.inj + (size_t)src * g.n_inj;
    PB_CLOCK(PC_ROW)
#define ROW(k) srow[IX(k)]
#define GEN_P(u) ((u) < nh ? 0.0 : (has_row ? (double)ROW(2 * nld + (u) - nh) : rec[(u) - nh]))
#define UNIT_VM(u) (has_row ? ((u) >= nh ? (double)PF_FDIV(ROW(2 * nld + ng + (u) - nh), unit_vn_[u]) : si[ng + (u)]) : rec[ng + (u)])
#define LOAD_P(k) (has_row ? (double)ROW(k) : rec[ng + nu + (k)])
#define LOAD_Q(k) (has_row ? (double)ROW(nld + (k)) : rec[ng + nu + nld + (k)])
#define STO_P(k) (has_row ? si[ng + nu + 2 * nld + (k)] : rec[ng + nu + 2 * nld + (k)])
#define SH_P(k) (has_row ? si[ng + nu + 2 * nld + nst + (k)] : rec[ng + nu + 2 * nld + nst + (k)])
#define SH_Q(k) (has_row ? si[ng + nu + 2 * nld + nst + nsh + (k)] : rec[ng + nu + 2 * nld + nst + nsh + (k)])

    // ---- 1. per-bus sums in element order; right-hand side of the DC system (lane = bus) -----------------
    {
        const uint16_t *bu_ptr = U16(o_bu_ptr), *bu = U16(o_bu), *bl_ptr = U16(o_bl_ptr), *bl = U16(o_bl);
        const uint16_t *bs_ptr = U16(o_bs_ptr), *bs = U16(o_bs), *bh_ptr = U16(o_bh_ptr), *bh = U16(o_bh);
        const uint16_t *vmunit = U16(o_vmunit);
        const double *dcshift = F64(o_dcshift);
        PF_PHASE {
            PB_LOOP for (int i = tid; i < nb; i += T) {
                double pg = 0.0, pd = 0.0, qd = 0.0, gs = 0.0, bsu = 0.0;
                PB_LOOP for (int e = bu_ptr[i]; e < bu_ptr[i + 1]; ++e) { const int u = bu[e]; pg += GEN_P(u); }
                PB_LOOP for (int e = bl_ptr[i]; e < bl_ptr[i + 1]; ++e) { const int k = bl[e]; pd += LOAD_P(k); qd += LOAD_Q(k); }
                PB_LOOP for (int e = bs_ptr[i]; e < bs_ptr[i + 1]; ++e) { const int k = bs[e]; pd += STO_P(k); qd += sto_q_[k]; }
                PB_LOOP for (int e = bh_ptr[i]; e < bh_ptr[i + 1]; ++e) { const int k = bh[e]; gs += SH_P(k) * sh_vratio_[k]; bsu -= SH_Q(k) * sh_vratio_[k]; }
                const int vu = vmunit[i];
                vm[IX(i)] = vu != 0xFFFF ? UNIT_VM(vu) : 1.0;
                const double ps = (pg - pd) * inv_base, gpu = gs * inv_base;      // (one division per lane instead of four per bus)
                psp[IX(i)] = ps; qsp[IX(i)] = -qd * inv_base;
                const int sx = shidx[i];
                if (sx != 0xFFFF) { gsh[IX(sx)] = gpu; bsh[IX(sx)] = bsu * inv_base; }
                const int c = p_dcidx[i];
                if (c != 0xFFFF) Pc[IX(c)] = ps - gpu - dcshift[i];
            }
        }
        PB_SYNC();
    }
    PB_CLOCK(PC_SUMS)
    // ---- 2. DC angles: theta = Bdc^-1 b with the plan's fp64 inverse (lane = row; Pc = right-hand side, Qc = result) ------
    {
        // staged: the plan's copy in shared memory (the 8 lanes of an instance read 8 consecutive doubles, the instances of a
        // warp the same ones: conflict free); otherwise streamed from global memory with evict-first loads
#define PB_INV(p) (STAGE ? *(p) : PF_LDCS(p))
        const double *inv = F64(o_dcinv);
        const int n1 = H.n1;
        PF_PHASE {
            PB_LOOP for (int i = tid; i < n1; i += T) {
                double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
                const double *col = inv + i;
                int j = 0;
                for (; j + 3 < n1; j += 4) {
                    const double a0 = PB_INV(col + (size_t)j * n1), a1 = PB_INV(col + (size_t)(j + 1) * n1), a2 = PB_INV(col + (size_t)(j + 2) * n1),
                                 a3 = PB_INV(col + (size_t)(j + 3) * n1);
                    s0 += a0 * Pc[IX(j)]; s1 += a1 * Pc[IX(j + 1)]; s2 += a2 * Pc[IX(j + 2)]; s3 += a3 * Pc[IX(j + 3)];
                }
                for (; j < n1; ++j) s0 += PB_INV(col + (size_t)j * n1) * Pc[IX(j)];
#undef PB_INV
                Qc[IX(i)] = (s0 + s1) + (s2 + s3);
            }
        }
        PB_SYNC();
    }
    PB_CLOCK(PC_DCINV)
    {
        int bad = 0;
        PF_PHASE {
            PB_LOOP for (int i = tid; i < nb; i += T) {
                const int c = p_dcidx[i];
                const double th = c != 0xFFFF ? Qc[IX(c)] : 0.0;
                va[IX(i)] = th;
                bad |= !(fabs(th) < 1e300);
                const double vmi = vm[IX(i)];
                if (is_dc) V[IX(i)] = make_double2(th, vmi);
                else {
                    double s, c2; PF_SINCOS(th, &s, &c2);
                    const double2 v = make_double2(vmi * c2, vmi * s);
                    V[IX(i)] = v; Vf[IX(i)] = make_float2((float)v.x, (float)v.y);
                }
            }
        }
        bad = PB_ANY(bad);
        if (bad) PB_FAIL(ST_DIV, 0)
    }
    // ---- 3. Newton-Raphson ---------------------------------------------------------------------------------
    // Three phases per iteration: [lane = bus: I = Y V from the plan's admittance row, S(V), mismatch, the bus's whole block
    // row + right-hand side; vote] [block operation stream] [lane = bus: state update; clear the fill-in blocks].
    int iters = 0;
    if (!is_dc) {
        const uint16_t *bzero = U16(o_bzero), *yptr = U16(o_yptr);
        const double *ydiag = F64(o_ydiag), *yval = F64(o_yval);
        const unsigned *yword = reinterpret_cast<const unsigned *>(blob + H.o_yword);
        const float2 *yf32 = reinterpret_cast<const float2 *>(blob + H.o_yf32);
        const uint2 *bdesc = reinterpret_cast<const uint2 *>(blob + H.o_bdesc);
        const uint2 *bops = reinterpret_cast<const uint2 *>(blob + H.o_bops);
        const int n_brow = H.n_brow, n_bzero = H.n_bzero;
        bool conv = false, running = fstat < 0;
        PF_PHASE { for (int k = tid; k < n_bzero; k += T) A4[IX(bzero[k])] = make_float4(0.f, 0.f, 0.f, 0.f); }
        PB_SYNC();
        PB_CLOCK(PC_DCANG)
        for (int it = 0;; ++it) {
            int viol = 0, wild = 0;
            PF_PHASE {                                         // lane = bus: S = V conj(I), mismatch, block row, right-hand side
                // A lane evaluates its buses i and i + T together, as two independent chains: the loads of both, then the
                // arithmetic of both, then the stores of both (the compiler cannot move a load above a shared-memory store).
                // Each bus keeps its own accumulators and summation order: (Y_ii + shunt) V_i, then its neighbours ascending.
                PB_LOOP for (int i = tid; i < nb; i += 2 * T) {
                    const int i2 = i + T < nb ? i + T : i;    // (no second bus: chain 2 re-reads bus i and stores nothing)
                    const bool two = i2 != i;
                    const uint2 da = bdesc[i], db = bdesc[i2];
                    const float2 Fa = Vf[IX(i)], Fb = Vf[IX(i2)];
                    double gsa = ydiag[2 * i], bsa = ydiag[2 * i + 1], gsb = ydiag[2 * i2], bsb = ydiag[2 * i2 + 1];   // Y_ii + shunt
                    const int ea = yptr[i], na = yptr[i + 1] - ea, eb = yptr[i2], nbb = two ? yptr[i2 + 1] - eb : 0;
                    unsigned wa = yword[na > 0 ? ea : 0], wb = yword[nbb > 0 ? eb : 0];      // (the plan stores at least one entry)
                    const int sxa = da.y & 0xFFFF, sxb = db.y & 0xFFFF;
                    if (sxa != 0xFFFF) { gsa += gsh[IX(sxa)]; bsa += bsh[IX(sxa)]; }
                    if (sxb != 0xFFFF) { gsb += gsh[IX(sxb)]; bsb += bsh[IX(sxb)]; }
                    double ira, iia, irb, iib;
                    {
                        const double2 Va = V[IX(i)], Vb = V[IX(i2)];
                        ira = gsa * Va.x - bsa * Va.y; iia = gsa * Va.y + bsa * Va.x;
                        irb = gsb * Vb.x - bsb * Vb.y; iib = gsb * Vb.y + bsb * Vb.x;
                    }
                    const float gfa = (float)gsa, bfa = (float)bsa, gfb = (float)gsb, bfb = (float)bsb;
                    // off-diagonal block (i, j) = [ti tr; -tr ti] with T = Vi conj(Y_ij Vj) (fp32), the Q row of a PV bus i and
                    // the |V| column of a PV bus j zero; written whole (the reference bus's row goes to the dummy block).  Entry k
                    // of both rows per round; the entry words of the next round are loaded before this round's stores.
                    const bool pqa = (da.y >> 16) != 0u, pqb = (db.y >> 16) != 0u;
                    // (at least one round, so that no branch separates the loads above from their use: two empty rows add
                    // nothing and store to the dummy block)
                    const int nk = na > nbb ? na : nbb;
                    int k = 0;
                    PB_LOOP do {
                        const bool ka = k < na, kb = k < nbb;
                        const int qa = ka ? ea + k : 0, qb = kb ? eb + k : 0;
                        const int ja = (wa >> 16) & 0x7FFF, jb = (wb >> 16) & 0x7FFF;
                        const double2 Vja = V[IX(ja)], Vjb = V[IX(jb)];
                        const float2 Fja = Vf[IX(ja)], Fjb = Vf[IX(jb)];
                        const double yra = yval[2 * qa], yia = yval[2 * qa + 1], yrb = yval[2 * qb], yib = yval[2 * qb + 1];
                        const float2 Ya = yf32[qa], Yb = yf32[qb];
                        const unsigned wna = yword[k + 1 < na ? ea + k + 1 : 0], wnb = yword[k + 1 < nbb ? eb + k + 1 : 0];
                        // (computed unconditionally, so that the compiler keeps every load of the round above its arithmetic;
                        // a chain past its row adds nothing and stores to the dummy block)
                        const double dra = yra * Vja.x - yia * Vja.y, dia = yra * Vja.y + yia * Vja.x;
                        const double drb = yrb * Vjb.x - yib * Vjb.y, dib = yrb * Vjb.y + yib * Vjb.x;
                        if (ka) { ira += dra; iia += dia; }
                        if (kb) { irb += drb; iib += dib; }
                        const float ara = Ya.x * Fja.x - Ya.y * Fja.y, aia = Ya.x * Fja.y + Ya.y * Fja.x;
                        const float arb = Yb.x * Fjb.x - Yb.y * Fjb.y, aib = Yb.x * Fjb.y + Yb.y * Fjb.x;
                        const float tra = Fa.x * ara + Fa.y * aia, tia = Fa.y * ara - Fa.x * aia;
                        const float trb = Fb.x * arb + Fb.y * aib, tib = Fb.y * arb - Fb.x * aib;
                        const bool pqja = (wa >> 31) != 0u, pqjb = (wb >> 31) != 0u;
                        A4[IX(ka ? (int)(wa & 0xFFFF) : nblkA)] = make_float4(tia, pqja ? tra : 0.f, pqa ? -tra : 0.f, (pqa && pqja) ? tia : 0.f);
                        A4[IX(kb ? (int)(wb & 0xFFFF) : nblkA)] = make_float4(tib, pqjb ? trb : 0.f, pqb ? -trb : 0.f, (pqb && pqjb) ? tib : 0.f);
                        wa = wna; wb = wnb;
                    } while (++k < nk);
                    const double2 Va = V[IX(i)], Vb = V[IX(i2)];            // (read again: fewer registers live through the rows)
                    const double Pa = Va.x * ira + Va.y * iia, Qa = Va.y * ira - Va.x * iia;
                    const double Pb = Vb.x * irb + Vb.y * iib, Qb = Vb.y * irb - Vb.x * iib;
                    const PbBusRow ra = pb_bus_row(Va, Pa, Qa, psp[IX(i)], qsp[IX(i)], gfa, bfa, pqa, a.tol_pu);
                    const PbBusRow rb = pb_bus_row(Vb, Pb, Qb, psp[IX(i2)], qsp[IX(i2)], gfb, bfb, pqb, a.tol_pu);
                    const int bda = da.x & 0xFFFF, bdb = db.x & 0xFFFF;            // (0xFFFF: reference bus)
                    Pc[IX(i)] = Pa; Qc[IX(i)] = Qa;
                    if (bda != 0xFFFF) { A4[IX(bda)] = ra.D; A4[IX(nblk + (da.x >> 16))] = ra.R; viol |= ra.viol; wild |= ra.wild; }
                    if (two) {
                        Pc[IX(i2)] = Pb; Qc[IX(i2)] = Qb;
                        if (bdb != 0xFFFF) { A4[IX(bdb)] = rb.D; A4[IX(nblk + (db.x >> 16))] = rb.R; viol |= rb.viol; wild |= rb.wild; }
                    }
                }
            }
            viol = PB_ANY(viol);
            PB_CLOCK(PC_BUSES)
#ifndef B200PF_EMULATE
            if (UNI) {
                // lockstep: an instance that is through (converged / given up) keeps running with the warp until all are; its
                // state is frozen (no update below), so the repeated evaluations reproduce the same currents and powers
                wild = PB_ANY(wild);
                if (running) {
                    if (!viol) { conv = true; iters = it; running = false; }
                    else if (it >= a.max_iter || wild) { iters = it; running = false; }
                }
                if (!__any_sync(0xffffffffu, running)) break;
            } else
#endif
            {
                if (!viol) { conv = true; iters = it; break; }
                wild = PB_ANY(wild);
                if (it >= a.max_iter || wild) { iters = it; break; }
            }
            // block LU + triangular solves: the plan's operation stream.  A row = T * U slots, lane j executes slots
            // j, j + T, ..., all loads of its U operations before any store; rows prefetched one ahead.
            {
                unsigned char *Ab = reinterpret_cast<unsigned char *>(A4) + (size_t)gi * 16;
#define PB_AT(off) (*reinterpret_cast<float4 *>(Ab + (off)))
#ifdef B200PF_EMULATE
                for (int r = 0; r < n_brow; ++r) {
                    for (int s = 0; s < T * U; ++s) {
                        const uint2 op = bops[(size_t)r * T * U + s];
                        const unsigned od = op.x & 0xffffu, oa = op.x >> 16, ob = op.y & 0xffffu, fl = op.y >> 16;
                        float4 D = PB_AT(od);
                        const float4 Aa = PB_AT(oa);
                        if (fl & 2u) {
                            const float rdet = PF_RCP(Aa.x * Aa.w - Aa.y * Aa.z);
                            const float nx = rdet * (Aa.w * D.x - Aa.y * D.z), ny = rdet * (Aa.w * D.y - Aa.y * D.w);
                            const float nz = rdet * (Aa.x * D.z - Aa.z * D.x), nw = rdet * (Aa.x * D.w - Aa.z * D.y);
                            D = make_float4(nx, ny, nz, nw);
                        } else {
                            const float4 Bb = PB_AT(ob);
                            D.x -= Aa.x * Bb.x + Aa.y * Bb.z; D.y -= Aa.x * Bb.y + Aa.y * Bb.w;
                            D.z -= Aa.z * Bb.x + Aa.w * Bb.z; D.w -= Aa.z * Bb.y + Aa.w * Bb.w;
                        }
                        PB_AT(od) = D;
                    }
                }
#else
                const uint2 *op_t = bops + tid;
                uint2 q[U], qn[U];
#pragma unroll
                for (int u = 0; u < U; ++u) q[u] = op_t[u * T];
                for (int r = 0; r < n_brow; ++r) {
                    op_t += T * U;
#pragma unroll
                    for (int u = 0; u < U; ++u) qn[u] = op_t[u * T];          // (the stream ends with a guard row)
                    const unsigned fl = q[0].y >> 16;
                    float4 D[U], Aa[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) { D[u] = PB_AT(q[u].x & 0xffffu); Aa[u] = PB_AT(q[u].x >> 16); }
                    if (fl & 2u) {
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const float rdet = PF_RCP(Aa[u].x * Aa[u].w - Aa[u].y * Aa[u].z);
                            const float nx = rdet * (Aa[u].w * D[u].x - Aa[u].y * D[u].z), ny = rdet * (Aa[u].w * D[u].y - Aa[u].y * D[u].w);
                            const float nz = rdet * (Aa[u].x * D[u].z - Aa[u].z * D[u].x), nw = rdet * (Aa[u].x * D[u].w - Aa[u].z * D[u].y);
                            D[u] = make_float4(nx, ny, nz, nw);
                        }
                    } else {
                        float4 Bb[U];
#pragma unroll
                        for (int u = 0; u < U; ++u) Bb[u] = PB_AT(q[u].y & 0xffffu);
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            D[u].x -= Aa[u].x * Bb[u].x + Aa[u].y * Bb[u].z; D[u].y -= Aa[u].x * Bb[u].y + Aa[u].y * Bb[u].w;
                            D[u].z -= Aa[u].z * Bb[u].x + Aa[u].w * Bb[u].z; D[u].w -= Aa[u].z * Bb[u].y + Aa[u].w * Bb[u].w;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) PB_AT(q[u].x & 0xffffu) = D[u];
                    if (fl & 1u) PB_SYNC();
#pragma unroll
                    for (int u = 0; u < U; ++u) q[u] = qn[u];
                }
#endif
#undef PB_AT
            }
            PB_CLOCK(PC_STREAM)
            PF_PHASE {                                         // lane = bus: state update from the solved right-hand-side blocks
                // buses i and i + T of a lane as two independent chains, like the evaluation above
                PB_LOOP for (int i = tid; i < ((!UNI || running) ? nb : 0); i += 2 * T) {
                    const int i2 = i + T < nb ? i + T : i;
                    const uint2 da = bdesc[i], db = bdesc[i2];
                    const int ca = da.x >> 16, cb = db.x >> 16;               // (0xFFFF: reference bus, no step)
                    const float4 Xa = A4[IX(ca != 0xFFFF ? nblk + ca : nblkA)], Xb = A4[IX(cb != 0xFFFF ? nblk + cb : nblkA)];
                    const double2 Voa = V[IX(i)], Vob = V[IX(i2)];
                    const double vma = vm[IX(i)], vaa = va[IX(i)], vmb = vm[IX(i2)], vab = va[IX(i2)];
                    const double dtha = ca != 0xFFFF ? (double)Xa.x : 0.0, dthb = cb != 0xFFFF ? (double)Xb.x : 0.0;
                    const double dvra = (ca != 0xFFFF && (da.y >> 16) != 0u) ? (double)Xa.z : 0.0;
                    const double dvrb = (cb != 0xFFFF && (db.y >> 16) != 0u) ? (double)Xb.z : 0.0;
                    PbUpd ua = pb_update_small(Voa, vma, vaa, dtha, dvra), ub = pb_update_small(Vob, vmb, vab, dthb, dvrb);
                    if (!ua.small) pb_update_slow(ua);
                    if (!ub.small) pb_update_slow(ub);
                    V[IX(i)] = ua.V; Vf[IX(i)] = make_float2((float)ua.V.x, (float)ua.V.y); vm[IX(i)] = ua.vm; va[IX(i)] = ua.va;
                    if (i2 != i) { V[IX(i2)] = ub.V; Vf[IX(i2)] = make_float2((float)ub.V.x, (float)ub.V.y); vm[IX(i2)] = ub.vm; va[IX(i2)] = ub.va; }
                }
                // (the bus lanes above read right-hand-side blocks only; the cleared set holds the fill-in blocks)
                PB_LOOP for (int k = tid; k < n_bzero; k += T) A4[IX(bzero[k])] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            PB_SYNC();
            PB_CLOCK(PC_UPDATE)
        }
        if (!conv) PB_FAIL(ST_DIV, iters)
    } else {
        // DC: line lanes compute flows from the angles, bus lanes sum them for the slack share
        PF_PHASE {
            PB_LOOP for (int l = tid; l < nl; l += T) {
                const int f = p_brf[l];
                if (f == 0xFFFF) continue;
                const double pfl = line_bdc_[l] * (V[IX(f)].x - V[IX(p_brt[l])].x) + line_pshift_[l];
                cur[IX(2 * l)] = make_double2(pfl, 0.0); cur[IX(2 * l + 1)] = make_double2(-pfl, 0.0);
            }
        }
        PB_SYNC();
        PF_PHASE {
            PB_LOOP for (int i = tid; i < nb; i += T) {
                const int sx = shidx[i];
                double p = sx != 0xFFFF ? gsh[IX(sx)] : 0.0;
                for (int e = adj_ptr[i]; e < adj_ptr[i + 1]; ++e) p += cur[IX(adj[e])].x;
                Pc[IX(i)] = p; Qc[IX(i)] = 0.0;
            }
        }
        PB_SYNC();
    }
    // ---- 4. results (same float32 rounding rules as the reference's read-back, pPB:1159-1183) ------------------
    PB_SYNC();
    if (!is_dc) {
        // pandapower reports Va = angle(V), i.e. angles in (-180, 180]; the Newton iteration accumulates them unwrapped
        PF_PHASE { for (int i = tid; i < nb; i += T) { const double x = va[IX(i)]; va[IX(i)] = x - 6.283185307179586477 * rint(x * 0.15915494309189533577); } }
        PB_SYNC();
    }
    const double RAD2DEG = 57.295779513082320877, SQRT3 = 1.7320508075688772935;
    {
        const uint16_t *unit_bus = U16(o_unit_bus), *load_bus = U16(o_load_bus), *sto_bus = U16(o_sto_bus), *sh_bus = U16(o_sh_bus);
        const uint16_t *bu_ptr = U16(o_bu_ptr), *bu = U16(o_bu), *bl_ptr = U16(o_bl_ptr), *bl = U16(o_bl);
        const uint16_t *bs_ptr = U16(o_bs_ptr), *bs = U16(o_bs), *p_cnt = U16(o_cnt), *p_nref = U16(o_nref), *p_slot = U16(o_slot);
        const double *qmins = F64(o_qmins), *qmaxs = F64(o_qmaxs);
        PF_PHASE {
          if (UNI && fstat >= 0) {                             // lockstep: the failure record, stored without leaving the warp
            if (tid == 0) { a.status[inst] = fstat; a.iters[inst] = fiters; if (fstat == ST_DIV) PF_REDO_ARM(g, a, rd); }
            if (out) for (int k = tid; k < g.n_out; k += T) out[k] = PF_QNANF();
            if (a.busv) for (int k = tid; k < 2 * g.n_slot; k += T) a.busv[(size_t)inst * 2 * g.n_slot + k] = PF_QNAN();
            if (a.rho) for (int k = tid; k < g.n_line; k += T) a.rho[(size_t)inst * g.n_line + k] = PF_QNANF();
          } else {
            if (tid == 0) { a.status[inst] = ST_OK; a.iters[inst] = iters; }
            PB_LOOP for (int l = tid; l < nl; l += T) {
                float r[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                const int f = p_brf[l];
                if (f != 0xFFFF) {
                    const int t = p_brt[l];
                    const double vmf = vm[IX(f)], vmt = vm[IX(t)];
                    double pf, qf, pt, qt, sf, st;
                    if (is_dc) { pf = cur[IX(2 * l)].x * base; pt = -pf; qf = 0.0; qt = 0.0; sf = fabs(pf); st = sf; }
                    else {
                        // branch currents at both ends from the converged V (the Newton loop works on bus currents only)
                        const double2 Aa = V[IX(f)], Bb = V[IX(t)];
                        const double *y = line_y + (size_t)l * 8;
                        const double2 If = make_double2(y[0] * Aa.x - y[1] * Aa.y + y[2] * Bb.x - y[3] * Bb.y,
                                                        y[0] * Aa.y + y[1] * Aa.x + y[2] * Bb.y + y[3] * Bb.x);
                        const double2 It = make_double2(y[4] * Aa.x - y[5] * Aa.y + y[6] * Bb.x - y[7] * Bb.y,
                                                        y[4] * Aa.y + y[5] * Aa.x + y[6] * Bb.y + y[7] * Bb.x);
                        pf = (Aa.x * If.x + Aa.y * If.y) * base; qf = (Aa.y * If.x - Aa.x * If.y) * base;
                        pt = (Bb.x * It.x + Bb.y * It.y) * base; qt = (Bb.y * It.x - Bb.x * It.y) * base;
                        sf = sqrt(pf * pf + qf * qf); st = sqrt(pt * pt + qt * qt);
                    }
                    const float vnf = line_or_vn_[l], vnt = line_ex_vn_[l];
                    float a1 = (float)(sf / (SQRT3 * (vmf * (double)vnf)) * 1000.0), a2 = (float)(st / (SQRT3 * (vmt * (double)vnt)) * 1000.0);
                    if (!(fabsf(a1) <= 3.4e38f)) a1 = 0.f;
                    if (!(fabsf(a2) <= 3.4e38f)) a2 = 0.f;
                    r[0] = (float)pf; r[1] = (float)qf; r[2] = PF_FMUL((float)vmf, vnf); r[3] = a1; r[4] = (float)(va[IX(f)] * RAD2DEG);
                    r[5] = (float)pt; r[6] = (float)qt; r[7] = PF_FMUL((float)vmt, vnt); r[8] = a2; r[9] = (float)(va[IX(t)] * RAD2DEG);
                }
                if (out) { PB_UNROLL for (int k = 0; k < 10; ++k) out[k * nl + l] = r[k]; }
                if (a.rho) a.rho[(size_t)inst * nl + l] = r[3] / th_lim_[l];
            }
            if (out) {
                float *o = out + 10 * nl;
                PB_LOOP for (int u = tid; u < nu; u += T) {
                    float p = 0.f, q = 0.f, v = 0.f, th = 0.f;
                    const int i = unit_bus[u];
                    if (i != 0xFFFF) {
                        double pd = 0.0, qd = 0.0, pnonref = 0.0;
                        PB_LOOP for (int e = bl_ptr[i]; e < bl_ptr[i + 1]; ++e) { const int k = bl[e]; pd += LOAD_P(k); qd += LOAD_Q(k); }
                        PB_LOOP for (int e = bs_ptr[i]; e < bs_ptr[i + 1]; ++e) { const int k = bs[e]; pd += STO_P(k); qd += sto_q_[k]; }
                        PB_LOOP for (int e = bu_ptr[i]; e < bu_ptr[i + 1]; ++e) { const int u2 = bu[e]; if (!unit_is_ref_[u2]) pnonref += GEN_P(u2); }
                        double pu = GEN_P(u);
                        if (unit_is_ref_[u]) pu = (Pc[IX(i)] * base + pd - pnonref) / (double)p_nref[i];     // slack share (pandapower pfsoln)
                        double qu = 0.0;
                        if (!is_dc) {
                            const double qtot = Qc[IX(i)] * base + qd, qmn = qmins[i], qmx = qmaxs[i];
                            const int cb = p_cnt[i];
                            if (cb <= 1 || qmn == qmx) qu = qtot / (double)cb;
                            else qu = unit_qmin_[u] + (qtot - qmn) / (qmx - qmn + 2.220446049250313e-16) * (unit_qmax_[u] - unit_qmin_[u]);
                        }
                        p = (float)pu; q = (float)qu; v = PF_FMUL((float)vm[IX(i)], unit_vn_[u]); th = (float)(va[IX(i)] * RAD2DEG);
                    }
                    o[u] = p; o[nu + u] = q; o[2 * nu + u] = v; o[3 * nu + u] = th;
                }
                o += 4 * nu;
                PB_LOOP for (int k = tid; k < nld; k += T) {
                    const int i = load_bus[k];
                    o[k] = i != 0xFFFF ? PF_FMUL((float)vm[IX(i)], load_vn_[k]) : 0.f;
                    o[nld + k] = i != 0xFFFF ? (float)(va[IX(i)] * RAD2DEG) : 0.f;
                }
                o += 2 * nld;
                PB_LOOP for (int k = tid; k < nst; k += T) { const int i = sto_bus[k]; o[k] = i != 0xFFFF ? PF_FMUL((float)vm[IX(i)], sto_vn_[k]) : 0.f; }
                o += nst;
                PB_LOOP for (int k = tid; k < nsh; k += T) {
                    const int i = sh_bus[k];
                    float p = 0.f, q = 0.f, v = 0.f;
                    if (i != 0xFFFF) {
                        const double v2 = is_dc ? 1.0 : vm[IX(i)] * vm[IX(i)];
                        p = (float)(SH_P(k) * sh_vratio_[k] * v2);
                        q = is_dc ? 0.f : (float)(SH_Q(k) * sh_vratio_[k] * v2);
                        v = PF_FMUL((float)vm[IX(i)], sh_vn_[k]);
                    }
                    o[k] = p; o[nsh + k] = q; o[2 * nsh + k] = v;
                }
            }
            if (a.busv) {
                double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
                PB_LOOP for (int s = tid; s < 2 * g.n_slot; s += T) bv[s] = PF_QNAN();
            }
          }
        }
        PB_SYNC();
        if (a.busv) {
            double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
            PF_PHASE { if (!(UNI && fstat >= 0)) PB_LOOP for (int i = tid; i < nb; i += T) { bv[p_slot[i]] = vm[IX(i)]; bv[g.n_slot + p_slot[i]] = va[IX(i)]; } }
            PB_SYNC();
        }
    }
    PB_CLOCK(PC_OUT)
#if PB_CLOCK_ON
    if (clk_lane0) atomicAdd(&pb_phase_clk[PC_SOLVES], 1ull);
#endif
    if (PROT) {
        // Cascading-failure round: same rules and bookkeeping as the PROT block of solve_sparse (reference
        // Backend.next_grid_state, backend.py:1466-1521; counters baseEnv.py:3361-3370)
        const size_t base_l = (size_t)inst * nl;
        int any_trip = 0;
        PF_PHASE {
            PB_LOOP for (int l = tid; l < nl; l += T) {
                const bool on = p_brf[l] != 0xFFFF;
                const float aor = out[3 * nl + l], lim = th_lim_[l];
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
        any_trip = PB_ANY(any_trip);
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
                PB_LOOP for (int l = tid; l < nl; l += T) {
                    const float aor = out[3 * nl + l], lim = th_lim_[l];
                    int *pcp = a.pcount + base_l, *tsp = a.ts_over + base_l;
                    pcp[l] = (!a.from_reset && aor > PF_FMUL(a.soft_thr, lim)) ? pcp[l] + 1 : 0;
                    tsp[l] = (!a.from_reset && aor > lim) ? tsp[l] + 1 : 0;
                    a.incdone[base_l + l] = 0;
                }
            }
        }
        PB_SYNC();
    }
    (void)imask;
#undef PB_FAIL
#undef U16
#undef F64
#undef IX
#undef ROW
#undef GEN_P
#undef UNIT_VM
#undef LOAD_P
#undef LOAD_Q
#undef STO_P
#undef SH_P
#undef SH_Q
}

#ifndef B200PF_EMULATE
// ---- TMA (bulk asynchronous copy) staging of a SHARED plan -------------------------------------------------------------
// When every instance of a launch uses the same plan (DoNothing rollouts), a CTA of WPC warps can fetch the plan blob
// once into its shared memory with one cp.async.bulk (the TMA unit; completion on an mbarrier) instead of every lane
// re-reading the index arrays and the operation stream through L1 for every instance (B200PF_BLOCK_STAGE=0 selects the L1
// path for comparison).
__device__ __forceinline__ uint32_t pb_smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// starts the two copies (the CTA's first barrier included); pb_stage_wait returns once both have landed
__device__ __forceinline__ void pb_stage_issue(unsigned char *dst, const unsigned char *src, uint32_t bytes, unsigned char *dst2,
                                               const unsigned char *src2, uint32_t bytes2, uint64_t *mbar) {
    const uint32_t mb = pb_smem_addr(mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mb), "r"(1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes + bytes2) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(pb_smem_addr(dst)), "l"(src), "r"(bytes), "r"(mb) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(pb_smem_addr(dst2)), "l"(src2), "r"(bytes2), "r"(mb) : "memory");
    }
}
__device__ __forceinline__ void pb_stage_wait(uint64_t *mbar) {
    const uint32_t mb = pb_smem_addr(mbar);
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(mb), "r"(0) : "memory");
    }
}

// WPC warps per CTA for T <= 32 (each warp: G = 32 / T instances interleaved), one CTA of T threads per instance beyond.
// Persistent: warp slot w of CTA c takes the instance groups c * WPC + w, + gridDim * WPC, ...
// ws_bytes: workspace of one warp; STAGE: the launch's single plan (plan_bytes at plan_src in global memory) is copied behind
// the workspaces first, and while that copy is in flight every warp loads the chronics rows of its first instance group
// (row_ahead = 1: the plan is a solvable one, so pa_in.lay_nb / lay_nblkA give the workspace layout without its header;
// 0: solve_block stops at the plan's status before it reads a row, only a.t advances).
// UNI (T < 32 only): lockstep warps — requires ONE plan for the launch and batch % G == 0 (the host checks both).
template <int T, int U, int MINB, bool PROT, int WPC = 1, bool STAGE = false, bool UNI = false, int MODE = 0>
__global__ void __launch_bounds__((T < 32 ? 32 : T) * WPC, MINB)
pf_kernel_block(const DevGrid g, const RunArgs a, const PlanArgs pa_in, const int ws_bytes, const int plan_bytes, const unsigned char *plan_src,
                const int row_ahead, const RedoDesc rd) {
    extern __shared__ __align__(16) unsigned char smem[];
#if PB_CLOCK_ON
    const bool clk_lane0 = (threadIdx.x & 31) == 0;
    const long long clk_entry = clock64();
    long long clk_last = clk_entry;
    unsigned long long gt_entry;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt_entry));
#endif
    constexpr int G = T < 32 ? 32 / T : 1;
    static_assert(WPC == 1 || T <= 32, "several instances groups per CTA only for warp-sized groups");
    const int lane = T <= 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
    const int warp = T <= 32 ? (int)(threadIdx.x >> 5) : 0;
    const int gi = T < 32 ? lane % G : 0;
    const int j = T < 32 ? lane / G : lane;
    unsigned imask = 0xffffffffu;
    if (T < 32) {
        unsigned m = 0;
#pragma unroll
        for (int q = 0; q < T; ++q) m |= 1u << (q * G);
        imask = m << gi;
    }
    PlanArgs pa = pa_in;
    if (!STAGE) pa.stat = nullptr;
    __shared__ int zero_off;
    __shared__ __align__(8) uint64_t mbar;
    unsigned char *ws = smem + (size_t)warp * ws_bytes;
    const int n_grp = (a.batch + G - 1) / G;
    // staged launches: the inputs of an instance group (its chronics rows; the advance of a.t) are loaded here, ahead of
    // solve_block — for the warp's first group while the plan's bulk copy is in flight
    auto load_rows = [&](int inst) {
        const float *grow = block_row<T, G, PROT, UNI, MODE>(g, a, inst, j, imask);
        if (grow && row_ahead)
            block_row_copy<T, G, UNI>(grow, 2 * g.n_load + 2 * g.n_gen,
                                      reinterpret_cast<float *>(ws + block_srow_off<G>(pa_in.lay_nb, pa_in.lay_nblkA, g.n_shunt, g.n_line)), gi, j, imask);
    };
    int w = blockIdx.x * WPC + warp;
    if (STAGE) {
        // behind the workspaces: the plan blob, then the blob of static grid arrays (pa_in.stat: its copy in global memory)
        unsigned char *dst = smem + (size_t)WPC * ws_bytes;
        unsigned char *dst2 = dst + plan_bytes;
        if (threadIdx.x == 0) zero_off = 0;             // (published by the barrier inside pb_stage_issue)
        pb_stage_issue(dst, plan_src, (uint32_t)plan_bytes, dst2, pa_in.stat, (uint32_t)pa_in.so.total, &mbar);
        if (w < n_grp && w * G + gi < a.batch) load_rows((PROT && a.inst_list) ? a.inst_list[w * G + gi] : w * G + gi);
        pb_stage_wait(&mbar);
        pa.stat = dst2;
        pa.blobs = dst; pa.plan_off = &zero_off; pa.inst_plan = nullptr;
    }
    PB_CLOCK(PC_STAGE)
    for (bool first = true; w < n_grp; w += gridDim.x * WPC, first = false) {
        const int k = w * G + gi;
        if (k < a.batch) {
            const int inst = (PROT && a.inst_list) ? a.inst_list[k] : k;
            if (STAGE && !first) load_rows(inst);
            solve_block<T, U, G, PROT, UNI, MODE, STAGE>(g, a, pa, inst, ws, gi, j, imask, rd);
            // free-running instances leave solve_block at their failure (block_fail); the safety net is armed here, once per
            // instance, outside the diverged code (lockstep warps arm it in solve_block's failure record)
            if (!UNI && rd.on && j == 0 && a.status[inst] == ST_DIV) redo_arm(g, a, rd);
        }
        if (T <= 32) __syncwarp(); else __syncthreads();
    }
#if PB_CLOCK_ON
    if (clk_lane0) {
        unsigned long long gt_end;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt_end));
        atomicAdd(&pb_phase_clk[PC_WARPS], 1ull);
        atomicAdd(&pb_phase_clk[PC_CYCLES], (unsigned long long)(clock64() - clk_entry));
        atomicAdd(&pb_phase_clk[PC_NS], gt_end - gt_entry);
    }
#endif
}
#endif

}  // namespace b200pf

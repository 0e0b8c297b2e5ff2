// b200pf_small.cuh — one WARP per grid instance, for grids whose every element class fits 32 lanes
// (rte_case5, the 14-substation family): <= 32 bus slots, lines, units, loads, storages, shunts, and
// instances with <= 17 active buses (Newton system <= 32 unknowns, DC system <= 16).
//
// Compared with the generic group kernel (b200pf_kernel.cuh) the per-instance dependent chain is cut:
//   * lanes change role per phase: lane = line (flows, Jacobian off-diagonals), lane = bus (injections,
//     mismatch, diagonals, state update), lane = matrix row (Gauss-Jordan), lane = unit/load (read-back);
//   * topology in registers: active-slot bitmask + popc/fns numbering, reachability by bitmask sweeps;
//   * bus state (|V|, angle, P/Q spec, Yii) lives in registers of the bus lane; V and branch currents
//     are exchanged through small shared-memory tables (one STS.128 / LDS.128 each);
//   * Gauss-Jordan with the matrix in registers, pivot row broadcast by SHFL, pivot choice by one REDUX
//     on (|a| bits, lane) keys — no shared-memory round trip, no divergent branch in the step.
// Numerics are those of the generic kernel: fp64 state / mismatch / flows, fp32 Jacobian and solve.
#pragma once
#include "b200pf_kernel.cuh"

namespace b200pf {

struct SmallLayout {
    int off_V;      // double2 [32]
    int off_cur;    // double2 [64]
    int off_x;      // float [32] / double [16]
    int off_adj;    // unsigned [32]
    int off_b;      // bytes: brf[32] brt[32] colth[32] colv[32]
    int off_hot;    // double [6][32]: bus-lane state parked around the Gauss-Jordan (register pressure)
    int off_mat;    // matrix region
    int pitch_j;    // floats per Jacobian row
    int pitch_d;    // doubles per DC row
    int total;
};

__host__ __device__ inline SmallLayout small_layout(int nb_cap) {
    SmallLayout L;
    int o = 0;
    L.off_V = o; o += 32 * 16;
    L.off_cur = o; o += 64 * 16;
    L.off_x = o; o += 128;
    L.off_adj = o; o += 128;
    L.off_b = o; o += 128;
    L.off_hot = o; o += 6 * 32 * 8;
    L.off_mat = o;
    int d_cap = 2 * nb_cap - 2; if (d_cap > 32) d_cap = 32; if (d_cap < 2) d_cap = 2;
    int n1_cap = nb_cap - 1; if (n1_cap > 16) n1_cap = 16; if (n1_cap < 1) n1_cap = 1;
    L.pitch_j = (d_cap + 1) | 1;
    L.pitch_d = (n1_cap + 1) | 1;
    int ac = d_cap * L.pitch_j * 4, dc = n1_cap * L.pitch_d * 8;
    o += ((ac > dc ? ac : dc) + 15) & ~15;
    L.total = o;
    return L;
}

__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ float rcp_approx(float x) {      // one MUFU.RCP (1 ulp-ish; the fp64 residual decides convergence)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}


// N shuffles issued back to back from ONE asm statement: the consumers below cannot be interleaved with
// them by the compiler, so the SHFL latency is paid once per batch instead of once per element.
template <int N> struct ShflBatch;
template <> struct ShflBatch<8> {
    static __device__ __forceinline__ void run(float *o, const float *v, int src) {
        asm volatile("{\n"
                     "shfl.sync.idx.b32 %0, %8, %16, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %1, %9, %16, 0x1f, 0xffffffff;\n"
                     "shfl.sync.idx.b32 %2, %10, %16, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %3, %11, %16, 0x1f, 0xffffffff;\n"
                     "shfl.sync.idx.b32 %4, %12, %16, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %5, %13, %16, 0x1f, 0xffffffff;\n"
                     "shfl.sync.idx.b32 %6, %14, %16, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %7, %15, %16, 0x1f, 0xffffffff;\n"
                     "}"
                     : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]), "=f"(o[4]), "=f"(o[5]), "=f"(o[6]), "=f"(o[7])
                     : "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7]), "r"(src));
    }
};
template <> struct ShflBatch<4> {
    static __device__ __forceinline__ void run(float *o, const float *v, int src) {
        asm volatile("{\n"
                     "shfl.sync.idx.b32 %0, %4, %8, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %1, %5, %8, 0x1f, 0xffffffff;\n"
                     "shfl.sync.idx.b32 %2, %6, %8, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %3, %7, %8, 0x1f, 0xffffffff;\n"
                     "}"
                     : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]) : "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "r"(src));
    }
};
template <> struct ShflBatch<2> {
    static __device__ __forceinline__ void run(float *o, const float *v, int src) {
        asm volatile("{\n"
                     "shfl.sync.idx.b32 %0, %2, %4, 0x1f, 0xffffffff;\n" "shfl.sync.idx.b32 %1, %3, %4, 0x1f, 0xffffffff;\n"
                     "}"
                     : "=f"(o[0]), "=f"(o[1]) : "f"(v[0]), "f"(v[1]), "r"(src));
    }
};
template <> struct ShflBatch<1> {
    static __device__ __forceinline__ void run(float *o, const float *v, int src) { o[0] = __shfl_sync(0xffffffffu, v[0], src); }
};

// a[c0 .. c0+N) -= m * (row p's a[c0 .. c0+N)), N in {8,4,2,1}, then the rest of the row recursively
template <int C0, int END>
__device__ __forceinline__ void gj_row_update(float *a, float m, int p) {
    if constexpr (C0 < END) {
        constexpr int REM = END - C0;
        constexpr int N = REM >= 8 ? 8 : (REM >= 4 ? 4 : (REM >= 2 ? 2 : 1));
        float pr[N];
        ShflBatch<N>::run(pr, a + C0, p);
#pragma unroll
        for (int j = 0; j < N; ++j) a[C0 + j] -= m * pr[j];
        gj_row_update<C0 + N, END>(a, m, p);
    }
}

// compile-time dispatch on the (unrolled, hence constant) step index k
template <int DMAX, int K = 0>
__device__ __forceinline__ void gj_step_update(float *a, float m, int p, int k) {
    if constexpr (K < DMAX) {
        if (k == K) gj_row_update<K + 1, DMAX + 1>(a, m, p);
        else gj_step_update<DMAX, K + 1>(a, m, p, k);
    }
}

// Gauss-Jordan, rows in registers, pivot row broadcast with SHFL (see header).  M is only read.
template <int DMAX, typename S>
__device__ __forceinline__ bool gj_warp_shfl(const S *M, int n, int pitch, S *xs, int lane) {
    S a[DMAX + 1];
    const bool mine = lane < n;
    const S *Mr = M + lane * pitch;
#pragma unroll
    for (int c = 0; c < DMAX; ++c) a[c] = (mine && c < n) ? Mr[c] : S(0);
    a[DMAX] = mine ? Mr[n] : S(0);
    bool used = !mine;
    int mycol = -1;
    S pivval = S(1);
#pragma unroll
    for (int k = 0; k < DMAX; ++k) {
        if (k >= n) break;                                            // warp-uniform
        const float mag = fabsf((float)a[k]);
        unsigned key = (__float_as_uint(mag) & 0xffffffe0u) | (unsigned)(31 - lane);
        if (used || !(mag == mag)) key = 0u;
        const unsigned mx = __reduce_max_sync(0xffffffffu, key);
        if (mx < 0x00800000u) return false;                           // |pivot| below the smallest normal: singular / NaN
        const int p = 31 - (int)(mx & 31u);
        const S piv = __shfl_sync(0xffffffffu, a[k], p);
        S inv;
        if (sizeof(S) == 4) inv = (S)rcp_approx((float)piv); else inv = S(1) / piv;
        const bool isp = lane == p;
        const S m = isp ? S(0) : a[k] * inv;
        // pivot row broadcast in batches (fp32: batched asm shuffles; fp64: plain)
        if constexpr (sizeof(S) == 4) {
            gj_step_update<DMAX>(reinterpret_cast<float *>(a), (float)m, p, k);
        } else {
#pragma unroll
            for (int c = k + 1; c < DMAX + 1; ++c) {
                const S pr = __shfl_sync(0xffffffffu, a[c], p);
                a[c] -= m * pr;
            }
        }
        if (isp) { used = true; mycol = k; pivval = a[k]; }
    }
    if (mycol >= 0) xs[mycol] = a[DMAX] / pivval;
    __syncwarp();
    return true;
}

__device__ __noinline__ bool gj_small_f(const float *M, int n, int pitch, float *xs, int lane) {
    if (n <= 16) return gj_warp_shfl<16, float>(M, n, pitch, xs, lane);
    if (n <= 24) return gj_warp_shfl<24, float>(M, n, pitch, xs, lane);
    return gj_warp_shfl<32, float>(M, n, pitch, xs, lane);
}
__device__ __forceinline__ bool gj_small_d(const double *M, int n, int pitch, double *xs, int lane) {
    if (n <= 8) return gj_warp_shfl<8, double>(M, n, pitch, xs, lane);
    return gj_warp_shfl<16, double>(M, n, pitch, xs, lane);
}

__device__ __forceinline__ void small_fail(const DevGrid &g, const RunArgs &a, int inst, int status, int iters, int lane) {
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
    if (lane == 0) { a.status[inst] = status; a.iters[inst] = iters; if (a.done) a.done[inst] = 1; }
    if (a.disc && status == ST_DONE) for (int k = lane; k < g.n_line; k += 32) a.disc[(size_t)inst * g.n_line + k] = -1;
    if (out) for (int k = lane; k < g.n_out; k += 32) out[k] = qnanf();
    if (a.busv) for (int k = lane; k < 2 * g.n_slot; k += 32) a.busv[(size_t)inst * 2 * g.n_slot + k] = __longlong_as_double(0x7ff8000000000000LL);
    if (a.rho) for (int k = lane; k < g.n_line; k += 32) a.rho[(size_t)inst * g.n_line + k] = qnanf();
    __syncwarp();
}

template <bool PROT>
__device__ void solve_small(const DevGrid &g, const RunArgs &a, const SmallLayout &L, int inst, unsigned char *sm, int lane) {
    const unsigned FULL = 0xffffffffu;
    double2 *Vs = reinterpret_cast<double2 *>(sm + L.off_V);
    double2 *cur = reinterpret_cast<double2 *>(sm + L.off_cur);
    float *xs = reinterpret_cast<float *>(sm + L.off_x);
    double *xd = reinterpret_cast<double *>(sm + L.off_x);
    unsigned *adj = reinterpret_cast<unsigned *>(sm + L.off_adj);
    signed char *brf = reinterpret_cast<signed char *>(sm + L.off_b);
    signed char *brt = brf + 32, *colth_s = brf + 64, *colv_s = brf + 96;
    double *hot = reinterpret_cast<double *>(sm + L.off_hot);
    float *J = reinterpret_cast<float *>(sm + L.off_mat);
    double *Md = reinterpret_cast<double *>(sm + L.off_mat);
    const int src = a.n1_lines > 0 ? inst / a.n1_lines : inst;          // record the inputs come from
    const int outage = a.n1_lines > 0 ? inst % a.n1_lines : -1;         // line forced out of service (N-1 sweep)
    const int8_t *tv = a.topo + (size_t)src * g.n_topo_in;
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
    const double base = g.base_mva;
    const int nl = g.n_line, nu = g.n_unit, nh = g.n_hidden, ng = g.n_gen, nld = g.n_load, nst = g.n_sto, nsh = g.n_shunt;
    const unsigned lt = (1u << lane) - 1u;

    // ---- 0. this lane's injections (lane = unit / load / storage / shunt index) ---------------------
    double u_p = 0.0, u_vm = 1.0, l_p = 0.0, l_q = 0.0, s_p = 0.0, sh_p = 0.0, sh_q = 0.0;
    if (a.series) {
        const int sc = a.rows ? 0 : a.scen[src], trow = a.rows ? 0 : a.t[src];
        const float *row = a.rows ? a.rows + (size_t)src * (size_t)(2 * nld + 2 * ng)
                                  : a.chron + ((size_t)sc * a.n_rows + trow) * (size_t)(2 * nld + 2 * ng);
        const double *si = a.static_inj;
        if (lane < nld) { l_p = (double)row[lane]; l_q = (double)row[nld + lane]; }
        if (lane < nu) {
            if (lane >= nh) {
                u_p = (double)row[2 * nld + lane - nh];
                u_vm = (double)__fdiv_rn(row[2 * nld + ng + lane - nh], g.unit_vn[lane]);   // float32 / float32, pPB:927
            } else u_vm = si[ng + lane];
        }
        if (lane < nst) s_p = si[ng + nu + 2 * nld + lane];
        if (lane < nsh) { sh_p = si[ng + nu + 2 * nld + nst + lane]; sh_q = si[ng + nu + 2 * nld + nst + nsh + lane]; }
        __syncwarp();
        if (lane == 0 && !a.rows && a.n1_lines <= 0) a.t[inst] = (trow + 1 >= a.n_rows) ? 0 : trow + 1;
    } else {
        const double *sp = a.inj + (size_t)src * g.n_inj;
        if (lane < nu) { u_vm = sp[ng + lane]; if (lane >= nh) u_p = sp[lane - nh]; }
        if (lane < nld) { l_p = sp[ng + nu + lane]; l_q = sp[ng + nu + nld + lane]; }
        if (lane < nst) s_p = sp[ng + nu + 2 * nld + lane];
        if (lane < nsh) { sh_p = sp[ng + nu + 2 * nld + nst + lane]; sh_q = sp[ng + nu + 2 * nld + nst + nsh + lane]; }
    }

    // protections state (lane = line)
    if (PROT && a.done[inst]) { small_fail(g, a, inst, ST_DONE, 0, lane); return; }
    int pc_env = 0, pc = 0, disc_it = -1;
    bool forced_off = false, inc_done = false;
    if (PROT && lane < nl) { pc_env = a.pcount[(size_t)inst * nl + lane]; pc = pc_env; }
    for (int casc = 0;; ++casc) {
    // ---- 1. topology: active bus slots as a bit mask ------------------------------------------------
    int slot_o = -1, slot_e = -1, slot_u = -1, slot_k = -1, slot_s = -1, slot_h = -1;
    if (lane < nl && lane != outage && !(PROT && forced_off)) {
        const int bo = tv[g.line_or_pos[lane]], be = tv[g.line_ex_pos[lane]];
        if (bo > 0) slot_o = g.line_or_sub[lane] + (bo - 1) * g.n_sub;
        if (be > 0) slot_e = g.line_ex_sub[lane] + (be - 1) * g.n_sub;
    }
    if (lane < nu) { const int b = tv[g.unit_pos[lane]]; if (b > 0) slot_u = g.unit_sub[lane] + (b - 1) * g.n_sub; }
    if (lane < nld) { const int b = tv[g.load_pos[lane]]; if (b > 0) slot_k = g.load_sub[lane] + (b - 1) * g.n_sub; }
    if (lane < nst) { const int b = tv[g.sto_pos[lane]]; if (b > 0) slot_s = g.sto_sub[lane] + (b - 1) * g.n_sub; }
    if (lane < nsh) { const int b = tv[g.dim_topo + lane]; if (b > 0) slot_h = g.sh_sub[lane] + (b - 1) * g.n_sub; }
    unsigned m = 0;
    if (slot_o >= 0) m |= 1u << slot_o;
    if (slot_e >= 0) m |= 1u << slot_e;
    if (slot_u >= 0) m |= 1u << slot_u;
    if (slot_k >= 0) m |= 1u << slot_k;
    if (slot_s >= 0) m |= 1u << slot_s;
    if (slot_h >= 0) m |= 1u << slot_h;
    const unsigned amask = __reduce_or_sync(FULL, m);
    const int nb = __popc(amask);
    if (nb > a.nb_cap || nb > 17) { small_fail(g, a, inst, ST_LARGE, 0, lane); return; }
#define CIDX(s) (__popc(amask & ((1u << (s)) - 1u)))
    const int bf = (slot_o >= 0 && slot_e >= 0) ? CIDX(slot_o) : -1;
    const int bt = (slot_o >= 0 && slot_e >= 0) ? CIDX(slot_e) : -1;
    const int bu = slot_u >= 0 ? CIDX(slot_u) : -1;
    const int bk = slot_k >= 0 ? CIDX(slot_k) : -1;
    const int bs = slot_s >= 0 ? CIDX(slot_s) : -1;
    const int bh = slot_h >= 0 ? CIDX(slot_h) : -1;
    const bool isbus = lane < nb;
    const int myslot = isbus ? (int)__fns(amask, 0, lane + 1) : 0;
    const int mysub = myslot % g.n_sub;
    brf[lane] = (signed char)bf; brt[lane] = (signed char)bt;
    adj[lane] = 0u;
    __syncwarp();
    if (bf >= 0) { atomicOr(&adj[bf], 1u << bt); atomicOr(&adj[bt], 1u << bf); }
    // per-bus list of the in-service line ends on this bus, packed 6 bits per entry (code = 2*line + side < 64):
    // built once, used by every mismatch pass instead of re-filtering the substation's static list
    unsigned long long adjc = 0ull;
    int adeg = 0;
    if (isbus) {
        for (int e = g.sub_end_ptr[mysub]; e < g.sub_end_ptr[mysub + 1]; ++e) {
            const int code = g.sub_end[e], l = code >> 1;
            const int f = brf[l];
            if (f < 0 || ((code & 1) ? brt[l] : f) != lane) continue;
            if (adeg < 10) adjc |= (unsigned long long)code << (6 * adeg);
            ++adeg;
        }
    }
    const bool adj_packed = !__any_sync(FULL, adeg > 10);      // (a bus with more than 10 line ends: generic path)

    // ---- 2. per-bus aggregates, in element order (deterministic; the later unit wins the set point) -
    int btype = BT_PQ, cnt = 0, nref = 0;
    double vm = 1.0, pg = 0.0, pd = 0.0, qd = 0.0, gsh = 0.0, bsh = 0.0, qmins = 0.0, qmaxs = 0.0, pnonref = 0.0;
    {
        const int isref = (lane < nu) ? g.unit_is_ref[lane] : 0;
        const double qmn = (lane < nu) ? g.unit_qmin[lane] : 0.0, qmx = (lane < nu) ? g.unit_qmax[lane] : 0.0;
        for (int u = 0; u < nu; ++u) {
            const int b = __shfl_sync(FULL, bu, u);
            const int r = __shfl_sync(FULL, isref, u);
            const double p = shfl_d(u_p, u), v = shfl_d(u_vm, u), q1 = shfl_d(qmn, u), q2 = shfl_d(qmx, u);
            if (b == lane && isbus) {
                vm = v; cnt++; qmins += q1; qmaxs += q2; pg += p;
                if (r) { btype = BT_REF; nref++; } else { if (btype != BT_REF) btype = BT_PV; pnonref += p; }
            }
        }
        for (int k = 0; k < nld; ++k) {
            const int b = __shfl_sync(FULL, bk, k);
            const double p = shfl_d(l_p, k), q = shfl_d(l_q, k);
            if (b == lane && isbus) { pd += p; qd += q; }
        }
        const double sq = (lane < nst) ? g.sto_q[lane] : 0.0;
        for (int k = 0; k < nst; ++k) {
            const int b = __shfl_sync(FULL, bs, k);
            const double p = shfl_d(s_p, k), q = shfl_d(sq, k);
            if (b == lane && isbus) { pd += p; qd += q; }
        }
        const double vr = (lane < nsh) ? g.sh_vratio[lane] : 0.0;
        for (int k = 0; k < nsh; ++k) {
            const int b = __shfl_sync(FULL, bh, k);
            const double p = shfl_d(sh_p * vr, k), q = shfl_d(sh_q * vr, k);
            if (b == lane && isbus) { gsh += p; bsh -= q; }
        }
    }
    // ---- 3. reachability from the reference buses -------------------------------------------------
    __syncwarp();
    const unsigned myadj = isbus ? adj[lane] : 0u;
    const unsigned refmask = __ballot_sync(FULL, isbus && btype == BT_REF);
    if (!refmask) { small_fail(g, a, inst, ST_NOREF, 0, lane); return; }
    unsigned reach = refmask;
    for (int sweep = 0; sweep < 32; ++sweep) {
        const unsigned nr = reach | __reduce_or_sync(FULL, ((reach >> lane) & 1u) ? myadj : 0u);
        if (nr == reach) break;
        reach = nr;
    }
    const unsigned allmask = (nb >= 32) ? FULL : ((1u << nb) - 1u);
    if ((reach & allmask) != allmask) { small_fail(g, a, inst, ST_UNSUP, 0, lane); return; }

    // ---- 4. unknown numbering ---------------------------------------------------------------------
    const unsigned nonref = __ballot_sync(FULL, isbus && btype != BT_REF);
    const unsigned pqm = __ballot_sync(FULL, isbus && btype == BT_PQ);
    const int n1 = __popc(nonref), d = n1 + __popc(pqm);
    const int colth = (isbus && btype != BT_REF) ? __popc(nonref & lt) : -1;
    const int colv = (isbus && btype == BT_PQ) ? n1 + __popc(pqm & lt) : -1;
    if (n1 > 16 || d > 32 || n1 * L.pitch_d * 8 > (L.total - L.off_mat) || (!a.is_dc && d * L.pitch_j * 4 > (L.total - L.off_mat))) {
        small_fail(g, a, inst, ST_LARGE, 0, lane); return;
    }
    colth_s[lane] = (signed char)colth; colv_s[lane] = (signed char)colv;
    double pspec = (pg - pd) / base, qspec = -qd / base;
    // values needed again only for the read-back are parked in thread-local memory so that they do not
    // occupy registers during the Newton loop (the register Gauss-Jordan needs them for shuffle batching)
    volatile double cold[8];
    volatile int coldi[2];
    cold[0] = pd; cold[1] = qd; cold[2] = pnonref; cold[3] = qmins; cold[4] = qmaxs; cold[5] = u_p; cold[6] = sh_p; cold[7] = sh_q;
    coldi[0] = cnt; coldi[1] = nref;
    __syncwarp();

    // ---- 5. Ybus diagonal and the DC system (bus lane = matrix row) ---------------------------------
    const double gs_pu = gsh / base, bs_pu = bsh / base;      // shunt admittance in p.u. (divided once)
    double gii = gs_pu, bii = bs_pu, va = 0.0;
    if (a.is_dc) {
        // DC mode: the angles ARE the result -> fp64 system
        const int pitch = (n1 + 1) | 1;
        double *Mr = Md + (colth >= 0 ? colth : 0) * pitch;
        if (colth >= 0) for (int c = 0; c <= n1; ++c) Mr[c] = 0.0;
        double rhs = pspec - gs_pu, dsum = 0.0;
        if (isbus) {
            for (int e = g.sub_end_ptr[mysub]; e < g.sub_end_ptr[mysub + 1]; ++e) {
                const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                const int f = brf[l];
                if (f < 0) continue;
                const int t = brt[l];
                if ((side ? t : f) != lane) continue;
                const int j = side ? f : t;
                const double *y = g.line_y + l * 8 + (side ? 6 : 0);
                gii += y[0]; bii += y[1];
                const double b = g.line_bdc[l];
                dsum += b;
                const int cj = colth_s[j];
                if (colth >= 0 && cj >= 0) Mr[cj] -= b;                 // reference angle is 0 (pPB:473)
                rhs -= side ? -g.line_pshift[l] : g.line_pshift[l];
            }
            // (+=: a line with both ends on this bus took b twice off the diagonal above, which cancels its 2 b in dsum)
            if (colth >= 0) { Mr[colth] += dsum; Mr[n1] = rhs; }
        }
        __syncwarp();
        if (!gj_small_d(Md, n1, pitch, xd, lane)) { small_fail(g, a, inst, ST_DIV, 0, lane); return; }
        if (colth >= 0) va = xd[colth];
    } else {
        // AC mode: the DC angles are only the Newton start (init="dc", pPB:1086) -> fp32 system, same solver as
        // the Jacobian (the converged state does not depend on the last bits of the start)
        const int pitch = (n1 + 1) | 1;
        float *Mr = J + (colth >= 0 ? colth : 0) * pitch;
        if (colth >= 0) for (int c = 0; c <= n1; ++c) Mr[c] = 0.f;
        float rhs = (float)(pspec - gs_pu), dsum = 0.f;
        if (isbus) {
            for (int e = g.sub_end_ptr[mysub]; e < g.sub_end_ptr[mysub + 1]; ++e) {
                const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                const int f = brf[l];
                if (f < 0) continue;
                const int t = brt[l];
                if ((side ? t : f) != lane) continue;
                const int j = side ? f : t;
                const double *y = g.line_y + l * 8 + (side ? 6 : 0);
                gii += y[0]; bii += y[1];
                const float b = (float)g.line_bdc[l];
                dsum += b;
                const int cj = colth_s[j];
                if (colth >= 0 && cj >= 0) Mr[cj] -= b;
                const float ps = (float)g.line_pshift[l];
                rhs -= side ? -ps : ps;
            }
            if (colth >= 0) { Mr[colth] += dsum; Mr[n1] = rhs; }            // (+=: as in the DC system)
        }
        __syncwarp();
        if (!gj_small_f(J, n1, pitch, xs, lane)) { small_fail(g, a, inst, ST_DIV, 0, lane); return; }
        if (colth >= 0) va = (double)xs[colth];
    }
    {
        const int bad = isbus && !isfinite(va);
        if (__any_sync(FULL, bad)) { small_fail(g, a, inst, ST_DIV, 0, lane); return; }
        __syncwarp();
    }

    // ---- 6. Newton-Raphson ----------------------------------------------------------------------------
    const double RAD2DEG = 57.295779513082320877, SQRT3 = 1.7320508075688772935;
    double ve = 0.0, vf = 0.0, P = 0.0, Q = 0.0;
    int iters = 0;
    if (!a.is_dc) {
        { double s, c; sincos(va, &s, &c); ve = vm * c; vf = vm * s; }
        bool conv = false;
        const int pitch = (d + 1) | 1;
        for (int it = 0;; ++it) {
            if (isbus) Vs[lane] = make_double2(ve, vf);
            __syncwarp();
            double2 Vf = make_double2(0, 0), Vt = make_double2(0, 0);
            if (bf >= 0) {                                            // lane = line: currents at both ends
                Vf = Vs[bf]; Vt = Vs[bt];
                const double4 *y4 = reinterpret_cast<const double4 *>(g.line_y + lane * 8);
                const double4 ya = y4[0], yb = y4[1];                   // (yff, yft), (ytf, ytt)
                cur[2 * lane] = make_double2(ya.x * Vf.x - ya.y * Vf.y + ya.z * Vt.x - ya.w * Vt.y,
                                             ya.x * Vf.y + ya.y * Vf.x + ya.z * Vt.y + ya.w * Vt.x);
                cur[2 * lane + 1] = make_double2(yb.x * Vf.x - yb.y * Vf.y + yb.z * Vt.x - yb.w * Vt.y,
                                                 yb.x * Vf.y + yb.y * Vf.x + yb.z * Vt.y + yb.w * Vt.x);
            }
            __syncwarp();
            int viol = 0, wild = 0;
            double dP = 0.0, dQ = 0.0;
            if (isbus) {                                              // lane = bus: S = V conj(I)
                double ir = gs_pu * ve - bs_pu * vf, ii = gs_pu * vf + bs_pu * ve;
                if (adj_packed) {
                    unsigned long long cc = adjc;
                    for (int j = 0; j < adeg; ++j, cc >>= 6) {
                        const double2 c2 = cur[(int)(cc & 63ull)];
                        ir += c2.x; ii += c2.y;
                    }
                } else {
                    for (int e = g.sub_end_ptr[mysub]; e < g.sub_end_ptr[mysub + 1]; ++e) {
                        const int code = g.sub_end[e], l = code >> 1;
                        const int f = brf[l];
                        if (f < 0 || ((code & 1) ? brt[l] : f) != lane) continue;
                        const double2 c2 = cur[code];
                        ir += c2.x; ii += c2.y;
                    }
                }
                P = ve * ir + vf * ii; Q = vf * ir - ve * ii;
                if (btype != BT_REF) { dP = P - pspec; const double m1 = fabs(dP); viol |= !(m1 < a.tol_pu); wild |= !(m1 < 1e200); }
                if (btype == BT_PQ) { dQ = Q - qspec; const double m2 = fabs(dQ); viol |= !(m2 < a.tol_pu); wild |= !(m2 < 1e200); }
            }
            if (!__any_sync(FULL, viol)) { conv = true; iters = it; break; }
            if (it >= a.max_iter || __any_sync(FULL, wild)) { iters = it; break; }
            // Jacobian (fp32): zero, diagonals by the bus lanes, off-diagonals by the line lanes
            if (lane < d) { float *Jr = J + lane * pitch; for (int c = 0; c <= d; ++c) Jr[c] = 0.f; }
            __syncwarp();
            if (colth >= 0) {
                const float vi2 = (float)(ve * ve + vf * vf), Pf = (float)P, Qf = (float)Q, gi = (float)gii, bi = (float)bii;
                float *JP = J + colth * pitch;
                JP[colth] = -Qf - bi * vi2; JP[d] = (float)(-dP);
                if (colv >= 0) {
                    float *JQ = J + colv * pitch;
                    JP[colv] = Pf + gi * vi2;
                    JQ[colth] = Pf - gi * vi2; JQ[colv] = Qf - bi * vi2; JQ[d] = (float)(-dQ);
                }
            }
            if (bf >= 0) {
                const double4 *y4 = reinterpret_cast<const double4 *>(g.line_y + lane * 8);
                const double4 ya = y4[0], yb = y4[1];
                const float ef = (float)Vf.x, ff = (float)Vf.y, et = (float)Vt.x, ft = (float)Vt.y;
                {   // rows of bus f, columns of bus t:  T = Vf conj(yft Vt)
                    const float yr = (float)ya.z, yi = (float)ya.w;
                    const float ar = yr * et - yi * ft, ai = yr * ft + yi * et;
                    const float tr = ef * ar + ff * ai, ti = ff * ar - ef * ai;
                    const int rp = colth_s[bf], rq = colv_s[bf], cth = colth_s[bt], cv = colv_s[bt];
                    if (rp >= 0) { if (cth >= 0) atomicAdd(&J[rp * pitch + cth], ti); if (cv >= 0) atomicAdd(&J[rp * pitch + cv], tr); }
                    if (rq >= 0) { if (cth >= 0) atomicAdd(&J[rq * pitch + cth], -tr); if (cv >= 0) atomicAdd(&J[rq * pitch + cv], ti); }
                }
                {   // rows of bus t, columns of bus f:  T = Vt conj(ytf Vf)
                    const float yr = (float)yb.x, yi = (float)yb.y;
                    const float ar = yr * ef - yi * ff, ai = yr * ff + yi * ef;
                    const float tr = et * ar + ft * ai, ti = ft * ar - et * ai;
                    const int rp = colth_s[bt], rq = colv_s[bt], cth = colth_s[bf], cv = colv_s[bf];
                    if (rp >= 0) { if (cth >= 0) atomicAdd(&J[rp * pitch + cth], ti); if (cv >= 0) atomicAdd(&J[rp * pitch + cv], tr); }
                    if (rq >= 0) { if (cth >= 0) atomicAdd(&J[rq * pitch + cth], -tr); if (cv >= 0) atomicAdd(&J[rq * pitch + cv], ti); }
                }
            }
            __syncwarp();
            hot[lane] = vm; hot[32 + lane] = va; hot[64 + lane] = pspec; hot[96 + lane] = qspec; hot[128 + lane] = gii; hot[160 + lane] = bii;
            const bool solved = gj_small_f(J, d, pitch, xs, lane);
            vm = hot[lane]; va = hot[32 + lane]; pspec = hot[64 + lane]; qspec = hot[96 + lane]; gii = hot[128 + lane]; bii = hot[160 + lane];
            if (!solved) { iters = it + 1; break; }
            if (isbus) {
                if (colth >= 0) va += (double)xs[colth];
                if (colv >= 0) vm *= 1.0 + (double)xs[colv];
                if (vm < 0.0) { vm = -vm; va += 3.14159265358979323846; }
                double s, c; sincos(va, &s, &c); ve = vm * c; vf = vm * s;
            }
            __syncwarp();
        }
        if (!conv) { small_fail(g, a, inst, ST_DIV, iters, lane); return; }
    } else {
        // DC: publish angles, line lanes compute flows, bus lanes sum them for the slack share
        if (isbus) Vs[lane] = make_double2(va, vm);
        __syncwarp();
        if (bf >= 0) {
            const double pfl = g.line_bdc[lane] * (Vs[bf].x - Vs[bt].x) + g.line_pshift[lane];
            cur[2 * lane] = make_double2(pfl, 0.0); cur[2 * lane + 1] = make_double2(-pfl, 0.0);
        }
        __syncwarp();
        if (isbus) {
            double p = gs_pu;
            for (int e = g.sub_end_ptr[mysub]; e < g.sub_end_ptr[mysub + 1]; ++e) {
                const int code = g.sub_end[e], l = code >> 1;
                const int f = brf[l];
                if (f < 0 || ((code & 1) ? brt[l] : f) != lane) continue;
                p += cur[code].x;
            }
            P = p; Q = 0.0;
        }
    }

    // ---- 7. results -------------------------------------------------------------------------------------
    if (!a.is_dc) va = va - 6.283185307179586477 * rint(va * 0.15915494309189533577);     // pandapower reports angle(V): (-180, 180]
    if (lane == 0) { a.status[inst] = ST_OK; a.iters[inst] = iters; }
    float r[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    {   // lines (lane = line): flows from the currents of the last mismatch evaluation
        const int sf_ = bf >= 0 ? bf : 0, st_ = bt >= 0 ? bt : 0;
        const double vmf = shfl_d(vm, sf_), vmt = shfl_d(vm, st_), vaf = shfl_d(va, sf_), vat = shfl_d(va, st_);
        if (lane < nl && bf >= 0) {
            double pf, qf, pt, qt, sf, st;
            if (a.is_dc) {
                pf = cur[2 * lane].x * base; pt = -pf; qf = 0.0; qt = 0.0; sf = fabs(pf); st = sf;
            } else {
                const double2 A = Vs[bf], B = Vs[bt], If = cur[2 * lane], It = cur[2 * lane + 1];
                pf = (A.x * If.x + A.y * If.y) * base; qf = (A.y * If.x - A.x * If.y) * base;
                pt = (B.x * It.x + B.y * It.y) * base; qt = (B.y * It.x - B.x * It.y) * base;
                sf = sqrt(pf * pf + qf * qf); st = sqrt(pt * pt + qt * qt);
            }
            const float vnf = g.line_or_vn[lane], vnt = g.line_ex_vn[lane];
            float a1 = (float)(sf / (SQRT3 * (vmf * (double)vnf)) * 1000.0), a2 = (float)(st / (SQRT3 * (vmt * (double)vnt)) * 1000.0);
            if (!isfinite(a1)) a1 = 0.f;
            if (!isfinite(a2)) a2 = 0.f;
            r[0] = (float)pf; r[1] = (float)qf; r[2] = __fmul_rn((float)vmf, vnf); r[3] = a1; r[4] = (float)(vaf * RAD2DEG);
            r[5] = (float)pt; r[6] = (float)qt; r[7] = __fmul_rn((float)vmt, vnt); r[8] = a2; r[9] = (float)(vat * RAD2DEG);
        }
    }
    if (PROT) {
        // cascading failure step (reference Backend.next_grid_state, backend.py:1466-1521), lane = line
        const bool on = lane < nl && bf >= 0;
        const float lim = lane < nl ? a.th_lim[lane] : 0.f;
        bool to_disc = on && (r[3] > __fmul_rn(a.hard_thr, lim));
        const bool mask_inc = !a.from_reset && on && (r[3] > __fmul_rn(a.soft_thr, lim)) && !inc_done;
        if (mask_inc) { pc += 1; inc_done = true; }
        if (on && pc > a.max_pc) to_disc = true;
        if (__any_sync(FULL, to_disc)) {
            if (to_disc) { forced_off = true; disc_it = casc; }
            __syncwarp();
            continue;                                   // re-solve with the lines removed
        }
        if (lane < nl) {
            int *pcp = a.pcount + (size_t)inst * nl, *tsp = a.ts_over + (size_t)inst * nl;
            // counters: baseEnv.py:3361-3370; Environment.reset() zeroes them after its step (baseEnv.py:3969-3970)
            pcp[lane] = (!a.from_reset && r[3] > __fmul_rn(a.soft_thr, lim)) ? pc_env + 1 : 0;
            tsp[lane] = (!a.from_reset && r[3] > lim) ? tsp[lane] + 1 : 0;
            a.disc[(size_t)inst * nl + lane] = disc_it;
            if (forced_off) {                           // persist the outage (_BackendAction.update_state)
                int8_t *tw = const_cast<int8_t *>(tv);
                tw[g.line_or_pos[lane]] = -1; tw[g.line_ex_pos[lane]] = -1;
            }
        }
    }
    if (lane < nl) {
        if (out) {
#pragma unroll
            for (int k = 0; k < 10; ++k) out[k * nl + lane] = r[k];
        }
        if (a.rho) a.rho[(size_t)inst * nl + lane] = r[3] / a.th_lim[lane];
    }
    {   // units (lane = unit), loads, storages, shunts: read their bus through shuffles
        const int su = bu >= 0 ? bu : 0;
        const double pd_ = cold[0], qd_ = cold[1], pnonref_ = cold[2], qmins_ = cold[3], qmaxs_ = cold[4];
        const int cnt_ = coldi[0], nref_ = coldi[1];
        const double Pb = shfl_d(P, su), Qb = shfl_d(Q, su), pdb = shfl_d(pd_, su), qdb = shfl_d(qd_, su), pnr = shfl_d(pnonref_, su);
        const double qmn = shfl_d(qmins_, su), qmx = shfl_d(qmaxs_, su), vmb = shfl_d(vm, su), vab = shfl_d(va, su);
        const int cb = __shfl_sync(FULL, cnt_, su), nrb = __shfl_sync(FULL, nref_, su);
        if (lane < nu && out) {
            float p = 0.f, q = 0.f, v = 0.f, th = 0.f;
            if (bu >= 0) {
                double pu = cold[5];
                if (g.unit_is_ref[lane]) pu = (Pb * base + pdb - pnr) / (double)nrb;     // slack share (pandapower pfsoln)
                double qu = 0.0;
                if (!a.is_dc) {
                    const double qtot = Qb * base + qdb;
                    if (cb <= 1 || qmn == qmx) qu = qtot / (double)cb;
                    else qu = g.unit_qmin[lane] + (qtot - qmn) / (qmx - qmn + 2.220446049250313e-16) * (g.unit_qmax[lane] - g.unit_qmin[lane]);
                }
                p = (float)pu; q = (float)qu; v = __fmul_rn((float)vmb, g.unit_vn[lane]); th = (float)(vab * RAD2DEG);
            }
            float *o = out + 10 * nl;
            o[lane] = p; o[nu + lane] = q; o[2 * nu + lane] = v; o[3 * nu + lane] = th;
        }
        const int sk = bk >= 0 ? bk : 0;
        const double vmk = shfl_d(vm, sk), vak = shfl_d(va, sk);
        if (lane < nld && out) {
            float *o = out + 10 * nl + 4 * nu;
            o[lane] = bk >= 0 ? __fmul_rn((float)vmk, g.load_vn[lane]) : 0.f;
            o[nld + lane] = bk >= 0 ? (float)(vak * RAD2DEG) : 0.f;
        }
        const int ss = bs >= 0 ? bs : 0;
        const double vms = shfl_d(vm, ss);
        if (lane < nst && out) out[10 * nl + 4 * nu + 2 * nld + lane] = bs >= 0 ? __fmul_rn((float)vms, g.sto_vn[lane]) : 0.f;
        const int sh = bh >= 0 ? bh : 0;
        const double vmh = shfl_d(vm, sh);
        if (lane < nsh && out) {
            float *o = out + 10 * nl + 4 * nu + 2 * nld + nst;
            float p = 0.f, q = 0.f, v = 0.f;
            if (bh >= 0) {
                const double v2 = a.is_dc ? 1.0 : vmh * vmh;
                p = (float)(cold[6] * g.sh_vratio[lane] * v2);
                q = a.is_dc ? 0.f : (float)(cold[7] * g.sh_vratio[lane] * v2);
                v = __fmul_rn((float)vmh, g.sh_vn[lane]);
            }
            o[lane] = p; o[nsh + lane] = q; o[2 * nsh + lane] = v;
        }
    }
    if (a.busv) {
        double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
        const double nanv = __longlong_as_double(0x7ff8000000000000LL);
        if (lane < g.n_slot && !((amask >> lane) & 1u)) { bv[lane] = nanv; bv[g.n_slot + lane] = nanv; }
        if (isbus) { bv[myslot] = vm; bv[g.n_slot + myslot] = va; }
    }
    __syncwarp();
    break;
    }   // cascade loop
#undef CIDX
}

template <bool PROT>
__global__ void __launch_bounds__(32, B200PF_MIN_WARP_CTAS)
pf_kernel_small(const DevGrid g, const RunArgs a, const SmallLayout L) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x;
    for (int inst = blockIdx.x; inst < a.batch; inst += gridDim.x) solve_small<PROT>(g, a, L, inst, smem, lane);
}

}  // namespace b200pf

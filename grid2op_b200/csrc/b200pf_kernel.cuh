// b200pf_kernel.cuh — the fused per-instance power-flow kernel (sm_90a).
//
// One thread group (a warp for 5/14-substation grids, a CTA for 36/118-substation grids) owns one
// grid instance for the WHOLE solve; nothing but the inputs and the result record touches HBM:
//
//   topo_vect -> active buses -> bus types -> reachability -> DC angles (fp64 Gauss-Jordan)
//   -> Newton-Raphson { S(V) and |F|inf in fp64 ; Jacobian in fp32 ; Gauss-Jordan with partial
//      pivoting in shared memory ; fp64 state update }  -> branch flows / unit P,Q / voltages.
//
// What it replaces: pandapower's pd2ppc + makeYbus + dcpf + newtonpf + pfsoln + result tables as
// called from grid2op/Backend/pandaPowerBackend.py:1090 / 1097-1105 and read back at :1122-1218.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef B200PF_MIN_WARP_CTAS
#define B200PF_MIN_WARP_CTAS 28   // register budget: 65536 / (28 * 32) = 73 per thread
#endif

namespace b200pf {

struct DevGrid {
    int n_sub, n_busbar, n_slot, n_line, n_gen, n_hidden, n_unit, n_load, n_sto, n_shunt, dim_topo;
    int n_topo_in, n_inj, n_out;
    double base_mva;
    const int *line_or_sub, *line_ex_sub, *line_or_pos, *line_ex_pos;
    const double *line_y, *line_bdc, *line_pshift;
    const float *line_or_vn, *line_ex_vn;
    const int *unit_sub, *unit_pos, *unit_is_ref;
    const double *unit_qmin, *unit_qmax;
    const float *unit_vn;
    const int *load_sub, *load_pos;
    const float *load_vn;
    const int *sto_sub, *sto_pos;
    const float *sto_vn;
    const double *sto_q;
    const int *sh_sub;
    const float *sh_vn;
    const double *sh_vratio;
    const int *sub_rank;      // [n_sub] position of a substation in the bandwidth-reducing (RCM) order
    const int *sub_order;     // [n_sub] inverse permutation
    const int *sub_end_ptr;   // [n_sub+1]  static incidence: line ends per substation
    const int *sub_end;       // [2 n_line] code = line*2 + side (0 = origin, 1 = extremity)
};

struct RunArgs {
    int batch;
    const int8_t *topo;
    const double *inj;
    int is_dc, max_iter;
    double tol_pu;
    int nb_cap;
    int mat_bytes;   // bytes of the per-instance matrix region
    float *out;
    int *status;
    int *iters;
    double *busv;
    // time-series mode
    int series;
    const float *chron;
    // protections / cascading failure (series mode; reference Backend.next_grid_state, backend.py:1433-1521)
    int prot, from_reset, max_pc;
    float hard_thr, soft_thr;
    int *pcount;            // [B][n_line] protection counters of the environment (in/out)
    int *ts_over;           // [B][n_line] consecutive time steps in overflow (in/out)
    int *disc;              // [B][n_line] out: cascade iteration at which the line was disconnected, else -1
    int *done;              // [B] in/out: 1 once an instance is game over
    int n1_lines;           // > 0: contingency mode, instance = (base state, outage line) pair, base = inst / n1_lines
    const float *rows;      // rows mode: float32 [batch][2 n_load + 2 n_gen] for this very step (overrides chron)
    int n_scen, n_rows;
    const int *scen;
    int *t;
    const double *static_inj;
    const float *th_lim;
    float *rho;
    // protections with the planned kernel: one launch per cascade round, the host re-plans the instances whose lines trip
    int casc;                // cascade round of this launch (0 = the step itself)
    const int *inst_list;    // instances of this launch (nullptr: 0 .. batch-1)
    int8_t *trip;            // [B][n_line] out: 1 = the line trips in this round
    int8_t *incdone;         // [B][n_line] in/out: the soft-overflow counter of the line was already incremented in this step
    int *n_flag;             // out: number of instances with at least one tripping line
    int *flag_list;          // out: those instances
    // safety net of the non-pivoting planned kernel (b200pf_redo.cuh): 1 = this launch re-solves, with partial pivoting,
    // the instances the planned kernel left as ST_DIV; the series row of such an instance was already advanced
    int redo;
    unsigned char *redo_mat;  // safety net on large grids: per-CTA matrix region in GLOBAL memory (an fp64 Jacobian of the 118-substation
    size_t redo_mat_stride;   // grid does not fit on chip; the path is rare, its speed does not matter), nullptr = shared memory
    int dbg_div_mod;         // test knob: > 0 makes the planned kernel give up (ST_DIV) on every instance with inst % mod == 0
};

enum { ST_OK = 0, ST_DIV = 1, ST_UNSUP = 2, ST_NOREF = 3, ST_LARGE = 4, ST_DONE = 5 };
enum { BT_PQ = 1, BT_PV = 2, BT_REF = 3 };

// ---------------------------------------------------------------------------------------------
// per-instance shared-memory workspace
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline size_t align16(size_t x) { return (x + 15) & ~size_t(15); }

struct WsLayout {
    size_t off_bus_d;    // 17 double arrays [nbc]
    size_t off_inj;      // double [n_inj]
    size_t off_x;        // float [2 nbc]
    size_t off_vf32;     // float [2 nbc]
    size_t off_short;    // shorts: cidx[n_slot] colth[nbc] colv[nbc] bsub[nbc] cntu[nbc] nrefu[nbc] rowbus[2nbc] used[2nbc] prow[2nbc] brf[n_line] brt[n_line]
    size_t off_byte;     // bytes: btype[nbc] reach[nbc] mark[n_slot]
    size_t off_red;      // reduction scratch (256 B) + pivot-row buffers of the register Gauss-Jordan (768 B)
    size_t off_mat;      // matrix region
    size_t total;
};

__host__ __device__ inline size_t ws_fixed_bytes(int nbc, int n_slot, int n_line, int n_inj) {
    size_t o = 0;
    o += align16(size_t(17) * nbc * 8);
    o += align16(size_t(n_inj) * 8);
    o += align16(size_t(2) * nbc * 4);
    o += align16(size_t(2) * nbc * 4);
    o += align16(size_t(n_slot + 7 * nbc + 6 * nbc + 2 * n_line) * 2);
    o += align16(size_t(2 * nbc + n_slot));
    o += 576;
    return o;
}

// matrix bytes needed for the worst case of nbc active buses
__host__ __device__ inline size_t ws_mat_worst(int nbc, int jt_size) {
    size_t d = size_t(2) * nbc;
    size_t ac = d * (d + 2) * jt_size;
    size_t dc = size_t(nbc) * (nbc + 2) * 8;
    return align16(ac > dc ? ac : dc);
}

__host__ __device__ inline WsLayout ws_layout(int nbc, int n_slot, int n_line, int n_inj, size_t mat_bytes) {
    WsLayout L;
    size_t o = 0;
    L.off_bus_d = o; o += align16(size_t(17) * nbc * 8);
    L.off_inj = o;   o += align16(size_t(n_inj) * 8);
    L.off_x = o;     o += align16(size_t(2) * nbc * 4);
    L.off_vf32 = o;  o += align16(size_t(2) * nbc * 4);
    L.off_short = o; o += align16(size_t(n_slot + 7 * nbc + 6 * nbc + 2 * n_line) * 2);
    L.off_byte = o;  o += align16(size_t(2 * nbc + n_slot));
    L.off_red = o;   o += 576;
    L.off_mat = o;
    o += align16(mat_bytes);
    L.total = o;
    return L;
}

struct Ws {
    double *vm, *va, *ve, *vf, *pspec, *qspec, *gsh, *bsh, *gii, *bii, *pcalc, *qcalc, *pd, *qd, *qmins, *qmaxs, *pnonref;
    double *inj;
    float *x, *ve32, *vf32;
    short *cidx, *colth, *colv, *bsub, *cntu, *nrefu, *dcol, *dbus, *rowbus, *used, *prow, *brf, *brt;
    unsigned char *btype, *reach, *mark;
    float *redf;
    int *redi;
    double *pivbuf;   // 2 x 36 scalars (float or double) for gj_warp_reg
    void *mat;
};

__device__ inline Ws ws_bind(unsigned char *base, int nbc, int n_slot, int n_line, int n_inj, size_t mat_bytes) {
    WsLayout L = ws_layout(nbc, n_slot, n_line, n_inj, mat_bytes);
    Ws w;
    double *d = reinterpret_cast<double *>(base + L.off_bus_d);
    w.vm = d; w.va = d + nbc; w.ve = d + 2 * nbc; w.vf = d + 3 * nbc; w.pspec = d + 4 * nbc; w.qspec = d + 5 * nbc;
    w.gsh = d + 6 * nbc; w.bsh = d + 7 * nbc; w.gii = d + 8 * nbc; w.bii = d + 9 * nbc; w.pcalc = d + 10 * nbc;
    w.qcalc = d + 11 * nbc; w.pd = d + 12 * nbc; w.qd = d + 13 * nbc; w.qmins = d + 14 * nbc; w.qmaxs = d + 15 * nbc;
    w.pnonref = d + 16 * nbc;
    w.inj = reinterpret_cast<double *>(base + L.off_inj);
    w.x = reinterpret_cast<float *>(base + L.off_x);
    w.ve32 = reinterpret_cast<float *>(base + L.off_vf32);
    w.vf32 = w.ve32 + nbc;
    short *s = reinterpret_cast<short *>(base + L.off_short);
    w.cidx = s; s += n_slot;
    w.colth = s; s += nbc; w.colv = s; s += nbc; w.bsub = s; s += nbc; w.cntu = s; s += nbc; w.nrefu = s; s += nbc;
    w.dcol = s; s += nbc; w.dbus = s; s += nbc;
    w.rowbus = s; s += 2 * nbc; w.used = s; s += 2 * nbc; w.prow = s; s += 2 * nbc;
    w.brf = s; s += n_line; w.brt = s; s += n_line;
    unsigned char *b = base + L.off_byte;
    w.btype = b; w.reach = b + nbc; w.mark = b + 2 * nbc;
    w.redf = reinterpret_cast<float *>(base + L.off_red);
    w.redi = reinterpret_cast<int *>(base + L.off_red + 128);
    w.pivbuf = reinterpret_cast<double *>(base + L.off_red + 256);
    w.mat = base + L.off_mat;
    return w;
}

// ---------------------------------------------------------------------------------------------
// group primitives: T == 32 -> one warp (shuffles, __syncwarp); T > 32 -> one CTA
// ---------------------------------------------------------------------------------------------
template <int T> __device__ __forceinline__ void gsync() {
    if (T == 32) __syncwarp(); else __syncthreads();
}

// any-of over the group
template <int T> __device__ __forceinline__ int gany(int pred, Ws &w) {
    if (T == 32) return __any_sync(0xffffffffu, pred);
    return __syncthreads_or(pred);
}

// max over the group of a non-negative double (returns to all)
template <int T> __device__ __forceinline__ double gmax(double v, Ws &w, int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (T == 32) return v;
    double *sc = reinterpret_cast<double *>(w.redf);   // 16 doubles available (128 B)
    __syncthreads();
    if ((tid & 31) == 0) sc[tid >> 5] = v;
    __syncthreads();
    double r = sc[0];
#pragma unroll
    for (int k = 1; k < T / 32; ++k) r = fmax(r, sc[k]);
    return r;
}

// argmax of (val,row) over the group; ties -> smaller row (deterministic)
template <int T> __device__ __forceinline__ void gargmax(float &val, int &row, Ws &w, int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, val, o);
        int orow = __shfl_xor_sync(0xffffffffu, row, o);
        if (ov > val || (ov == val && orow < row)) { val = ov; row = orow; }
    }
    if (T == 32) return;
    __syncthreads();
    if ((tid & 31) == 0) { w.redf[tid >> 5] = val; w.redi[tid >> 5] = row; }
    __syncthreads();
    float bv = w.redf[0];
    int br = w.redi[0];
#pragma unroll
    for (int k = 1; k < T / 32; ++k) {
        float ov = w.redf[k];
        int orow = w.redi[k];
        if (ov > bv || (ov == bv && orow < br)) { bv = ov; br = orow; }
    }
    val = bv; row = br;
}

// ---------------------------------------------------------------------------------------------
// Warp Gauss-Jordan with the matrix in REGISTERS (n <= DMAX <= 32): lane r owns row r (DMAX columns +
// right-hand side), everything statically unrolled so that column indices are register names.  Per
// elimination step: pivot = max |a[r][k]| over unused rows via one REDUX (IEEE bit pattern of a
// non-negative float is monotonic) + ballot; the pivot lane publishes its row tail to shared memory
// (STS.128), all lanes read it back as broadcast LDS.128 and do DMAX-k FFMAs.  Two alternating
// row buffers -> one __syncwarp per step.  `prow` : 2*(DMAX+4) scalars of per-warp scratch.
// ---------------------------------------------------------------------------------------------
template <int DMAX, typename S>
__device__ __forceinline__ bool gj_warp_reg(const S *M, int n, int pitch, S *xs, S *prow, int lane) {
    static_assert(DMAX % 4 == 0 && DMAX <= 32, "DMAX");
    constexpr int W = DMAX + 4;          // buffer stride (rhs lives at index DMAX)
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
        if (k >= n) break;                                   // warp-uniform
        const float mag = fabsf((float)a[k]);
        const unsigned bits = (used || !(mag == mag)) ? 0u : __float_as_uint(mag);
        const unsigned mx = __reduce_max_sync(0xffffffffu, bits);
        if (mx < 0x00800000u) return false;                  // below the smallest normal: singular / NaN
        const unsigned who = __ballot_sync(0xffffffffu, bits == mx && !used);
        const int p = __ffs(who) - 1;
        S *buf = prow + (k & 1) * W;
        if (lane == p) {
#pragma unroll
            for (int c = (k & ~3); c < DMAX + 1; ++c) buf[c] = a[c];
            used = true; mycol = k; pivval = a[k];
        }
        __syncwarp();
        const S piv = buf[k];
        S inv;
        if (sizeof(S) == 4) inv = (S)__frcp_rn((float)piv); else inv = S(1) / piv;
        const S m = (lane == p) ? S(0) : a[k] * inv;
#pragma unroll
        for (int c = k + 1; c < DMAX + 1; ++c) a[c] -= m * buf[c];
    }
    if (mycol >= 0) xs[mycol] = a[DMAX] / pivval;
    __syncwarp();
    return true;
}

// pick the smallest unrolled variant that holds n
template <typename S>
__device__ __forceinline__ bool gj_warp_dispatch(const S *M, int n, int pitch, S *xs, S *prow, int lane) {
    if (n <= 8) return gj_warp_reg<8, S>(M, n, pitch, xs, prow, lane);
    if (n <= 16) return gj_warp_reg<16, S>(M, n, pitch, xs, prow, lane);
    if (sizeof(S) == 8) return false;     // fp64 rows wider than 16 would blow the register budget (caller falls back)
    if (n <= 24) return gj_warp_reg<24, S>(M, n, pitch, xs, prow, lane);
    return gj_warp_reg<32, S>(M, n, pitch, xs, prow, lane);
}

// ---------------------------------------------------------------------------------------------
// dense Gauss-Jordan with partial (row) pivoting on the augmented matrix M[n][pitch] (column n =
// right-hand side), rows distributed over the group.  Solution -> xs[0..n).  false if singular.
// ---------------------------------------------------------------------------------------------
template <int T, typename S>
__device__ bool gauss_jordan(S *M, int n, int pitch, float *xs, Ws &w, int tid) {
    for (int r = tid; r < n; r += T) w.used[r] = -1;
    gsync<T>();
    for (int k = 0; k < n; ++k) {
        float best = -1.0f;
        int brow = 0x7fffffff;
        for (int r = tid; r < n; r += T) {
            if (w.used[r] < 0) {
                float a = fabsf((float)M[(size_t)r * pitch + k]);
                if (a > best || (a == best && r < brow)) { best = a; brow = r; }   // NaN never wins
            }
        }
        gargmax<T>(best, brow, w, tid);
        if (!(best > 1e-30f)) return false;
        const int p = brow;
        const S *Mp = M + (size_t)p * pitch;
        const S inv = S(1) / Mp[k];
        for (int r = tid; r < n; r += T) {
            if (r == p) continue;
            S *Mr = M + (size_t)r * pitch;
            const S m = Mr[k] * inv;
            if (m != S(0)) {
                for (int c = k + 1; c <= n; ++c) Mr[c] -= m * Mp[c];
            }
        }
        if (tid == 0) { w.used[p] = (short)k; w.prow[k] = (short)p; }
        gsync<T>();
    }
    for (int k = tid; k < n; k += T) {
        const S *Mp = M + (size_t)w.prow[k] * pitch;
        xs[k] = (float)(Mp[n] / Mp[k]);
    }
    gsync<T>();
    return true;
}

// double-precision solution vector variant (DC): xs as double
template <int T>
__device__ bool gauss_jordan_d(double *M, int n, int pitch, double *xs, Ws &w, int tid) {
    for (int r = tid; r < n; r += T) w.used[r] = -1;
    gsync<T>();
    for (int k = 0; k < n; ++k) {
        float best = -1.0f;
        int brow = 0x7fffffff;
        for (int r = tid; r < n; r += T) {
            if (w.used[r] < 0) {
                float a = (float)fabs(M[(size_t)r * pitch + k]);
                if (a > best || (a == best && r < brow)) { best = a; brow = r; }
            }
        }
        gargmax<T>(best, brow, w, tid);
        if (!(best > 1e-30f)) return false;
        const int p = brow;
        const double *Mp = M + (size_t)p * pitch;
        const double inv = 1.0 / Mp[k];
        for (int r = tid; r < n; r += T) {
            if (r == p) continue;
            double *Mr = M + (size_t)r * pitch;
            const double m = Mr[k] * inv;
            if (m != 0.0) {
                for (int c = k + 1; c <= n; ++c) Mr[c] -= m * Mp[c];
            }
        }
        if (tid == 0) { w.used[p] = (short)k; w.prow[k] = (short)p; }
        gsync<T>();
    }
    for (int k = tid; k < n; k += T) {
        const double *Mp = M + (size_t)w.prow[k] * pitch;
        xs[k] = Mp[n] / Mp[k];
    }
    gsync<T>();
    return true;
}

// ---------------------------------------------------------------------------------------------
// Band-limited LU with partial pivoting on the augmented matrix M[n][pitch] (dense storage, column n
// = right-hand side).  The matrix has half band width bw in the (RCM bus order, interleaved unknowns)
// numbering; rows are never moved: an explicit list of ACTIVE rows (rows that can still hold a non-zero
// in the current column: at most bw+1) replaces the sliding window of a swap-based band LU, and the
// fill stays within columns (k, k + 2 bw].  Work per step = (#active rows) x (2 bw + 1) instead of n x n.
// Warps own rows, lanes own columns (conflict-free shared-memory access).  Back substitution by warp 0.
// xv: work vector of n scalars of type S; xout: solution (may alias xv when the types match).
// ---------------------------------------------------------------------------------------------
template <int T, typename S, typename X>
__device__ bool band_lu_solve(S *M, int n, int pitch, int bw, S *xv, X *xout, Ws &w, int tid) {
    short *act = w.used;                                   // active row list (<= bw + 1 <= n entries)
    const int lane = tid & 31, wid = tid >> 5;
    constexpr int NW = T / 32;
    int *pinfo = w.redi + 20;                              // [0] pivot row, [1] its index in act, [2] status
    if (bw < 1) bw = 1;
    int na = min(n, bw + 1);
    for (int r = tid; r < na; r += T) act[r] = (short)r;
    gsync<T>();
    for (int k = 0; k < n; ++k) {
        // warp 0: pivot search among the active rows (one REDUX on the |a| bit patterns + ballot); the other
        // warps wait at the barrier.  Two barriers per elimination step in total.
        if (wid == 0) {
            float best = -1.0f;
            int bidx_l = 0;
            for (int t = lane; t < na; t += 32) {
                const float a = fabsf((float)M[(size_t)act[t] * pitch + k]);
                if (a > best) { best = a; bidx_l = t; }          // NaN never wins
            }
            const unsigned bits = best > 0.0f ? __float_as_uint(best) : 0u;
            const unsigned mx = __reduce_max_sync(0xffffffffu, bits);
            const unsigned who = __ballot_sync(0xffffffffu, bits == mx);
            const int src = __ffs(who) - 1;
            const int bidx_w = __shfl_sync(0xffffffffu, bidx_l, src);
            if (lane == 0) {
                pinfo[2] = (mx < 0x00800000u) ? 1 : 0;        // |pivot| below the smallest normal: singular / NaN
                pinfo[1] = bidx_w;
                pinfo[0] = act[bidx_w];
            }
        }
        gsync<T>();
        if (pinfo[2]) return false;
        const int bidx = pinfo[1];
        const int p = pinfo[0];
        const S *Mp = M + (size_t)p * pitch;
        const S inv = S(1) / Mp[k];
        const int c_last = min(n - 1, k + 2 * bw);          // fill never goes beyond k + 2 bw
        const int ncols = c_last - k;                        // columns k+1 .. c_last
        const int nchunk = (ncols + 1 + 31) >> 5;            // 32-column chunks per row (incl. the right-hand side)
        if (nchunk <= 4) {
            // warp = two rows per pass, lane = column within each of (up to) 4 chunks: all loads of a pass are
            // issued before the first dependent FFMA
            for (int t0 = wid; t0 < na; t0 += 2 * NW) {
                const int tA = t0, tB = t0 + NW;
                const bool vA = tA != bidx, vB = tB < na && tB != bidx;
                S *MrA = M + (size_t)act[tA] * pitch;
                S *MrB = M + (size_t)act[vB ? tB : tA] * pitch;
                const S mA = vA ? MrA[k] * inv : S(0), mB = vB ? MrB[k] * inv : S(0);
                if (mA == S(0) && mB == S(0)) continue;
                S pa[4], ra[4], rb[4];
                int cj[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int cc = j * 32 + lane;
                    cj[j] = (cc < ncols) ? k + 1 + cc : ((cc == ncols) ? n : -1);
                    if (cj[j] >= 0) { pa[j] = Mp[cj[j]]; ra[j] = MrA[cj[j]]; rb[j] = MrB[cj[j]]; }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (cj[j] >= 0) {
                        if (mA != S(0)) MrA[cj[j]] = ra[j] - mA * pa[j];
                        if (mB != S(0)) MrB[cj[j]] = rb[j] - mB * pa[j];
                    }
                }
            }
        } else {
            for (int task = wid; task < na * nchunk; task += NW) {   // warp = (row, chunk), lane = column
                const int t = task / nchunk, cc = (task - t * nchunk) * 32 + lane;
                if (t == bidx || cc > ncols) continue;
                S *Mr = M + (size_t)act[t] * pitch;
                const S m = Mr[k] * inv;
                if (m == S(0)) continue;
                const int c = (cc == ncols) ? n : k + 1 + cc;      // last item = right-hand side
                Mr[c] -= m * Mp[c];
            }
        }
        gsync<T>();
        // bookkeeping: the pivot row leaves the active set, the next row enters (one thread; the next
        // reader of act is warp 0 itself in the pivot search, the others pass a barrier first)
        if (tid == 0) {
            w.prow[k] = (short)p;
            act[bidx] = act[na - 1];
            if (k + bw + 1 < n) act[na - 1] = (short)(k + bw + 1);
        }
        if (!(k + bw + 1 < n)) --na;
        if (T == 32) __syncwarp();
    }
    gsync<T>();
    // back substitution, reverse pivot order
    if (wid == 0) {
        for (int k = n - 1; k >= 0; --k) {
            const S *Mp = M + (size_t)w.prow[k] * pitch;
            const int c_last = min(n - 1, k + 2 * bw);
            S s = S(0);
            for (int c = k + 1 + lane; c <= c_last; c += 32) s += Mp[c] * xv[c];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) xv[k] = (Mp[n] - s) / Mp[k];
            __syncwarp();
        }
    }
    gsync<T>();
    if ((void *)xout != (void *)xv) {
        for (int k = tid; k < n; k += T) xout[k] = (X)xv[k];
        gsync<T>();
    }
    return true;
}

__device__ __forceinline__ float qnanf() { return __int_as_float(0x7fc00000); }

// ---------------------------------------------------------------------------------------------
// the instance solver
// ---------------------------------------------------------------------------------------------
template <int T, typename JT>
__device__ void solve_instance(const DevGrid &g, const RunArgs &a, int inst, unsigned char *wsbase, int tid) {
    const int nbc = a.nb_cap;
    Ws w = ws_bind(wsbase, nbc, g.n_slot, g.n_line, g.n_inj, (size_t)a.mat_bytes);
    if (a.redo_mat) w.mat = a.redo_mat + (size_t)blockIdx.x * a.redo_mat_stride;
    const int src = a.n1_lines > 0 ? inst / a.n1_lines : inst;          // record the inputs come from
    const int outage = a.n1_lines > 0 ? inst % a.n1_lines : -1;         // line forced out of service (N-1 sweep)
    const int8_t *tv = a.topo + (size_t)src * g.n_topo_in;
    float *out = a.out ? a.out + (size_t)inst * g.n_out : nullptr;
    const double base = g.base_mva;
    const int nl = g.n_line;

    // ---- 0. stage the injection record -----------------------------------------------------
    if (a.series) {
        const int sc = a.rows ? 0 : a.scen[src];
        int trow = a.rows ? 0 : a.t[src];
        if (a.redo && !a.rows) trow = trow == 0 ? a.n_rows - 1 : trow - 1;     // the planned kernel advanced the row already
        const float *row = a.rows ? a.rows + (size_t)src * (size_t)(2 * g.n_load + 2 * g.n_gen)
                                  : a.chron + ((size_t)sc * a.n_rows + trow) * (size_t)(2 * g.n_load + 2 * g.n_gen);
        for (int k = tid; k < g.n_inj; k += T) w.inj[k] = a.static_inj[k];
        gsync<T>();
        for (int k = tid; k < g.n_load; k += T) {
            w.inj[g.n_gen + g.n_unit + k] = (double)row[k];
            w.inj[g.n_gen + g.n_unit + g.n_load + k] = (double)row[g.n_load + k];
        }
        for (int k = tid; k < g.n_gen; k += T) {
            w.inj[k] = (double)row[2 * g.n_load + k];
            // set point in p.u.: float32 / float32 like the reference (pandaPowerBackend.py:927)
            w.inj[g.n_gen + g.n_hidden + k] = (double)__fdiv_rn(row[2 * g.n_load + g.n_gen + k], g.unit_vn[g.n_hidden + k]);
        }
        gsync<T>();
        if (tid == 0 && !a.rows && a.n1_lines <= 0 && !a.redo) a.t[inst] = (trow + 1 >= a.n_rows) ? 0 : trow + 1;
    } else {
        const double *srcp = a.inj + (size_t)src * g.n_inj;
        for (int k = tid; k < g.n_inj; k += T) w.inj[k] = srcp[k];
    }
    const double *gen_p = w.inj;
    const double *unit_vm = w.inj + g.n_gen;
    const double *load_p = unit_vm + g.n_unit;
    const double *load_q = load_p + g.n_load;
    const double *sto_p = load_q + g.n_load;
    const double *sh_p = sto_p + g.n_sto;
    const double *sh_q = sh_p + g.n_shunt;

    // ---- 1. active bus slots and their compact numbering -----------------------------------
    for (int s = tid; s < g.n_slot; s += T) w.mark[s] = 0;
    gsync<T>();
    for (int l = tid; l < nl; l += T) {
        if (l == outage) continue;
        const int bo = tv[g.line_or_pos[l]], be = tv[g.line_ex_pos[l]];
        if (bo > 0) w.mark[g.sub_rank[g.line_or_sub[l]] * g.n_busbar + (bo - 1)] = 1;
        if (be > 0) w.mark[g.sub_rank[g.line_ex_sub[l]] * g.n_busbar + (be - 1)] = 1;
    }
    for (int u = tid; u < g.n_unit; u += T) {
        const int b = tv[g.unit_pos[u]];
        if (b > 0) w.mark[g.sub_rank[g.unit_sub[u]] * g.n_busbar + (b - 1)] = 1;
    }
    for (int k = tid; k < g.n_load; k += T) {
        const int b = tv[g.load_pos[k]];
        if (b > 0) w.mark[g.sub_rank[g.load_sub[k]] * g.n_busbar + (b - 1)] = 1;
    }
    for (int k = tid; k < g.n_sto; k += T) {
        const int b = tv[g.sto_pos[k]];
        if (b > 0) w.mark[g.sub_rank[g.sto_sub[k]] * g.n_busbar + (b - 1)] = 1;
    }
    for (int k = tid; k < g.n_shunt; k += T) {
        const int b = tv[g.dim_topo + k];
        if (b > 0) w.mark[g.sub_rank[g.sh_sub[k]] * g.n_busbar + (b - 1)] = 1;
    }
    gsync<T>();
    int nb = 0;
    if (tid < 32) {   // ordered compaction by the first warp
        for (int s0 = 0; s0 < g.n_slot; s0 += 32) {
            const int s = s0 + tid;
            const int on = (s < g.n_slot) ? (int)w.mark[s] : 0;
            const unsigned m = __ballot_sync(0xffffffffu, on);
            if (s < g.n_slot) {
                const int ci = nb + __popc(m & ((1u << tid) - 1u));
                w.cidx[s] = on ? (short)ci : (short)-1;
                if (on && ci < nbc) w.bsub[ci] = (short)g.sub_order[s / g.n_busbar];
            }
            nb += __popc(m);
        }
        if (tid == 0) w.redi[16] = nb;
    }
    gsync<T>();
    nb = w.redi[16];
    int status = ST_OK;
    if (nb > nbc) status = ST_LARGE;

    int n1 = 0, npq = 0, d = 0, iters = 0, bw_dc = 0, bw_ac = 1;
    if (status == ST_OK) {
        // ---- 2. per-bus initialisation ------------------------------------------------------
        for (int i = tid; i < nb; i += T) {
            w.btype[i] = BT_PQ; w.reach[i] = 0; w.vm[i] = 1.0; w.va[i] = 0.0;
            w.pspec[i] = 0.0; w.qspec[i] = 0.0; w.gsh[i] = 0.0; w.bsh[i] = 0.0;
            w.pd[i] = 0.0; w.qd[i] = 0.0; w.qmins[i] = 0.0; w.qmaxs[i] = 0.0; w.pnonref[i] = 0.0;
            w.cntu[i] = 0; w.nrefu[i] = 0;
        }
        gsync<T>();
        // serial accumulation in table order: deterministic, and "the later unit wins" for the
        // voltage set point exactly like the ppc generator table (pandapower build_gen)
        if (tid == 0) {
            for (int u = 0; u < g.n_unit; ++u) {
                const int b = tv[g.unit_pos[u]];
                if (b <= 0) continue;
                const int i = w.cidx[g.sub_rank[g.unit_sub[u]] * g.n_busbar + (b - 1)];
                const double pu = (u >= g.n_hidden) ? gen_p[u - g.n_hidden] : 0.0;
                w.vm[i] = unit_vm[u];
                w.cntu[i] += 1;
                w.qmins[i] += g.unit_qmin[u];
                w.qmaxs[i] += g.unit_qmax[u];
                if (g.unit_is_ref[u]) { w.btype[i] = BT_REF; w.nrefu[i] += 1; }
                else { if (w.btype[i] != BT_REF) w.btype[i] = BT_PV; w.pnonref[i] += pu; }
                w.pspec[i] += pu;
            }
        } else if (tid == 1) {
            for (int k = 0; k < g.n_load; ++k) {
                const int b = tv[g.load_pos[k]];
                if (b <= 0) continue;
                const int i = w.cidx[g.sub_rank[g.load_sub[k]] * g.n_busbar + (b - 1)];
                w.pd[i] += load_p[k]; w.qd[i] += load_q[k];
            }
            for (int k = 0; k < g.n_sto; ++k) {
                const int b = tv[g.sto_pos[k]];
                if (b <= 0) continue;
                const int i = w.cidx[g.sub_rank[g.sto_sub[k]] * g.n_busbar + (b - 1)];
                w.pd[i] += sto_p[k]; w.qd[i] += g.sto_q[k];
            }
        } else if (tid == 2) {
            for (int k = 0; k < g.n_shunt; ++k) {
                const int b = tv[g.dim_topo + k];
                if (b <= 0) continue;
                const int i = w.cidx[g.sub_rank[g.sh_sub[k]] * g.n_busbar + (b - 1)];
                w.gsh[i] += sh_p[k] * g.sh_vratio[k];
                w.bsh[i] -= sh_q[k] * g.sh_vratio[k];
            }
        }
        // branches -> compact end buses
        for (int l = tid; l < nl; l += T) {
            const int bo = tv[g.line_or_pos[l]], be = tv[g.line_ex_pos[l]];
            if (bo > 0 && be > 0 && l != outage) {
                w.brf[l] = w.cidx[g.sub_rank[g.line_or_sub[l]] * g.n_busbar + (bo - 1)];
                w.brt[l] = w.cidx[g.sub_rank[g.line_ex_sub[l]] * g.n_busbar + (be - 1)];
            } else { w.brf[l] = -1; w.brt[l] = -1; }
        }
        gsync<T>();
        // ---- 3. reachability from the reference buses ---------------------------------------
        int anyref = 0;
        for (int i = tid; i < nb; i += T) if (w.btype[i] == BT_REF) { w.reach[i] = 1; anyref = 1; }
        anyref = gany<T>(anyref, w);
        if (!anyref) status = ST_NOREF;
        else {
            for (int sweep = 0; sweep < nb; ++sweep) {
                int ch = 0;
                for (int l = tid; l < nl; l += T) {
                    const int f = w.brf[l];
                    if (f < 0) continue;
                    const int t = w.brt[l];
                    const int rf = w.reach[f], rt = w.reach[t];
                    if (rf != rt) { w.reach[f] = 1; w.reach[t] = 1; ch = 1; }
                }
                gsync<T>();
                if (!gany<T>(ch, w)) break;
            }
            int bad = 0;
            for (int i = tid; i < nb; i += T) if (!w.reach[i]) bad = 1;
            if (gany<T>(bad, w)) status = ST_UNSUP;
        }
    }

    if (status == ST_OK) {
        // ---- 4. unknown numbering, bus by bus in the (RCM-ordered) bus order: Newton system interleaved
        //         [theta_i, |V|_i] so that the Jacobian is banded; the DC system numbers the non-ref buses
        if (tid == 0) {
            int c = 0, c1 = 0;
            for (int i = 0; i < nb; ++i) {
                if (w.btype[i] != BT_REF) {
                    w.dcol[i] = (short)c1; w.dbus[c1] = (short)i; ++c1;
                    w.colth[i] = (short)c; w.rowbus[c] = (short)i; ++c;
                    if (w.btype[i] == BT_PQ) { w.colv[i] = (short)c; w.rowbus[c] = (short)i; ++c; } else w.colv[i] = -1;
                } else { w.dcol[i] = -1; w.colth[i] = -1; w.colv[i] = -1; }
            }
            w.redi[17] = c1; w.redi[18] = c;
        }
        // specified injections (p.u.) and diagonal of Ybus
        for (int i = tid; i < nb; i += T) {
            w.pspec[i] = (w.pspec[i] - w.pd[i]) / base;
            w.qspec[i] = -w.qd[i] / base;
            double gs = w.gsh[i] / base, bs = w.bsh[i] / base;
            const int s = w.bsub[i];
            for (int e = g.sub_end_ptr[s]; e < g.sub_end_ptr[s + 1]; ++e) {
                const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                if (w.brf[l] < 0) continue;
                if ((side ? w.brt[l] : w.brf[l]) != i) continue;
                const double *y = g.line_y + (size_t)l * 8 + (side ? 6 : 0);
                gs += y[0]; bs += y[1];
            }
            w.gii[i] = gs; w.bii[i] = bs;
        }
        gsync<T>();
        n1 = w.redi[17]; d = w.redi[18]; npq = d - n1;
        {   // half band widths of the DC matrix and of the Jacobian (max over in-service lines)
            int b1 = 0, b2 = 1;
            for (int l = tid; l < nl; l += T) {
                const int f = w.brf[l];
                if (f < 0) continue;
                const int t = w.brt[l];
                if (w.dcol[f] >= 0 && w.dcol[t] >= 0) {
                    const int a1 = abs(w.dcol[f] - w.dcol[t]), a2 = abs(w.colth[f] - w.colth[t]) + 1;
                    b1 = max(b1, a1); b2 = max(b2, a2);
                }
            }
            bw_dc = (int)gmax<T>((double)b1, w, tid);
            bw_ac = (int)gmax<T>((double)b2, w, tid);
        }
        if ((size_t)n1 * ((n1 + 1) | 1) * 8 > (size_t)a.mat_bytes ||
            (!a.is_dc && (size_t)d * ((d + 1) | 1) * sizeof(JT) > (size_t)a.mat_bytes)) status = ST_LARGE;
    }
    if (status == ST_OK) {

        // ---- 5. DC angles (init="dc", and the DC mode itself) ---------------------------------
        {
            double *M = reinterpret_cast<double *>(w.mat);
            const int pitch = (n1 + 1) | 1;
            for (int r = tid; r < n1; r += T) {
                const int i = w.dbus[r];
                double *Mr = M + (size_t)r * pitch;
                for (int c = 0; c <= n1; ++c) Mr[c] = 0.0;
                double rhs = w.pspec[i] - w.gsh[i] / base;
                const int s = w.bsub[i];
                for (int e = g.sub_end_ptr[s]; e < g.sub_end_ptr[s + 1]; ++e) {
                    const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                    if (w.brf[l] < 0) continue;
                    if ((side ? w.brt[l] : w.brf[l]) != i) continue;
                    const int j = side ? w.brf[l] : w.brt[l];
                    const double b = g.line_bdc[l];
                    Mr[r] += b;
                    if (w.dcol[j] >= 0) Mr[w.dcol[j]] -= b;        // reference angle is 0 (pPB:473)
                    rhs -= side ? -g.line_pshift[l] : g.line_pshift[l];
                }
                Mr[n1] = rhs;
            }
            gsync<T>();
            double *th = w.pcalc;   // scratch
            bool ok;
            if (T == 32 && n1 <= 16) ok = gj_warp_dispatch<double>(M, n1, pitch, th, w.pivbuf, tid);
            else ok = band_lu_solve<T, double, double>(M, n1, pitch, bw_dc, th, th, w, tid);
            if (!ok) status = ST_DIV;
            else {
                for (int r = tid; r < n1; r += T) w.va[w.dbus[r]] = th[r];
                gsync<T>();
                int bad = 0;
                for (int i = tid; i < nb; i += T) if (!isfinite(w.va[i])) bad = 1;
                if (gany<T>(bad, w)) status = ST_DIV;
            }
        }
    }

    if (status == ST_OK && !a.is_dc) {
        // ---- 6. Newton-Raphson -----------------------------------------------------------------
        for (int i = tid; i < nb; i += T) {
            double s, c;
            sincos(w.va[i], &s, &c);
            w.ve[i] = w.vm[i] * c; w.vf[i] = w.vm[i] * s;
            w.ve32[i] = (float)w.ve[i]; w.vf32[i] = (float)w.vf[i];
        }
        gsync<T>();
        JT *J = reinterpret_cast<JT *>(w.mat);
        const int pitch = (d + 1) | 1;
        bool conv = false;
        for (int it = 0;; ++it) {
            // (a) S(V) and the mismatch norm, fp64, one thread per bus
            double fmx = 0.0;
            for (int i = tid; i < nb; i += T) {
                const double ei = w.ve[i], fi = w.vf[i];
                double ir = w.gii[i] * ei - w.bii[i] * fi;
                double ii = w.gii[i] * fi + w.bii[i] * ei;
                const int s = w.bsub[i];
                for (int e = g.sub_end_ptr[s]; e < g.sub_end_ptr[s + 1]; ++e) {
                    const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                    if (w.brf[l] < 0) continue;
                    if ((side ? w.brt[l] : w.brf[l]) != i) continue;
                    const int j = side ? w.brf[l] : w.brt[l];
                    const double *y = g.line_y + (size_t)l * 8 + (side ? 4 : 2);
                    const double ej = w.ve[j], fj = w.vf[j];
                    ir += y[0] * ej - y[1] * fj;
                    ii += y[0] * fj + y[1] * ej;
                }
                const double P = ei * ir + fi * ii;
                const double Q = fi * ir - ei * ii;
                w.pcalc[i] = P; w.qcalc[i] = Q;
                const int bt = w.btype[i];
                if (bt != BT_REF) {
                    double m = fabs(P - w.pspec[i]);
                    if (!(m == m)) m = 1e300;
                    fmx = fmax(fmx, m);
                    if (bt == BT_PQ) {
                        double mq = fabs(Q - w.qspec[i]);
                        if (!(mq == mq)) mq = 1e300;
                        fmx = fmax(fmx, mq);
                    }
                }
            }
            fmx = gmax<T>(fmx, w, tid);
            if (fmx < a.tol_pu) { conv = true; iters = it; break; }
            if (it >= a.max_iter || !(fmx < 1e200)) { iters = it; break; }
            gsync<T>();
            // (b) Jacobian rows in the solver's precision, one thread per row
            for (int r = tid; r < d; r += T) {
                const int i = w.rowbus[r];
                const bool isq = (r == w.colv[i]);
                JT *Jr = J + (size_t)r * pitch;
                for (int c = 0; c < d; ++c) Jr[c] = JT(0);
                const JT ei = (JT)w.ve32[i], fi = (JT)w.vf32[i];
                const JT vi2 = ei * ei + fi * fi;
                const JT P = (JT)w.pcalc[i], Q = (JT)w.qcalc[i];
                const JT gi = (JT)w.gii[i], bi = (JT)w.bii[i];
                if (!isq) {
                    Jr[w.colth[i]] = -Q - bi * vi2;
                    if (w.colv[i] >= 0) Jr[w.colv[i]] = P + gi * vi2;
                    Jr[d] = (JT)(w.pspec[i] - w.pcalc[i]);
                } else {
                    Jr[w.colth[i]] = P - gi * vi2;
                    Jr[w.colv[i]] = Q - bi * vi2;
                    Jr[d] = (JT)(w.qspec[i] - w.qcalc[i]);
                }
                const int s = w.bsub[i];
                for (int e = g.sub_end_ptr[s]; e < g.sub_end_ptr[s + 1]; ++e) {
                    const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                    if (w.brf[l] < 0) continue;
                    if ((side ? w.brt[l] : w.brf[l]) != i) continue;
                    const int j = side ? w.brf[l] : w.brt[l];
                    const double *y = g.line_y + (size_t)l * 8 + (side ? 4 : 2);
                    const JT yr = (JT)y[0], yi = (JT)y[1];
                    const JT ej = (JT)w.ve32[j], fj = (JT)w.vf32[j];
                    const JT ar = yr * ej - yi * fj, ai = yr * fj + yi * ej;     // Y_ij V_j
                    const JT tr = ei * ar + fi * ai, ti = fi * ar - ei * ai;     // V_i conj(Y_ij V_j)
                    const int cth = w.colth[j], cv = w.colv[j];
                    if (!isq) { if (cth >= 0) Jr[cth] += ti; if (cv >= 0) Jr[cv] += tr; }
                    else      { if (cth >= 0) Jr[cth] -= tr; if (cv >= 0) Jr[cv] += ti; }
                }
            }
            gsync<T>();
            // (c) solve J dx = -F
            bool solved;
            if (T == 32 && d <= 32 && sizeof(JT) == 4)
                solved = gj_warp_dispatch<float>(reinterpret_cast<float *>(J), d, pitch, w.x, reinterpret_cast<float *>(w.pivbuf), tid);
            else {
                JT *xv = (sizeof(JT) == 4) ? reinterpret_cast<JT *>(w.x) : reinterpret_cast<JT *>(w.pcalc);   // work vector (2 nbc)
                solved = band_lu_solve<T, JT, float>(J, d, pitch, bw_ac, xv, w.x, w, tid);
            }
            if (!solved) { iters = it + 1; break; }
            // (d) fp64 state update; |V| unknown is relative (dV/V)
            for (int i = tid; i < nb; i += T) {
                double vm = w.vm[i], va = w.va[i];
                if (w.colth[i] >= 0) va += (double)w.x[w.colth[i]];
                if (w.colv[i] >= 0) vm *= 1.0 + (double)w.x[w.colv[i]];
                if (vm < 0.0) { vm = -vm; va += 3.14159265358979323846; }
                double s, c;
                sincos(va, &s, &c);
                w.vm[i] = vm; w.va[i] = va;
                w.ve[i] = vm * c; w.vf[i] = vm * s;
                w.ve32[i] = (float)w.ve[i]; w.vf32[i] = (float)w.vf[i];
            }
            gsync<T>();
        }
        if (!conv) status = ST_DIV;
    }

    // ---- 7. results ----------------------------------------------------------------------------
    if (a.redo && status == ST_LARGE) status = ST_DIV;      // the safety net could not hold the system: the first verdict stands
    if (tid == 0) { a.status[inst] = status; a.iters[inst] = iters; }
    if (status != ST_OK) {
        if (out) for (int k = tid; k < g.n_out; k += T) out[k] = qnanf();
        if (a.busv) for (int k = tid; k < 2 * g.n_slot; k += T) a.busv[(size_t)inst * 2 * g.n_slot + k] = __longlong_as_double(0x7ff8000000000000LL);
        if (a.rho) for (int k = tid; k < nl; k += T) a.rho[(size_t)inst * nl + k] = qnanf();
        gsync<T>();
        return;
    }
    const double RAD2DEG = 57.295779513082320877;
    const double SQRT3 = 1.7320508075688772935;
    if (!a.is_dc) {        // pandapower reports Va = angle(V), i.e. angles in (-180, 180]
        for (int i = tid; i < nb; i += T) { const double x = w.va[i]; w.va[i] = x - 6.283185307179586477 * rint(x * 0.15915494309189533577); }
        gsync<T>();
    }
    if (a.is_dc) {
        // DC: injections at every bus from the angles (needed for the slack share)
        for (int i = tid; i < nb; i += T) {
            double p = w.gsh[i] / base;
            const int s = w.bsub[i];
            for (int e = g.sub_end_ptr[s]; e < g.sub_end_ptr[s + 1]; ++e) {
                const int code = g.sub_end[e], l = code >> 1, side = code & 1;
                if (w.brf[l] < 0) continue;
                if ((side ? w.brt[l] : w.brf[l]) != i) continue;
                const int j = side ? w.brf[l] : w.brt[l];
                p += g.line_bdc[l] * (w.va[i] - w.va[j]) + (side ? -g.line_pshift[l] : g.line_pshift[l]);
            }
            w.pcalc[i] = p; w.qcalc[i] = 0.0;
        }
        gsync<T>();
    }
    float *const outw = out;
    float *o_p_or = out, *o_q_or = out + nl, *o_v_or = out + 2 * nl, *o_a_or = out + 3 * nl, *o_t_or = out + 4 * nl;
    float *o_p_ex = out + 5 * nl, *o_q_ex = out + 6 * nl, *o_v_ex = out + 7 * nl, *o_a_ex = out + 8 * nl, *o_t_ex = out + 9 * nl;
    for (int l = tid; l < nl; l += T) {
        const int f = w.brf[l];
        float p1 = 0.f, q1 = 0.f, v1 = 0.f, a1 = 0.f, t1 = 0.f, p2 = 0.f, q2 = 0.f, v2 = 0.f, a2 = 0.f, t2 = 0.f;
        if (f >= 0) {
            const int t = w.brt[l];
            double pf, qf, pt, qt, sf, st;
            if (a.is_dc) {
                pf = (g.line_bdc[l] * (w.va[f] - w.va[t]) + g.line_pshift[l]) * base;
                pt = -pf; qf = 0.0; qt = 0.0; sf = fabs(pf); st = fabs(pt);
            } else {
                const double *y = g.line_y + (size_t)l * 8;
                const double ef = w.ve[f], ff = w.vf[f], et = w.ve[t], ft = w.vf[t];
                const double ifr = y[0] * ef - y[1] * ff + y[2] * et - y[3] * ft;
                const double ifi = y[0] * ff + y[1] * ef + y[2] * ft + y[3] * et;
                const double itr = y[4] * ef - y[5] * ff + y[6] * et - y[7] * ft;
                const double iti = y[4] * ff + y[5] * ef + y[6] * ft + y[7] * et;
                pf = (ef * ifr + ff * ifi) * base; qf = (ff * ifr - ef * ifi) * base;
                pt = (et * itr + ft * iti) * base; qt = (ft * itr - et * iti) * base;
                sf = sqrt(pf * pf + qf * qf); st = sqrt(pt * pt + qt * qt);
            }
            const double vmf = w.vm[f], vmt = w.vm[t];
            const double ika_f = sf / (SQRT3 * (vmf * (double)g.line_or_vn[l]));
            const double ika_t = st / (SQRT3 * (vmt * (double)g.line_ex_vn[l]));
            p1 = (float)pf; q1 = (float)qf; p2 = (float)pt; q2 = (float)qt;
            a1 = (float)(ika_f * 1000.0); a2 = (float)(ika_t * 1000.0);
            if (!isfinite(a1)) a1 = 0.f;
            if (!isfinite(a2)) a2 = 0.f;
            v1 = __fmul_rn((float)vmf, g.line_or_vn[l]); v2 = __fmul_rn((float)vmt, g.line_ex_vn[l]);
            t1 = (float)(w.va[f] * RAD2DEG); t2 = (float)(w.va[t] * RAD2DEG);
        }
        if (outw) {
            o_p_or[l] = p1; o_q_or[l] = q1; o_v_or[l] = v1; o_a_or[l] = a1; o_t_or[l] = t1;
            o_p_ex[l] = p2; o_q_ex[l] = q2; o_v_ex[l] = v2; o_a_ex[l] = a2; o_t_ex[l] = t2;
        }
        if (a.rho) a.rho[(size_t)inst * nl + l] = a1 / a.th_lim[l];
    }
    float *o_up = out + 10 * nl, *o_uq = o_up + g.n_unit, *o_uv = o_uq + g.n_unit, *o_ut = o_uv + g.n_unit;
    for (int u = tid; u < (outw ? g.n_unit : 0); u += T) {
        const int b = tv[g.unit_pos[u]];
        float p = 0.f, q = 0.f, v = 0.f, th = 0.f;
        if (b > 0) {
            const int i = w.cidx[g.sub_rank[g.unit_sub[u]] * g.n_busbar + (b - 1)];
            double pu = (u >= g.n_hidden) ? gen_p[u - g.n_hidden] : 0.0;
            if (g.unit_is_ref[u]) {
                // slack power of the bus shared equally by its reference units (pandapower pfsoln)
                pu = (w.pcalc[i] * base + w.pd[i] - w.pnonref[i]) / (double)w.nrefu[i];
            }
            double qu = 0.0;
            if (!a.is_dc) {
                const double qtot = w.qcalc[i] * base + w.qd[i];
                if (w.cntu[i] <= 1 || w.qmins[i] == w.qmaxs[i]) qu = qtot / (double)w.cntu[i];
                else qu = g.unit_qmin[u] + (qtot - w.qmins[i]) / (w.qmaxs[i] - w.qmins[i] + 2.220446049250313e-16) * (g.unit_qmax[u] - g.unit_qmin[u]);
            }
            p = (float)pu; q = (float)qu;
            v = __fmul_rn((float)w.vm[i], g.unit_vn[u]);
            th = (float)(w.va[i] * RAD2DEG);
        }
        o_up[u] = p; o_uq[u] = q; o_uv[u] = v; o_ut[u] = th;
    }
    float *o_lv = o_ut + g.n_unit, *o_lt = o_lv + g.n_load;
    for (int k = tid; k < (outw ? g.n_load : 0); k += T) {
        const int b = tv[g.load_pos[k]];
        float v = 0.f, th = 0.f;
        if (b > 0) {
            const int i = w.cidx[g.sub_rank[g.load_sub[k]] * g.n_busbar + (b - 1)];
            v = __fmul_rn((float)w.vm[i], g.load_vn[k]);
            th = (float)(w.va[i] * RAD2DEG);
        }
        o_lv[k] = v; o_lt[k] = th;
    }
    float *o_sv = o_lt + g.n_load;
    for (int k = tid; k < (outw ? g.n_sto : 0); k += T) {
        const int b = tv[g.sto_pos[k]];
        float v = 0.f;
        if (b > 0) v = __fmul_rn((float)w.vm[w.cidx[g.sub_rank[g.sto_sub[k]] * g.n_busbar + (b - 1)]], g.sto_vn[k]);
        o_sv[k] = v;
    }
    float *o_shp = o_sv + g.n_sto, *o_shq = o_shp + g.n_shunt, *o_shv = o_shq + g.n_shunt;
    for (int k = tid; k < (outw ? g.n_shunt : 0); k += T) {
        const int b = tv[g.dim_topo + k];
        float p = 0.f, q = 0.f, v = 0.f;
        if (b > 0) {
            const int i = w.cidx[g.sub_rank[g.sh_sub[k]] * g.n_busbar + (b - 1)];
            const double v2 = a.is_dc ? 1.0 : w.vm[i] * w.vm[i];
            p = (float)(sh_p[k] * g.sh_vratio[k] * v2);
            q = a.is_dc ? 0.f : (float)(sh_q[k] * g.sh_vratio[k] * v2);
            v = __fmul_rn((float)w.vm[i], g.sh_vn[k]);
        }
        o_shp[k] = p; o_shq[k] = q; o_shv[k] = v;
    }
    if (a.busv) {
        double *bv = a.busv + (size_t)inst * 2 * g.n_slot;
        for (int s = tid; s < g.n_slot; s += T) {
            const int i = w.cidx[g.sub_rank[s % g.n_sub] * g.n_busbar + s / g.n_sub];      // slot = sub + (busbar-1)*n_sub
            bv[s] = (i >= 0) ? w.vm[i] : __longlong_as_double(0x7ff8000000000000LL);
            bv[g.n_slot + s] = (i >= 0) ? w.va[i] : __longlong_as_double(0x7ff8000000000000LL);
        }
    }
    gsync<T>();
}

// persistent kernel: each group (warp / CTA) strides over the instances of the batch
template <int T, typename JT>
__global__ void __launch_bounds__(T, (T == 32) ? B200PF_MIN_WARP_CTAS : 1)
pf_kernel(const DevGrid g, const RunArgs a, const int ws_bytes) {
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr int BLOCK = T;                // one group per CTA (a warp-CTA for the small grids: finest SM balance)
    constexpr int GPB = 1;
    const int gid = threadIdx.x / T;
    const int tid = threadIdx.x % T;
    unsigned char *wsbase = smem + (size_t)gid * ws_bytes;
    for (int inst = blockIdx.x * GPB + gid; inst < a.batch; inst += gridDim.x * GPB) {
        solve_instance<T, JT>(g, a, inst, wsbase, tid);
    }
}

}  // namespace b200pf

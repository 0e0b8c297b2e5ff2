// b200pf_plan.hpp — host-side "topology plan" of the sparse kernel (b200pf_sparse.cuh).
//
// Everything of a power flow that depends on the TOPOLOGY only (reference: what pandapower's pd2ppc does on
// every runpp call, grid2op/Backend/pandaPowerBackend.py:1097-1105 — bus fusion, bus types, connectivity
// check, Ybus / Bdc structure — plus what a sparse direct solver's symbolic phase does) is computed ONCE per
// distinct topology vector on the host and cached:
//   * active buses, bus types, reachability from the reference buses -> static status of the class
//   * per-bus element lists (units, loads, storages, shunts, line ends) in element order (deterministic sums)
//   * a minimum-degree elimination order of the non-reference buses, unknowns (theta_i, |V|_i) interleaved
//   * the filled pattern of the Newton Jacobian in that order, positions of every entry in a packed value
//     array, the positions each line / bus writes at assembly time
//   * the numeric factorisation as a list of passes of independent multiply-subtract operations
//     A[ij] -= A[ik] * A[kj] / A[kk]  (right-looking LU without pivoting, right-hand side carried along)
//     and the level schedule of the back substitution
//   * the DC matrix Bdc of the topology, INVERTED here in fp64 (it only depends on the topology): the DC start of
//     every Newton solve, and the DC power flow itself, is one matrix-vector product on the device.
// The device kernel is then a numeric interpreter of the plan: one warp (or CTA) per instance, all values in
// shared memory.  Instances that share a topology share a plan; a launch may mix plans freely.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#ifdef B200PF_PLAN_PROFILE
#include <chrono>
#include <map>
#include <string>
namespace b200pf { inline std::map<std::string, double> &plan_prof() { static std::map<std::string, double> m; return m; }
inline std::chrono::steady_clock::time_point &plan_prof_t() { static std::chrono::steady_clock::time_point t; return t; } }
#define PLAN_TICK(name) { auto now_ = std::chrono::steady_clock::now(); b200pf::plan_prof()[name] += std::chrono::duration<double>(now_ - b200pf::plan_prof_t()).count(); b200pf::plan_prof_t() = now_; }
#define PLAN_TICK0() { b200pf::plan_prof_t() = std::chrono::steady_clock::now(); }
#else
#define PLAN_TICK(name)
#define PLAN_TICK0()
#endif

namespace b200pf {

struct HostGrid {
    int n_sub = 0, n_busbar = 0, n_slot = 0, n_line = 0, n_gen = 0, n_hidden = 0, n_unit = 0, n_load = 0, n_sto = 0,
        n_shunt = 0, dim_topo = 0, n_topo_in = 0;
    double base_mva = 1.0;
    std::vector<int> line_or_sub, line_ex_sub, line_or_pos, line_ex_pos;
    std::vector<double> line_y, line_bdc, line_pshift;
    std::vector<int> unit_sub, unit_pos, unit_is_ref;
    std::vector<double> unit_qmin, unit_qmax;
    std::vector<int> load_sub, load_pos, sto_sub, sto_pos, sh_sub;
};

// Header of a plan blob.  All offsets are BYTES from the start of the blob (which is 16-byte aligned on the
// device); u16 arrays hold 0xFFFF for "none".
struct PlanHeader {
    int status;            // static status of the class: ST_OK / ST_UNSUP / ST_NOREF
    int nb, n1, d;         // active buses, non-reference buses (DC unknowns), Newton unknowns
    int nnzF, nA;          // entries of the filled Jacobian; nA = nnzF + d (right-hand side appended) ; A[nA] = dummy
    int n_round;           // assembly rounds of the line lanes (parallel lines write the same entries)
    int n_pass, n_op;      // LU passes / operation slots (passes padded to whole rows of op_width slots)
    int op_width, n_oprow; // threads per instance the operation stream is laid out for; rows of op_width slots
    int n_zero;            // entries the line lanes add into + pure fill (cleared after every solve; the bus lanes assign the rest)
    int smem_bytes;        // per-instance workspace this plan needs
    int total_bytes;
    // per bus (nb entries each)
    int o_slot, o_btype, o_colth, o_colv, o_dcidx, o_vmunit, o_cnt, o_nref, o_dpos /* [nb][4] */;
    // ydiag: sum of y_ff / y_tt over the bus's line ends; block plans: the full Y_ii (a line with both ends on the bus adds
    // y_ft + y_tf too)
    int o_qmins, o_qmaxs, o_ydiag /* [nb][2] */, o_dcshift;                               // doubles
    int o_adj_ptr, o_adj, o_bu_ptr, o_bu, o_bl_ptr, o_bl, o_bs_ptr, o_bs, o_bh_ptr, o_bh;  // CSR lists (u16)
    // per line
    int o_brf, o_brt, o_round, o_jpos /* [n_line][8] */;
    // per element: bus index (u16, 0xFFFF = disconnected)
    int o_unit_bus, o_load_bus, o_sto_bus, o_sh_bus;
    // LU
    // operation stream: rows of op_width slots, thread t of the instance's group executes slot t of every row; a slot is
    // 4 x u16 BYTE offsets into the value array (ij, ik, kj, kk | 1 on the LAST row of a pass: group barrier after it);
    // padding slots work on A[dummy]
    int o_zero, o_pass_ptr /* int32 [n_pass + 1]: slot range of every pass (diagnostics / validation) */, o_ops;
    // DC: the inverse of Bdc (fp64, [n1][n1], stored transposed: entry (j, i) at j * n1 + i so that lanes = rows read
    // consecutive addresses) — Bdc depends on the topology only, so its solve is a matrix-vector product at run time
    int o_dcinv;
    int o_shidx;           // u16 [nb]: index of the bus among the buses that carry a shunt (0xFFFF: none)
    int n_shb;
    int o_late, n_late;    // u16 pairs (line, round) of the lines of assembly rounds >= 1 (parallel lines), sorted by round
    // ---- BLOCK plans (b200pf_block.cuh): the Jacobian as 2x2 blocks per bus pair, values = float4 per block -------------
    int blk;               // 0: scalar plan (b200pf_sparse.cuh), 1: block plan
    int blk_T, blk_U, blk_G;   // lanes per instance, operations per lane and row, instances per warp the streams are laid out for
    int nblk, nblkA;       // blocks of the filled pattern; nblkA = nblk + n1 (right-hand-side blocks); block nblkA = dummy
    int n_brow, n_bpass;   // rows of blk_T * blk_U slots; passes
    int o_bops;            // 8-byte slots {u16 d, a, b, flags}: BYTE offsets (16 * blk_G * block index) into the value array;
                           // flags bit 0: barrier after this row, bit 1: row type (0: D -= A B, 1: D = inv(A) D)
    int o_bdpos;           // u16 [nb]: block index of the diagonal block of the bus (0xFFFF: reference bus)
    int o_bjpos;           // u16 [n_line][2]: block (from,to) and (to,from) of the line (dummy when an end is a reference bus;
                           // validation: the kernel assembles from the admittance rows)
    int o_bzero, n_bzero;  // u16 block indices cleared before every assembly (the pure fill-in blocks)
    int o_bpass_ptr;       // int32 [n_bpass + 1] slot range of every pass (validation)
    // admittance rows of the buses, CSR, neighbours in ascending bus order: Y_ij summed over the lines between i and j in line
    // order (y_ft at a from end, y_tf at a to end), and the off-diagonal block (dcidx i, dcidx j) the lane of bus i writes
    // (dummy when either end is a reference bus)
    int o_yptr, o_ynb;     // u16 [nb + 1] row pointer, u16 neighbour bus per entry
    int o_yval;            // fp64 [entries][2]: Y_ij
    int o_yblk;            // u16 per entry: block index
    // the same rows packed for the kernel's bus phase (one load per entry and per bus instead of one per field):
    int o_yword;           // u32 per entry: block index (bits 0-15) | neighbour bus (bits 16-30) | bit 31: the neighbour is a PQ bus
    int o_yf32;            // fp32 [entries][2]: (float) of Y_ij, the operands of the off-diagonal blocks
    int o_bdesc;           // u32 [nb][2]: {bdpos | dcidx << 16, shidx | bit 16: the bus is a PQ bus}
    int pad2[2];
};
static_assert(sizeof(PlanHeader) % 16 == 0, "plan blobs are concatenated 16-byte aligned");

enum { PLAN_ST_OK = 0, PLAN_ST_UNSUP = 2, PLAN_ST_NOREF = 3 };
enum { PLAN_BT_PQ = 1, PLAN_BT_PV = 2, PLAN_BT_REF = 3 };

// per-instance shared-memory workspace of the sparse kernel for (nb buses, n_line lines, nA values)
inline int plan_smem_bytes(int nb, int n_line, int nA, int n_rowcol, int n_shunt) {
    size_t o = 0;
    o += ((size_t)(nA + 1) * 4 + 15) & ~(size_t)15;   // Jacobian values + right-hand side + dummy (first: shared-memory offset 0)
    o += (size_t)6 * nb * 8;                 // vm va pspec qspec P Q
    o += (size_t)2 * n_shunt * 8;            // shunt admittance (g, b) of the buses that carry one
    o += (size_t)nb * 16;                    // V (e, f)
    o += (size_t)2 * n_line * 16;            // branch currents, both ends
    o += ((size_t)n_rowcol * 4 + 15) & ~(size_t)15;   // this step's chronics row (load_p, load_q, prod_p, prod_v)
    return (int)((o + 15) & ~(size_t)15);
}

// per-INSTANCE workspace of the block kernel (a warp holds blk_G of them, element-interleaved)
inline int plan_block_smem_bytes(int nb, int n_line, int nblkA, int n_rowcol, int n_shunt) {
    size_t o = 0;
    o += (size_t)(nblkA + 1) * 16;           // blocks + right-hand-side blocks + dummy
    o += (size_t)6 * nb * 8;                 // vm va pspec qspec P Q
    o += (size_t)2 * n_shunt * 8;            // shunt admittance (g, b) of the buses that carry one
    o += (size_t)nb * 16;                    // V (e, f)
    o += (size_t)2 * n_line * 16;            // branch currents, both ends
    o += (size_t)nb * 8;                     // V in fp32 (the operands of the off-diagonal blocks)
    o += ((size_t)n_rowcol * 4 + 15) & ~(size_t)15;
    return (int)((o + 15) & ~(size_t)15);
}

// takes the tripped lines (trip[l] != 0) out of a topology row: both ends disconnected, like
// PandaPowerBackend._disconnect_line (reference pandaPowerBackend.py:1464-1475) / _BackendAction.update_state
inline void apply_trips(const HostGrid &g, int8_t *topo_row, const int8_t *trip) {
    for (int l = 0; l < g.n_line; ++l)
        if (trip[l]) { topo_row[g.line_or_pos[l]] = -1; topo_row[g.line_ex_pos[l]] = -1; }
}

class PlanBuilder {
public:
    // optimize_layout: spend ~1 ms per plan on a bank-conflict-reducing layout of the value array (plans that are re-used by
    // many solves: device-resident rollouts; not worth it when hundreds of plans are built for one call)
    explicit PlanBuilder(const HostGrid &g, int op_width = 32, bool optimize_layout = false, int order_seed = 0)
        : g_(g), op_width_(op_width), optimize_layout_(optimize_layout), order_seed_(order_seed) {}
    // block plans: T lanes per instance, U operations per lane and row, G instances per warp (G = 32 / T for T < 32, else 1)
    PlanBuilder &block_mode(int T, int U) { blk_ = 1; blk_T_ = T; blk_U_ = U < 1 ? 1 : U; blk_G_ = T < 32 ? 32 / T : 1; return *this; }

    // topo: int8 [n_topo_in]; outage: line forced out of service (N-1 sweep) or -1.  Returns the blob.
    std::vector<unsigned char> build(const int8_t *tv, int outage) const {
        PLAN_TICK0();
        const HostGrid &g = g_;
        const int nsub = g.n_sub, nl = g.n_line, nu = g.n_unit, nld = g.n_load, nst = g.n_sto, nsh = g.n_shunt, dt = g.dim_topo;
        const int ns = g.n_slot;
        // ---- active slots -> compact bus numbers (slot order) --------------------------------------
        std::vector<int> cidx(ns, 0);
        auto mark = [&](int sub, int b) { if (b > 0 && b <= g.n_busbar) cidx[sub + (b - 1) * nsub] = 1; };
        auto lbus = [&](int l, int side) -> int {
            if (l == outage) return -1;
            return side ? tv[g.line_ex_pos[l]] : tv[g.line_or_pos[l]];
        };
        for (int l = 0; l < nl; ++l) { mark(g.line_or_sub[l], lbus(l, 0)); mark(g.line_ex_sub[l], lbus(l, 1)); }
        for (int u = 0; u < nu; ++u) mark(g.unit_sub[u], tv[g.unit_pos[u]]);
        for (int k = 0; k < nld; ++k) mark(g.load_sub[k], tv[g.load_pos[k]]);
        for (int k = 0; k < nst; ++k) mark(g.sto_sub[k], tv[g.sto_pos[k]]);
        for (int k = 0; k < nsh; ++k) mark(g.sh_sub[k], tv[dt + k]);
        int nb = 0;
        std::vector<int> slot_of;
        for (int s = 0; s < ns; ++s) { if (cidx[s]) { cidx[s] = nb++; slot_of.push_back(s); } else cidx[s] = -1; }
        auto bus_of = [&](int sub, int b) -> int { return (b > 0 && b <= g.n_busbar) ? cidx[sub + (b - 1) * nsub] : -1; };

        std::vector<int> unit_bus(nu), load_bus(nld), sto_bus(nst), sh_bus(nsh), brf(nl), brt(nl);
        for (int u = 0; u < nu; ++u) unit_bus[u] = bus_of(g.unit_sub[u], tv[g.unit_pos[u]]);
        for (int k = 0; k < nld; ++k) load_bus[k] = bus_of(g.load_sub[k], tv[g.load_pos[k]]);
        for (int k = 0; k < nst; ++k) sto_bus[k] = bus_of(g.sto_sub[k], tv[g.sto_pos[k]]);
        for (int k = 0; k < nsh; ++k) sh_bus[k] = bus_of(g.sh_sub[k], tv[dt + k]);
        for (int l = 0; l < nl; ++l) {
            const int bo = lbus(l, 0), be = lbus(l, 1);
            if (bo > 0 && be > 0) { brf[l] = bus_of(g.line_or_sub[l], bo); brt[l] = bus_of(g.line_ex_sub[l], be); }
            else { brf[l] = -1; brt[l] = -1; }
        }
        PLAN_TICK("decode");
        // ---- bus types, static per-bus unit data --------------------------------------------------
        std::vector<int> btype(nb, PLAN_BT_PQ), cnt(nb, 0), nref(nb, 0), vmunit(nb, -1);
        std::vector<double> qmins(nb, 0.0), qmaxs(nb, 0.0);
        for (int u = 0; u < nu; ++u) {
            const int i = unit_bus[u];
            if (i < 0) continue;
            vmunit[i] = u; cnt[i]++; qmins[i] += g.unit_qmin[u]; qmaxs[i] += g.unit_qmax[u];
            if (g.unit_is_ref[u]) { btype[i] = PLAN_BT_REF; nref[i]++; }
            else if (btype[i] != PLAN_BT_REF) btype[i] = PLAN_BT_PV;
        }
        int status = PLAN_ST_OK;
        {
            std::vector<char> reach(nb, 0);
            bool anyref = false;
            for (int i = 0; i < nb; ++i) if (btype[i] == PLAN_BT_REF) { reach[i] = 1; anyref = true; }
            if (!anyref) status = PLAN_ST_NOREF;
            else {
                for (int sweep = 0; sweep < nb + 1; ++sweep) {
                    bool ch = false;
                    for (int l = 0; l < nl; ++l) {
                        const int f = brf[l], t = brt[l];
                        if (f < 0) continue;
                        if (reach[f] != reach[t]) { reach[f] = 1; reach[t] = 1; ch = true; }
                    }
                    if (!ch) break;
                }
                for (int i = 0; i < nb; ++i) if (!reach[i]) status = PLAN_ST_UNSUP;
            }
        }
        if (status != PLAN_ST_OK) {
            PlanHeader H;
            memset(&H, 0, sizeof(H));
            H.status = status; H.nb = nb; H.total_bytes = (int)sizeof(PlanHeader);
            H.smem_bytes = 16;
            std::vector<unsigned char> blob(sizeof(PlanHeader));
            memcpy(blob.data(), &H, sizeof(H));
            return blob;
        }
        PLAN_TICK("types+reach");
        // ---- bus graph and minimum-degree elimination order of the non-reference buses -------------
        std::vector<char> adjm((size_t)nb * nb, 0);
        for (int l = 0; l < nl; ++l) {
            const int f = brf[l], t = brt[l];
            if (f < 0 || f == t) continue;
            adjm[(size_t)f * nb + t] = 1; adjm[(size_t)t * nb + f] = 1;
        }
        std::vector<int> order;         // non-reference buses in elimination order
        {
            // minimum degree, ties broken by minimum LENGTH (MD-ML: the longest elimination path that ends in the node) —
            // the factorisation runs as passes of independent operations, so the height of the elimination tree, not the
            // fill alone, sets its run time.  Degrees are maintained incrementally (O(nb) per elimination + the clique).
            std::vector<char> w(adjm);  // working copy; edges to reference / eliminated buses are ignored through `alive`
            std::vector<char> alive(nb, 0);
            int n_alive = 0;
            for (int i = 0; i < nb; ++i) if (btype[i] != PLAN_BT_REF) { alive[i] = 1; ++n_alive; }
            std::vector<int> nbrs, length(nb, 0), deg(nb, 0);
            uint32_t ord_state = 0x2545F491u * (uint32_t)(order_seed_ + 1);
            auto ord_rng = [&]() { ord_state ^= ord_state << 13; ord_state ^= ord_state >> 17; ord_state ^= ord_state << 5; return ord_state >> 7; };
            for (int i = 0; i < nb; ++i) {
                if (!alive[i]) continue;
                const char *row = &w[(size_t)i * nb];
                int dg = 0;
                for (int j = 0; j < nb; ++j) dg += (row[j] && alive[j]);
                deg[i] = dg;
            }
            while (n_alive > 0) {
                int best = -1, bestdeg = 1 << 30, bestlen = 1 << 30;
                for (int i = 0; i < nb; ++i) {
                    if (!alive[i]) continue;
                    const bool tie = deg[i] == bestdeg && length[i] == bestlen;
                    if (deg[i] < bestdeg || (deg[i] == bestdeg && length[i] < bestlen) || (tie && order_seed_ && (ord_rng() & 1u))) { bestdeg = deg[i]; bestlen = length[i]; best = i; }
                }
                nbrs.clear();
                const char *rb = &w[(size_t)best * nb];
                for (int j = 0; j < nb; ++j) if (rb[j] && alive[j]) nbrs.push_back(j);
                alive[best] = 0; --n_alive;
                for (size_t a = 0; a < nbrs.size(); ++a) {
                    const int u = nbrs[a];
                    --deg[u];                                   // its edge to the eliminated bus
                    length[u] = std::max(length[u], length[best] + 1);
                    for (size_t b = a + 1; b < nbrs.size(); ++b) {
                        const int v = nbrs[b];
                        if (!w[(size_t)u * nb + v]) { w[(size_t)u * nb + v] = 1; w[(size_t)v * nb + u] = 1; ++deg[u]; ++deg[v]; }
                    }
                }
                order.push_back(best);
            }
        }
        const int n1 = (int)order.size();
        std::vector<int> dcidx(nb, -1), colth(nb, -1), colv(nb, -1);
        int d = 0;
        for (int k = 0; k < n1; ++k) {
            const int i = order[k];
            dcidx[i] = k;
            colth[i] = d++;
            if (btype[i] == PLAN_BT_PQ) colv[i] = d++;
        }
        PLAN_TICK("ordering");
        struct Op { uint16_t ij, ik, kj, kk; };
        struct BOp { uint16_t d, a, b, fl; };
        int n_oprow = 0, nnzF = 0, nA = 0, n_pass = 0, n_round = 0;
        std::vector<Op> ops;
        std::vector<int> pass_ptr(1, 0), round(nl, 0);
        std::vector<uint16_t> dpos, jpos, zero;
        int nblk = 0, nblkA = 0, n_brow = 0, n_bpass = 0;            // block plans
        std::vector<BOp> bops;
        std::vector<int> bdpos(nb, -1), bjpos((size_t)nl * 2, -1), bzero, bpass_ptr(1, 0), yptr, ynb, yblk;
        std::vector<double> yval;
        if (!blk_) {
        // ---- scalar pattern of the Jacobian, symbolic LU --------------------------------------------
        std::vector<char> S((size_t)d * d, 0);
        auto setblk = [&](int i, int j) {   // rows of bus i, columns of bus j
            const int r[2] = {colth[i], colv[i]}, c[2] = {colth[j], colv[j]};
            for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) if (r[a] >= 0 && c[b] >= 0) S[(size_t)r[a] * d + c[b]] = 1;
        };
        for (int i = 0; i < nb; ++i) if (colth[i] >= 0) setblk(i, i);
        for (int l = 0; l < nl; ++l) {
            const int f = brf[l], t = brt[l];
            if (f < 0) continue;
            setblk(f, t); setblk(t, f);
        }
        std::vector<std::vector<int>> rowU(d), colL(d);   // columns j > k of row k ; rows i > k of column k (filled pattern)
        {
            std::vector<int> lst;
            for (int k = 0; k < d; ++k) {
                lst.clear();
                for (int j = k + 1; j < d; ++j) if (S[(size_t)k * d + j]) lst.push_back(j);
                rowU[k] = lst;
                colL[k] = lst;              // the pattern is structurally symmetric (block pattern of the bus graph) and stays so under fill
                for (int i : lst) { char *Si = &S[(size_t)i * d]; for (int j : lst) Si[j] = 1; }
            }
        }
        std::vector<int> pos((size_t)d * d, -1);
        nnzF = 0;
        for (int i = 0; i < d; ++i) for (int j = 0; j < d; ++j) if (S[(size_t)i * d + j]) pos[(size_t)i * d + j] = nnzF++;
        nA = nnzF + d;
        const int DUMMY = nA;
        auto P = [&](int i, int j) -> int { return (i >= 0 && j >= 0) ? pos[(size_t)i * d + j] : -1; };
        PLAN_TICK("symbolic");
        // ---- LU + both triangular solves as ONE list of multiply-subtract operations A[ij] -= A[ik] A[kj] / A[kk]
        //      (right-looking elimination with the right-hand side carried along, then column-oriented back
        //      substitution on the right-hand side), list-scheduled into passes: an operation goes to the earliest
        //      pass after the last write of everything it reads (RAW), after the previous write of its target (WAW:
        //      two updates of one entry never share a pass, and keep their sequential order, so the rounding is that
        //      of the sequential algorithm) and after the last read of its target (WAR).  The number of passes is
        //      the depth of the dependency graph (about twice the height of the elimination tree), not the number
        //      of columns.  The solution is x_k = rhs_k / A[kk] (taken by the bus lanes in the state update).
        {
            std::vector<Op> seq;
            seq.reserve((size_t)nnzF * 4 + 64);
            for (int k = 0; k < d; ++k) {
                const int kk = P(k, k);
                for (int i : colL[k]) {
                    const int ik = P(i, k);
                    for (int j : rowU[k]) seq.push_back({(uint16_t)P(i, j), (uint16_t)ik, (uint16_t)P(k, j), (uint16_t)kk});
                    seq.push_back({(uint16_t)(nnzF + i), (uint16_t)ik, (uint16_t)(nnzF + k), (uint16_t)kk});
                }
            }
            for (int k = d - 1; k >= 0; --k) {
                const int kk = P(k, k);
                for (int i = k - 1; i >= 0; --i)
                    if (S[(size_t)i * d + k]) seq.push_back({(uint16_t)(nnzF + i), (uint16_t)P(i, k), (uint16_t)(nnzF + k), (uint16_t)kk});
            }
            PLAN_TICK("ops: seq");
            std::vector<int> wlev(nA + 1, 0), rlev(nA + 1, 0), lev(seq.size(), 0);
            // For the row balancing below: the earliest pass of any successor of an operation in the dependency graph (RAW, WAW,
            // WAR edges).  Flat arrays only (this is the builder's hot loop: the cost of a new topology in a single environment):
            // the readers of an entry since its last write are a linked list threaded through the three read slots of every
            // operation.
            const int NOSUCC = 1 << 30;
            std::vector<int> minsucc(seq.size(), NOSUCC), lastw(nA + 1, -1), rd_head(nA + 1, -1), rd_next(seq.size() * 3, -1);
            int nlev = 0;
            for (size_t q = 0; q < seq.size(); ++q) {
                const Op &o = seq[q];
                const int lv = std::max(std::max(wlev[o.ik], wlev[o.kj]), std::max(wlev[o.kk], std::max(wlev[o.ij], rlev[o.ij]))) + 1;
                lev[q] = lv; nlev = std::max(nlev, lv);
                wlev[o.ij] = lv;
                rlev[o.ik] = std::max(rlev[o.ik], lv); rlev[o.kj] = std::max(rlev[o.kj], lv); rlev[o.kk] = std::max(rlev[o.kk], lv);
                const int rd[3] = {o.ik, o.kj, o.kk};
                for (int r : rd) { const int p = lastw[r]; if (p >= 0 && lv < minsucc[p]) minsucc[p] = lv; }            // RAW
                { const int p = lastw[o.ij]; if (p >= 0 && lv < minsucc[p]) minsucc[p] = lv; }                          // WAW
                for (int nd = rd_head[o.ij]; nd >= 0; nd = rd_next[nd]) { const int p = nd / 3; if (lv < minsucc[p]) minsucc[p] = lv; }   // WAR
                rd_head[o.ij] = -1;
                for (int s3 = 0; s3 < 3; ++s3) { const int nd = (int)q * 3 + s3; rd_next[nd] = rd_head[rd[s3]]; rd_head[rd[s3]] = nd; }
                lastw[o.ij] = (int)q;
            }
            PLAN_TICK("ops: levels");
            const int W = op_width_;
            {   // Row balancing: a pass costs ceil(n / W) rows.  Going down the passes, the operations of the last, partly
                // filled row move to the next pass when they have slack (every successor at least two passes later; those with
                // the most slack first): that saves a row here and costs at most one there, where the remainder rolls on.
                // Dependencies are untouched by construction (tests/ validate every stream).  (The successors of the operations of
                // pass l sit in later passes, which have not been touched yet when l is balanced: their passes are still the ones
                // of the scan above, which is what minsucc holds.)
                std::vector<int> cnt(nlev + 2, 0), off(nlev + 3, 0);
                for (int lv : lev) cnt[lv]++;
                for (int l = 0; l <= nlev + 1; ++l) off[l + 1] = off[l] + cnt[l] + W;      // room for what moves in from the pass before
                std::vector<int> at((size_t)off[nlev + 2]), fill(off.begin(), off.end() - 1);
                for (size_t q = 0; q < seq.size(); ++q) at[fill[lev[q]]++] = (int)q;
                std::vector<std::pair<int, int>> cand;
                for (int l = 1; l < nlev; ++l) {
                    const int n_here = fill[l] - off[l];
                    const int r = n_here % W;
                    if (r == 0) continue;
                    cand.clear();
                    for (int k = off[l]; k < fill[l]; ++k) { const int q = at[k]; if (minsucc[q] >= l + 2) cand.push_back({-minsucc[q], q}); }
                    if ((int)cand.size() < r) continue;
                    std::sort(cand.begin(), cand.end());
                    for (int c = 0; c < r; ++c) { const int q = cand[c].second; lev[q] = l + 1; at[fill[l + 1]++] = q; }
                    int w = off[l];
                    for (int k = off[l]; k < fill[l]; ++k) if (lev[at[k]] == l) at[w++] = at[k];
                    fill[l] = w;
                }
            }
            PLAN_TICK("ops: balance");
            // passes padded to whole rows of op_width slots; the last row of a pass carries the barrier flag
            std::vector<int> lv_ptr(nlev + 2, 0);
            for (int lv : lev) lv_ptr[lv + 1]++;
            for (int l = 1; l <= nlev + 1; ++l) lv_ptr[l] += lv_ptr[l - 1];
            std::vector<Op> sorted_ops(seq.size());
            {
                std::vector<int> fillp(lv_ptr.begin(), lv_ptr.end() - 1);
                for (size_t q = 0; q < seq.size(); ++q) sorted_ops[fillp[lev[q]]++] = seq[q];
            }
            const Op nop = {(uint16_t)DUMMY, (uint16_t)DUMMY, (uint16_t)DUMMY, (uint16_t)DUMMY};
            pass_ptr.assign(1, 0);
            ops.reserve(seq.size() + (size_t)(nlev + 8) * W);
            for (int l = 1; l <= nlev; ++l) {
                Op *b0 = sorted_ops.data() + lv_ptr[l], *b1 = sorted_ops.data() + lv_ptr[l + 1];
                // neighbouring slots work on neighbouring entries (fewer shared-memory bank conflicts); targets are unique
                // within a pass, so the order inside a pass is free
                std::sort(b0, b1, [](const Op &a, const Op &b) { return a.ij < b.ij; });
                const size_t first = ops.size();
                ops.insert(ops.end(), b0, b1);
                while ((ops.size() - first) % (size_t)W) ops.push_back(nop);
                for (size_t q = ops.size() - (size_t)W; q < ops.size(); ++q) ops[q].kk |= 0x4000u;   // becomes bit 0 of the byte offset below
                pass_ptr.push_back((int)ops.size());
            }
            while ((ops.size() / (size_t)W) % 4) ops.insert(ops.end(), (size_t)W, nop);     // whole blocks of 4 rows (prefetch unit)
            n_oprow = (int)(ops.size() / (size_t)W);
            ops.insert(ops.end(), (size_t)W * 4, nop);      // guard block: the prefetch of "the block after the last" reads it, nothing executes it
        }
        n_pass = (int)pass_ptr.size() - 1;
        PLAN_TICK("ops+schedule");
        // ---- assembly positions ------------------------------------------------------------------
        dpos.assign((size_t)nb * 4, (uint16_t)DUMMY); jpos.assign((size_t)nl * 8, (uint16_t)DUMMY);
        std::vector<char> is_buslane(nA + 1, 0);
        for (int i = 0; i < nb; ++i) {
            const int r[2] = {colth[i], colv[i]};
            for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) {
                const int p = P(r[a], r[b]);
                if (p >= 0) { dpos[(size_t)i * 4 + a * 2 + b] = (uint16_t)p; is_buslane[p] = 1; }
            }
        }
        for (int k = 0; k < d; ++k) is_buslane[nnzF + k] = 1;      // right-hand side: written by the bus lanes
        {
            std::vector<std::vector<char>> used;   // per round: position used
            for (int l = 0; l < nl; ++l) {
                const int f = brf[l], t = brt[l];
                if (f < 0) continue;
                const int rf[2] = {colth[f], colv[f]}, rt[2] = {colth[t], colv[t]};
                uint16_t *jp = &jpos[(size_t)l * 8];
                for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) {
                    int p = P(rf[a], rt[b]); if (p >= 0) jp[a * 2 + b] = (uint16_t)p;
                    p = P(rt[a], rf[b]);     if (p >= 0) jp[4 + a * 2 + b] = (uint16_t)p;
                }
                // round 0 is added BEFORE the bus lanes assign the diagonal blocks: a line with both ends on one bus (it
                // writes into a diagonal block) must come later
                int r = (f == t) ? 1 : 0;
                for (;; ++r) {
                    while (r >= (int)used.size()) used.emplace_back(nA + 1, 0);
                    bool clash = false;
                    for (int q = 0; q < 8; ++q) if (jp[q] != DUMMY && used[r][jp[q]]) clash = true;
                    // a line whose two ends sit on the same bus writes the same entry twice: keep it alone in a round
                    if (!clash) break;
                }
                for (int q = 0; q < 8; ++q) if (jp[q] != DUMMY) used[r][jp[q]] = 1;
                round[l] = r; n_round = std::max(n_round, r + 1);
            }
        }
        for (int p = 0; p < nnzF; ++p) if (!is_buslane[p]) zero.push_back((uint16_t)p);
        PLAN_TICK("assembly pos");
        } else {
            // ---- BLOCK plan: the Jacobian as 2x2 blocks (rows P_i, Q_i x columns theta_j, |V|_j) per bus pair in elimination
            //      order; a PV bus keeps its block shape with an identity Q row / a zero |V| column (b200pf_block.cuh), so every
            //      block is a float4 and every operation of the factorisation a 2x2 product:
            //        row k normalised     U'_kj = inv(A_kk) A_kj ,  r'_k = inv(A_kk) r_k                       (type 1)
            //        rows below updated   A_ij -= A_ik U'_kj     ,  r_i -= A_ik r'_k                            (type 0)
            //        back substitution    r'_i -= U'_ik x_k  (x_k = r'_k once all its updates are done)         (type 0)
            //      list-scheduled into passes exactly like the scalar stream (RAW / WAW / WAR levels).  One block operation
            //      replaces ~8 scalar ones at 3 vector loads + 1 vector store instead of 8 x (4 loads + 1 store).
            std::vector<char> SBk((size_t)n1 * n1, 0);
            for (int k = 0; k < n1; ++k) SBk[(size_t)k * n1 + k] = 1;
            for (int l = 0; l < nl; ++l) {
                const int f = brf[l], t = brt[l];
                if (f < 0) continue;
                const int cf = dcidx[f], ct = dcidx[t];
                if (cf >= 0 && ct >= 0 && cf != ct) { SBk[(size_t)cf * n1 + ct] = 1; SBk[(size_t)ct * n1 + cf] = 1; }
            }
            std::vector<std::vector<int>> rowUb(n1);
            {
                std::vector<int> lst;
                for (int k = 0; k < n1; ++k) {
                    lst.clear();
                    for (int j = k + 1; j < n1; ++j) if (SBk[(size_t)k * n1 + j]) lst.push_back(j);
                    rowUb[k] = lst;
                    for (int i : lst) { char *Si = &SBk[(size_t)i * n1]; for (int j : lst) Si[j] = 1; }
                }
            }
            std::vector<int> bpos((size_t)n1 * n1, -1);
            for (int i = 0; i < n1; ++i) for (int j = 0; j < n1; ++j) if (SBk[(size_t)i * n1 + j]) bpos[(size_t)i * n1 + j] = nblk++;
            nblkA = nblk + n1;
            const int BD = nblkA;
            auto BP = [&](int r, int c) -> int { return bpos[(size_t)r * n1 + c]; };
            struct SOp { int d, a, b, type; };
            std::vector<SOp> seq;
            seq.reserve((size_t)nblk * 6 + 64);
            for (int k = 0; k < n1; ++k) {
                const int kk = BP(k, k);
                for (int j : rowUb[k]) seq.push_back({BP(k, j), kk, BD, 1});
                seq.push_back({nblk + k, kk, BD, 1});
                for (int i : rowUb[k]) {
                    const int ik = BP(i, k);
                    for (int j : rowUb[k]) seq.push_back({BP(i, j), ik, BP(k, j), 0});
                    seq.push_back({nblk + i, ik, nblk + k, 0});
                }
            }
            for (int k = n1 - 1; k >= 0; --k)
                for (int i = k - 1; i >= 0; --i)
                    if (SBk[(size_t)i * n1 + k]) seq.push_back({nblk + i, BP(i, k), nblk + k, 0});
            std::vector<int> wlev(nblkA + 1, 0), rlev(nblkA + 1, 0), lev(seq.size(), 0);
            int nlev = 0;
            for (size_t q = 0; q < seq.size(); ++q) {
                const SOp &o = seq[q];
                int lv = std::max(std::max(wlev[o.a], wlev[o.d]), rlev[o.d]);
                if (o.type == 0) lv = std::max(lv, wlev[o.b]);
                lv += 1;
                lev[q] = lv; nlev = std::max(nlev, lv);
                wlev[o.d] = lv;
                rlev[o.a] = std::max(rlev[o.a], lv);
                if (o.type == 0) rlev[o.b] = std::max(rlev[o.b], lv);
            }
            const int W = blk_T_ * blk_U_;
            const size_t osc = (size_t)16 * blk_G_;
            auto emit = [&](int dd, int aa, int bb, int type) {
                BOp r;
                r.d = (uint16_t)((size_t)dd * osc); r.a = (uint16_t)((size_t)aa * osc); r.b = (uint16_t)((size_t)bb * osc);
                r.fl = (uint16_t)(type ? 2 : 0);
                bops.push_back(r);
            };
            {
                std::vector<std::vector<int>> at(nlev + 1);
                for (size_t q = 0; q < seq.size(); ++q) at[lev[q]].push_back((int)q);
                for (int l = 1; l <= nlev; ++l) {
                    for (int type = 1; type >= 0; --type) {
                        std::vector<int> grp;
                        for (int q : at[l]) if (seq[q].type == type) grp.push_back(q);
                        if (grp.empty()) continue;
                        std::sort(grp.begin(), grp.end(), [&](int x, int y) { return seq[x].d < seq[y].d; });
                        for (int q : grp) emit(seq[q].d, seq[q].a, seq[q].b, type);
                        while (bops.size() % (size_t)W) emit(BD, BD, BD, type);
                    }
                    for (size_t q = bops.size() - (size_t)W; q < bops.size(); ++q) bops[q].fl |= 1;     // barrier after the last row of the pass
                    bpass_ptr.push_back((int)bops.size());
                }
            }
            n_brow = (int)(bops.size() / (size_t)W);
            n_bpass = (int)bpass_ptr.size() - 1;
            for (int q = 0; q < W; ++q) emit(BD, BD, BD, 0);          // guard row: the prefetch of "the row after the last" reads it
            // ---- assembly positions ------------------------------------------------------------------------
            for (int i = 0; i < nb; ++i) if (dcidx[i] >= 0) bdpos[i] = BP(dcidx[i], dcidx[i]);
            for (int l = 0; l < nl; ++l) {
                const int f = brf[l], t = brt[l];
                bjpos[(size_t)2 * l] = BD; bjpos[(size_t)2 * l + 1] = BD;
                if (f < 0) continue;
                const int cf = dcidx[f], ct = dcidx[t];
                if (cf >= 0 && ct >= 0) { bjpos[(size_t)2 * l] = BP(cf, ct); bjpos[(size_t)2 * l + 1] = BP(ct, cf); }
            }
            // ---- admittance rows: the bus lane of bus i computes its current from them and writes the off-diagonal blocks of
            //      its block row whole, so every block of the bus graph has exactly one writer per Newton evaluation (parallel
            //      lines are summed here; a line with both ends on one bus is part of Y_ii, below) and only the fill is cleared
            {
                std::vector<std::vector<std::pair<int, int>>> ends(nb);          // (neighbour bus, 2 * line + side)
                for (int l = 0; l < nl; ++l) {
                    const int f = brf[l], t = brt[l];
                    if (f < 0 || f == t) continue;
                    ends[f].push_back({t, 2 * l}); ends[t].push_back({f, 2 * l + 1});
                }
                std::vector<char> written(nblk, 0);
                yptr.assign(1, 0);
                for (int i = 0; i < nb; ++i) {
                    std::sort(ends[i].begin(), ends[i].end());                   // neighbours ascending, then line order
                    for (size_t e = 0; e < ends[i].size();) {
                        const int j = ends[i][e].first;
                        double yr = 0.0, yi = 0.0;
                        for (; e < ends[i].size() && ends[i][e].first == j; ++e) {
                            const int l = ends[i][e].second >> 1, side = ends[i][e].second & 1;
                            const double *y = &g.line_y[(size_t)l * 8 + (side ? 4 : 2)];     // y_ft at the from end, y_tf at the to end
                            yr += y[0]; yi += y[1];
                        }
                        const int ci = dcidx[i], cj = dcidx[j];
                        const int b = (ci >= 0 && cj >= 0) ? BP(ci, cj) : BD;
                        if (b != BD) written[b] = 1;
                        ynb.push_back(j); yval.push_back(yr); yval.push_back(yi); yblk.push_back(b);
                    }
                    yptr.push_back((int)ynb.size());
                }
                for (int k = 0; k < n1; ++k) written[BP(k, k)] = 1;
                for (int p = 0; p < nblk; ++p) if (!written[p]) bzero.push_back(p);
            }
        }
        // ---- static per-bus line data ------------------------------------------------------------------
        std::vector<double> ydiag((size_t)nb * 2, 0.0), dcshift(nb, 0.0);
        std::vector<std::vector<int>> adj(nb), bu(nb), bl(nb), bs(nb), bh(nb);
        for (int l = 0; l < nl; ++l) {
            const int f = brf[l], t = brt[l];
            if (f < 0) continue;
            const double *y = &g.line_y[(size_t)l * 8];
            ydiag[(size_t)f * 2] += y[0]; ydiag[(size_t)f * 2 + 1] += y[1];
            ydiag[(size_t)t * 2] += y[6]; ydiag[(size_t)t * 2 + 1] += y[7];
            if (blk_ && f == t) { ydiag[(size_t)f * 2] += y[2] + y[4]; ydiag[(size_t)f * 2 + 1] += y[3] + y[5]; }
            dcshift[f] += g.line_pshift[l]; dcshift[t] -= g.line_pshift[l];
            adj[f].push_back(2 * l); adj[t].push_back(2 * l + 1);
        }
        for (int i = 0; i < nb; ++i) std::sort(adj[i].begin(), adj[i].end());
        for (int u = 0; u < nu; ++u) if (unit_bus[u] >= 0) bu[unit_bus[u]].push_back(u);
        for (int k = 0; k < nld; ++k) if (load_bus[k] >= 0) bl[load_bus[k]].push_back(k);
        for (int k = 0; k < nst; ++k) if (sto_bus[k] >= 0) bs[sto_bus[k]].push_back(k);
        for (int k = 0; k < nsh; ++k) if (sh_bus[k] >= 0) bh[sh_bus[k]].push_back(k);
        PLAN_TICK("perbus");
        // ---- DC matrix, factorised (fp64, no pivoting: Bdc is symmetric and, for positive series reactances,
        //      positive definite), in the elimination order of the buses --------------------------------------
        std::vector<double> B((size_t)n1 * n1, 0.0);
        std::vector<char> SB((size_t)n1 * n1, 0);
        for (int l = 0; l < nl; ++l) {
            const int f = brf[l], t = brt[l];
            if (f < 0) continue;
            const double b = g.line_bdc[l];
            const int cf = dcidx[f], ct = dcidx[t];
            if (cf >= 0) { B[(size_t)cf * n1 + cf] += b; SB[(size_t)cf * n1 + cf] = 1; if (ct >= 0) { B[(size_t)cf * n1 + ct] -= b; SB[(size_t)cf * n1 + ct] = 1; } }
            if (ct >= 0) { B[(size_t)ct * n1 + ct] += b; SB[(size_t)ct * n1 + ct] = 1; if (cf >= 0) { B[(size_t)ct * n1 + cf] -= b; SB[(size_t)ct * n1 + cf] = 1; } }
        }
        {
            std::vector<int> cj;
            for (int k = 0; k < n1; ++k) {
                cj.clear();
                for (int j = k + 1; j < n1; ++j) if (SB[(size_t)k * n1 + j]) cj.push_back(j);
                const double piv = B[(size_t)k * n1 + k];
                for (int i = k + 1; i < n1; ++i) {
                    if (!SB[(size_t)i * n1 + k]) continue;
                    const double m = B[(size_t)i * n1 + k] / piv;
                    B[(size_t)i * n1 + k] = m;                    // L (unit diagonal)
                    for (int j : cj) { B[(size_t)i * n1 + j] -= m * B[(size_t)k * n1 + j]; SB[(size_t)i * n1 + j] = 1; }
                }
            }
        }
        PLAN_TICK("dc factor");
        std::vector<double> dcinv((size_t)n1 * n1, 0.0);
        {
            // row lists of the factors (non-zeros only), then one sparse forward + backward solve per unit vector
            std::vector<int> lptr(n1 + 1, 0), uptr(n1 + 1, 0), lcol, ucol;
            std::vector<double> lval, uval, udiag(n1, 1.0);
            for (int i = 0; i < n1; ++i) {
                const double *Bi = &B[(size_t)i * n1];
                const char *Si = &SB[(size_t)i * n1];
                for (int j = 0; j < i; ++j) if (Si[j]) { lcol.push_back(j); lval.push_back(Bi[j]); }
                for (int j = i + 1; j < n1; ++j) if (Si[j]) { ucol.push_back(j); uval.push_back(Bi[j]); }
                lptr[i + 1] = (int)lcol.size(); uptr[i + 1] = (int)ucol.size();
                udiag[i] = 1.0 / Bi[i];
            }
            std::vector<double> x(n1);
            for (int c = 0; c < n1; ++c) {
                for (int i = 0; i < c; ++i) x[i] = 0.0;
                x[c] = 1.0;
                for (int i = c + 1; i < n1; ++i) {                 // L y = e_c (unit lower; y_i = 0 for i < c)
                    double sacc = 0.0;
                    for (int e = lptr[i]; e < lptr[i + 1]; ++e) if (lcol[e] >= c) sacc -= lval[e] * x[lcol[e]];
                    x[i] = sacc;
                }
                for (int i = n1 - 1; i >= 0; --i) {                // U x = y
                    double sacc = x[i];
                    for (int e = uptr[i]; e < uptr[i + 1]; ++e) sacc -= uval[e] * x[ucol[e]];
                    x[i] = sacc * udiag[i];
                }
                double *dst = &dcinv[(size_t)c * n1];              // column c of the inverse = row c of the transposed store
                for (int i = 0; i < n1; ++i) dst[i] = x[i];
            }
        }
        PLAN_TICK("dc inverse");
        // ---- physical layout of the matrix entries: a permutation of the slots [0, nnzF) that spreads the entries one warp-row
        //      of the operation stream touches together over the 32 shared-memory banks (right-hand side and dummy keep their
        //      slots: the kernel addresses them implicitly).  Local search over swaps, cost = wavefronts of the stream.
        if (optimize_layout_ && nnzF > 32) {
            const int W = op_width_;
            const int n_wrow = n_oprow * (W / 32);
            // groups: (warp-row, stream) -> distinct movable positions + fixed per-bank counts of the rest
            struct Group { std::vector<int> pos; int fixed[32]; int cnt[32]; int weight; };
            std::vector<Group> groups((size_t)n_wrow * 4);
            std::vector<std::vector<int>> memb(nnzF);
            std::vector<int> mark(nA + 1, -1);
            for (int wr = 0; wr < n_wrow; ++wr)
                for (int st = 0; st < 4; ++st) {
                    Group &G = groups[(size_t)wr * 4 + st];
                    for (int b = 0; b < 32; ++b) G.fixed[b] = 0;
                    G.weight = st == 0 ? 2 : 1;
                    const int gid = wr * 4 + st;
                    for (int l = 0; l < 32; ++l) {
                        const Op &o = ops[(size_t)wr * 32 + l];
                        const int p = st == 0 ? o.ij : (st == 1 ? o.ik : (st == 2 ? o.kj : (o.kk & 0x3fff)));
                        if (mark[p] == gid) continue;
                        mark[p] = gid;
                        if (p < nnzF) { G.pos.push_back(p); memb[p].push_back(gid); } else G.fixed[p % 32]++;
                    }
                }
            std::vector<int> slot(nnzF), owner(nnzF);
            for (int p = 0; p < nnzF; ++p) { slot[p] = p; owner[p] = p; }
            auto gcost = [](const Group &G) { int m = 1; for (int b = 0; b < 32; ++b) m = std::max(m, G.cnt[b]); return m * G.weight; };
            for (Group &G : groups) { for (int b = 0; b < 32; ++b) G.cnt[b] = G.fixed[b]; for (int p : G.pos) G.cnt[slot[p] % 32]++; }
            uint32_t rng = 0x9E3779B9u ^ (uint32_t)nnzF;
            auto rnd = [&]() { rng ^= rng << 13; rng ^= rng >> 17; rng ^= rng << 5; return rng; };
            std::vector<int> touched;
            for (int sweep = 0; sweep < 6; ++sweep) {
                int improved = 0;
                for (size_t gi = 0; gi < groups.size(); ++gi) {
                    Group &G = groups[gi];
                    int bmax = 0;
                    for (int b = 1; b < 32; ++b) if (G.cnt[b] > G.cnt[bmax]) bmax = b;
                    if (G.cnt[bmax] <= 1) continue;
                    for (int p : G.pos) {
                        if (slot[p] % 32 != bmax) continue;
                        bool done = false;
                        for (int trial = 0; trial < 12 && !done; ++trial) {
                            const int s2 = (int)(rnd() % (uint32_t)nnzF);
                            const int q = owner[s2], bp = slot[p] % 32, bq = s2 % 32;
                            if (q == p || bq == bp || G.cnt[bq] >= G.cnt[bmax] - 1) continue;
                            // cost change over the groups of p and q
                            touched.clear();
                            for (int g2 : memb[p]) touched.push_back(g2);
                            for (int g2 : memb[q]) touched.push_back(g2);
                            std::sort(touched.begin(), touched.end());
                            touched.erase(std::unique(touched.begin(), touched.end()), touched.end());
                            int before = 0, after = 0;
                            for (int g2 : touched) before += gcost(groups[g2]);
                            for (int g2 : memb[p]) { groups[g2].cnt[bp]--; groups[g2].cnt[bq]++; }
                            for (int g2 : memb[q]) { groups[g2].cnt[bq]--; groups[g2].cnt[bp]++; }
                            for (int g2 : touched) after += gcost(groups[g2]);
                            if (after < before) {
                                std::swap(slot[p], slot[q]); owner[slot[p]] = p; owner[slot[q]] = q;
                                ++improved; done = true;
                            } else {
                                for (int g2 : memb[p]) { groups[g2].cnt[bp]++; groups[g2].cnt[bq]--; }
                                for (int g2 : memb[q]) { groups[g2].cnt[bq]++; groups[g2].cnt[bp]--; }
                            }
                        }
                        if (done) break;
                    }
                }
                if (!improved) break;
            }
            auto mp = [&](uint16_t v) -> uint16_t { return v < nnzF ? (uint16_t)slot[v] : v; };
            for (Op &o : ops) { o.ij = mp(o.ij); o.ik = mp(o.ik); o.kj = mp(o.kj); o.kk = (uint16_t)((o.kk & 0x4000u) | mp((uint16_t)(o.kk & 0x3fffu))); }
            for (uint16_t &v : dpos) v = mp(v);
            for (uint16_t &v : jpos) v = mp(v);
            for (uint16_t &v : zero) v = mp(v);
        }
        // slots hold BYTE offsets into the value array (4 * position; the barrier flag moves to bit 0 of kk)
        for (Op &o : ops) {
            const unsigned flag = (o.kk & 0x4000u) ? 1u : 0u;
            o.ij = (uint16_t)(o.ij * 4u); o.ik = (uint16_t)(o.ik * 4u); o.kj = (uint16_t)(o.kj * 4u);
            o.kk = (uint16_t)(((o.kk & 0x3fffu) * 4u) | flag);
        }
        PLAN_TICK("layout");
        // ---- serialise ------------------------------------------------------------------------------------
        PlanHeader H;
        memset(&H, 0, sizeof(H));
        H.status = PLAN_ST_OK; H.nb = nb; H.n1 = n1; H.d = d; H.nnzF = nnzF; H.nA = nA; H.n_round = n_round;
        H.n_pass = n_pass; H.n_op = (int)ops.size();
        H.op_width = op_width_; H.n_oprow = n_oprow;
        H.n_zero = (int)zero.size();
        H.smem_bytes = plan_smem_bytes(nb, nl, nA, 2 * nld + 2 * g.n_gen, nsh);
        if (blk_) {
            H.blk = 1; H.blk_T = blk_T_; H.blk_U = blk_U_; H.blk_G = blk_G_; H.nblk = nblk; H.nblkA = nblkA; H.n_brow = n_brow;
            H.n_bpass = n_bpass; H.n_bzero = (int)bzero.size();
            H.smem_bytes = plan_block_smem_bytes(nb, nl, nblkA, 2 * nld + 2 * g.n_gen, nsh);
        }
        std::vector<unsigned char> blob(sizeof(PlanHeader));
        blob.reserve(sizeof(PlanHeader) + (size_t)n1 * n1 * 8 + ops.size() * 8 + (size_t)nl * 32 + (size_t)nb * 96 + 4096);
        auto align = [&](size_t a) { while (blob.size() % a) blob.push_back(0); };
        auto put_d = [&](const std::vector<double> &v) -> int {
            align(8);
            const int off = (int)blob.size();
            blob.resize(blob.size() + v.size() * 8);
            if (!v.empty()) memcpy(&blob[off], v.data(), v.size() * 8);
            return off;
        };
        auto put_u16 = [&](const std::vector<int> &v) -> int {
            align(4);
            const int off = (int)blob.size();
            blob.resize(blob.size() + v.size() * 2);
            uint16_t *dst = reinterpret_cast<uint16_t *>(blob.data() + off);
            for (size_t q = 0; q < v.size(); ++q) dst[q] = v[q] < 0 ? (uint16_t)0xFFFF : (uint16_t)v[q];
            return off;
        };
        auto put_u16v = [&](const std::vector<uint16_t> &v) -> int {
            align(4);
            const int off = (int)blob.size();
            blob.resize(blob.size() + v.size() * 2);
            if (!v.empty()) memcpy(&blob[off], v.data(), v.size() * 2);
            return off;
        };
        auto put_i32 = [&](const std::vector<int> &v) -> int {
            align(4);
            const int off = (int)blob.size();
            blob.resize(blob.size() + v.size() * 4);
            if (!v.empty()) memcpy(&blob[off], v.data(), v.size() * 4);
            return off;
        };
        auto put_csr = [&](const std::vector<std::vector<int>> &lists, int &o_ptr, int &o_idx) {
            std::vector<int> ptr(1, 0), idx;
            for (const auto &l : lists) { idx.insert(idx.end(), l.begin(), l.end()); ptr.push_back((int)idx.size()); }
            o_ptr = put_u16(ptr); o_idx = put_u16(idx);
        };
        H.o_qmins = put_d(qmins); H.o_qmaxs = put_d(qmaxs); H.o_ydiag = put_d(ydiag); H.o_dcshift = put_d(dcshift);
        H.o_dcinv = put_d(dcinv);
        {   // ops: 8-byte records
            align(8);
            H.o_ops = (int)blob.size();
            blob.resize(blob.size() + ops.size() * sizeof(Op));
            if (!ops.empty()) memcpy(&blob[H.o_ops], ops.data(), ops.size() * sizeof(Op));
        }
        H.o_pass_ptr = put_i32(pass_ptr);
        H.o_slot = put_u16(slot_of); H.o_btype = put_u16(btype); H.o_colth = put_u16(colth); H.o_colv = put_u16(colv);
        H.o_dcidx = put_u16(dcidx); H.o_vmunit = put_u16(vmunit); H.o_cnt = put_u16(cnt); H.o_nref = put_u16(nref);
        H.o_dpos = put_u16v(dpos);
        put_csr(adj, H.o_adj_ptr, H.o_adj); put_csr(bu, H.o_bu_ptr, H.o_bu); put_csr(bl, H.o_bl_ptr, H.o_bl);
        put_csr(bs, H.o_bs_ptr, H.o_bs); put_csr(bh, H.o_bh_ptr, H.o_bh);
        H.o_brf = put_u16(brf); H.o_brt = put_u16(brt);
        if (!blk_) { H.o_round = put_u16(round); H.o_jpos = put_u16v(jpos); }
        H.o_unit_bus = put_u16(unit_bus); H.o_load_bus = put_u16(load_bus); H.o_sto_bus = put_u16(sto_bus); H.o_sh_bus = put_u16(sh_bus);
        std::vector<int> shidx(nb, -1);
        {
            int n_shb = 0;
            for (int i = 0; i < nb; ++i) if (!bh[i].empty()) shidx[i] = n_shb++;
            H.o_shidx = put_u16(shidx); H.n_shb = n_shb;
        }
        if (!blk_) {
            std::vector<int> late;
            for (int r = 1; r < n_round; ++r) for (int l = 0; l < nl; ++l) if (brf[l] >= 0 && round[l] == r) { late.push_back(l); late.push_back(r); }
            H.o_late = put_u16(late); H.n_late = (int)late.size() / 2;
            H.o_zero = put_u16v(zero);
        }
        if (blk_) {
            align(8);
            H.o_bops = (int)blob.size();
            blob.resize(blob.size() + bops.size() * sizeof(BOp));
            if (!bops.empty()) memcpy(&blob[H.o_bops], bops.data(), bops.size() * sizeof(BOp));
            H.o_yval = put_d(yval);
            H.o_bdpos = put_u16(bdpos); H.o_bjpos = put_u16(bjpos); H.o_bzero = put_u16(bzero); H.o_bpass_ptr = put_i32(bpass_ptr);
            H.o_yptr = put_u16(yptr); H.o_ynb = put_u16(ynb); H.o_yblk = put_u16(yblk);
            const size_t ne = ynb.size();
            // (at least one entry: the kernel's first round of a bus pair reads entry 0 even when both rows are empty)
            std::vector<int> yword(ne > 0 ? ne : 1, 0), bdesc((size_t)nb * 2);
            std::vector<float> yf32(ne > 0 ? 2 * ne : 2, 0.f);
            for (size_t e = 0; e < ne; ++e) {
                yword[e] = (int)((unsigned)yblk[e] | (unsigned)ynb[e] << 16 | (colv[ynb[e]] >= 0 ? 1u << 31 : 0u));
                yf32[2 * e] = (float)yval[2 * e]; yf32[2 * e + 1] = (float)yval[2 * e + 1];
            }
            for (int i = 0; i < nb; ++i) {
                bdesc[(size_t)2 * i] = (int)((bdpos[i] < 0 ? 0xFFFFu : (unsigned)bdpos[i]) | (dcidx[i] < 0 ? 0xFFFFu : (unsigned)dcidx[i]) << 16);
                bdesc[(size_t)2 * i + 1] = (int)((shidx[i] < 0 ? 0xFFFFu : (unsigned)shidx[i]) | (colv[i] >= 0 ? 1u << 16 : 0u));
            }
            H.o_yword = put_i32(yword);
            align(8);                                                  // (uint2 / float2 loads)
            H.o_bdesc = put_i32(bdesc);
            H.o_yf32 = (int)blob.size();
            blob.resize(blob.size() + yf32.size() * 4);
            if (!yf32.empty()) memcpy(&blob[H.o_yf32], yf32.data(), yf32.size() * 4);
        }
        PLAN_TICK("serialise");
        align(16);
        H.total_bytes = (int)blob.size();
        memcpy(blob.data(), &H, sizeof(H));
        return blob;
    }

    // the plan format addresses values and list entries with 16 bits
    static bool fits(const PlanHeader &H) {
        if (H.blk) return (size_t)(H.nblkA + 1) * 16 * (size_t)H.blk_G <= 0xFFFF && H.nb < 0x8000;
        return H.nA + 1 < 0x3FFF && H.n_op < (1 << 30);
    }

private:
    const HostGrid &g_;
    int op_width_;
    bool optimize_layout_;
    int order_seed_;      // 0: deterministic tie-breaking of the elimination order; > 0: randomised ties (plan search)
    int blk_ = 0, blk_T_ = 32, blk_U_ = 1, blk_G_ = 1;
};

// Plan for a topology that many solves will re-use (batched launches): the elimination order's ties are broken in
// `n_seeds` different ways, the variant whose operation stream needs the fewest rows (then the fewest operations) wins —
// case14: 29 -> 25 rows, 36 substations: 48 -> 43 — and gets the bank-conflict-aware layout.  Deterministic (fixed seeds).
inline std::vector<unsigned char> build_plan_searched(const HostGrid &g, int op_width, const int8_t *tv, int outage, int n_seeds,
                                                      int blk_T = 0, int blk_U = 1) {
    int best_seed = 0;
    long best_cost = -1;
    for (int seed = 0; seed < n_seeds; ++seed) {
        PlanBuilder pb(g, op_width, false, seed);
        if (blk_T > 0) pb.block_mode(blk_T, blk_U);
        const std::vector<unsigned char> blob = pb.build(tv, outage);
        const PlanHeader *H = reinterpret_cast<const PlanHeader *>(blob.data());
        if (H->status != PLAN_ST_OK) return blob;                       // nothing to optimise
        const long cost = blk_T > 0 ? (long)H->n_brow * 100000L + H->nblk : (long)H->n_oprow * 100000L + H->nnzF;
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_seed = seed; }
    }
    PlanBuilder pb(g, op_width, blk_T <= 0, best_seed);
    if (blk_T > 0) pb.block_mode(blk_T, blk_U);
    return pb.build(tv, outage);
}

}  // namespace b200pf

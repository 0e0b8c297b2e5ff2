// TEST INFRASTRUCTURE (never part of the product): the block plan builder of grid2op_b200/csrc/b200pf_plan.hpp on the host,
// so that tests can read a plan blob's arrays (tests/test_block_ybus_cpu.py: the admittance rows against a dense Ybus).
#include "../../grid2op_b200/csrc/b200pf_plan.hpp"
#include "../../include/b200pf.h"

using namespace b200pf;

static HostGrid host_grid(const b200pf_grid_desc *gd) {
    HostGrid g;
    g.n_sub = gd->n_sub; g.n_busbar = gd->n_busbar; g.n_slot = gd->n_sub * gd->n_busbar; g.n_line = gd->n_line;
    g.n_gen = gd->n_gen; g.n_hidden = gd->n_hidden; g.n_unit = gd->n_gen + gd->n_hidden; g.n_load = gd->n_load;
    g.n_sto = gd->n_storage; g.n_shunt = gd->n_shunt; g.dim_topo = gd->dim_topo;
    g.n_topo_in = g.dim_topo + g.n_shunt + g.n_hidden; g.base_mva = gd->sn_mva;
#define CP(dst, src, n) g.dst.assign(gd->src, gd->src + (n))
    CP(line_or_sub, line_or_sub, g.n_line); CP(line_ex_sub, line_ex_sub, g.n_line); CP(line_or_pos, line_or_pos, g.n_line);
    CP(line_ex_pos, line_ex_pos, g.n_line); CP(line_y, line_y, 8 * g.n_line); CP(line_bdc, line_bdc, g.n_line);
    CP(line_pshift, line_pshift, g.n_line); CP(unit_sub, unit_sub, g.n_unit); CP(unit_pos, unit_pos, g.n_unit);
    CP(unit_is_ref, unit_is_ref, g.n_unit); CP(unit_qmin, unit_qmin, g.n_unit); CP(unit_qmax, unit_qmax, g.n_unit);
    CP(load_sub, load_sub, g.n_load); CP(load_pos, load_pos, g.n_load); CP(sto_sub, storage_sub, g.n_sto);
    CP(sto_pos, storage_pos, g.n_sto); CP(sh_sub, shunt_sub, g.n_shunt);
#undef CP
    return g;
}

// Builds the block plan of one topology record for (T, U) into buf (cap bytes); returns the blob size (or -size when cap is too
// small).  fields[0..17]: status, nb, n1, nblk, nblkA, blk_G, n_bzero, and the byte offsets o_yptr, o_ynb, o_yval, o_yblk,
// o_ydiag, o_dcidx, o_bdpos, o_bjpos, o_bzero, o_brf, o_brt.
extern "C" int plan_rows_block(const b200pf_grid_desc *gd, const int8_t *topo, int outage, int T, int U, unsigned char *buf, int cap,
                               int32_t *fields) {
    HostGrid hg = host_grid(gd);
    PlanBuilder pb(hg, 32);
    pb.block_mode(T, U);
    const std::vector<unsigned char> blob = pb.build(topo, outage);
    const PlanHeader &H = *reinterpret_cast<const PlanHeader *>(blob.data());
    const int32_t f[18] = {H.status, H.nb, H.n1, H.nblk, H.nblkA, H.blk_G, H.n_bzero, H.o_yptr, H.o_ynb, H.o_yval, H.o_yblk,
                           H.o_ydiag, H.o_dcidx, H.o_bdpos, H.o_bjpos, H.o_bzero, H.o_brf, H.o_brt};
    for (int k = 0; k < 18; ++k) fields[k] = f[k];
    if ((int)blob.size() > cap) return -(int)blob.size();
    memcpy(buf, blob.data(), blob.size());
    return (int)blob.size();
}

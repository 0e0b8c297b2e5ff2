// TEST INFRASTRUCTURE (never part of the product): the block plan builder of grid2op_b200/csrc/b200pf_plan.hpp on the host,
// so that tests can read the packed words of the bus phase next to the arrays they are packed from
// (tests/test_bus_chains_cpu.py).
#include "plan_rows.cpp"

// Same as plan_rows_block; fields[0..8]: status, nb, n_entries (yptr[nb]), and the byte offsets o_yword, o_yf32, o_bdesc,
// o_colv, o_shidx, o_yptr.
extern "C" int plan_bus_words(const b200pf_grid_desc *gd, const int8_t *topo, int outage, int T, int U, unsigned char *buf, int cap,
                              int32_t *fields) {
    HostGrid hg = host_grid(gd);
    PlanBuilder pb(hg, 32);
    pb.block_mode(T, U);
    const std::vector<unsigned char> blob = pb.build(topo, outage);
    const PlanHeader &H = *reinterpret_cast<const PlanHeader *>(blob.data());
    const int ne = H.status == PLAN_ST_OK ? reinterpret_cast<const uint16_t *>(blob.data() + H.o_yptr)[H.nb] : 0;
    const int32_t f[9] = {H.status, H.nb, ne, H.o_yword, H.o_yf32, H.o_bdesc, H.o_colv, H.o_shidx, H.o_yptr};
    for (int k = 0; k < 9; ++k) fields[k] = f[k];
    if ((int)blob.size() > cap) return -(int)blob.size();
    memcpy(buf, blob.data(), blob.size());
    return (int)blob.size();
}

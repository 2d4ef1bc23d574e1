/* chain_emul_extend.cpp -- TEST INFRASTRUCTURE: chain_emul.cpp plus the extend-mode fuse of abpoa_b200/csrc/poa_chain.cuh
 * (chain_fuse's KO instantiation: the reference's Kahn order, chain_kahn_order, instead of the splice), compiled for the
 * host into its own library.  Nothing in the product links this file. */
#include "chain_emul.cpp"

/* chain_emul_fuse on the extend runs' instantiation */
extern "C" int chain_emul_x_fuse(Emul *e, const uint64_t *ops, int n_ops, int best_score, int64_t cells) {
    memcpy(e->s.jd.cigar, ops, (size_t)n_ops * 8);
    PoaResultDev *res = e->s.jd.result;
    memset(res, 0, sizeof *res);
    res->status = POA_ST_OK; res->n_ops = n_ops; res->best_score = best_score; res->cells = cells;
    chain_fuse<false, false, true>(&e->s, &e->cp, e->s.fused);
    return e->s.failed;
}
/* the Kahn walk alone on the current graph, into a caller's buffer (order) -- and the current order untouched */
extern "C" int chain_emul_kahn(Emul *e, int32_t *order) {
    std::vector<int32_t> row((size_t)e->s.n_nodes);
    memcpy(row.data(), e->s.node_row, row.size() * 4);
    chain_kahn_order(&e->s, &e->cp, order, e->s.n_nodes);
    memcpy(e->s.node_row, row.data(), row.size() * 4);
    return e->s.failed;
}

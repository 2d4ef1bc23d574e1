/* chain_emul_msa.cpp -- TEST INFRASTRUCTURE: chain_emul.cpp plus the RC-MSA part of abpoa_b200/csrc/poa_chain.cuh
 * (per-node read sets, chain_msa_rank, chain_msa_rows), compiled for the host into its own library so that the CPU
 * suite can compare it with the host graph layer.  Nothing in the product links this file. */
#include "chain_emul.cpp"

/* RC-MSA on: W words per read set (poisoned, nothing may rely on zeroed memory); call before chain_emul_seed */
extern "C" void chain_emul_enable_msa(Emul *e, int W) {
    e->cp.W = W;
    const size_t n = (size_t)e->s.n_cap * W;
    e->s.read_set = (uint64_t *)malloc(n * sizeof(uint64_t) + 8);
    for (size_t i = 0; i < n; ++i) e->s.read_set[i] = 0xcdcdcdcdcdcdcdcdull;
}
extern "C" void chain_emul_msa_free(Emul *e) { free(e->s.read_set); chain_emul_free(e); }
extern "C" const uint64_t *chain_emul_read_set(Emul *e) { return e->s.read_set; }
extern "C" const int32_t *chain_emul_msa_ranks(Emul *e) { return e->s.scr[5]; }
/* ranks + rows after the last read, as poa_chain_msa_kernel runs them (with_cons: chain_consensus first, for its path);
 * returns msa_len (-1: no MSA, -2: `rows` holds fewer than (n_reads + with_cons) * msa_len bytes) */
extern "C" int chain_emul_msa(Emul *e, int with_cons, uint8_t *rows, int64_t cap) {
    if (with_cons) { std::vector<int32_t> tmp((size_t)e->s.n_cap + 1); chain_consensus(&e->s, &e->cp, tmp.data(), e->s.n_cap); }
    const int msa_len = chain_msa_rank(&e->s, &e->cp);
    if (msa_len < 0) return -1;
    if ((int64_t)(e->s.n_reads + with_cons) * msa_len > cap) return -2;
    chain_msa_rows(&e->s, &e->cp, msa_len, with_cons, rows);
    return msa_len;
}

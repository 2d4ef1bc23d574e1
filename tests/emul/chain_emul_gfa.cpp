/* chain_emul_gfa.cpp -- TEST INFRASTRUCTURE: chain_emul.cpp plus the GFA part of abpoa_b200/csrc/poa_chain.cuh
 * (chain_gfa_order, chain_gfa_size, chain_gfa_record), compiled for the host into its own library so that the CPU suite
 * can format the device record with the product's formatter and compare it with the host writer.  Nothing in the
 * product links this file. */
#include "chain_emul.cpp"

extern "C" const int32_t *chain_emul_gfa_queue(Emul *e) { return e->s.scr[4]; }
/* the record after the last read, as poa_chain_gfa_kernel writes it (with_cons: chain_consensus first, for its path);
 * returns its size in int32 words (-1: no record, -2: `rec` holds fewer than that many words) */
extern "C" int64_t chain_emul_gfa(Emul *e, int with_cons, int32_t *rec, int64_t cap) {
    if (with_cons) { std::vector<int32_t> tmp((size_t)e->s.n_cap + 1); chain_consensus(&e->s, &e->cp, tmp.data(), e->s.n_cap); }
    int32_t hdr[POA_GFA_HDR_WORDS];
    const int64_t words = chain_gfa_size(&e->s, &e->cp, with_cons, hdr);
    if (words < 0) return -1;
    if (words > cap) return -2;
    chain_gfa_record(&e->s, &e->cp, hdr, rec);
    return words;
}

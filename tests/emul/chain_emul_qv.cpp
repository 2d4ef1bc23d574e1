/* chain_emul_qv.cpp -- TEST INFRASTRUCTURE: chain_emul_strand.cpp plus what -Q (use_qv) adds to
 * abpoa_b200/csrc/poa_chain.cuh: the per-base weight bytes that chain_seed and chain_fuse add to the edges
 * (chain_read_weight), and the reads region with them.  Compiled for the host into its own library.  Nothing in the
 * product links this file. */
#include "chain_emul_strand.cpp"

/* -Q: one weight byte per read base at the reads' offsets, owned by the caller; NULL: unit weights */
extern "C" void chain_emul_set_read_qw(Emul *e, const uint8_t *read_qw) { e->s.read_qw = read_qw; }

/* chain_slot_reads with and without the weight bytes: every request of a run without -Q weights must be the same, and the
 * weights (one byte per base) must come behind them; a slot laid out without them has no weights.  Returns 0, or the index
 * of the first request that breaks it. */
extern "C" int chain_emul_reads_layout_check(int n_reads, int64_t bases) {
    std::vector<size_t> plain, qv;
    PoaChainSlot s; memset(&s, 0, sizeof s);
    chain_slot_reads(&s, n_reads, bases, [&](size_t b) { plain.push_back(b); return (uint8_t *)NULL; });
    if (s.read_qw) return -1;
    chain_slot_reads(&s, n_reads, bases, [&](size_t b) { qv.push_back(b); return (uint8_t *)&s; }, true);
    for (size_t k = 0; k < plain.size(); ++k) if (k >= qv.size() || plain[k] != qv[k]) return (int)k + 1;
    if (qv.size() != plain.size() + 1 || qv.back() != (size_t)bases || !s.read_qw) return (int)qv.size() + 1;
    return 0;
}

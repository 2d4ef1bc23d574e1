/* chain_emul_strand.cpp -- TEST INFRASTRUCTURE: chain_emul.cpp plus what -s (amb_strand) adds to
 * abpoa_b200/csrc/poa_chain.cuh: the weak-hit predicate the alignment warp uses, the per-read strand bytes that
 * chain_fuse reads its bases through (chain_read_base), and the slot layout with the strand arrays.  Compiled for the
 * host into its own library.  Nothing in the product links this file. */
#include "chain_emul.cpp"

/* the alignment warp's test (poa_kernels.cu: chain_align_read) */
extern "C" int chain_emul_weak_hit(int best_score, int qlen, int node_n, int max_mat) { return chain_weak_hit(best_score, qlen, node_n, max_mat); }

/* -s: the slot's strand bytes, one per read (bit 0: fused as the reverse complement), owned by the caller */
extern "C" void chain_emul_set_read_rc(Emul *e, uint8_t *read_rc) { e->s.read_rc = read_rc; }

/* the -r 1 / -r 2 rows (with_cons: after the heaviest-bundling consensus row) after the last read, as poa_chain_msa_kernel
 * writes them; returns msa_len (-1: no MSA, -2: `rows` holds too few bytes) */
extern "C" int chain_emul_msa(Emul *e, int with_cons, uint8_t *rows, int64_t cap) {
    if (with_cons) { std::vector<int32_t> tmp((size_t)e->s.n_cap + 1); chain_consensus(&e->s, &e->cp, tmp.data(), e->s.n_cap); if (tmp[0] < 0) return -1; }
    const int msa_len = chain_msa_rank(&e->s, &e->cp);
    if (msa_len < 0) return -1;
    if ((int64_t)(e->s.n_reads + with_cons) * msa_len > cap) return -2;
    chain_msa_rows(&e->s, &e->cp, msa_len, with_cons, rows);
    return msa_len;
}
/* the -r 3 / -r 4 GFA record after the last read, as poa_chain_gfa_kernel writes it; returns its size in int32 words
 * (-1: no record, -2: `rec` holds fewer than that many words) */
extern "C" int64_t chain_emul_gfa(Emul *e, int with_cons, int32_t *rec, int64_t cap) {
    if (with_cons) { std::vector<int32_t> tmp((size_t)e->s.n_cap + 1); chain_consensus(&e->s, &e->cp, tmp.data(), e->s.n_cap); if (tmp[0] < 0) return -1; }
    int32_t hdr[POA_GFA_HDR_WORDS];
    const int64_t words = chain_gfa_size(&e->s, &e->cp, with_cons, hdr);
    if (words < 0) return -1;
    if (words > cap) return -2;
    chain_gfa_record(&e->s, &e->cp, hdr, rec);
    return words;
}

/* chain_slot_layout with and without the strand arrays: every request up to the last one of a run without -s must be the
 * same (offset and size), and the three strand arrays must come behind it.  Returns 0, or the index of the first
 * request that breaks it. */
extern "C" int chain_emul_layout_check(int n_cap, int qmax, int n_reads, int K, int A, int m, int W, int record) {
    std::vector<size_t> plain, strand;
    PoaChainSlot s;
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, record != 0, [&](size_t b) { plain.push_back(b); return (uint8_t *)NULL; });
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, record != 0, [&](size_t b) { strand.push_back(b); return (uint8_t *)NULL; }, true);
    for (size_t k = 0; k < plain.size(); ++k) if (k >= strand.size() || plain[k] != strand[k]) return (int)k + 1;
    if (strand.size() != plain.size() + 3) return (int)strand.size() + 1;
    const size_t want[3] = { (size_t)n_reads, (size_t)s.jd.cigar_cap * 8, sizeof(PoaResultDev) };
    for (int k = 0; k < 3; ++k) if (strand[plain.size() + k] != want[k]) return (int)(plain.size() + k) + 1;
    return 0;
}

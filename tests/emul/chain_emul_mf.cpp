/* chain_emul_mf.cpp -- TEST INFRASTRUCTURE: chain_emul.cpp plus the most-frequent-base consensus of
 * abpoa_b200/csrc/poa_chain.cuh (chain_mf_consensus through chain_cons_path), compiled for the host into its own library
 * so that the CPU suite can compare the device record, its path, the -r 2 consensus row and the GFA consensus path with
 * the host's most_frequent.  Nothing in the product links this file. */
#include "chain_emul.cpp"

/* the record after the last read, as poa_chain_consensus_kernel writes it with -a 1; returns its length (-1: none) */
extern "C" int chain_emul_mf(Emul *e, int32_t *out, int cap) {
    e->cp.cons_algrm = 1;
    chain_cons_path(&e->s, &e->cp, out, cap);
    return out[0];
}
/* the consensus path the record left in scr[1]: node ids into `ids`, returns their number (-1: longer than cap) */
extern "C" int chain_emul_cons_path(Emul *e, int32_t *ids, int cap) {
    const int32_t *nxt = e->s.scr[1];
    int len = 0;
    for (int cur = nxt[0]; cur != 1 && cur >= 0; cur = nxt[cur]) { if (len >= cap) return -1; ids[len++] = cur; }
    return len;
}
/* What the vote relies on, on the ranks chain_msa_rank left in scr[5]: every aligned set shares one rank, its bases are
 * pairwise distinct, and no two sets share a rank.  Returns 0, or the first node id that breaks it. */
extern "C" int chain_emul_mf_check_columns(Emul *e) {
    const PoaChainSlot &s = e->s;
    const int A = e->cp.A, n = s.n_nodes;
    const int32_t *rank = s.scr[5];
    std::vector<int> owner((size_t)n + 2, -1);
    for (int v = 2; v < n; ++v) {
        const int32_t *al = s.aln_id + (size_t)v * A;
        int lead = v;
        for (int a = 0; a < s.aln_cnt[v]; ++a) {
            if (rank[al[a]] != rank[v] || s.base[al[a]] == s.base[v]) return v;
            if (al[a] < lead) lead = al[a];
        }
        if (rank[v] < 1 || rank[v] > n) return v;
        if (owner[rank[v]] < 0) owner[rank[v]] = lead;
        else if (owner[rank[v]] != lead) return v;
    }
    return 0;
}
/* the -r 2 rows after the last read, as poa_chain_msa_kernel writes them behind the -a 1 consensus kernel; returns msa_len
 * (-1: no MSA, -2: `rows` holds fewer than (n_reads + 1) * msa_len bytes) */
extern "C" int chain_emul_mf_msa(Emul *e, uint8_t *rows, int64_t cap) {
    std::vector<int32_t> tmp((size_t)e->s.n_cap + 1);
    if (chain_emul_mf(e, tmp.data(), e->s.n_cap) < 0) return -1;
    const int msa_len = chain_msa_rank(&e->s, &e->cp);
    if (msa_len < 0) return -1;
    if ((int64_t)(e->s.n_reads + 1) * msa_len > cap) return -2;
    chain_msa_rows(&e->s, &e->cp, msa_len, 1, rows);
    return msa_len;
}
/* the -r 4 GFA record after the last read, as poa_chain_gfa_kernel writes it behind the -a 1 consensus kernel; returns its
 * size in int32 words (-1: no record, -2: `rec` holds fewer than that many words) */
extern "C" int64_t chain_emul_mf_gfa(Emul *e, int32_t *rec, int64_t cap) {
    std::vector<int32_t> tmp((size_t)e->s.n_cap + 1);
    if (chain_emul_mf(e, tmp.data(), e->s.n_cap) < 0) return -1;
    int32_t hdr[POA_GFA_HDR_WORDS];
    const int64_t words = chain_gfa_size(&e->s, &e->cp, 1, hdr);
    if (words < 0) return -1;
    if (words > cap) return -2;
    chain_gfa_record(&e->s, &e->cp, hdr, rec);
    return words;
}

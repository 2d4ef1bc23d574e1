/* chain_emul_ps.cpp -- TEST INFRASTRUCTURE: chain_emul_qv.cpp plus what -G (inc_path_score) adds to
 * abpoa_b200/csrc/poa_chain.cuh: the predscore section chain_flatten writes into the job blob (chain_path_score of every
 * in-edge), and the room chain_slot_layout makes for it.  Compiled for the host into its own library.  Nothing in the
 * product links this file. */
#include "chain_emul_qv.cpp"

/* chain_emul_new with -G on: the slot laid out with room for the predscore section (drive it with chain_emul_ps_seed /
 * chain_emul_ps_fuse) */
extern "C" Emul *chain_emul_ps_new(int n_reads, const int32_t *lens, const uint8_t *const *seqs, const int32_t *w, int n_cap, int K, int A,
                                   int m, int max_mat, int min_mis, int o1, int e1, int oe1, int oe2, int W) {
    Emul *e = new Emul();
    memset(&e->s, 0, sizeof e->s); memset(&e->cp, 0, sizeof e->cp);
    e->cp.K = K; e->cp.A = A; e->cp.m = m; e->cp.max_mat = max_mat; e->cp.min_mis = min_mis; e->cp.o1 = o1; e->cp.e1 = e1; e->cp.oe1 = oe1; e->cp.oe2 = oe2; e->cp.record = 1;
    e->cp.W = W;
    int qmax = 1; int64_t bases = 0;
    for (int i = 0; i < n_reads; ++i) { bases += lens[i]; if (lens[i] > qmax) qmax = lens[i]; }
    PoaChainSlot &s = e->s;
    size_t bytes = 0;
    auto count = [&](size_t b) { bytes += (b + 15) & ~(size_t)15; return (uint8_t *)NULL; };
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, true, count, false, true);
    chain_slot_reads(&s, n_reads, bases, count);
    e->mem.assign(bytes, 0xcd);                            /* poison: nothing may rely on zeroed memory */
    uint8_t *p = e->mem.data();
    auto take = [&](size_t b) { uint8_t *q = p; p += (b + 15) & ~(size_t)15; return q; };
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, true, take, false, true);
    chain_slot_reads(&s, n_reads, bases, take);
    uint8_t *reads = const_cast<uint8_t *>(s.reads);
    int32_t *off = const_cast<int32_t *>(s.read_off), *rw = const_cast<int32_t *>(s.read_w);
    off[0] = 0;
    for (int i = 0; i < n_reads; ++i) { memcpy(reads + off[i], seqs[i], (size_t)lens[i]); off[i + 1] = off[i] + lens[i]; rw[i] = w[i]; }
    return e;
}

/* chain_emul_seed / chain_emul_fuse on the path-score instantiation of the graph code (every job flattened with scores) */
extern "C" void chain_emul_ps_seed(Emul *e) { chain_seed<true>(&e->s, &e->cp); }
extern "C" int chain_emul_ps_fuse(Emul *e, const uint64_t *ops, int n_ops, int best_score, int64_t cells) {
    memcpy(e->s.jd.cigar, ops, (size_t)n_ops * 8);
    PoaResultDev *res = e->s.jd.result;
    memset(res, 0, sizeof *res);
    res->status = POA_ST_OK; res->n_ops = n_ops; res->best_score = best_score; res->cells = cells;
    chain_fuse<true>(&e->s, &e->cp, e->s.fused);
    return e->s.failed;
}

/* the shared score function (chain_path_score) on n pairs */
extern "C" void chain_emul_path_scores(const int32_t *edge_w, const int32_t *node_w, int n, int32_t *out) {
    for (int i = 0; i < n; ++i) out[i] = chain_path_score(edge_w[i], node_w[i]);
}

/* chain_slot_layout with and without -G, with and without -s: without -G every request is the one of the old call; with
 * it only the job blob grows, by one int per predecessor slot plus the section's padding.  Returns 0, or the index of the
 * first request that breaks it. */
extern "C" int chain_emul_ps_layout_check(int n_cap, int qmax, int n_reads, int K, int A, int m, int W, int record, int strand) {
    std::vector<size_t> old_, plain, ps;
    PoaChainSlot s0, s1, s2;
    chain_slot_layout(&s0, n_cap, qmax, n_reads, K, A, m, W, record != 0, [&](size_t b) { old_.push_back(b); return (uint8_t *)NULL; }, strand != 0);
    chain_slot_layout(&s1, n_cap, qmax, n_reads, K, A, m, W, record != 0, [&](size_t b) { plain.push_back(b); return (uint8_t *)NULL; }, strand != 0, false);
    chain_slot_layout(&s2, n_cap, qmax, n_reads, K, A, m, W, record != 0, [&](size_t b) { ps.push_back(b); return (uint8_t *)NULL; }, strand != 0, true);
    if (old_ != plain || s0.blob_cap != s1.blob_cap) return -1;
    if (ps.size() != plain.size()) return -2;
    const size_t grow = (size_t)s1.pred_cap * 4 + 4 + 16;
    if ((size_t)s2.blob_cap != (size_t)s1.blob_cap + grow) return -3;
    for (size_t k = 0; k < plain.size(); ++k) {
        const bool blob = plain[k] == (size_t)s1.blob_cap && ps[k] == (size_t)s2.blob_cap;
        if (ps[k] != plain[k] && !blob) return (int)k + 1;
    }
    return 0;
}

/* chain_emul.cpp -- TEST INFRASTRUCTURE: the device-side graph code of abpoa_b200/csrc/poa_chain.cuh compiled
 * for the host (-DPOA_CHAIN_EMUL: PAR_FOR = plain loop, barrier = nothing) behind a tiny C interface, so that
 * the CPU suite can drive it read by read next to the host graph layer (poa_graph.c / poa_flat.c) and compare
 * every array.  Nothing in the product links this file. */
#define POA_CHAIN_EMUL 1
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "poa_chain.cuh"

struct Emul {
    PoaChainSlot s; PoaChainParams cp;
    std::vector<uint8_t> mem;                              /* the group's arrays and reads, laid out by chain_slot_layout / chain_slot_reads */
};

/* W > 0: RC-MSA on, W words per read set */
extern "C" Emul *chain_emul_new(int n_reads, const int32_t *lens, const uint8_t *const *seqs, const int32_t *w, int n_cap, int K, int A,
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
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, true, count);
    chain_slot_reads(&s, n_reads, bases, count);
    e->mem.assign(bytes, 0xcd);                            /* poison: nothing may rely on zeroed memory */
    uint8_t *p = e->mem.data();
    auto take = [&](size_t b) { uint8_t *q = p; p += (b + 15) & ~(size_t)15; return q; };
    chain_slot_layout(&s, n_cap, qmax, n_reads, K, A, m, W, true, take);
    chain_slot_reads(&s, n_reads, bases, take);
    uint8_t *reads = const_cast<uint8_t *>(s.reads);
    int32_t *off = const_cast<int32_t *>(s.read_off), *rw = const_cast<int32_t *>(s.read_w);
    off[0] = 0;
    for (int i = 0; i < n_reads; ++i) { memcpy(reads + off[i], seqs[i], (size_t)lens[i]); off[i + 1] = off[i] + lens[i]; rw[i] = w[i]; }
    return e;
}
extern "C" void chain_emul_free(Emul *e) { delete e; }
extern "C" void chain_emul_seed(Emul *e) { chain_seed(&e->s, &e->cp); }
/* ops: graph-CIGAR words in BACKTRACK order with DP rows (what the alignment kernel leaves in jd.cigar) */
extern "C" int chain_emul_fuse(Emul *e, const uint64_t *ops, int n_ops, int best_score, int64_t cells) {
    memcpy(e->s.jd.cigar, ops, (size_t)n_ops * 8);
    PoaResultDev *res = e->s.jd.result;                    /* what the alignment kernel reports */
    memset(res, 0, sizeof *res);
    res->status = POA_ST_OK; res->n_ops = n_ops; res->best_score = best_score; res->cells = cells;
    chain_fuse(&e->s, &e->cp, e->s.fused);
    return e->s.failed;
}
extern "C" const PoaChainSlot *chain_emul_slot(Emul *e) { return &e->s; }
extern "C" int chain_emul_n_nodes(Emul *e) { return e->s.n_nodes; }
extern "C" int chain_emul_failed(Emul *e) { return e->s.failed; }
extern "C" const int32_t *chain_emul_array(Emul *e, int which) {
    PoaChainSlot &s = e->s;
    switch (which) {
    case 0: return s.in_cnt; case 1: return s.out_cnt; case 2: return s.aln_cnt; case 3: return s.n_read;
    case 4: return s.in_id; case 5: return s.in_w; case 6: return s.out_id; case 7: return s.out_w; case 8: return s.aln_id;
    case 9: return s.order[s.cur]; case 10: return s.node_row; case 11: return s.rem_row;
    case 12: return s.rec_score; case 13: return s.rec_nops;
    }
    return NULL;
}
extern "C" const uint8_t *chain_emul_bases(Emul *e) { return e->s.base; }
extern "C" const uint8_t *chain_emul_blob(Emul *e) { return e->s.jd.blob; }
extern "C" const uint64_t *chain_emul_hashes(Emul *e) { return e->s.rec_hash; }
extern "C" int64_t chain_emul_cells(Emul *e) { return e->s.cells; }
extern "C" int chain_emul_consensus(Emul *e, int32_t *out, int cap) { chain_consensus(&e->s, &e->cp, out, cap); return out[0]; }

/* poa_chain.cuh -- the partial-order graph ON THE DEVICE: fusing a graph-CIGAR, keeping the
 * topological order, the edge order and the band centre, and flattening the graph into the
 * next alignment job, all without a host round trip (SURVEY 8f row f1).
 *
 * What is reproduced (same observable graph, node id for node id, as the host layer in
 * poa_graph.c, which is pinned to the reference):
 *   abpoa_add_subgraph_alignment   reference src/abpoa_graph.c:689-774   (whole graph, inc_both_ends)
 *   abpoa_add_graph_edge           reference src/abpoa_graph.c:480-556
 *   aligned-node sets              reference src/abpoa_graph.c:439-463
 *   edge order (exchange pass)     reference src/abpoa_graph.c:192-219
 *   max_remain                     reference src/abpoa_graph.c:268-309
 *   pre_index / query set-up       reference src/abpoa_align_simd.c:463-560
 * The topological order is the SPLICED order of poa_graph.c in global mode (the DP result does not
 * depend on which topological order the rows follow), and the reference's FIFO Kahn order in extend
 * mode (chain_kahn_order: the best cell and the z-drop stop are the first row in row order that meets them).
 *
 * How it is written: one CTA per read group; the body is a sequence of data-parallel PHASES
 * (POA_PAR_FOR loops separated by CTA barriers) plus block scans.  A read's path visits every
 * node at most once, so "item qi" (query base qi) owns the in-list of its target node and the
 * out-list of the previous target: all list updates of one read are conflict-free.
 * The same source compiles for the host with -DPOA_CHAIN_EMUL (PAR_FOR = plain loop, barrier =
 * nothing), which is how tests/ pins this logic on the CPU against poa_graph.c / poa_flat.c.
 */
#ifndef POA_CHAIN_CUH
#define POA_CHAIN_CUH

#include <math.h>
#include <stdint.h>
#include "poa_device.cuh"

#ifdef POA_CHAIN_EMUL
#define POA_DEV static inline
#define POA_PAR_FOR(i, n) for (int i = 0; i < (n); ++i)
#define POA_CTA_SYNC() do { } while (0)
#define POA_TID0 1
#define POA_SHARED static
#define POA_ATOMIC_OR(p, v) (*(p) |= (v))
#define POA_CTZ64(x) __builtin_ctzll(x)
#define POA_CHAIN_T 256
#else
#define POA_DEV __device__ __forceinline__
#define POA_PAR_FOR(i, n) for (int i = (int)threadIdx.x; i < (n); i += (int)blockDim.x)
#define POA_CTA_SYNC() __syncthreads()
#define POA_TID0 (threadIdx.x == 0)
#define POA_SHARED __shared__
#define POA_ATOMIC_OR(p, v) atomicOr((p), (v))
#define POA_CTZ64(x) (__ffsll((long long)(x)) - 1)
#define POA_CHAIN_T 256                 /* threads per CTA of the fuse kernel */
#endif

/* why a group left the device chain (it is then finished by the host-path engine) */
#define POA_CF_NODE_CAP   0x01          /* node capacity of the slot exhausted            */
#define POA_CF_EDGE_CAP   0x02          /* a node needs more than K in- or out-edges       */
#define POA_CF_ALN_CAP    0x04          /* an aligned set needs more than A members        */
#define POA_CF_ORDER      0x08          /* the spliced / Kahn order would not be topological */
#define POA_CF_BLOB_CAP   0x10          /* flattened job does not fit the slot's blob      */
#define POA_CF_DP_STATUS  0x20          /* the DP kernel reported RANGE / PLANE_OVF / ...  */
#define POA_CF_CIGAR      0x40          /* graph-CIGAR inconsistent with the read          */
#define POA_CF_POOL       0x80          /* the round's plane pool is exhausted             */

#define POA_ST_SKIP       9             /* DP kernel: the slot has no job this round       */

typedef struct PoaChainParams {         /* one per batch call */
    int32_t K, A;                       /* inline edge slots per node and direction / aligned-set slots */
    int32_t m, max_mat, min_mis, o1, e1, oe1, oe2;      /* for the reference's score-width rule (pn) */
    int32_t record;                     /* keep per-read score / CIGAR length / FNV-1a hash */
    int32_t P;                          /* plane units per 8-cell group of a DP row (compact layout:
                                           H and the E planes; 1 / 2 / 3) */
    int32_t W;                          /* 64-bit words per read set (ceil(n_reads / 64) of the largest group); 0: no RC-MSA */
    int32_t cons_algrm;                 /* consensus: 0 heaviest bundling (ABPOA_HB), 1 most frequent base (ABPOA_MF) */
    int32_t amb_strand;                 /* -s: a weak forward hit is re-aligned as the reverse complement (chain_weak_hit) */
} PoaChainParams;

typedef struct PoaChainSlot {           /* one per read group; every pointer aims into the group's HBM region */
    /* graph, indexed by node id */
    int32_t n_nodes, n_cap, pred_cap, blob_cap;
    int32_t failed;                     /* POA_CF_* bits; non-zero: the slot is inert       */
    int32_t n_reads, fused;             /* reads of the group / reads already in the graph  */
    int32_t retry;                      /* the pending job is the generous re-run of an alignment whose band outgrew its plane slab */
    int32_t cur;                        /* which of order[2] is current                     */
    int64_t cells;                      /* DP cells of all alignments so far                */
    int64_t fwd_clk, bt_clk;            /* SM cycles of the forward DP / the backtrace, summed over the alignments */
    uint8_t *base;
    int32_t *in_cnt, *out_cnt, *aln_cnt, *n_read;
    int32_t *in_id, *in_w, *out_id, *out_w;             /* [n_cap * K] */
    int32_t *aln_id;                                    /* [n_cap * A] */
    int32_t *order[2];                  /* row -> node                                      */
    int32_t *node_row;                  /* node -> row                                      */
    int32_t *rem_row;                   /* row -> max_remain                                */
    int32_t *scr[6];                    /* scratch, each max(q_cap + 2, n_cap) ints         */
    /* reads of the group, concatenated */
    const uint8_t *reads; const int32_t *read_off;      /* [n_reads + 1] */
    const int32_t *read_w;                              /* [n_reads] band half width w per read */
    /* the alignment job the DP kernel runs for this slot */
    PoaJobDesc jd;
    /* score planes live only while an alignment runs: every round the jobs of a cohort carve theirs out of one
     * pool (exact size: rows x band estimate x planes).  Two cursors alternate by round parity -- the DP kernel of
     * round r zeroes the one the fuse kernel of round r fills for round r + 1 -- over the SAME memory. */
    uint8_t *pool_base; unsigned long long *pool_cursor; uint64_t pool_units;
    /* free-running mode (no rounds): pool_cursor == NULL, [pool_base, pool_units) is the group's PRIVATE plane slab, and the
     * alignment warp and the fuse workers hand the slot back and forth through `turn` (PoaChainSync below) */
    int32_t turn;                       /* 0: the alignment warp's move, 1: a fuse worker's move */
    int32_t rsv0;
    unsigned long long wait_ns, fuse_ns;        /* time the alignment warp waited for its fuse tasks / time inside chain_fuse */
    int64_t prof[6];                    /* -DPOA_KPROF builds: per-phase cycles of the forward row loop, summed over the alignments */
    int64_t btdiag[5];                  /* -DPOA_KPROF builds: PoaResultDev.btdiag summed */
    /* per-read records (record mode) */
    int32_t *rec_score, *rec_nops; uint64_t *rec_hash;
    /* RC-MSA (PoaChainParams::W > 0): bit r of node v's set = read r's path passes through v, i.e. the union of the read
     * sets of v's out-edges in the host graph -- all the row-column MSA needs (reference src/abpoa_output.c:105-192) */
    uint64_t *read_set;                                 /* [n_cap * W] */
    /* -s (PoaChainParams::amb_strand): per read, bit 0 = fused as the reverse complement, bit 1 = the reverse complement was
     * aligned too (a weak forward hit); the alignment warp runs that second pass into rc_cigar / rc_result */
    uint8_t *read_rc;                                   /* [n_reads] */
    uint64_t *rc_cigar;                                 /* [jd.cigar_cap] */
    PoaResultDev *rc_result;
    /* -Q (use_qv): the weight of every read base (the edge that enters the base's node gets it), at the reads' offsets;
     * NULL: unit weights */
    const uint8_t *read_qw;                             /* [sum of the read lengths] */
} PoaChainSlot;

/* A group's memory, host side: the slot's capacities and every per-group array, taken in one fixed order from the
 * caller's allocator `take(bytes)`, which also decides the alignment.  The engine carves a wave's HBM with it, its
 * wave planner sums the same requests, and the CPU emulator lays out its host buffer with it, so the three cannot
 * disagree.  The reads (chain_slot_reads) live in a region of their own: they are staged and uploaded in one copy.
 * `strand` (-s runs) adds the strand bytes and the second CIGAR buffer and result behind everything else.  `ps` (-G runs)
 * makes the job blob room for the predscore section, one int per in-edge like pred. */
template <class Take>
static inline void chain_slot_layout(PoaChainSlot *s, int n_cap, int qmax, int n_reads, int K, int A, int m, int W, bool record, Take take,
                                     bool strand = false, bool ps = false) {
    const size_t nc = (size_t)n_cap, scr_n = nc > (size_t)qmax + 2 ? nc : (size_t)qmax + 2;
    s->n_cap = n_cap; s->pred_cap = (int32_t)(nc * 3); s->n_reads = n_reads;
    s->blob_cap = (int32_t)(256 + (nc + 1) * 8 + (size_t)s->pred_cap * 4 + 4 + (size_t)qmax + 64);
    if (ps) s->blob_cap += (int32_t)((size_t)s->pred_cap * 4 + 4 + 16);
    s->jd.cigar_cap = (int32_t)(qmax + n_cap + 8);
    s->base = (uint8_t *)take(nc);
    s->in_cnt = (int32_t *)take(nc * 4); s->out_cnt = (int32_t *)take(nc * 4); s->aln_cnt = (int32_t *)take(nc * 4); s->n_read = (int32_t *)take(nc * 4);
    s->in_id = (int32_t *)take(nc * K * 4); s->in_w = (int32_t *)take(nc * K * 4); s->out_id = (int32_t *)take(nc * K * 4); s->out_w = (int32_t *)take(nc * K * 4);
    s->aln_id = (int32_t *)take(nc * A * 4);
    s->order[0] = (int32_t *)take(nc * 4); s->order[1] = (int32_t *)take(nc * 4); s->node_row = (int32_t *)take(nc * 4); s->rem_row = (int32_t *)take(nc * 4);
    for (int k = 0; k < 6; ++k) s->scr[k] = (int32_t *)take(scr_n * 4);
    s->jd.blob = (uint8_t *)take((size_t)s->blob_cap);
    s->jd.rowinfo = (PoaRowInfo *)take(nc * sizeof(PoaRowInfo)); s->jd.rowoff = (PoaRowOff *)take(nc * sizeof(PoaRowOff));
    s->jd.cigar = (uint64_t *)take((size_t)s->jd.cigar_cap * 8);
    s->jd.qprof = (int16_t *)take((size_t)m * ((((size_t)qmax + 1 + 7) & ~(size_t)7) + 8) * 2);
    s->jd.result = (PoaResultDev *)take(sizeof(PoaResultDev));
    s->jd.btrec = (PoaBtRec *)take(nc * sizeof(PoaBtRec));
    if (record) { s->rec_score = (int32_t *)take((size_t)n_reads * 4); s->rec_nops = (int32_t *)take((size_t)n_reads * 4); s->rec_hash = (uint64_t *)take((size_t)n_reads * 8); }
    if (W > 0) s->read_set = (uint64_t *)take(nc * W * 8);
    if (strand) {
        s->read_rc = (uint8_t *)take((size_t)n_reads);
        s->rc_cigar = (uint64_t *)take((size_t)s->jd.cigar_cap * 8);
        s->rc_result = (PoaResultDev *)take(sizeof(PoaResultDev));
    }
}

/* the group's reads: `bases` bytes back to back, n_reads + 1 offsets, n_reads band half widths; `qv` (-Q runs with
 * weights) adds one weight byte per base behind them */
template <class Take>
static inline void chain_slot_reads(PoaChainSlot *s, int n_reads, int64_t bases, Take take, bool qv = false) {
    s->reads = (const uint8_t *)take((size_t)bases);
    s->read_off = (const int32_t *)take(((size_t)n_reads + 1) * 4);
    s->read_w = (const int32_t *)take((size_t)n_reads * 4);
    if (qv) s->read_qw = (const uint8_t *)take((size_t)bases);
}

/* Free-running chain: every group advances at its own pace.  One resident warp per group runs its alignments back to back;
 * after each one it appends the group to `tasks` and waits; persistent fuse CTAs draw tickets, fuse + flatten the group and
 * hand it back.  `total` = fuse tasks that will ever be appended (lowered when a group leaves the chain early): a worker
 * whose ticket is >= total exits. */
typedef struct PoaChainSync {
    /* every word that is polled or bumped sits in its own 128-byte line: a thousand waiting warps must not queue up on the
     * L2 line the queue counters live in (they poll their OWN slot / task word, and look at `abort` / `total` only now and then) */
    unsigned int q_head; int32_t pad0[31];      /* next ticket */
    unsigned int q_tail; int32_t pad1[31];      /* next free task slot */
    int32_t total; int32_t pad2[31];
    int32_t abort; int32_t pad3[31];            /* set by a waiter whose partner did not answer within the watchdog time */
    unsigned long long watchdog_ns;
    int32_t *tasks;                             /* [sum over groups of (n_reads - 1)], initialised to -1 */
} PoaChainSync;

/* ------------------------------------------------------------------ block-wide helpers */
#ifdef POA_CHAIN_EMUL
POA_DEV int cta_excl_scan(int32_t *a, int n) {             /* in place; returns the total */
    int run = 0;
    for (int i = 0; i < n; ++i) { const int v = a[i]; a[i] = run; run += v; }
    return run;
}
POA_DEV void cta_incl_maxscan(int32_t *a, int n) {
    int run = INT32_MIN;
    for (int i = 0; i < n; ++i) { if (a[i] > run) run = a[i]; a[i] = run; }
}
#else
/* exclusive sum scan of a[0..n) in place (global memory), chunk by chunk with a running carry */
__device__ inline int cta_excl_scan(int32_t *a, int n) {
    __shared__ int warp_sum[32];
    __shared__ int carry_s;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int v = i < n ? a[i] : 0;
        int x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += t; }
        if (lane == 31) warp_sum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int s = lane < nw ? warp_sum[lane] : 0;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += t; }
            warp_sum[lane] = s;                             /* inclusive over warps */
        }
        __syncthreads();
        const int carry = carry_s;
        const int before = carry + (wid > 0 ? warp_sum[wid - 1] : 0) + x - v;
        if (i < n) a[i] = before;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + warp_sum[nw - 1];
        __syncthreads();
    }
    return carry_s;
}
__device__ inline void cta_incl_maxscan(int32_t *a, int n) {
    __shared__ int warp_max[32];
    __shared__ int carry_m;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (threadIdx.x == 0) carry_m = INT32_MIN;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        int x = i < n ? a[i] : INT32_MIN;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x = max(x, t); }
        if (lane == 31) warp_max[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int s = lane < nw ? warp_max[lane] : INT32_MIN;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s = max(s, t); }
            warp_max[lane] = s;
        }
        __syncthreads();
        int r = max(carry_m, x);
        if (wid > 0) r = max(r, warp_max[wid - 1]);
        if (i < n) a[i] = r;
        __syncthreads();
        if (threadIdx.x == 0) carry_m = max(carry_m, warp_max[nw - 1]);
        __syncthreads();
    }
}
#endif

/* ------------------------------------------------------------------ small per-thread helpers */
/* the reference's in-place exchange pass (src/abpoa_graph.c:192-219): swap whenever w[j] < w[k], j < k */
POA_DEV void chain_exchange_order(int32_t *ids, int32_t *ws, int n) {
    for (int j = 0; j + 1 < n; ++j)
        for (int k = j + 1; k < n; ++k)
            if (ws[j] < ws[k]) { int32_t t = ids[j]; ids[j] = ids[k]; ids[k] = t; t = ws[j]; ws[j] = ws[k]; ws[k] = t; }
}

/* row of the last member of v's aligned group in the CURRENT order (groups occupy consecutive rows) */
POA_DEV int chain_group_last_row(const PoaChainSlot *s, int A, const int32_t *order, int old_n, int v) {
    int r = s->node_row[v];
    const int na = s->aln_cnt[v];
    if (na == 0) return r;
    const int32_t *al = s->aln_id + (size_t)v * A;
    for (; r + 1 < old_n; ++r) {
        const int u = order[r + 1];
        int member = 0;
        for (int a = 0; a < na; ++a) if (al[a] == u) { member = 1; break; }
        if (!member) break;
    }
    return r;
}

/* reference src/abpoa_align_simd.c:1293-1303: lanes of the AVX2 vector for the width the reference would pick */
POA_DEV int chain_ref_pn(const PoaChainParams *cp, int qlen, int n_rows) {
    const int len = qlen > n_rows ? qlen : n_rows;
    const int a = qlen * cp->max_mat, b = len * cp->e1 + cp->o1;
    const int max_score = a > b ? a : b;
    return max_score <= 32767 - cp->min_mis - cp->oe1 - cp->oe2 ? 16 : 8;
}

/* linear gaps: cells a DP row stores beyond its band at most -- the band rounded out to whole vectors of pn lanes on both
 * sides (the reference's banded linear-gap rows, p16_run_job's LGX rows) */
#define POA_LG_ROW_CELLS(pn) (2 * ((pn) - 1))

POA_DEV size_t chain_al16(size_t x) { return (x + 15) & ~(size_t)15; }

/* -s, reference src/abpoa_align.c:323-325: the forward hit is weak, so the reverse complement is aligned too.  node_n counts
 * SRC and SINK (the job's n_rows); the bound is an int product times a double, as the reference evaluates it. */
POA_DEV bool chain_weak_hit(int best_score, int qlen, int node_n, int max_mat) {
    const int lim = qlen < node_n - 2 ? qlen : node_n - 2;
    return best_score < lim * max_mat * .3333;
}

/* -G: the score of an in-edge of weight edge_w whose tail's out-edges weigh node_w in all, max(round(ln(edge_w / node_w)), -20),
 * 0 if either weight is 0 (reference src/abpoa_graph.c:429-437; host twin poa_edge_path_score in poa_graph.c).  The device's
 * log may differ from glibc's in the last bit; the chain admits node weights up to POA_PS_MAX_NODE_W only, and for those no
 * ratio lies within 1024 ulp of a rounding boundary -(k + 1/2) (tests/test_chain_emul_ps.py proves it), so both round
 * alike. */
#define POA_PS_MAX_NODE_W (1 << 20)
POA_DEV int chain_path_score(int edge_w, int node_w) {
    if (node_w == 0 || edge_w == 0) return 0;
    const int s = (int)round(log((double)edge_w / (double)node_w));
    return s > -20 ? s : -20;
}

/* complement of a base code (reference src/abpoa_align.c:329): 0..3 -> 3..0, everything else -> 4, with -c too */
POA_DEV uint8_t chain_comp(uint8_t b) { return b < 4 ? (uint8_t)(3 - b) : (uint8_t)4; }

/* read r as the graph code fuses it, looked up once per read: its bases, its -Q weights (NULL: unit weights), its length
 * and whether it is fused as the reverse complement (read_rc[r]) */
typedef struct ChainRead { const uint8_t *q, *w; int len; bool rc; } ChainRead;

POA_DEV ChainRead chain_read(const PoaChainSlot *s, int r) {
    ChainRead rd;
    rd.q = s->reads + s->read_off[r]; rd.w = s->read_qw ? s->read_qw + s->read_off[r] : NULL;
    rd.len = s->read_off[r + 1] - s->read_off[r]; rd.rc = s->read_rc && (s->read_rc[r] & 1);
    return rd;
}

/* base qi on the strand the read is fused on: the reverse complement, computed on the fly */
POA_DEV uint8_t chain_read_base(const ChainRead &rd, int qi) { return rd.rc ? chain_comp(rd.q[rd.len - 1 - qi]) : rd.q[qi]; }

/* -Q: weight of base qi on the strand the read is fused on (a reverse-complemented read's weights are reversed, as in
 * poa_msa.c and the launch engine), 1 without weights */
POA_DEV int chain_read_weight(const ChainRead &rd, int qi) { return !rd.w ? 1 : rd.w[rd.rc ? rd.len - 1 - qi : qi]; }

/* ------------------------------------------------------------------ order-dependent passes */
/* max_remain by row: remain[row] = remain[row of heaviest out-neighbour] + 1, SINK = -1 (reference
 * src/abpoa_graph.c:268-309; out-lists are weight-ordered here, so the heaviest, first on ties, is slot 0).
 * Tiles of POA_CHAIN_T rows from the sink end; inside a tile the chain is resolved by pointer jumping. */
POA_DEV void chain_set_remain(PoaChainSlot *s, int K, const int32_t *order, int n) {
    POA_SHARED int t_ptr[POA_CHAIN_T], t_val[POA_CHAIN_T], t_np[POA_CHAIN_T], t_nv[POA_CHAIN_T];
    int32_t *rem = s->rem_row;
    if (POA_TID0) rem[n - 1] = -1;                        /* SINK is always the last row */
    POA_CTA_SYNC();
    for (int hi = n - 1; hi > 0; hi -= POA_CHAIN_T) {     /* rows [lo, hi) */
        const int lo = hi - POA_CHAIN_T > 0 ? hi - POA_CHAIN_T : 0;
        const int cnt = hi - lo;
        POA_PAR_FOR(l, POA_CHAIN_T) {
            if (l < cnt) {
                const int v = order[lo + l];
                const int sr = s->node_row[s->out_id[(size_t)v * K]];
                if (sr >= hi) { t_ptr[l] = -1; t_val[l] = rem[sr] + 1; }
                else { t_ptr[l] = sr - lo; t_val[l] = 1; }
            } else { t_ptr[l] = -1; t_val[l] = 0; }
        }
        POA_CTA_SYNC();
        for (int step = 1; step < POA_CHAIN_T; step <<= 1) {
            POA_PAR_FOR(l, POA_CHAIN_T) {
                const int p = t_ptr[l];
                if (p >= 0) { t_nv[l] = t_val[l] + t_val[p]; t_np[l] = t_ptr[p]; } else { t_nv[l] = t_val[l]; t_np[l] = -1; }
            }
            POA_CTA_SYNC();
            POA_PAR_FOR(l, POA_CHAIN_T) { t_val[l] = t_nv[l]; t_ptr[l] = t_np[l]; }
            POA_CTA_SYNC();
        }
        POA_PAR_FOR(l, POA_CHAIN_T) { if (l < cnt) rem[lo + l] = t_val[l]; }
        POA_CTA_SYNC();
    }
}

/* Extend mode: the reference's row order (host twin abpoa_BFS_set_node_index in poa_graph.c, reference
 * src/abpoa_graph.c:221-266) into order[] / node_row[]: FIFO Kahn from SRC, stopping when SINK is dequeued; out-edges in
 * list order; a node in an aligned set becomes ready only when every member's in-degree is 0, and the set is then
 * enqueued as the trigger node followed by its aligned list.  The host walks the out-lists BEFORE the read's weight
 * changes are re-ordered (order_edges_by_weight runs after the walk), so chain_fuse<.., KO> leaves its out-lists in
 * append / bump order and re-orders them behind this walk.  The queue is order[] itself.
 * The CTA precomputes, per node, its in-degree counter (a byte in scr[2]; CHAIN_KAHN_LINK for a "chain link": one in-edge
 * and no aligned set, ready as soon as its predecessor is dequeued) and, when the node's only out-edge enters a chain
 * link, that successor (scr[3]); the walk itself is serial on thread 0 (a POA graph is about as deep as it is long) and
 * costs one dependent load per node on a run of chain links.  Needs K <= 254 (plan_groups).  Needs the whole CTA. */
#define CHAIN_KAHN_LINK 0xff
POA_DEV void chain_kahn_order(PoaChainSlot *s, const PoaChainParams *cp, int32_t *order, int n) {
    const int K = cp->K, A = cp->A;
    uint8_t *deg = reinterpret_cast<uint8_t *>(s->scr[2]);
    int32_t *nx = s->scr[3];
    POA_PAR_FOR(v, n) {
        const int ni = s->in_cnt[v];
        deg[v] = (ni == 1 && s->aln_cnt[v] == 0) ? (uint8_t)CHAIN_KAHN_LINK : (uint8_t)ni;
    }
    POA_CTA_SYNC();
    POA_PAR_FOR(u, n) {
        int x = -1;
        if (s->out_cnt[u] == 1) { const int v = s->out_id[(size_t)u * K]; if (deg[v] == CHAIN_KAHN_LINK) x = v; }
        nx[u] = x;
    }
    POA_CTA_SYNC();
    if (POA_TID0) {
        int head = 0, tail = 1, last = 0, done = 0;
        order[0] = 0;
        while (head < tail) {
            const int cur = head + 1 == tail ? last : order[head];      /* a queue of one: the node just pushed, from a register */
            s->node_row[cur] = head++;
            if (cur == 1) { done = head == n; break; }
            const int x = nx[cur];
            if (x >= 0) {                                                /* a run of chain links */
                if (tail >= n) break;
                order[tail++] = last = x;
                continue;
            }
            const int ne = s->out_cnt[cur];
            const int32_t *oid = s->out_id + (size_t)cur * K;
            int full = 0;
            for (int e = 0; e < ne && !full; ++e) {
                const int v = oid[e];
                int d = deg[v];
                if (d != CHAIN_KAHN_LINK) {
                    deg[v] = (uint8_t)--d;
                    if (d != 0) continue;
                    const int na = s->aln_cnt[v];
                    const int32_t *al = s->aln_id + (size_t)v * A;
                    int ready = 1;
                    for (int a = 0; a < na; ++a) if (deg[al[a]] != 0) { ready = 0; break; }
                    if (!ready) continue;
                    if (tail + 1 + na > n) { full = 1; break; }
                    order[tail++] = last = v;
                    for (int a = 0; a < na; ++a) order[tail++] = last = al[a];
                } else {
                    if (tail >= n) { full = 1; break; }
                    order[tail++] = last = v;
                }
            }
            if (full) break;
        }
        if (!done) POA_ATOMIC_OR(&s->failed, POA_CF_ORDER);     /* not a DAG, or SINK came before a node: not a POA graph */
    }
    POA_CTA_SYNC();
}

/* Flatten the graph + read `r` into the slot's job blob (layout: PoaJobHeader; the host twin is
 * poa_blob_fill in poa_flat.c).  Also the last line of defence for the order: every predecessor row
 * must be smaller than its row.  PS (-G runs; the host picks the fuse kernels' instantiation, so a run without -G compiles
 * to the bare flatten): the predscore section behind pred, every in-edge's chain_path_score.  LG (linear-gap runs, picked
 * the same way): the DP stores a row in whole reference vectors of pn cells around its band, up to 2 (pn - 1) cells more
 * (POA_LG_ROW_CELLS). */
template <bool PS = false, bool LG = false>
POA_DEV void chain_flatten(PoaChainSlot *s, const PoaChainParams *cp, const int32_t *order, int n, int r, int pool_parity, int generous) {
    const int K = cp->K;
    int32_t *cnt = s->scr[0];
    POA_PAR_FOR(i, n) cnt[i] = i == 0 ? 0 : s->in_cnt[order[i]];
    POA_CTA_SYNC();
    const int n_pred = cta_excl_scan(cnt, n);
    POA_CTA_SYNC();
    const int qlen = s->read_off[r + 1] - s->read_off[r];
    uint8_t *blob = const_cast<uint8_t *>(s->jd.blob);
    PoaJobHeader *h = reinterpret_cast<PoaJobHeader *>(blob);
    size_t off = chain_al16(sizeof(PoaJobHeader));
    const size_t off_rowmeta = off; off += chain_al16(((size_t)n + 1) * 8);
    const size_t off_pred = off; off += chain_al16((size_t)n_pred * 4 + 4);
    const size_t off_ps = off; if (PS) off += chain_al16((size_t)n_pred * 4 + 4);
    const size_t off_qs = off; off += chain_al16((size_t)qlen + 1) + 16;
    if (off > (size_t)s->blob_cap || n_pred > s->pred_cap) {
        if (POA_TID0) { POA_ATOMIC_OR(&s->failed, POA_CF_BLOB_CAP); h->n_rows = 0; }
        POA_CTA_SYNC();
        return;
    }
    int32_t *rowmeta = reinterpret_cast<int32_t *>(blob + off_rowmeta), *pred = reinterpret_cast<int32_t *>(blob + off_pred);
    int32_t *pscore = reinterpret_cast<int32_t *>(blob + off_ps);
    uint8_t *qs = blob + off_qs;
    POA_PAR_FOR(i, n) {
        const int v = order[i];
        const int po = cnt[i];
        rowmeta[2 * i] = po;
        rowmeta[2 * i + 1] = (int32_t)((uint32_t)s->rem_row[i] << 8) | s->base[v];
        if (i > 0) {
            const int ni = s->in_cnt[v];
            const int32_t *iid = s->in_id + (size_t)v * K;
            for (int e = 0; e < ni; ++e) {
                const int pr = s->node_row[iid[e]];
                if (pr >= i) POA_ATOMIC_OR(&s->failed, POA_CF_ORDER);
                pred[po + e] = pr;
                if (PS) {                                       /* the in-edge's weight over its tail's out-edge weights */
                    const int u = iid[e], no = s->out_cnt[u];
                    const int32_t *ow = s->out_w + (size_t)u * K;
                    int node_w = 0;
                    for (int o = 0; o < no; ++o) node_w += ow[o];
                    pscore[po + e] = chain_path_score(s->in_w[(size_t)v * K + e], node_w);
                }
            }
        }
    }
    const uint8_t *q = s->reads + s->read_off[r];
    const int qpad = (int)(off - off_qs);
    POA_PAR_FOR(j, qpad) qs[j] = (j >= 1 && j <= qlen) ? q[j - 1] : (uint8_t)0;
    if (POA_TID0) {
        rowmeta[2 * n] = n_pred; rowmeta[2 * n + 1] = 0;
        h->qlen = qlen; h->w = s->read_w[r]; h->node_n = n;
        h->off_rowmeta = (int32_t)off_rowmeta; h->off_pred = (int32_t)off_pred; h->off_predscore = PS ? (int32_t)off_ps : -1; h->off_live = -1;
        h->off_qs = (int32_t)off_qs; h->rsv[0] = h->rsv[1] = h->rsv[2] = h->rsv[3] = 0;
        h->blob_bytes = (int32_t)off; h->pn = chain_ref_pn(cp, qlen, n); h->pad[0] = h->pad[1] = 0;
#ifndef POA_CHAIN_EMUL
        if (s->pool_base) {
            /* planes of the job.  Band of a row = [min(ml, c) - w, max(mr, c) + w] with c the remain-centre: when read and graph
             * differ in length the arg-max drifts away from c by up to that difference, so the estimate carries it; a band
             * that still outgrows the slab comes back as PLANE_OVF and is re-run once with the full rectangle (generous). */
            const int w = s->read_w[r];
            const int drift = qlen > s->rem_row[0] ? qlen - s->rem_row[0] : s->rem_row[0] - qlen;
            unsigned long long per_row = (unsigned long long)((2 * w + 1 + drift + 64 + (LG ? POA_LG_ROW_CELLS(h->pn) : 0) + 7) / 8 + 2);
            const unsigned long long full = (unsigned long long)((qlen + 1 + 7) / 8 + 1);
            if (generous || per_row > full) per_row = full;
            const unsigned long long units = per_row * (unsigned long long)cp->P * (unsigned long long)n;
            if (!s->pool_cursor) {                                     /* private slab: the job may use all of it */
                s->jd.planes = s->pool_base; s->jd.plane_cap_units = s->pool_units;
            } else {
                const unsigned long long at = atomicAdd(&s->pool_cursor[pool_parity & 1], units);
                if (at + units > s->pool_units) POA_ATOMIC_OR(&s->failed, POA_CF_POOL);
                else { s->jd.planes = s->pool_base + (size_t)at * (POA_GROUP * 2); s->jd.plane_cap_units = units; }
            }
        }
#endif
    }
    POA_CTA_SYNC();
    if (POA_TID0) h->n_rows = s->failed ? 0 : n;          /* n_rows == 0: the DP kernel skips the slot */
    POA_CTA_SYNC();
}

/* ------------------------------------------------------------------ first read of a group */
/* a chain SRC -> b0 -> b1 ... -> SINK (reference src/abpoa_graph.c:573-593): the edge into b_i weighs w[i], the edge into
 * SINK w[len - 1]; PS: see chain_flatten */
template <bool PS = false, bool LG = false>
POA_DEV void chain_seed(PoaChainSlot *s, const PoaChainParams *cp) {
    const int K = cp->K;
    ChainRead rd = chain_read(s, 0);
    rd.rc = false;                                       /* read 0 is fused forward (its strand byte is cleared below) */
    const int len = rd.len;
    const uint8_t *q = rd.q;
    const int n = len + 2;
    if (n > s->n_cap || len < 1) {
        if (POA_TID0) { POA_ATOMIC_OR(&s->failed, POA_CF_NODE_CAP); reinterpret_cast<PoaJobHeader *>(const_cast<uint8_t *>(s->jd.blob))->n_rows = 0; }
        POA_CTA_SYNC();
        return;
    }
    int32_t *order = s->order[0];
    POA_PAR_FOR(v, n) {
        /* node ids: 0 SRC, 1 SINK, 2 + i = base i */
        s->aln_cnt[v] = 0;
        if (v == 0) { s->base[v] = 0; s->in_cnt[v] = 0; s->out_cnt[v] = 1; s->out_id[0] = 2; s->out_w[0] = chain_read_weight(rd, 0); s->n_read[v] = 1; order[0] = 0; s->node_row[0] = 0; }
        else if (v == 1) {
            s->base[v] = 0; s->out_cnt[v] = 0; s->in_cnt[v] = 1; s->in_id[(size_t)K] = len + 1; s->in_w[(size_t)K] = chain_read_weight(rd, len - 1); s->n_read[v] = 0;
            order[n - 1] = 1; s->node_row[1] = n - 1;
        } else {
            const int i = v - 2;
            s->base[v] = q[i];
            s->in_cnt[v] = 1; s->in_id[(size_t)v * K] = i == 0 ? 0 : v - 1; s->in_w[(size_t)v * K] = chain_read_weight(rd, i);
            s->out_cnt[v] = 1; s->out_id[(size_t)v * K] = i == len - 1 ? 1 : v + 1; s->out_w[(size_t)v * K] = chain_read_weight(rd, i == len - 1 ? i : i + 1);
            s->n_read[v] = 1;
            order[i + 1] = v; s->node_row[v] = i + 1;
        }
    }
    if (cp->W > 0) {                                     /* read 0 passes through SRC and every node it created; SINK has no out-edge */
        const int W = cp->W;
        POA_PAR_FOR(v, n) { uint64_t *rs = s->read_set + (size_t)v * W; for (int wd = 0; wd < W; ++wd) rs[wd] = (wd == 0 && v != 1) ? 1ull : 0ull; }
    }
    if (POA_TID0) { s->n_nodes = n; s->cur = 0; s->fused = 1; s->retry = 0; if (s->read_rc) s->read_rc[0] = 0; }   /* read 0 seeds: no strand test */
    POA_CTA_SYNC();
    chain_set_remain(s, K, order, n);
    if (s->n_reads > 1) chain_flatten<PS, LG>(s, cp, order, n, 1, /*pool_parity=*/1, 0);
}

/* ------------------------------------------------------------------ fuse read r, prepare read r + 1 */
/* item kinds */
#define CK_OLD  0       /* the read reuses an existing node (equal base, or an aligned sibling with its base) */
#define CK_NEWM 1       /* mismatch: new node aligned with the matched column                                 */
#define CK_NEWI 2       /* inserted base: new unaligned node                                                  */

/* `round`: the round of the cohort's schedule that just ran (the next alignment kernel is round + 1; its plane pool is
 * the one with that parity).  A group normally fuses read `round`, but one that had to re-run an alignment lags behind.
 * PS: see chain_flatten.  KO (extend runs; the host picks the fuse kernels' instantiation): the new order is the
 * reference's Kahn order (chain_kahn_order) instead of the splice of steps 4 and 8, and the out-lists are re-ordered by
 * weight behind it.  The seed's chain order is already the Kahn order of a path. */
template <bool PS = false, bool LG = false, bool KO = false>
POA_DEV void chain_fuse(PoaChainSlot *s, const PoaChainParams *cp, int round) {
    const int K = cp->K, A = cp->A;
    const int r = s->fused;                                /* the read whose alignment just finished */
    PoaJobHeader *hdr = reinterpret_cast<PoaJobHeader *>(const_cast<uint8_t *>(s->jd.blob));
    if (s->failed || r >= s->n_reads) return;
    const PoaResultDev *res = s->jd.result;
    if (res->status == POA_ST_SKIP) return;               /* nothing ran for this slot in this round */
    if (res->status == POA_ST_PLANE_OVF && !s->retry && s->pool_cursor) {   /* band wider than the slab: same read again, full-rectangle slab */
        POA_CTA_SYNC();
        if (POA_TID0) s->retry = 1;
        chain_flatten<PS, LG>(s, cp, s->order[s->cur], s->n_nodes, r, round + 1, 1);
        return;
    }
    if (res->status != POA_ST_OK) {
        if (POA_TID0) { POA_ATOMIC_OR(&s->failed, POA_CF_DP_STATUS); hdr->n_rows = 0; }
        POA_CTA_SYNC();
        return;
    }
    const ChainRead rd = chain_read(s, r);
    const int qlen = rd.len;
    const uint64_t *ops = s->jd.cigar;
    const int n_ops = res->n_ops;
    const int old_n = s->n_nodes;
    const int32_t *order = s->order[s->cur];
    int32_t *order_new = s->order[s->cur ^ 1];
    int32_t *item_row = s->scr[0], *tgt = s->scr[1], *isnew = s->scr[2], *kind_anchor = s->scr[3], *defidx = s->scr[4], *new_anchor = s->scr[5];

    /* ---- record mode: score, CIGAR length and the FNV-1a hash of the words the host API would return
     *      (forward order, DP rows translated to node ids; poa_job_to_res in poa_cuda.cu) ---- */
    if (POA_TID0) {
        s->cells += res->cells; s->fwd_clk += res->fwd_clk; s->bt_clk += res->bt_clk;
#ifdef POA_KPROF
        for (int z = 0; z < 6; ++z) s->prof[z] += res->prof[z];
        for (int z = 0; z < 5; ++z) s->btdiag[z] += res->btdiag[z];
#endif
        if (cp->record) {
            s->rec_score[r] = res->best_score; s->rec_nops[r] = n_ops;
            uint64_t hsh = 1469598103934665603ull;
            for (int t = n_ops - 1; t >= 0; --t) {
                uint64_t w = ops[t];
                if ((w & 0xf) != 1) w = ((uint64_t)(uint32_t)order[w >> 34] << 34) | (w & 0x3ffffffffull);
                for (int b = 0; b < 8; ++b) { hsh ^= (w >> (8 * b)) & 0xff; hsh *= 1099511628211ull; }
            }
            s->rec_hash[r] = hsh;
        }
    }

    /* ---- 1. one item per query base: the DP row it is matched to, or -1 (inserted) ---- */
    POA_PAR_FOR(qi, qlen + 1) { item_row[qi] = -2; }
    POA_CTA_SYNC();
    POA_PAR_FOR(t, n_ops) {
        const uint64_t w = ops[t];
        const int op = (int)(w & 0xf);
        if (op == 0) {                                       /* MATCH: row << 34 | qpos << 4 */
            const int qp = (int)((w >> 4) & 0x3fffffff), row = (int)(w >> 34);
            if (qp < qlen && row > 0 && row < old_n - 1) item_row[qp] = row; else POA_ATOMIC_OR(&s->failed, POA_CF_CIGAR);
        } else if (op == 1) {                                /* INS: last qpos << 34 | len << 4 | 1 */
            const int qp = (int)(w >> 34), len = (int)((w >> 4) & 0x3fffffff);
            if (qp < qlen && qp - len + 1 >= 0) { for (int k = 0; k < len; ++k) item_row[qp - k] = -1; } else POA_ATOMIC_OR(&s->failed, POA_CF_CIGAR);
        }
    }
    POA_CTA_SYNC();

    /* ---- 2. classify (reads only the OLD graph) ---- */
    POA_PAR_FOR(qi, qlen) {
        const int row = item_row[qi];
        int kind = CK_NEWI, target = -1, anchor = -1;
        if (row == -2) POA_ATOMIC_OR(&s->failed, POA_CF_CIGAR);          /* global mode: every base is M or I */
        if (row >= 0) {
            const int v = order[row];
            const uint8_t b = chain_read_base(rd, qi);
            if (s->base[v] == b) { kind = CK_OLD; target = v; }
            else {
                const int na = s->aln_cnt[v]; const int32_t *al = s->aln_id + (size_t)v * A;
                for (int a = 0; a < na; ++a) if (s->base[al[a]] == b) { target = al[a]; break; }
                if (target >= 0) kind = CK_OLD;
                else { kind = CK_NEWM; anchor = KO ? -1 : chain_group_last_row(s, A, order, old_n, v); target = v; }   /* target: the column's node for now */
            }
        }
        tgt[qi] = target; isnew[qi] = kind != CK_OLD;
        kind_anchor[qi] = (kind << 28) | (anchor & 0x0fffffff);
    }
    POA_CTA_SYNC();
    if (s->failed) { if (POA_TID0) hdr->n_rows = 0; POA_CTA_SYNC(); return; }

    /* ---- 3. ids of the new nodes: old_n + rank among the new items (the host creates them in this order) ---- */
    int32_t *newidx = defidx;                                /* borrowed until step 5 */
    POA_PAR_FOR(qi, qlen) newidx[qi] = isnew[qi];
    POA_CTA_SYNC();
    const int n_new = cta_excl_scan(newidx, qlen);
    POA_CTA_SYNC();
    const int n = old_n + n_new;
    if (n > s->n_cap) { if (POA_TID0) { POA_ATOMIC_OR(&s->failed, POA_CF_NODE_CAP); hdr->n_rows = 0; } POA_CTA_SYNC(); return; }

    /* ---- 4. anchors of the new nodes in the OLD order (spliced order, poa_graph.c):
     *         mismatch node      -> behind the aligned group of its column
     *         inserted after old -> behind the aligned group of the previous path node
     *         inserted after new -> inherits the previous new node's anchor                      ---- */
    if (!KO) {
    POA_PAR_FOR(qi, qlen) {
        const int kind = kind_anchor[qi] >> 28;
        int anchor = -1;
        if (kind == CK_NEWM) anchor = kind_anchor[qi] & 0x0fffffff;
        else if (kind == CK_NEWI && !(qi > 0 && isnew[qi - 1])) anchor = chain_group_last_row(s, A, order, old_n, qi == 0 ? 0 : tgt[qi - 1]);
        new_anchor[qi] = anchor;                             /* by item for now */
    }
    POA_CTA_SYNC();
    {   /* nearest definer at or before each item */
        int32_t *d = item_row;                               /* item_row is no longer needed */
        POA_PAR_FOR(qi, qlen) d[qi] = new_anchor[qi] >= 0 ? qi : -1;
        POA_CTA_SYNC();
        cta_incl_maxscan(d, qlen);
        POA_CTA_SYNC();
        POA_PAR_FOR(qi, qlen) {
            if (isnew[qi]) {
                const int a = d[qi] >= 0 ? new_anchor[d[qi]] : -1;
                if (a < 0) POA_ATOMIC_OR(&s->failed, POA_CF_ORDER);
                kind_anchor[qi] = (kind_anchor[qi] & (int32_t)0xf0000000) | (a & 0x0fffffff);
            }
        }
        POA_CTA_SYNC();
    }
    }

    /* ---- 5. create the new nodes; final targets ---- */
    POA_PAR_FOR(qi, qlen) {
        if (isnew[qi]) {
            const int id = old_n + newidx[qi];
            const int col = tgt[qi];                         /* CK_NEWM: the column's node */
            s->base[id] = chain_read_base(rd, qi); s->in_cnt[id] = 0; s->out_cnt[id] = 0; s->aln_cnt[id] = 0; s->n_read[id] = 0;
            if (cp->W > 0) for (int wd = 0; wd < cp->W; ++wd) s->read_set[(size_t)id * cp->W + wd] = 0;
            new_anchor[newidx[qi]] = kind_anchor[qi] & 0x0fffffff;      /* compacted: by new-node rank (anchors are non-decreasing) */
            item_row[qi] = col;                              /* remember the column for the aligned-set update */
            tgt[qi] = id;
        }
    }
    POA_CTA_SYNC();
    /* new_anchor was written by rank while being read by item in the loop above only through kind_anchor: safe */

    /* ---- 6. edges: item qi owns in-list(tgt[qi]) and out-list(tgt[qi-1]); item qlen is the closing edge to SINK.
     *         Weights (-Q) add to the edges; n_read counts reads ---- */
    POA_PAR_FOR(qi, qlen + 1) {
        const int from = qi == 0 ? 0 : tgt[qi - 1], to = qi < qlen ? tgt[qi] : 1;
        const int from_new = qi > 0 && isnew[qi - 1], to_new = qi < qlen && isnew[qi];
        const int w = chain_read_weight(rd, qi < qlen ? qi : qlen - 1);       /* the closing edge: the last base's */
        int32_t *iid = s->in_id + (size_t)to * K, *iw = s->in_w + (size_t)to * K;
        int32_t *oid = s->out_id + (size_t)from * K, *ow = s->out_w + (size_t)from * K;
        int nin = s->in_cnt[to], nout = s->out_cnt[from];
        int found = 0;
        if (!from_new && !to_new) {
            for (int i = 0; i < nin; ++i)
                if (iid[i] == from) { iw[i] += w; found = 1; if (i > 0 && iw[i - 1] < iw[i]) chain_exchange_order(iid, iw, nin); break; }
            if (found)
                for (int i = 0; i < nout; ++i)
                    if (oid[i] == to) { ow[i] += w; if (!KO && i > 0 && ow[i - 1] < ow[i]) chain_exchange_order(oid, ow, nout); break; }
        }
        if (!found) {
            if (nin >= K || nout >= K) POA_ATOMIC_OR(&s->failed, POA_CF_EDGE_CAP);
            else {
                iid[nin] = from; iw[nin] = w; s->in_cnt[to] = ++nin;
                if (nin > 1 && iw[nin - 2] < w) chain_exchange_order(iid, iw, nin);
                oid[nout] = to; ow[nout] = w; s->out_cnt[from] = ++nout;
                if (!KO && nout > 1 && ow[nout - 2] < w) chain_exchange_order(oid, ow, nout);
            }
        }
        s->n_read[from] += 1;
        if (cp->W > 0) s->read_set[(size_t)from * cp->W + (r >> 6)] |= 1ull << (r & 63);      /* item qi owns node `from` */
    }
    POA_CTA_SYNC();

    /* ---- 7. aligned sets of the new mismatch nodes (reference src/abpoa_graph.c:455-463) ---- */
    POA_PAR_FOR(qi, qlen) {
        if ((kind_anchor[qi] >> 28) == CK_NEWM) {
            const int col = item_row[qi], id = tgt[qi];
            const int na = s->aln_cnt[col];
            if (na + 1 > A) POA_ATOMIC_OR(&s->failed, POA_CF_ALN_CAP);
            else {
                int32_t *mine = s->aln_id + (size_t)id * A; int nm = 0;
                for (int a = 0; a < na; ++a) {
                    const int sib = s->aln_id[(size_t)col * A + a];
                    s->aln_id[(size_t)sib * A + s->aln_cnt[sib]] = id; s->aln_cnt[sib] += 1;
                    mine[nm++] = sib;
                }
                s->aln_id[(size_t)col * A + na] = id; s->aln_cnt[col] = na + 1;
                mine[nm++] = col; s->aln_cnt[id] = nm;
            }
        }
    }
    POA_CTA_SYNC();
    if (s->failed) { if (POA_TID0) hdr->n_rows = 0; POA_CTA_SYNC(); return; }

    /* ---- 8. splice: old row i moves up by the number of new nodes anchored in front of it; the k-th new node
     *         (anchors non-decreasing along the path) lands at anchor_k + 1 + k.
     *         KO: the Kahn walk instead, then the out-lists by weight (the exchange pass leaves a sorted list alone) ---- */
    if (KO) {
        chain_kahn_order(s, cp, order_new, n);
        POA_PAR_FOR(v, n) { const int no = s->out_cnt[v]; if (no > 1) chain_exchange_order(s->out_id + (size_t)v * K, s->out_w + (size_t)v * K, no); }
        POA_CTA_SYNC();
        if (s->failed) { if (POA_TID0) hdr->n_rows = 0; POA_CTA_SYNC(); return; }
    } else {
    POA_PAR_FOR(k, n_new) { if (k > 0 && new_anchor[k] < new_anchor[k - 1]) POA_ATOMIC_OR(&s->failed, POA_CF_ORDER); }
    POA_CTA_SYNC();
    if (s->failed) { if (POA_TID0) hdr->n_rows = 0; POA_CTA_SYNC(); return; }
    POA_PAR_FOR(i, old_n) {
        int lo = 0, hi = n_new;                              /* new nodes with anchor < i */
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (new_anchor[mid] < i) lo = mid + 1; else hi = mid; }
        const int v = order[i], nr = i + lo;
        order_new[nr] = v; s->node_row[v] = nr;
    }
    POA_PAR_FOR(k, n_new) {
        const int nr = new_anchor[k] + 1 + k, v = old_n + k;
        order_new[nr] = v; s->node_row[v] = nr;
    }
    POA_CTA_SYNC();
    }
    if (POA_TID0) { s->n_nodes = n; s->cur ^= 1; s->fused = r + 1; s->retry = 0; }
    POA_CTA_SYNC();

    /* ---- 9. band centres and the next job ---- */
    chain_set_remain(s, K, order_new, n);
    if (r + 1 < s->n_reads) chain_flatten<PS, LG>(s, cp, order_new, n, r + 1, round + 1, 0);
    else if (POA_TID0) hdr->n_rows = 0;
    POA_CTA_SYNC();
}

/* ------------------------------------------------------------------ consensus on the device (SURVEY 8f row f2)
 * Heaviest bundling (most frequent base: chain_mf_consensus below), single cluster (reference src/abpoa_output.c:477-547; host twin: heaviest_bundling in
 * poa_cons.c): score[v] = w(best out-edge) + score[its head], best = largest weight, among equal weights an inner
 * node keeps the LAST edge whose head scores >= the current pick, SRC keeps the first unless strictly better.
 * The reference visits nodes in reverse Kahn order; the values depend only on the out-neighbours, so one backward
 * sweep over the (spliced) topological order gives the same picks.  It runs once per group, serially on one
 * thread (every group has its own CTA; ~25 k dependent steps against ~1 M row steps of DP per group).
 * out[0] = consensus length, out[1 + k] = base | coverage << 8 of consensus position k. */
POA_DEV void chain_consensus(PoaChainSlot *s, const PoaChainParams *cp, int32_t *out, int out_cap) {
    if (!POA_TID0) return;
    const int K = cp->K, n = s->n_nodes;
    const int32_t *order = s->order[s->cur];
    int32_t *score = s->scr[0], *nxt = s->scr[1];
    if (s->failed || n < 3) { out[0] = -1; return; }
    for (int r = n - 1; r >= 0; --r) {
        const int v = order[r];
        const int ne = s->out_cnt[v];
        const int32_t *oid = s->out_id + (size_t)v * K, *ow = s->out_w + (size_t)v * K;
        if (v == 1) { score[v] = 0; nxt[v] = -1; }
        else if (v == 0) {
            int pick = -1, pick_score = -1, pick_w = -1;
            for (int e = 0; e < ne; ++e) {
                const int u = oid[e], w = ow[e];
                if (w > pick_w || (w == pick_w && score[u] > pick_score)) { pick = u; pick_score = score[u]; pick_w = w; }
            }
            nxt[v] = pick;
        } else {
            int pick = -1, pick_w = INT32_MIN;
            for (int e = 0; e < ne; ++e) {
                const int u = oid[e], w = ow[e];
                if (pick_w < w) { pick_w = w; pick = u; }
                else if (pick_w == w && score[pick] <= score[u]) pick = u;
            }
            score[v] = pick_w + score[pick];
            nxt[v] = pick;
        }
    }
    int len = 0;
    for (int cur = nxt[0]; cur != 1 && cur >= 0; cur = nxt[cur]) {
        if (1 + len >= out_cap) { out[0] = -1; return; }
        out[1 + len++] = (int32_t)s->base[cur] | (s->n_read[cur] << 8);
    }
    out[0] = len;
}

/* ------------------------------------------------------------------ row-column MSA on the device
 * Ranks (host twin: poa_set_msa_rank in poa_graph.c): Kahn from SRC with a LIFO stack; a node is pushed, together with
 * its aligned set, when its in-degree and that of every aligned sibling have reached 0; a popped node without a rank
 * takes the next one together with its aligned set.  Out-edges and aligned sets are visited in list order, which is the
 * host's order node for node.  Serial, on one thread per group (like chain_consensus).  Leaves rank[] in scr[5] and
 * returns msa_len = rank[SINK] - 1, or -1. */
POA_DEV int chain_msa_rank(PoaChainSlot *s, const PoaChainParams *cp) {
    if (!POA_TID0) return -1;
    const int K = cp->K, A = cp->A, n = s->n_nodes;
    int32_t *deg = s->scr[3], *st = s->scr[4], *rank = s->scr[5];
    if (s->failed || n < 3) return -1;
    for (int v = 0; v < n; ++v) deg[v] = s->in_cnt[v];
    int top = 0, next_rank = 0;
    st[top++] = 0; rank[0] = -1;
    while (top > 0) {
        const int cur = st[--top];
        const int na = s->aln_cnt[cur];
        const int32_t *al = s->aln_id + (size_t)cur * A;
        if (rank[cur] < 0) {
            rank[cur] = next_rank;
            for (int a = 0; a < na; ++a) rank[al[a]] = next_rank;
            ++next_rank;
        }
        if (cur == 1) return rank[1] - 1;
        const int ne = s->out_cnt[cur];
        const int32_t *oid = s->out_id + (size_t)cur * K;
        for (int e = 0; e < ne; ++e) {
            const int v = oid[e];
            if (--deg[v] != 0) continue;
            const int nv = s->aln_cnt[v];
            const int32_t *av = s->aln_id + (size_t)v * A;
            int ready = 1;
            for (int a = 0; a < nv; ++a) if (deg[av[a]] != 0) { ready = 0; break; }
            if (!ready) continue;
            if (top + 1 + nv > n) return -1;                  /* every node is pushed once: a graph that breaks this is not a DAG */
            st[top++] = v; rank[v] = -1;
            for (int a = 0; a < nv; ++a) { st[top++] = av[a]; rank[av[a]] = -1; }
        }
    }
    return -1;
}

/* Most frequent base per RC-MSA column, single cluster (reference src/abpoa_output.c:393-451, :549-586; host twin:
 * most_frequent in poa_cons.c).  Ranks on one thread (chain_msa_rank: scr[3..5]), the vote and the compaction by the
 * whole CTA.  An aligned set takes one rank when it is pushed and popped, and every column is exactly one aligned set:
 * its members' bases are pairwise distinct (a read reuses a sibling with its base before it adds a node), so the
 * reference's per-column table, where a later node overwrites an earlier one of the same base, never overwrites.  The
 * set's smallest id votes it: codes 0..m-2 only, the largest n_read wins, the lowest code among equal counts; the column
 * is kept iff that count >= n_reads minus the votes.  Writes the record of chain_consensus (out[0] = length, then
 * base | coverage << 8) and leaves the path as nxt[] in scr[1] (nxt[0] = first node, the last points to SINK) for
 * chain_msa_rows and chain_gfa_record; scr[0] holds the kept ids.  Needs the whole CTA. */
POA_DEV void chain_mf_consensus(PoaChainSlot *s, const PoaChainParams *cp, int32_t *out, int out_cap) {
    POA_SHARED int msa_len_s;
    if (POA_TID0) msa_len_s = chain_msa_rank(s, cp);
    POA_CTA_SYNC();
    const int msa_len = msa_len_s;
    if (msa_len < 0) { if (POA_TID0) out[0] = -1; POA_CTA_SYNC(); return; }
    const int A = cp->A, m = cp->m, n = s->n_nodes, n_seq = s->n_reads;
    const int32_t *rank = s->scr[5];
    int32_t *win = s->scr[3], *pos = s->scr[4], *kept = s->scr[0], *nxt = s->scr[1];       /* the rank pass's deg / stack are dead */
    POA_PAR_FOR(j, msa_len) win[j] = -1;
    POA_CTA_SYNC();
    POA_PAR_FOR(v, n) {
        const int na = s->aln_cnt[v];
        const int32_t *al = s->aln_id + (size_t)v * A;
        int lead = v >= 2, r = rank[v];
        for (int a = 0; a < na; ++a) { if (al[a] < v) lead = 0; if (rank[al[a]] > r) r = rank[al[a]]; }
        if (lead) {
            int max_c = 0, max_b = m, total_c = 0, pick = -1;
            for (int a = -1; a < na; ++a) {
                const int u = a < 0 ? v : al[a], b = s->base[u];
                if (b >= m - 1) continue;
                const int c = s->n_read[u];
                total_c += c;
                if (c > max_c || (c == max_c && c > 0 && b < max_b)) { max_c = c; max_b = b; pick = u; }
            }
            if (pick >= 0 && max_c >= n_seq - total_c) win[r - 1] = pick;
        }
    }
    POA_CTA_SYNC();
    POA_PAR_FOR(j, msa_len) pos[j] = win[j] >= 0;
    POA_CTA_SYNC();
    const int len = cta_excl_scan(pos, msa_len);
    POA_CTA_SYNC();
    if (1 + len > out_cap) { if (POA_TID0) out[0] = -1; POA_CTA_SYNC(); return; }
    POA_PAR_FOR(j, msa_len) {
        const int v = win[j];
        if (v >= 0) { out[1 + pos[j]] = (int32_t)s->base[v] | (s->n_read[v] << 8); kept[pos[j]] = v; }
    }
    POA_CTA_SYNC();
    POA_PAR_FOR(k, len) nxt[kept[k]] = k + 1 < len ? kept[k + 1] : 1;
    if (POA_TID0) { out[0] = len; nxt[0] = len > 0 ? kept[0] : 1; }
    POA_CTA_SYNC();
}

/* The consensus the call asked for (PoaChainParams::cons_algrm): the record in `out`, the path in scr[1].  Heaviest
 * bundling runs on thread 0 (the other threads return at once), most frequent base on the whole CTA: every thread of
 * the CTA calls this. */
POA_DEV void chain_cons_path(PoaChainSlot *s, const PoaChainParams *cp, int32_t *out, int out_cap) {
    if (cp->cons_algrm == 1) chain_mf_consensus(s, cp, out, out_cap);
    else chain_consensus(s, cp, out, out_cap);
}

/* Rows of the RC-MSA (host twin: abpoa_generate_rc_msa in poa_cons.c) from the ranks of chain_msa_rank: n_reads rows (+ the
 * consensus row if with_cons) of msa_len codes, gaps = cp->m.  The column of a node is the largest rank in its aligned set,
 * minus one.  Every node id >= 2 writes its base into the rows of the reads in its read set; the consensus row takes the
 * consensus path chain_consensus left in scr[1] (nxt).  Needs the whole CTA. */
POA_DEV void chain_msa_rows(PoaChainSlot *s, const PoaChainParams *cp, int msa_len, int with_cons, uint8_t *rows) {
    const int A = cp->A, W = cp->W, n = s->n_nodes, nr = s->n_reads;
    const int32_t *rank = s->scr[5], *nxt = s->scr[1];
    int32_t *col = s->scr[4];                            /* the rank pass's stack is dead */
    POA_PAR_FOR(v, n) {
        int r = rank[v];
        const int32_t *al = s->aln_id + (size_t)v * A;
        for (int a = 0; a < s->aln_cnt[v]; ++a) if (rank[al[a]] > r) r = rank[al[a]];
        col[v] = r - 1;
    }
    for (int i = 0; i < nr + with_cons; ++i) {
        uint8_t *row = rows + (size_t)i * msa_len;
        POA_PAR_FOR(j, msa_len) row[j] = (uint8_t)cp->m;   /* code m prints as '-' */
    }
    POA_CTA_SYNC();
    POA_PAR_FOR(v, n) {
        if (v >= 2) {                                    /* every node is ranked before SINK, which takes the last rank */
            const uint8_t b = s->base[v];
            const size_t c = (size_t)col[v];
            const uint64_t *rs = s->read_set + (size_t)v * W;
            for (int wd = 0; wd < W; ++wd)
                for (uint64_t bits = rs[wd]; bits; bits &= bits - 1) {
                    const int rd = wd * 64 + POA_CTZ64(bits);
                    rows[(size_t)rd * msa_len + c] = b;
                }
        }
    }
    if (with_cons && POA_TID0) {
        uint8_t *row = rows + (size_t)nr * msa_len;
        for (int cur = nxt[0]; cur != 1 && cur >= 0; cur = nxt[cur]) row[col[cur]] = s->base[cur];
    }
    POA_CTA_SYNC();
}

/* ------------------------------------------------------------------ GFA on the device
 * The record abpoa_generate_gfa prints (layout: poa_gfa_t in poa_internal.h; text: poa_gfa_format in poa_cons.c).  The
 * reference's writer (src/abpoa_output.c:194-294) lists the nodes in FIFO Kahn order from SRC and builds each read's path
 * from the union of the read sets of a node's out-edges, which is the node's read set here.
 *
 * chain_gfa_order (host twin: gfa_describe_host): Kahn from SRC with a FIFO queue, out-edges in list order, stopping when
 * SINK is dequeued -- not the LIFO order of chain_msa_rank.  Serial, on one thread.  Leaves the queue in scr[4] (SRC, then
 * the segments) and returns the number of segments, or -1; *n_link = the segments' in-links from nodes other than SRC.
 * scr[3] holds the in-degrees; scr[1] (the consensus path of chain_consensus) is left alone. */
#define POA_GFA_HDR_WORDS 6             /* header words of a record (POA_GFA_HDR in poa_internal.h) */

POA_DEV int chain_gfa_order(PoaChainSlot *s, const PoaChainParams *cp, int *n_link) {
    if (!POA_TID0) return -1;
    const int K = cp->K, n = s->n_nodes;
    int32_t *deg = s->scr[3], *q = s->scr[4];
    if (s->failed || n < 3) return -1;
    for (int v = 0; v < n; ++v) deg[v] = s->in_cnt[v];
    int head = 0, tail = 0, links = 0;
    q[tail++] = 0;
    while (head < tail) {
        const int cur = q[head++];
        if (cur == 1) { *n_link = links; return head - 2; }
        if (cur != 0) {
            const int32_t *iid = s->in_id + (size_t)cur * K;
            for (int e = 0; e < s->in_cnt[cur]; ++e) links += iid[e] != 0;
        }
        const int32_t *oid = s->out_id + (size_t)cur * K;
        for (int e = 0; e < s->out_cnt[cur]; ++e) {
            const int v = oid[e];
            if (--deg[v] == 0) { if (tail >= n) return -1; q[tail++] = v; }
        }
    }
    return -1;
}

/* The header of a group's record (order on one thread: chain_gfa_order; with_cons: the path chain_consensus left in
 * scr[1]) and its size in int32 words, or -1.  Read sets take the group's own ceil(n_reads / 64) words, not W. */
POA_DEV int64_t chain_gfa_size(PoaChainSlot *s, const PoaChainParams *cp, int with_cons, int32_t *hdr) {
    int n_link = 0;
    const int n_seg = chain_gfa_order(s, cp, &n_link);
    if (n_seg < 0) return -1;
    const int n = s->n_nodes, words = (s->n_reads + 63) / 64;
    int nl = -s->out_cnt[0];
    for (int v = 2; v < n; ++v) nl += s->in_cnt[v];
    int cons_len = -1;
    if (with_cons) {
        const int32_t *nxt = s->scr[1];
        cons_len = 0;
        for (int cur = nxt[0]; cur != 1 && cur >= 0; cur = nxt[cur]) if (++cons_len > n) return -1;
    }
    hdr[0] = n_seg; hdr[1] = n_link; hdr[2] = n - 2; hdr[3] = nl; hdr[4] = words; hdr[5] = cons_len;
    int64_t w = POA_GFA_HDR_WORDS + 3ll * n_seg + n_link + (cons_len > 0 ? cons_len : 0);
    return (w + 1) / 2 * 2 + 2ll * n_seg * words;
}

/* The record itself (header from chain_gfa_size) at `rec`, 8-byte aligned.  Needs the whole CTA; scr[3] becomes the
 * link offsets (the in-degrees are dead). */
POA_DEV void chain_gfa_record(PoaChainSlot *s, const PoaChainParams *cp, const int32_t *hdr, int32_t *rec) {
    const int K = cp->K, W = cp->W;
    const int n_seg = hdr[0], n_link = hdr[1], words = hdr[4], cons_len = hdr[5];
    const int32_t *q = s->scr[4] + 1, *nxt = s->scr[1];
    int32_t *lo = s->scr[3];
    int32_t *seg_id = rec + POA_GFA_HDR_WORDS, *seg_base = seg_id + n_seg, *link_cnt = seg_base + n_seg, *link_from = link_cnt + n_seg;
    int32_t *cons_id = link_from + n_link;
    const int64_t w = POA_GFA_HDR_WORDS + 3ll * n_seg + n_link + (cons_len > 0 ? cons_len : 0);
    uint64_t *sets = reinterpret_cast<uint64_t *>(rec + (w + 1) / 2 * 2);
    if (POA_TID0) for (int k = 0; k < POA_GFA_HDR_WORDS; ++k) rec[k] = hdr[k];
    POA_PAR_FOR(i, n_seg) {
        const int v = q[i];
        const int32_t *iid = s->in_id + (size_t)v * K;
        int c = 0;
        for (int e = 0; e < s->in_cnt[v]; ++e) c += iid[e] != 0;
        seg_id[i] = v; seg_base[i] = s->base[v]; link_cnt[i] = c; lo[i] = c;
    }
    POA_CTA_SYNC();
    cta_excl_scan(lo, n_seg);
    POA_CTA_SYNC();
    POA_PAR_FOR(i, n_seg) {
        const int v = q[i];
        const int32_t *iid = s->in_id + (size_t)v * K;
        int32_t *to = link_from + lo[i];
        for (int e = 0; e < s->in_cnt[v]; ++e) if (iid[e] != 0) *to++ = iid[e];
    }
    POA_PAR_FOR(k, n_seg * words) {
        const int i = k / words, wd = k - i * words;
        sets[k] = s->read_set[(size_t)q[i] * W + wd];
    }
    if (cons_len > 0 && POA_TID0) {
        int j = 0;
        for (int cur = nxt[0]; cur != 1 && cur >= 0 && j < cons_len; cur = nxt[cur]) cons_id[j++] = cur;
    }
    POA_CTA_SYNC();
}

#endif

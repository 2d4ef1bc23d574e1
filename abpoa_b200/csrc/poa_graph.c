/* poa_graph.c -- the partial-order graph on the host.
 *
 * The sequence-to-graph DP runs on the GPU; what stays on the host is the (cheap,
 * strictly sequential) graph bookkeeping between two alignments of a read group:
 * fusing a graph-CIGAR into the graph, re-deriving the topological order, the edge
 * order and the `max_remain` band centre.  Those three decide the DP's row order, its
 * predecessor order and therefore every tie-break, so their behaviour follows the
 * reference exactly (same observable results for the same call sequence):
 *
 *   abpoa_add_graph_edge            reference src/abpoa_graph.c:480-556
 *   abpoa_add_subgraph_alignment    reference src/abpoa_graph.c:689-774
 *   abpoa_BFS_set_node_index        reference src/abpoa_graph.c:221-266  (FIFO Kahn, aligned groups)
 *   edge order (weight, exchange)   reference src/abpoa_graph.c:192-219
 *   abpoa_BFS_set_node_remain       reference src/abpoa_graph.c:268-309
 *   abpoa_topological_sort          reference src/abpoa_graph.c:322-357
 *   MSA column ranks (LIFO Kahn)    reference src/abpoa_graph.c:359-418
 *   abpoa_reset / init / free       reference src/abpoa_graph.c:99-189, 783-875
 *
 * Layout note: abpoa_graph_t / abpoa_node_t are ABI (callers walk them), so nodes keep
 * their per-node edge arrays.  Scratch that the reference re-mallocs on every sort
 * (degree counters, BFS queue) lives in a private tail of the graph object instead.
 */
#include <math.h>
#include <time.h>
#include "poa_internal.h"

/* optional per-thread phase timers (ABPOA_GPU_PROFILE): where does host graph time go */
__thread double poa_prof_ms[8];
static inline double prof_now(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }

#define POA_INL 4                 /* inline edge slots per node and direction */
#define POA_FUSE_AHEAD 12          /* graph-CIGAR ops of look-ahead for the fusion loop's prefetches */

typedef struct {
    abpoa_graph_t pub;          /* must stay first: callers hold &pub */
    int *deg;                   /* degree counters for the Kahn passes */
    int *queue;                 /* BFS queue / DFS stack storage        */
    int scratch_m;
    /* Compact, node-id-indexed mirror of what the per-read passes (two Kahn traversals, edge
     * ordering, flattening for the device) read.  abpoa_node_t is 120 B with separately
     * malloc'ed edge arrays; walking 25 k of those per read is cache-miss bound.  Here the edge
     * lists of nodes with <= POA_INL edges per direction LIVE in four dense slabs (the ABI
     * pointers node[].in_id etc. point into them; capacity field == POA_INL), and degrees /
     * residues / aligned-set sizes are mirrored in dense arrays, so a pass touches ~40 B per node. */
    int slab_m;
    int *in_id4, *in_w4, *out_id4, *out_w4;     /* [slab_m][POA_INL] */
    int *aln4;                                  /* [slab_m][POA_INL] first aligned-group members (copy of node[].aligned_node_id) */
    int *cin, *cout;                            /* == node[].in_edge_n / out_edge_n */
    int *caln;                                  /* == node[].aligned_node_n          */
    uint8_t *cbase;                             /* == node[].base                    */
    int *cnread, *cspan;                        /* AUTHORITATIVE n_read / n_span_read while public_stale is set */
    int span_pending;                           /* whole-graph "+1 span read on every node" not yet folded into cspan */
    int public_stale;                           /* node[].n_read / n_span_read lag behind the dense arrays */
    int has_read_ids;                           /* some out-edge carries a read-id bitset */
    int msa_installed;                          /* abc holds RC-MSA rows computed elsewhere (poa_msa_install) for this graph */
    const int32_t *gfa_rec;                     /* borrowed GFA record computed elsewhere (poa_gfa_install), or NULL */
    int *touched; int n_touched, touched_m; uint8_t *touch_mark;   /* nodes whose edge lists changed since the last ordering */
    int64_t n_edges;                            /* total in-edges in the graph        */
    /* nodes the Kahn passes must COUNT for: in-degree >= 2 or member of an aligned group (forward
     * pass), out-degree >= 2 (reverse pass).  Everything else is a plain chain link and is pushed
     * the moment its only neighbour is dequeued, without touching a counter. */
    int *fwd_list, n_fwd, fwd_m; uint8_t *fwd_mark;
    int *rev_list, n_rev, rev_m; uint8_t *rev_mark;
    /* Spliced topological order (poa_graph_set_fast_order).  The DP result does not depend on
     * WHICH topological order the rows follow in global mode, so instead of a full Kahn pass
     * after every read the previous order is kept and the nodes the read created are spliced in
     * behind their anchors (see splice_order).  Recorded while a read is threaded: */
    int fast_order;                             /* enabled by the batch engine for this handle      */
    int tracking, old_n;                        /* a fusion onto a sorted graph is being recorded    */
    int *new_ids, *new_anchor; int n_new, new_m;
    int *new_edges; int n_new_edges, new_edges_m;   /* (from,to) pairs of new edges between old nodes */
    int64_t n_spliced, n_splice_fallback;
} poa_graph_x;

static inline poa_graph_x *gx(abpoa_graph_t *abg) { return (poa_graph_x *)abg; }
static inline const poa_graph_x *cgx(const abpoa_graph_t *abg) { return (const poa_graph_x *)abg; }

static void scratch_reserve(abpoa_graph_t *abg, int n) {
    poa_graph_x *x = gx(abg);
    if (n <= x->scratch_m) return;
    int m = poa_roundup32(n);
    x->deg = (int *)poa_xrealloc(x->deg, (size_t)m * sizeof(int));
    x->queue = (int *)poa_xrealloc(x->queue, (size_t)m * sizeof(int));
    x->scratch_m = m;
}

/* ------------------------------------------------------------------ nodes */
static void node_blank(abpoa_node_t *nd, int id) {
    memset(nd, 0, sizeof *nd);
    nd->node_id = id;
}

static void node_release(abpoa_node_t *nd) {
    if (nd->in_edge_m > POA_INL) { free(nd->in_id); free(nd->in_edge_weight); }
    if (nd->out_edge_m > POA_INL) { free(nd->out_id); free(nd->out_edge_weight); }
    if (nd->read_ids) {
        if (nd->read_ids_n > 0)
            for (int j = 0; j < nd->out_edge_m; ++j) free(nd->read_ids[j]);
        free(nd->read_ids);
    }
    if (nd->m_read > 0) free(nd->read_weight);
    if (nd->aligned_node_m > 0) free(nd->aligned_node_id);
}

/* grow the node array and the mirror; inline edge pointers are re-aimed at the moved slabs */
static void nodes_reserve(abpoa_graph_t *abg, int want) {
    if (want <= abg->node_m) return;
    poa_graph_x *x = gx(abg);
    const int old = abg->node_m, m = poa_roundup32(want);
    abg->node = (abpoa_node_t *)poa_xrealloc(abg->node, (size_t)m * sizeof(abpoa_node_t));
    for (int i = old; i < m; ++i) node_blank(&abg->node[i], i);
    abg->node_m = m;
    x->in_id4 = (int *)poa_xrealloc(x->in_id4, (size_t)m * POA_INL * sizeof(int));
    x->in_w4 = (int *)poa_xrealloc(x->in_w4, (size_t)m * POA_INL * sizeof(int));
    x->out_id4 = (int *)poa_xrealloc(x->out_id4, (size_t)m * POA_INL * sizeof(int));
    x->out_w4 = (int *)poa_xrealloc(x->out_w4, (size_t)m * POA_INL * sizeof(int));
    x->aln4 = (int *)poa_xrealloc(x->aln4, (size_t)m * POA_INL * sizeof(int));
    x->cin = (int *)poa_xrealloc(x->cin, (size_t)m * sizeof(int));
    x->cout = (int *)poa_xrealloc(x->cout, (size_t)m * sizeof(int));
    x->caln = (int *)poa_xrealloc(x->caln, (size_t)m * sizeof(int));
    x->cbase = (uint8_t *)poa_xrealloc(x->cbase, (size_t)m);
    x->cnread = (int *)poa_xrealloc(x->cnread, (size_t)m * sizeof(int)); x->cspan = (int *)poa_xrealloc(x->cspan, (size_t)m * sizeof(int));
    memset(x->cnread + old, 0, (size_t)(m - old) * sizeof(int)); memset(x->cspan + old, 0, (size_t)(m - old) * sizeof(int));
    x->touch_mark = (uint8_t *)poa_xrealloc(x->touch_mark, (size_t)m);
    x->fwd_mark = (uint8_t *)poa_xrealloc(x->fwd_mark, (size_t)m); x->rev_mark = (uint8_t *)poa_xrealloc(x->rev_mark, (size_t)m);
    memset(x->fwd_mark + old, 0, (size_t)(m - old)); memset(x->rev_mark + old, 0, (size_t)(m - old));
    memset(x->cin + old, 0, (size_t)(m - old) * sizeof(int)); memset(x->cout + old, 0, (size_t)(m - old) * sizeof(int));
    memset(x->caln + old, 0, (size_t)(m - old) * sizeof(int)); memset(x->cbase + old, 0, (size_t)(m - old));
    memset(x->touch_mark + old, 0, (size_t)(m - old));
    x->slab_m = m;
    for (int i = 0; i < old; ++i) {
        abpoa_node_t *nd = &abg->node[i];
        if (nd->in_edge_m == POA_INL) { nd->in_id = x->in_id4 + (size_t)i * POA_INL; nd->in_edge_weight = x->in_w4 + (size_t)i * POA_INL; }
        if (nd->out_edge_m == POA_INL) { nd->out_id = x->out_id4 + (size_t)i * POA_INL; nd->out_edge_weight = x->out_w4 + (size_t)i * POA_INL; }
    }
}

static inline void list_push(int **list, int *n, int *m, int id) {
    if (*n == *m) { *m = *m ? *m << 1 : 1024; *list = (int *)poa_xrealloc(*list, (size_t)*m * sizeof(int)); }
    (*list)[(*n)++] = id;
}
static inline void mark_fwd_counted(poa_graph_x *x, int id) { if (!x->fwd_mark[id]) { x->fwd_mark[id] = 1; list_push(&x->fwd_list, &x->n_fwd, &x->fwd_m, id); } }
static inline void mark_rev_counted(poa_graph_x *x, int id) { if (!x->rev_mark[id]) { x->rev_mark[id] = 1; list_push(&x->rev_list, &x->n_rev, &x->rev_m, id); } }

static inline void touch(poa_graph_x *x, int id) {
    if (x->touch_mark[id]) return;
    x->touch_mark[id] = 1;
    if (x->n_touched == x->touched_m) {
        x->touched_m = x->touched_m ? x->touched_m << 1 : 1024;
        x->touched = (int *)poa_xrealloc(x->touched, (size_t)x->touched_m * sizeof(int));
    }
    x->touched[x->n_touched++] = id;
}

abpoa_graph_t *poa_graph_new(void) {
    poa_graph_x *x = (poa_graph_x *)poa_xcalloc(1, sizeof(poa_graph_x));
    abpoa_graph_t *abg = &x->pub;
    abg->node_m = 0;
    nodes_reserve(abg, 2);
    abg->node_n = 2;                 /* SRC = 0, SINK = 1 always exist */
    return abg;
}

void poa_graph_free(abpoa_graph_t *abg) {
    if (!abg) return;
    poa_graph_x *x = gx(abg);
    for (int i = 0; i < abg->node_m; ++i) node_release(&abg->node[i]);
    free(abg->node);
    free(abg->index_to_node_id); free(abg->node_id_to_index); free(abg->node_id_to_msa_rank);
    free(abg->node_id_to_max_pos_left); free(abg->node_id_to_max_pos_right); free(abg->node_id_to_max_remain);
    free(x->deg); free(x->queue);
    free(x->in_id4); free(x->in_w4); free(x->out_id4); free(x->out_w4); free(x->aln4);
    free(x->cin); free(x->cout); free(x->caln); free(x->cbase); free(x->cnread); free(x->cspan); free(x->touched); free(x->touch_mark); free(x->fwd_list); free(x->fwd_mark); free(x->rev_list); free(x->rev_mark); free(x->new_ids); free(x->new_anchor); free(x->new_edges);
    free(x);
}

/* per-node index arrays: grow together, allocate the optional ones on first need */
static void index_arrays_reserve(abpoa_graph_t *abg, const abpoa_para_t *abpt, int n) {
    int m = abg->index_rank_m;
    if (n > m) {
        m = poa_roundup32(n);
        abg->index_to_node_id = (int *)poa_xrealloc(abg->index_to_node_id, (size_t)m * sizeof(int));
        abg->node_id_to_index = (int *)poa_xrealloc(abg->node_id_to_index, (size_t)m * sizeof(int));
        if (abg->node_id_to_msa_rank) abg->node_id_to_msa_rank = (int *)poa_xrealloc(abg->node_id_to_msa_rank, (size_t)m * sizeof(int));
        if (abg->node_id_to_max_pos_left) {
            abg->node_id_to_max_pos_left = (int *)poa_xrealloc(abg->node_id_to_max_pos_left, (size_t)m * sizeof(int));
            abg->node_id_to_max_pos_right = (int *)poa_xrealloc(abg->node_id_to_max_pos_right, (size_t)m * sizeof(int));
        }
        if (abg->node_id_to_max_remain) abg->node_id_to_max_remain = (int *)poa_xrealloc(abg->node_id_to_max_remain, (size_t)m * sizeof(int));
        abg->index_rank_m = m;
    }
    if (abpt) {
        if ((abpt->out_msa || abpt->max_n_cons > 1 || abpt->cons_algrm == ABPOA_MF) && !abg->node_id_to_msa_rank)
            abg->node_id_to_msa_rank = (int *)poa_xmalloc((size_t)m * sizeof(int));
        if (abpt->wb >= 0 && !abg->node_id_to_max_pos_left) {
            abg->node_id_to_max_pos_left = (int *)poa_xmalloc((size_t)m * sizeof(int));
            abg->node_id_to_max_pos_right = (int *)poa_xmalloc((size_t)m * sizeof(int));
        }
        if ((abpt->wb >= 0 || abpt->zdrop > 0) && !abg->node_id_to_max_remain)
            abg->node_id_to_max_remain = (int *)poa_xmalloc((size_t)m * sizeof(int));
    }
}

abpoa_cons_t *poa_cons_new(void) { return (abpoa_cons_t *)poa_xcalloc(1, sizeof(abpoa_cons_t)); }

void poa_cons_clear(abpoa_cons_t *abc) {
    if (abc->n_cons > 0) {
        free(abc->clu_n_seq); free(abc->cons_len);
        for (int i = 0; i < abc->n_cons; ++i) {
            if (abc->cons_node_ids) free(abc->cons_node_ids[i]);
            if (abc->cons_base) free(abc->cons_base[i]);
            if (abc->cons_cov) free(abc->cons_cov[i]);
            if (abc->clu_read_ids) free(abc->clu_read_ids[i]);
            if (abc->cons_phred_score) free(abc->cons_phred_score[i]);
        }
        free(abc->cons_node_ids); free(abc->cons_base); free(abc->cons_cov);
        free(abc->clu_read_ids); free(abc->cons_phred_score);
    }
    if (abc->msa_len > 0 && abc->msa_base) {
        for (int i = 0; i < abc->n_seq + abc->n_cons; ++i) free(abc->msa_base[i]);
        free(abc->msa_base);
    }
    memset(abc, 0, sizeof *abc);
}

void poa_cons_free(abpoa_cons_t *abc) { if (abc) { poa_cons_clear(abc); free(abc); } }

void abpoa_clean_msa_cons(abpoa_t *ab) { poa_cons_clear(ab->abc); }

/* ------------------------------------------------------------------ handle */
abpoa_t *abpoa_init(void) {
    abpoa_t *ab = (abpoa_t *)poa_xmalloc(sizeof(abpoa_t));
    ab->abg = poa_graph_new();
    ab->abs = poa_seq_new();
    ab->abm = (abpoa_simd_matrix_t *)poa_xcalloc(1, sizeof(abpoa_simd_matrix_t));
    ab->abc = poa_cons_new();
    return ab;
}

void abpoa_free(abpoa_t *ab) {
    if (!ab) return;
    poa_graph_free(ab->abg);
    poa_seq_free(ab->abs);
    if (ab->abm) {
        if (ab->abm->s_mem) poa_dev_ctx_free((poa_dev_ctx *)ab->abm->s_mem);
        free(ab->abm->dp_beg); free(ab->abm->dp_end); free(ab->abm->dp_beg_sn); free(ab->abm->dp_end_sn);
        free(ab->abm);
    }
    poa_cons_free(ab->abc);
    free(ab);
}

/* Empty the graph but keep every allocation for the next read group. */
void abpoa_reset(abpoa_t *ab, abpoa_para_t *abpt, int qlen) {
    abpoa_graph_t *abg = ab->abg;
    abg->is_topological_sorted = abg->is_called_cons = abg->is_set_msa_rank = 0;
    for (int i = 0; i < abg->node_n; ++i) {
        abpoa_node_t *nd = &abg->node[i];
        if (nd->read_ids_n > 0)
            for (int j = 0; j < nd->out_edge_n; ++j) memset(nd->read_ids[j], 0, (size_t)nd->read_ids_n * sizeof(uint64_t));
        nd->in_edge_n = nd->out_edge_n = nd->aligned_node_n = 0;
        nd->n_read = nd->n_span_read = 0;
        /* invariant of the dense mirror: "degree <= POA_INL  <=>  edges live in the slabs".
         * A node that spilled to the heap goes back to its inline slots for the next group. */
        if (nd->in_edge_m > POA_INL) {
            free(nd->in_id); free(nd->in_edge_weight);
            nd->in_id = gx(abg)->in_id4 + (size_t)i * POA_INL; nd->in_edge_weight = gx(abg)->in_w4 + (size_t)i * POA_INL; nd->in_edge_m = POA_INL;
        }
        if (nd->out_edge_m > POA_INL) {
            free(nd->out_id); free(nd->out_edge_weight);
            if (nd->read_ids && nd->read_ids_n > 0)
                for (int j = POA_INL; j < nd->out_edge_m; ++j) free(nd->read_ids[j]);
            nd->out_id = gx(abg)->out_id4 + (size_t)i * POA_INL; nd->out_edge_weight = gx(abg)->out_w4 + (size_t)i * POA_INL; nd->out_edge_m = POA_INL;
        }
    }
    {
        poa_graph_x *x = gx(abg);
        memset(x->cin, 0, (size_t)abg->node_n * sizeof(int)); memset(x->cout, 0, (size_t)abg->node_n * sizeof(int));
        memset(x->caln, 0, (size_t)abg->node_n * sizeof(int));
        memset(x->cnread, 0, (size_t)abg->node_n * sizeof(int)); memset(x->cspan, 0, (size_t)abg->node_n * sizeof(int));
        x->span_pending = 0; x->public_stale = 0; x->has_read_ids = 0; x->msa_installed = 0; x->gfa_rec = NULL;
        for (int t = 0; t < x->n_touched; ++t) x->touch_mark[x->touched[t]] = 0;
        x->n_touched = 0; x->n_edges = 0;
        for (int t = 0; t < x->n_fwd; ++t) x->fwd_mark[x->fwd_list[t]] = 0;
        for (int t = 0; t < x->n_rev; ++t) x->rev_mark[x->rev_list[t]] = 0;
        x->n_fwd = x->n_rev = 0;
        x->tracking = 0; x->n_new = x->n_new_edges = 0;
    }
    abg->node_n = 2;
    nodes_reserve(abg, qlen + 2);
    index_arrays_reserve(abg, abpt, abg->node_m);
    ab->abs->n_seq = 0;
    poa_cons_clear(ab->abc);
}

/* ------------------------------------------------------------------ edges */
/* edge storage: the first POA_INL edges live inline in the slabs, more spill to the heap */
static void in_edges_reserve(poa_graph_x *x, int id, int want) {
    abpoa_node_t *nd = &x->pub.node[id];
    if (want <= nd->in_edge_m) return;
    if (want <= POA_INL) {
        nd->in_id = x->in_id4 + (size_t)id * POA_INL; nd->in_edge_weight = x->in_w4 + (size_t)id * POA_INL; nd->in_edge_m = POA_INL;
        return;
    }
    const int m = poa_roundup32(want);
    int *ids = (int *)poa_xmalloc((size_t)m * sizeof(int)), *ws = (int *)poa_xmalloc((size_t)m * sizeof(int));
    memcpy(ids, nd->in_id, (size_t)nd->in_edge_n * sizeof(int)); memcpy(ws, nd->in_edge_weight, (size_t)nd->in_edge_n * sizeof(int));
    if (nd->in_edge_m > POA_INL) { free(nd->in_id); free(nd->in_edge_weight); }
    nd->in_id = ids; nd->in_edge_weight = ws; nd->in_edge_m = m;
}

static void out_edges_reserve(poa_graph_x *x, int id, int want, int want_read_ids) {
    abpoa_node_t *nd = &x->pub.node[id];
    if (want > nd->out_edge_m) {
        const int old = nd->out_edge_m;
        int m;
        if (want <= POA_INL) {
            m = POA_INL;
            nd->out_id = x->out_id4 + (size_t)id * POA_INL; nd->out_edge_weight = x->out_w4 + (size_t)id * POA_INL;
        } else {
            m = poa_roundup32(want);
            int *ids = (int *)poa_xmalloc((size_t)m * sizeof(int)), *ws = (int *)poa_xmalloc((size_t)m * sizeof(int));
            memcpy(ids, nd->out_id, (size_t)nd->out_edge_n * sizeof(int)); memcpy(ws, nd->out_edge_weight, (size_t)nd->out_edge_n * sizeof(int));
            if (old > POA_INL) { free(nd->out_id); free(nd->out_edge_weight); }
            nd->out_id = ids; nd->out_edge_weight = ws;
        }
        if (nd->read_ids) {
            nd->read_ids = (uint64_t **)poa_xrealloc(nd->read_ids, (size_t)m * sizeof(uint64_t *));
            for (int j = old; j < m; ++j)
                nd->read_ids[j] = nd->read_ids_n > 0 ? (uint64_t *)poa_xcalloc(nd->read_ids_n, sizeof(uint64_t)) : NULL;
        }
        nd->out_edge_m = m;
    }
    if (want_read_ids && !nd->read_ids)
        nd->read_ids = (uint64_t **)poa_xcalloc(nd->out_edge_m, sizeof(uint64_t *));
}

/* make every out-edge slot of `nd` hold a bitset of at least `words` 64-bit words */
static void read_ids_widen(abpoa_node_t *nd, int words) {
    if (nd->read_ids_n >= words) return;
    for (int j = 0; j < nd->out_edge_m; ++j) {
        if (nd->read_ids_n == 0) nd->read_ids[j] = (uint64_t *)poa_xcalloc(words, sizeof(uint64_t));
        else {
            nd->read_ids[j] = (uint64_t *)poa_xrealloc(nd->read_ids[j], (size_t)words * sizeof(uint64_t));
            memset(nd->read_ids[j] + nd->read_ids_n, 0, (size_t)(words - nd->read_ids_n) * sizeof(uint64_t));
        }
    }
    nd->read_ids_n = words;
}

int abpoa_add_graph_node(abpoa_graph_t *abg, uint8_t base) {
    int id = abg->node_n;
    nodes_reserve(abg, id + 1);
    abg->node[id].base = base;
    gx(abg)->cbase[id] = base;
    abg->node_n = id + 1;
    return id;
}

/* Fold the dense n_read / n_span_read counters back into the ABI node structs.  The per-read
 * fusion loop only updates the dense arrays (it would otherwise drag every 120-byte node of
 * the path through the cache once more); every PUBLIC entry point that finishes a mutation,
 * and everything that reads the counters, calls this first. */
void poa_graph_sync_public(abpoa_graph_t *abg) {
    poa_graph_x *x = gx(abg);
    if (!x->public_stale && !x->span_pending) return;
    const int n = abg->node_n, add = x->span_pending;
    for (int i = 0; i < n; ++i) {
        x->cspan[i] += add;
        abg->node[i].n_read = x->cnread[i]; abg->node[i].n_span_read = x->cspan[i];
    }
    x->span_pending = 0; x->public_stale = 0;
}

static int edge_add(abpoa_graph_t *abg, int from_id, int to_id, int check_edge, int w, uint8_t add_read_id,
                    uint8_t add_read_weight, int read_id, int read_ids_n, int tot_read_n);

int abpoa_add_graph_edge(abpoa_graph_t *abg, int from_id, int to_id, int check_edge, int w, uint8_t add_read_id,
                         uint8_t add_read_weight, int read_id, int read_ids_n, int tot_read_n) {
    const int r = edge_add(abg, from_id, to_id, check_edge, w, add_read_id, add_read_weight, read_id, read_ids_n, tot_read_n);
    abg->node[from_id].n_read = gx(abg)->cnread[from_id];
    return r;
}

static int edge_add(abpoa_graph_t *abg, int from_id, int to_id, int check_edge, int w, uint8_t add_read_id,
                    uint8_t add_read_weight, int read_id, int read_ids_n, int tot_read_n) {
    if (from_id < 0 || from_id >= abg->node_n || to_id < 0 || to_id >= abg->node_n)
        poa_die(__func__, "node_n: %d\tfrom_id: %d\tto_id: %d.", abg->node_n, from_id, to_id);
    poa_graph_x *x = gx(abg);
    abpoa_node_t *from = &abg->node[from_id], *to = &abg->node[to_id];
    int slot = -1;
    if (check_edge) {            /* the edge may exist already: bump both copies of its weight */
        /* degrees and inline edge lists come from the dense mirror: no 120-byte node structs touched */
        const int nin = x->cin[to_id], nout = x->cout[from_id];
        int *iid = nin <= POA_INL ? x->in_id4 + (size_t)to_id * POA_INL : to->in_id;
        int *iw = nin <= POA_INL ? x->in_w4 + (size_t)to_id * POA_INL : to->in_edge_weight;
        int *oid = nout <= POA_INL ? x->out_id4 + (size_t)from_id * POA_INL : from->out_id;
        int *ow = nout <= POA_INL ? x->out_w4 + (size_t)from_id * POA_INL : from->out_edge_weight;
        /* A list in non-increasing weight order is a fixed point of the exchange pass, so a node
         * needs re-ordering only when a bump (or an append) breaks that order. */
        for (int i = 0; i < nin; ++i)
            if (iid[i] == from_id) { iw[i] += w; if (i > 0 && iw[i - 1] < iw[i]) touch(x, to_id); break; }
        for (int i = 0; i < nout; ++i)
            if (oid[i] == to_id) { ow[i] += w; slot = i; if (i > 0 && ow[i - 1] < ow[i]) touch(x, from_id); break; }
    }
    if (slot < 0) {              /* new edge, appended after the existing ones */
        in_edges_reserve(x, to_id, to->in_edge_n + 1);
        to->in_id[to->in_edge_n] = from_id; to->in_edge_weight[to->in_edge_n] = w; x->cin[to_id] = ++to->in_edge_n;
        if (to->in_edge_n == 2) mark_fwd_counted(x, to_id);
        out_edges_reserve(x, from_id, from->out_edge_n + 1, add_read_id);
        slot = from->out_edge_n;
        from->out_id[slot] = to_id; from->out_edge_weight[slot] = w; x->cout[from_id] = ++from->out_edge_n;
        x->n_edges += 1;
        if (x->tracking && from_id < x->old_n && to_id < x->old_n) {
            if (x->n_new_edges + 2 > x->new_edges_m) { x->new_edges_m = x->new_edges_m ? x->new_edges_m << 1 : 256; x->new_edges = (int *)poa_xrealloc(x->new_edges, (size_t)x->new_edges_m * sizeof(int)); }
            x->new_edges[x->n_new_edges++] = from_id; x->new_edges[x->n_new_edges++] = to_id;
        }
        if (to->in_edge_n > 1 && to->in_edge_weight[to->in_edge_n - 2] < w) touch(x, to_id);
        if (slot > 0 && from->out_edge_weight[slot - 1] < w) touch(x, from_id);
    }
    if (add_read_id) {           /* which reads run through this edge: feeds the RC-MSA */
        if (read_ids_n <= 0) poa_die(__func__, "Unexpected read_ids_n: %d.", read_ids_n);
        out_edges_reserve(x, from_id, from->out_edge_n, 1);
        read_ids_widen(from, read_ids_n);
        from->read_ids[slot][read_id >> 6] |= 1ULL << (read_id & 63);
        x->has_read_ids = 1;
    }
    x->cnread[from_id] += 1; x->public_stale = 1;
    if (add_read_weight) {
        if (tot_read_n > from->m_read) {
            from->read_weight = (int *)poa_xrealloc(from->read_weight, (size_t)tot_read_n * sizeof(int));
            memset(from->read_weight + from->m_read, 0, (size_t)(tot_read_n - from->m_read) * sizeof(int));
            from->m_read = tot_read_n;
        }
        from->read_weight[read_id] = w;
    }
    return 1;
}

/* nodes that occupy the same MSA column ("aligned" = mismatch alternatives) */
static void aligned_push_raw(abpoa_node_t *nd, int id);
static inline void aligned_push(abpoa_graph_t *abg, int owner, int id) {
    abpoa_node_t *nd = &abg->node[owner];
    if (nd->aligned_node_n < POA_INL) gx(abg)->aln4[(size_t)owner * POA_INL + nd->aligned_node_n] = id;
    aligned_push_raw(nd, id);
}
static void aligned_push_raw(abpoa_node_t *nd, int id) {
    if (nd->aligned_node_n == nd->aligned_node_m) {
        int m = nd->aligned_node_m ? nd->aligned_node_m << 1 : 2;
        nd->aligned_node_id = (int *)(nd->aligned_node_m ? poa_xrealloc(nd->aligned_node_id, (size_t)m * sizeof(int)) : poa_xmalloc((size_t)m * sizeof(int)));
        nd->aligned_node_m = m;
    }
    nd->aligned_node_id[nd->aligned_node_n++] = id;
}

static void aligned_join(abpoa_graph_t *abg, int node_id, int new_id) {
    abpoa_node_t *node = abg->node; int *caln = gx(abg)->caln;
    mark_fwd_counted(gx(abg), node_id); mark_fwd_counted(gx(abg), new_id);
    for (int i = 0; i < node[node_id].aligned_node_n; ++i) {
        int sib = node[node_id].aligned_node_id[i];
        mark_fwd_counted(gx(abg), sib);
        aligned_push(abg, sib, new_id); caln[sib] = node[sib].aligned_node_n;
        aligned_push(abg, new_id, sib);
    }
    aligned_push(abg, node_id, new_id); caln[node_id] = node[node_id].aligned_node_n;
    aligned_push(abg, new_id, node_id); caln[new_id] = node[new_id].aligned_node_n;
}

static int aligned_with_base(const abpoa_graph_t *abg, int node_id, uint8_t base) {
    const poa_graph_x *x = cgx(abg);
    const int na = x->caln[node_id];
    if (na == 0) return -1;
    const int *al = na <= POA_INL ? x->aln4 + (size_t)node_id * POA_INL : abg->node[node_id].aligned_node_id;
    for (int i = 0; i < na; ++i)
        if (x->cbase[al[i]] == base) return al[i];
    return -1;
}

/* ------------------------------------------------------------------ orders */
/* Topological index = dequeue order of a FIFO Kahn traversal in which a node becomes
 * ready only together with all nodes of its aligned group; the group is enqueued as
 * (trigger node, then its aligned list in stored order). */
/* edge list of node v in direction `out`: inline slab row or the heap spill */
static inline const int *out_ids_of(const poa_graph_x *x, int v) { return x->cout[v] <= POA_INL ? x->out_id4 + (size_t)v * POA_INL : x->pub.node[v].out_id; }
static inline const int *out_ws_of(const poa_graph_x *x, int v) { return x->cout[v] <= POA_INL ? x->out_w4 + (size_t)v * POA_INL : x->pub.node[v].out_edge_weight; }
static inline const int *in_ids_of(const poa_graph_x *x, int v) { return x->cin[v] <= POA_INL ? x->in_id4 + (size_t)v * POA_INL : x->pub.node[v].in_id; }

void abpoa_BFS_set_node_index(abpoa_graph_t *abg, int src_id, int sink_id) {
    const int n = abg->node_n;
    scratch_reserve(abg, n);
    const poa_graph_x *x = gx(abg);
    int *deg = gx(abg)->deg, *q = gx(abg)->queue;
    const abpoa_node_t *node = abg->node;
    const int *cin = x->cin, *cout = x->cout, *caln = x->caln;
    /* only "counted" nodes (in-degree >= 2 or in an aligned group) need an in-degree counter */
    for (int t = 0; t < x->n_fwd; ++t) { const int v = x->fwd_list[t]; deg[v] = cin[v]; }
    int *index_to_node_id = abg->index_to_node_id, *node_id_to_index = abg->node_id_to_index;
    int head = 0, tail = 0, index = 0;
    q[tail++] = src_id;
    while (head < tail) {
        const int cur = q[head++];
        index_to_node_id[index] = cur;
        node_id_to_index[cur] = index++;
        if (cur == sink_id) return;
        const int ne = cout[cur]; const int *oid = out_ids_of(x, cur);
        for (int e = 0; e < ne; ++e) {
            const int v = oid[e];
            const int na = caln[v];
            if (cin[v] == 1 && na == 0) { q[tail++] = v; continue; }       /* chain link: ready at once */
            if (--deg[v] != 0) continue;
            if (na) {                                   /* ready only together with its whole aligned group */
                const int *al = na <= POA_INL ? x->aln4 + (size_t)v * POA_INL : node[v].aligned_node_id;
                int ready = 1;
                for (int a = 0; a < na; ++a) if (deg[al[a]] != 0) { ready = 0; break; }
                if (!ready) continue;
                q[tail++] = v;
                for (int a = 0; a < na; ++a) q[tail++] = al[a];
            } else q[tail++] = v;
        }
    }
    poa_die(__func__, "Failed to set node index.");
}

/* Edge lists ordered by weight, heaviest first.  This is the DP's predecessor order and
 * the order every tie is broken in, so the permutation must be the one the reference's
 * in-place exchange pass produces (swap whenever w[j] < w[k], j < k; not stable).  The pass
 * is idempotent (a list it produced is left unchanged), so only nodes whose lists changed
 * since the previous ordering need it. */
static void order_edges_of(abpoa_node_t *nd) {
    for (int j = 0; j + 1 < nd->in_edge_n; ++j)
        for (int k = j + 1; k < nd->in_edge_n; ++k)
            if (nd->in_edge_weight[j] < nd->in_edge_weight[k]) {
                int t = nd->in_id[j]; nd->in_id[j] = nd->in_id[k]; nd->in_id[k] = t;
                t = nd->in_edge_weight[j]; nd->in_edge_weight[j] = nd->in_edge_weight[k]; nd->in_edge_weight[k] = t;
            }
    for (int j = 0; j + 1 < nd->out_edge_n; ++j)
        for (int k = j + 1; k < nd->out_edge_n; ++k)
            if (nd->out_edge_weight[j] < nd->out_edge_weight[k]) {
                int t = nd->out_id[j]; nd->out_id[j] = nd->out_id[k]; nd->out_id[k] = t;
                t = nd->out_edge_weight[j]; nd->out_edge_weight[j] = nd->out_edge_weight[k]; nd->out_edge_weight[k] = t;
                if (nd->read_ids_n > 0) { uint64_t *r = nd->read_ids[j]; nd->read_ids[j] = nd->read_ids[k]; nd->read_ids[k] = r; }
            }
}

static inline void exchange_order(int *ids, int *ws, int n) {
    for (int j = 0; j + 1 < n; ++j)
        for (int k = j + 1; k < n; ++k)
            if (ws[j] < ws[k]) { int t = ids[j]; ids[j] = ids[k]; ids[k] = t; t = ws[j]; ws[j] = ws[k]; ws[k] = t; }
}

static void order_edges_by_weight(abpoa_graph_t *abg) {
    poa_graph_x *x = gx(abg);
    for (int t = 0; t < x->n_touched; ++t) {
        const int id = x->touched[t];
        x->touch_mark[id] = 0;
        if (id >= abg->node_n) continue;
        const int ni = x->cin[id], no = x->cout[id];
        if (!x->has_read_ids && ni <= POA_INL && no <= POA_INL) {       /* common case: all in the slabs */
            if (ni > 1) exchange_order(x->in_id4 + (size_t)id * POA_INL, x->in_w4 + (size_t)id * POA_INL, ni);
            if (no > 1) exchange_order(x->out_id4 + (size_t)id * POA_INL, x->out_w4 + (size_t)id * POA_INL, no);
        } else order_edges_of(&abg->node[id]);
    }
    x->n_touched = 0;
}

/* max_remain[v] = 1 + max_remain[heaviest out-neighbour, first on ties]; SINK = -1: the centre
 * line of the adaptive band.  The reference runs a reverse Kahn traversal from the sink
 * (src/abpoa_graph.c:333-389); the values depend only on the out-neighbours, so one backward sweep
 * over the topological order just computed gives the same numbers without queue or counters. */
void abpoa_BFS_set_node_remain(abpoa_graph_t *abg, int src_id, int sink_id) {
    const poa_graph_x *x = gx(abg);
    int *remain = abg->node_id_to_max_remain;
    const int *cout = x->cout, *order = abg->index_to_node_id;
    const int lo = abg->node_id_to_index[src_id], hi = abg->node_id_to_index[sink_id];
    if (lo < 0 || hi >= abg->node_n || lo > hi) poa_die(__func__, "Failed to set node remain.");
    remain[sink_id] = -1;
    for (int i = hi - 1; i >= lo; --i) {
        const int cur = order[i];
        if (i - 16 >= lo) {                          /* the order is known: fetch the mirror rows of the nodes ahead */
            const size_t v = (size_t)order[i - 16];
            __builtin_prefetch(cout + v, 0); __builtin_prefetch(x->out_id4 + v * POA_INL, 0); __builtin_prefetch(x->out_w4 + v * POA_INL, 0);
            __builtin_prefetch(remain + v, 1);
        }
        const int ne = cout[cur]; const int *oid = out_ids_of(x, cur);
        if (ne == 1) remain[cur] = remain[oid[0]] + 1;
        else {
            const int *ow = out_ws_of(x, cur);
            int best_w = -1, best = sink_id;
            for (int e = 0; e < ne; ++e) if (ow[e] > best_w) { best_w = ow[e]; best = oid[e]; }
            remain[cur] = remain[best] + 1;
        }
    }
}

/* ------------------------------------------------------------------ spliced order
 * Invariant shared with the Kahn order above: the members of an aligned group occupy consecutive
 * rows.  A read's path is monotone in the rows of the order it was aligned in, so
 *   - a new node aligned to x goes right behind x's group,
 *   - a new unaligned (inserted) node goes right behind the group of the previous path node
 *     (or inherits the anchor of the previous node if that one is new as well),
 * which keeps every old and every new edge pointing forward and the groups consecutive.  Anchors
 * come out in non-decreasing order along the path, so the splice is one backward merge.  New
 * edges between OLD nodes are re-checked; a violation falls back to the full Kahn pass. */
void poa_graph_set_fast_order(abpoa_graph_t *abg, int on) { gx(abg)->fast_order = on; }
void poa_graph_order_stats(const abpoa_graph_t *abg, int64_t *spliced, int64_t *fallback) { *spliced = cgx(abg)->n_spliced; *fallback = cgx(abg)->n_splice_fallback; }

static inline int group_last_row(const abpoa_graph_t *abg, int v) {
    const poa_graph_x *x = cgx(abg);
    int r = abg->node_id_to_index[v];
    const int na = x->caln[v];
    if (na == 0) return r;
    const int *al = na <= POA_INL ? x->aln4 + (size_t)v * POA_INL : abg->node[v].aligned_node_id;
    for (; r + 1 < x->old_n; ++r) {
        const int u = abg->index_to_node_id[r + 1];
        int member = 0;
        for (int a = 0; a < na; ++a) if (al[a] == u) { member = 1; break; }
        if (!member) break;
    }
    return r;
}
static inline void record_new_node(poa_graph_x *x, int id, int anchor) {
    if (x->n_new == x->new_m) {
        x->new_m = x->new_m ? x->new_m << 1 : 256;
        x->new_ids = (int *)poa_xrealloc(x->new_ids, (size_t)x->new_m * sizeof(int));
        x->new_anchor = (int *)poa_xrealloc(x->new_anchor, (size_t)x->new_m * sizeof(int));
    }
    x->new_ids[x->n_new] = id; x->new_anchor[x->n_new++] = anchor;
}
static int splice_order(abpoa_graph_t *abg) {
    poa_graph_x *x = gx(abg);
    const int old_n = x->old_n, n = abg->node_n;
    if (old_n + x->n_new != n) return 0;              /* nodes were created behind our back */
    int *order = abg->index_to_node_id, *idx = abg->node_id_to_index;
    int w = n - 1, k = x->n_new - 1;
    for (int i = old_n - 1; i >= 0 && k >= 0; --i) {  /* rows in front of the first anchor keep their index */
        while (k >= 0 && x->new_anchor[k] == i) { const int v = x->new_ids[k--]; order[w] = v; idx[v] = w--; }
        const int v = order[i]; order[w] = v; idx[v] = w--;
    }
    if (k >= 0) return 0;
    for (int e = 0; e < x->n_new_edges; e += 2)
        if (idx[x->new_edges[e]] >= idx[x->new_edges[e + 1]]) return 0;
    return 1;
}

/* ABPOA_GPU_CHECK_ORDER=1 (tests): after a splice, verify what the splice relies on -- every edge points forward in the
 * order and the members of every aligned group occupy consecutive rows -- instead of letting a violation show up as parity drift. */
static void check_spliced_order(const abpoa_graph_t *abg) {
    const poa_graph_x *x = cgx(abg);
    const int n = abg->node_n;
    for (int v = 0; v < n; ++v) {
        const int ne = x->cout[v]; const int *oid = out_ids_of(x, v);
        for (int e = 0; e < ne; ++e)
            if (abg->node_id_to_index[v] >= abg->node_id_to_index[oid[e]])
                poa_die(__func__, "spliced order: edge %d -> %d points backwards (rows %d -> %d)", v, oid[e], abg->node_id_to_index[v], abg->node_id_to_index[oid[e]]);
        const int na = x->caln[v];
        if (na) {
            const int *al = na <= POA_INL ? x->aln4 + (size_t)v * POA_INL : abg->node[v].aligned_node_id;
            int lo = abg->node_id_to_index[v], hi = lo;
            for (int a = 0; a < na; ++a) { const int r = abg->node_id_to_index[al[a]]; if (r < lo) lo = r; if (r > hi) hi = r; }
            if (hi - lo != na) poa_die(__func__, "spliced order: aligned group of node %d spans rows %d..%d for %d members", v, lo, hi, na + 1);
        }
    }
    for (int i = 0; i < n; ++i) if (abg->node_id_to_index[abg->index_to_node_id[i]] != i) poa_die(__func__, "spliced order: index arrays are not inverse at row %d", i);
}

void abpoa_topological_sort(abpoa_graph_t *abg, abpoa_para_t *abpt) {
    if (abg->node_n <= 0) { fprintf(stderr, "[%s] Empty graph.\n", __func__); return; }
    const int n = abg->node_n;
    index_arrays_reserve(abg, abpt, n);
    double t0 = prof_now();
    {
        poa_graph_x *x = gx(abg);
        int spliced = 0;
        if (x->tracking) {
            spliced = splice_order(abg);
            if (spliced) x->n_spliced += 1; else x->n_splice_fallback += 1;
            if (spliced) { static int check = -1; if (check < 0) { const char *e = getenv("ABPOA_GPU_CHECK_ORDER"); check = e && *e == '1'; } if (check) check_spliced_order(abg); }
            x->tracking = 0;
        }
        if (!spliced) abpoa_BFS_set_node_index(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID);
    }
    double t1 = prof_now(); poa_prof_ms[0] += t1 - t0;
    order_edges_by_weight(abg);
    double t2 = prof_now(); poa_prof_ms[1] += t2 - t1;
    if (abpt->wb >= 0) {
        for (int i = 0; i < n; ++i) { abg->node_id_to_max_pos_right[i] = 0; abg->node_id_to_max_pos_left[i] = n; }
        abpoa_BFS_set_node_remain(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID);
        poa_prof_ms[2] += prof_now() - t2;
    } else if (abpt->zdrop > 0) {
        abpoa_BFS_set_node_remain(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID);
    }
    abg->is_topological_sorted = 1;
}

/* MSA column rank: Kahn traversal with a LIFO; a popped node that has no rank yet
 * takes the next rank together with its whole aligned group. */
void poa_set_msa_rank(abpoa_graph_t *abg, int src_id, int sink_id) {
    if (abg->is_set_msa_rank) return;
    const int n = abg->node_n;
    scratch_reserve(abg, n);
    index_arrays_reserve(abg, NULL, n);
    if (!abg->node_id_to_msa_rank) abg->node_id_to_msa_rank = (int *)poa_xmalloc((size_t)abg->index_rank_m * sizeof(int));
    int *deg = gx(abg)->deg, *st = gx(abg)->queue, *rank = abg->node_id_to_msa_rank;
    const abpoa_node_t *node = abg->node;
    for (int i = 0; i < n; ++i) deg[i] = node[i].in_edge_n;
    int top = 0, next_rank = 0;
    st[top++] = src_id; rank[src_id] = -1;
    while (top > 0) {
        int cur = st[--top];
        if (rank[cur] < 0) {
            rank[cur] = next_rank;
            for (int a = 0; a < node[cur].aligned_node_n; ++a) rank[node[cur].aligned_node_id[a]] = next_rank;
            ++next_rank;
        }
        if (cur == sink_id) { abg->is_set_msa_rank = 1; return; }
        for (int e = 0; e < node[cur].out_edge_n; ++e) {
            int v = node[cur].out_id[e];
            if (--deg[v] != 0) continue;
            int ready = 1;
            for (int a = 0; a < node[v].aligned_node_n; ++a)
                if (deg[node[v].aligned_node_id[a]] != 0) { ready = 0; break; }
            if (!ready) continue;
            st[top++] = v; rank[v] = -1;
            for (int a = 0; a < node[v].aligned_node_n; ++a) { st[top++] = node[v].aligned_node_id[a]; rank[node[v].aligned_node_id[a]] = -1; }
        }
    }
    poa_die(__func__, "Error in set_msa_rank.");
}

/* -G: per-in-edge additive path score max(round(ln(edge_w / node_w)), -20)
 * (reference src/abpoa_graph.c:421-437) */
int poa_edge_path_score(const abpoa_graph_t *abg, int node_id, int in_idx) {
    const abpoa_node_t *nd = &abg->node[node_id];
    if (in_idx < 0 || in_idx >= nd->in_edge_n) poa_die(__func__, "Unexpected in_id_idx: %d.", in_idx);
    const abpoa_node_t *pre = &abg->node[nd->in_id[in_idx]];
    int node_w = 0;
    for (int e = 0; e < pre->out_edge_n; ++e) node_w += pre->out_edge_weight[e];
    int edge_w = nd->in_edge_weight[in_idx];
    if (node_w == 0 || edge_w == 0) return 0;
    int s = (int)round(log((double)edge_w / (double)node_w));
    return POA_MAX(s, -20);
}

/* ------------------------------------------------------------------ fusion */
/* every node strictly between src and sink (topologically) is spanned by one more read.  For
 * the whole graph with both ends included that is "every node": only counted, folded in later. */
static void bump_span_reads(abpoa_graph_t *abg, int src_id, int sink_id, int inc_both_ends) {
    poa_graph_x *x = gx(abg);
    if (src_id == ABPOA_SRC_NODE_ID && sink_id == ABPOA_SINK_NODE_ID && inc_both_ends) { x->span_pending += 1; return; }
    int lo = abg->node_id_to_index[src_id], hi = abg->node_id_to_index[sink_id];
    for (int i = lo + 1; i < hi; ++i) x->cspan[abg->index_to_node_id[i]] += 1;
    if (inc_both_ends) { x->cspan[src_id] += 1; x->cspan[sink_id] += 1; }
    x->public_stale = 1;
}

/* first read of a group: a simple chain SRC -> b0 -> b1 ... -> SINK */
static void seed_graph_with_sequence(abpoa_graph_t *abg, abpoa_para_t *abpt, const uint8_t *seq, const int *weight, int seq_l,
                                     int *qpos_to_node_id, uint8_t add_read_id, uint8_t add_read_weight,
                                     int read_id, int read_ids_n, int tot_read_n) {
    if (seq_l <= 0) return;
    int last = ABPOA_SRC_NODE_ID;
    for (int i = 0; i < seq_l; ++i) {
        int cur = abpoa_add_graph_node(abg, seq[i]);
        if (qpos_to_node_id) qpos_to_node_id[i] = cur;
        edge_add(abg, last, cur, 0, weight[i], add_read_id, add_read_weight, read_id, read_ids_n, tot_read_n);
        gx(abg)->cspan[cur] = gx(abg)->cspan[last];
        last = cur;
    }
    edge_add(abg, last, ABPOA_SINK_NODE_ID, 0, weight[seq_l - 1], add_read_id, add_read_weight, read_id, read_ids_n, tot_read_n);
    abg->is_called_cons = abg->is_set_msa_rank = abg->is_topological_sorted = 0; gx(abg)->msa_installed = 0; gx(abg)->gfa_rec = NULL;
    abpoa_topological_sort(abg, abpt);
    bump_span_reads(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, 1);
}

/* Thread one aligned read through the graph:
 *   M on an equal base     -> reuse the node (edge weight += w)
 *   M on a different base  -> reuse the aligned sibling with that base, else new node
 *                             registered as aligned with the whole sibling set
 *   I                      -> one new node per inserted base
 *   D                      -> nothing
 * then close with an edge to end_node_id and re-sort. */
int poa_add_alignment_nosync(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id, uint8_t *seq, int *_weight,
                             int seq_l, int *qpos_to_node_id, abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends) {
    abpoa_graph_t *abg = ab->abg;
    poa_graph_x *x = gx(abg);
    const int read_ids_n = 1 + ((tot_read_n - 1) >> 6);
    const uint8_t add_read_id = abpt->use_read_ids, add_read_weight = abpt->use_qv & (abpt->max_n_cons > 1);
    int *weight = _weight;
    if (!weight) {
        weight = (int *)poa_xmalloc((size_t)POA_MAX(seq_l, 1) * sizeof(int));
        for (int i = 0; i < seq_l; ++i) weight[i] = 1;
    }
    if (abg->node_n < 2) poa_die(__func__, "Graph node: %d.", abg->node_n);
    if (abg->node_n == 2) {
        seed_graph_with_sequence(abg, abpt, seq, weight, seq_l, qpos_to_node_id, add_read_id, add_read_weight, read_id, read_ids_n, tot_read_n);
    } else if (res.n_cigar > 0) {
        const double tf0 = prof_now();
        int qi = -1, last_id = beg_node_id, last_is_new = 0, last_anchor = -1;
        x->tracking = x->fast_order && abg->is_topological_sorted && abpt->align_mode == ABPOA_GLOBAL_MODE &&
                      beg_node_id == ABPOA_SRC_NODE_ID && end_node_id == ABPOA_SINK_NODE_ID;
        x->old_n = abg->node_n; x->n_new = 0; x->n_new_edges = 0;
        const int fast_ok = !add_read_id && !add_read_weight;       /* no per-edge read sets / read weights to maintain */
        x->public_stale = 1;
        for (int c = 0; c < res.n_cigar; ++c) {
            const abpoa_cigar_t cg = res.graph_cigar[c];
            const int op = (int)(cg & 0xf);
            if (c + POA_FUSE_AHEAD < res.n_cigar) {      /* the path's node ids are known in advance: pull their mirror rows in early */
                const abpoa_cigar_t ca = res.graph_cigar[c + POA_FUSE_AHEAD];
                if ((ca & 0xf) == ABPOA_CMATCH) {
                    const size_t v = (size_t)((ca >> 34) & 0x3fffffff);
                    __builtin_prefetch(x->in_id4 + v * POA_INL, 1); __builtin_prefetch(x->in_w4 + v * POA_INL, 1);
                    __builtin_prefetch(x->out_id4 + v * POA_INL, 1); __builtin_prefetch(x->out_w4 + v * POA_INL, 1);
                    __builtin_prefetch(x->cin + v, 0); __builtin_prefetch(x->cout + v, 0); __builtin_prefetch(x->cnread + v, 1);
                    __builtin_prefetch(x->cbase + v, 0);
                }
            }
            if (op == ABPOA_CMATCH) {
                const int node_id = (int)((cg >> 34) & 0x3fffffff);
                ++qi;
                /* by far the most common step: the read follows the heaviest edge between two nodes it matches
                 * (first slot of both inline lists).  Bumping a first slot cannot break the weight order. */
                if (fast_ok && !last_is_new && x->cbase[node_id] == seq[qi] && (last_id != beg_node_id || inc_both_ends)) {
                    const size_t v = (size_t)node_id * POA_INL, u = (size_t)last_id * POA_INL;
                    if (x->cin[node_id] <= POA_INL && x->cout[last_id] <= POA_INL && x->in_id4[v] == last_id && x->out_id4[u] == node_id) {
                        x->in_w4[v] += weight[qi]; x->out_w4[u] += weight[qi];
                        x->cnread[last_id] += 1;
                        last_id = node_id;
                        if (qpos_to_node_id) qpos_to_node_id[qi] = last_id;
                        continue;
                    }
                }
                const uint8_t add = (last_id != beg_node_id || inc_both_ends) ? 1 : 0;
                int target, target_is_new = 0;
                if (gx(abg)->cbase[node_id] == seq[qi]) target = node_id;
                else if ((target = aligned_with_base(abg, node_id, seq[qi])) < 0) {
                    target = abpoa_add_graph_node(abg, seq[qi]); target_is_new = 1;
                    if (x->tracking) { last_anchor = group_last_row(abg, node_id); record_new_node(x, target, last_anchor); }
                }
                edge_add(abg, last_id, target, target_is_new ? 0 : 1 - last_is_new, weight[qi], add_read_id & add, add_read_weight, read_id, read_ids_n, tot_read_n);
                if (target_is_new) x->cspan[target] = x->cspan[last_id];
                if (!add) x->cnread[last_id]--;
                if (target_is_new) aligned_join(abg, node_id, target);
                last_id = target; last_is_new = target_is_new;
                if (qpos_to_node_id) qpos_to_node_id[qi] = last_id;
            } else if (op == ABPOA_CINS || op == ABPOA_CSOFT_CLIP || op == ABPOA_CHARD_CLIP) {
                const int len = (int)((cg >> 4) & 0x3fffffff);
                for (int k = 0; k < len; ++k) {
                    ++qi;
                    const uint8_t add = (last_id != beg_node_id || inc_both_ends) ? 1 : 0;
                    int nid = abpoa_add_graph_node(abg, seq[qi]);
                    if (x->tracking) { if (!last_is_new) last_anchor = group_last_row(abg, last_id); record_new_node(x, nid, last_anchor); }
                    edge_add(abg, last_id, nid, 0, weight[qi], add_read_id & add, add_read_weight, read_id, read_ids_n, tot_read_n);
                    x->cspan[nid] = x->cspan[last_id];
                    if (!add) x->cnread[last_id]--;
                    last_id = nid; last_is_new = 1;
                    if (qpos_to_node_id) qpos_to_node_id[qi] = last_id;
                }
            } /* ABPOA_CDEL: the read skips this node */
        }
        edge_add(abg, last_id, end_node_id, 1 - last_is_new, weight[seq_l - 1], add_read_id, add_read_weight, read_id, read_ids_n, tot_read_n);
        abg->is_called_cons = abg->is_set_msa_rank = abg->is_topological_sorted = 0; x->msa_installed = 0; x->gfa_rec = NULL;
        poa_prof_ms[3] += prof_now() - tf0;
        abpoa_topological_sort(abg, abpt);
        const double tf1 = prof_now();
        bump_span_reads(abg, beg_node_id, end_node_id, inc_both_ends);
        poa_prof_ms[4] += prof_now() - tf1;
    }
    if (!_weight) free(weight);
    return 0;
}

int abpoa_add_subgraph_alignment(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id, uint8_t *seq, int *weight,
                                 int seq_l, int *qpos_to_node_id, abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends) {
    const int r = poa_add_alignment_nosync(ab, abpt, beg_node_id, end_node_id, seq, weight, seq_l, qpos_to_node_id, res, read_id, tot_read_n, inc_both_ends);
    poa_graph_sync_public(ab->abg);          /* public API: leave the ABI structs coherent */
    return r;
}

int abpoa_add_graph_alignment(abpoa_t *ab, abpoa_para_t *abpt, uint8_t *seq, int *weight, int seq_l, int *qpos_to_node_id,
                              abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends) {
    return abpoa_add_subgraph_alignment(ab, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, seq, weight, seq_l, qpos_to_node_id,
                                        res, read_id, tot_read_n, inc_both_ends);
}

/* ------------------------------------------------------------------ import of a device-built graph
 * The device chain (poa_chain.cuh) builds the same graph, node id for node id, on the GPU; at the end of
 * a read group it is exported as int32 words
 *   [0] n  [1] total in-edges E  [2] total aligned-set entries  [3] reads fused
 *   base[n] n_read[n] in_cnt[n] out_cnt[n] aln_cnt[n]  in_id[E] in_w[E] out_id[E] out_w[E]  aln[..]
 * (edge lists node by node, in list order) and rebuilt here so that consensus / output run on the
 * ordinary host structures.  The handle must be freshly abpoa_reset(). */
void poa_graph_import(abpoa_t *ab, abpoa_para_t *abpt, const int32_t *ex) {
    abpoa_graph_t *abg = ab->abg;
    poa_graph_x *x = gx(abg);
    const int n = ex[0], n_in = ex[1], n_fused = ex[3];
    if (abg->node_n != 2 || n < 2) poa_die(__func__, "import needs an empty graph (node_n %d) and n >= 2 (%d)", abg->node_n, n);
    const int32_t *base = ex + 4, *n_read = base + n, *in_cnt = n_read + n, *out_cnt = in_cnt + n, *aln_cnt = out_cnt + n;
    const int32_t *in_id = aln_cnt + n, *in_w = in_id + n_in, *out_id = in_w + n_in, *out_w = out_id + n_in, *aln = out_w + n_in;
    nodes_reserve(abg, n);
    index_arrays_reserve(abg, abpt, abg->node_m);
    for (int v = 2; v < n; ++v) { abg->node[v].base = (uint8_t)base[v]; x->cbase[v] = (uint8_t)base[v]; }
    abg->node_n = n;
    int pi = 0, po = 0, pa = 0;
    for (int v = 0; v < n; ++v) {
        abpoa_node_t *nd = &abg->node[v];
        if (in_cnt[v] > 0) {
            in_edges_reserve(x, v, in_cnt[v]);
            memcpy(nd->in_id, in_id + pi, (size_t)in_cnt[v] * sizeof(int)); memcpy(nd->in_edge_weight, in_w + pi, (size_t)in_cnt[v] * sizeof(int));
        }
        nd->in_edge_n = in_cnt[v]; x->cin[v] = in_cnt[v]; pi += in_cnt[v];
        if (in_cnt[v] >= 2) mark_fwd_counted(x, v);
        if (out_cnt[v] > 0) {
            out_edges_reserve(x, v, out_cnt[v], 0);
            memcpy(nd->out_id, out_id + po, (size_t)out_cnt[v] * sizeof(int)); memcpy(nd->out_edge_weight, out_w + po, (size_t)out_cnt[v] * sizeof(int));
        }
        nd->out_edge_n = out_cnt[v]; x->cout[v] = out_cnt[v]; po += out_cnt[v];
        for (int a = 0; a < aln_cnt[v]; ++a) aligned_push(abg, v, aln[pa + a]);
        x->caln[v] = nd->aligned_node_n; pa += aln_cnt[v];
        if (aln_cnt[v] > 0) mark_fwd_counted(x, v);
        x->cnread[v] = n_read[v]; x->cspan[v] = n_fused;
    }
    if (pi != n_in || po != n_in) poa_die(__func__, "inconsistent export: %d in-edges, %d out-edges, header says %d", pi, po, n_in);
    x->n_edges = n_in; x->public_stale = 1; x->span_pending = 0; x->msa_installed = 0; x->gfa_rec = NULL;
    abg->is_topological_sorted = abg->is_called_cons = abg->is_set_msa_rank = 0;
    poa_graph_sync_public(abg);
}

int poa_graph_msa_installed(const abpoa_graph_t *abg) { return cgx(abg)->msa_installed; }
void poa_graph_set_msa_installed(abpoa_graph_t *abg) { gx(abg)->msa_installed = 1; }
const int32_t *poa_graph_gfa_record(const abpoa_graph_t *abg) { return cgx(abg)->gfa_rec; }
void poa_graph_set_gfa_record(abpoa_graph_t *abg, const int32_t *rec) { gx(abg)->gfa_rec = rec; }

/* ------------------------------------------------------------------ sub-graph windows
 * abpoa_subgraph_nodes (reference src/abpoa_graph.c:595-687): widen the index window
 * [inc_beg, inc_end] until no edge enters it from outside, and return the node ids just
 * outside it as the exclusive begin / end of a sub-graph alignment. */
static int window_closed_upstream(const abpoa_graph_t *abg, int up, int down, int lo, int hi) {
    const int min_i = POA_MIN(up, lo), max_i = POA_MAX(down, hi);
    for (int i = up + 1; i <= down; ++i) {
        const abpoa_node_t *nd = &abg->node[abg->index_to_node_id[i]];
        for (int e = 0; e < nd->in_edge_n; ++e) {
            const int pi = abg->node_id_to_index[nd->in_id[e]];
            if (pi < min_i || pi > max_i) return 0;
        }
    }
    return 1;
}

static int widen_upstream(const abpoa_graph_t *abg, int lo, int hi) {
    for (;;) {
        int min_i = lo;
        for (int i = lo; i <= hi; ++i) {
            const abpoa_node_t *nd = &abg->node[abg->index_to_node_id[i]];
            for (int e = 0; e < nd->in_edge_n; ++e) min_i = POA_MIN(min_i, abg->node_id_to_index[nd->in_id[e]]);
        }
        if (window_closed_upstream(abg, min_i, lo, lo, hi)) return min_i;
        hi = lo; lo = min_i;
    }
}

static int widen_downstream(const abpoa_graph_t *abg, int lo, int hi) {
    for (;;) {
        int max_i = hi;
        for (int i = lo; i <= hi; ++i) {
            const abpoa_node_t *nd = &abg->node[abg->index_to_node_id[i]];
            for (int e = 0; e < nd->out_edge_n; ++e) max_i = POA_MAX(max_i, abg->node_id_to_index[nd->out_id[e]]);
        }
        if (window_closed_upstream(abg, hi, max_i, lo, hi)) return max_i;
        lo = hi; hi = max_i;
    }
}

void abpoa_subgraph_nodes(abpoa_t *ab, abpoa_para_t *abpt, int inc_beg, int inc_end, int *exc_beg, int *exc_end) {
    abpoa_graph_t *abg = ab->abg;
    if (abg->is_topological_sorted == 0) abpoa_topological_sort(abg, abpt);
    const int lo = abg->node_id_to_index[inc_beg], hi = abg->node_id_to_index[inc_end];
    const int up = widen_upstream(abg, lo, hi), down = widen_downstream(abg, lo, hi);
    if (up < 0 || down >= abg->node_n) poa_die(__func__, "Error in subgraph_nodes");
    *exc_beg = abg->index_to_node_id[up];
    *exc_end = abg->index_to_node_id[down];
}

/* ------------------------------------------------------------------ compact views for the flattener */
int64_t poa_graph_edge_count(const abpoa_graph_t *abg) { return cgx(abg)->n_edges; }
const uint8_t *poa_graph_bases(const abpoa_graph_t *abg) { return cgx(abg)->cbase; }
const int *poa_graph_in_degrees(const abpoa_graph_t *abg) { return cgx(abg)->cin; }
const int *poa_graph_in_ids(const abpoa_graph_t *abg, int id) { return in_ids_of(cgx(abg), id); }
/* address of the node's inline in-edge slots (valid to PREFETCH even when the list has spilled to the heap) */
const int *poa_graph_in_ids_inline(const abpoa_graph_t *abg, int id) { return cgx(abg)->in_id4 + (size_t)id * POA_INL; }

/* debugging aid: copy out / clear this thread's phase timers */
void poa_prof_snapshot(double *out8, int clear) {
    for (int i = 0; i < 8; ++i) { out8[i] = poa_prof_ms[i]; if (clear) poa_prof_ms[i] = 0; }
}

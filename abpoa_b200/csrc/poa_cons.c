/* poa_cons.c -- consensus (heaviest bundling) and row-column MSA from the final graph.
 *
 * These run once per read group after the last alignment; they exist on the host so
 * that parity with the reference can be expressed on its own outputs (consensus FASTA,
 * RC-MSA).  Behaviour follows
 *   heaviest bundling   reference src/abpoa_output.c:477-547 (tie rules!), :375-391
 *   phred of a column   reference src/abpoa_output.c:296-302
 *   RC-MSA              reference src/abpoa_output.c:105-192
 *   writers             reference src/abpoa_output.c:72-103, :588-627
 *   abpoa_output        reference src/abpoa_align.c:354-370
 * Out of the hot-path scope and therefore not provided (they abort with a message):
 * most-frequent-base consensus, multi-consensus clustering (max_n_cons > 1), GFA, dot.
 */
#include <math.h>
#include "poa_internal.h"

/* tables exported under the reference's names (src/abpoa_output.c:13-14) */
char ab_LogTable65536[65536];
char ab_bit_table16[65536];
extern char ab_char256_table[256];

void poa_set_65536_table(void) {
    ab_LogTable65536[0] = -1;
    for (int i = 1; i < 65536; ++i) ab_LogTable65536[i] = (char)(31 - __builtin_clz((unsigned)i));
}
void poa_set_bit_table16(void) {
    for (int i = 0; i < 65536; ++i) ab_bit_table16[i] = (char)__builtin_popcount((unsigned)i);
}

static int column_phred(int n_cov, int n_seq) {
    if (n_cov > n_seq) poa_die("abpoa_cons_phred_score", "Error: unexpected n_cov/n_seq (%d/%d).", n_cov, n_seq);
    double x = 13.8 * (1.25 * n_cov / n_seq - 0.25);
    double p = 1 - 1.0 / (1.0 + pow(2.718281828459045, -1 * x));
    return 33 + (int)(-10 * log10(p) + 0.499);
}

static void cons_alloc(abpoa_cons_t *abc, int n_node, int n_seq, int n_cons) {
    abc->n_cons = n_cons; abc->n_seq = n_seq;
    abc->clu_n_seq = (int *)poa_xcalloc(n_cons, sizeof(int));
    abc->cons_len = (int *)poa_xcalloc(n_cons, sizeof(int));
    abc->cons_node_ids = (int **)poa_xmalloc(n_cons * sizeof(int *));
    abc->cons_base = (uint8_t **)poa_xmalloc(n_cons * sizeof(uint8_t *));
    abc->cons_cov = (int **)poa_xmalloc(n_cons * sizeof(int *));
    abc->clu_read_ids = (int **)poa_xmalloc(n_cons * sizeof(int *));
    abc->cons_phred_score = (int **)poa_xmalloc(n_cons * sizeof(int *));
    for (int i = 0; i < n_cons; ++i) {
        abc->cons_node_ids[i] = (int *)poa_xmalloc((size_t)n_node * sizeof(int));
        abc->cons_base[i] = (uint8_t *)poa_xmalloc((size_t)n_node);
        abc->cons_cov[i] = (int *)poa_xmalloc((size_t)n_node * sizeof(int));
        abc->clu_read_ids[i] = (int *)poa_xmalloc((size_t)POA_MAX(n_seq, 1) * sizeof(int));
        abc->cons_phred_score[i] = (int *)poa_xmalloc((size_t)n_node * sizeof(int));
    }
}

/* Heaviest bundling, single cluster.  Reverse Kahn from SINK; score[v] = w(best out
 * edge) + score[its head].  Ties: an inner node keeps the LAST edge among equal weights
 * whose head scores >= the current pick; SRC keeps the first unless strictly better. */
static void heaviest_bundling(abpoa_graph_t *abg, abpoa_cons_t *abc) {
    const int n = abg->node_n, src = ABPOA_SRC_NODE_ID, sink = ABPOA_SINK_NODE_ID;
    const abpoa_node_t *node = abg->node;
    int *deg = (int *)poa_xmalloc((size_t)n * sizeof(int)), *score = (int *)poa_xmalloc((size_t)n * sizeof(int));
    int *next = (int *)poa_xmalloc((size_t)n * sizeof(int)), *q = (int *)poa_xmalloc((size_t)n * sizeof(int));
    for (int i = 0; i < n; ++i) deg[i] = node[i].out_edge_n;
    abc->clu_n_seq[0] = abc->n_seq;
    for (int i = 0; i < abc->n_seq; ++i) abc->clu_read_ids[0][i] = i;

    int head = 0, tail = 0;
    q[tail++] = sink;
    while (head < tail) {
        int cur = q[head++];
        if (cur == sink) { next[cur] = -1; score[cur] = 0; }
        else if (cur == src) {
            int pick = -1, pick_score = -1, pick_w = -1;
            for (int e = 0; e < node[cur].out_edge_n; ++e) {
                int v = node[cur].out_id[e], w = node[cur].out_edge_weight[e];
                if (w > pick_w || (w == pick_w && score[v] > pick_score)) { pick = v; pick_score = score[v]; pick_w = w; }
            }
            next[cur] = pick;
            break;
        } else {
            int pick = -1, pick_w = INT32_MIN;
            for (int e = 0; e < node[cur].out_edge_n; ++e) {
                int v = node[cur].out_id[e], w = node[cur].out_edge_weight[e];
                if (pick_w < w) { pick_w = w; pick = v; }
                else if (pick_w == w && score[pick] <= score[v]) pick = v;
            }
            score[cur] = pick_w + score[pick];
            next[cur] = pick;
        }
        for (int e = 0; e < node[cur].in_edge_n; ++e) {
            int u = node[cur].in_id[e];
            if (--deg[u] == 0) q[tail++] = u;
        }
    }
    int len = 0;
    for (int cur = next[src]; cur != sink; cur = next[cur], ++len) {
        abc->cons_node_ids[0][len] = cur;
        abc->cons_base[0][len] = node[cur].base;
        abc->cons_cov[0][len] = node[cur].n_read;
        abc->cons_phred_score[0][len] = column_phred(node[cur].n_read, abc->clu_n_seq[0]);
    }
    abc->cons_len[0] = len;
    free(deg); free(score); free(next); free(q);
}

void abpoa_generate_consensus(abpoa_t *ab, abpoa_para_t *abpt) {
    abpoa_graph_t *abg = ab->abg;
    poa_graph_sync_public(abg);
    if (abg->is_called_cons == 1 || abg->node_n <= 2) return;
    if (abpt->max_n_cons > 1) poa_die(__func__, "multi-consensus clustering (max_n_cons > 1) is outside the scope of the GPU hot-path library.");
    if (abpt->cons_algrm != ABPOA_HB) poa_die(__func__, "most-frequent-base consensus is outside the scope of the GPU hot-path library.");
    cons_alloc(ab->abc, abg->node_n, ab->abs->n_seq, 1);
    heaviest_bundling(abg, ab->abc);
    abg->is_called_cons = 1;
}

/* A consensus that was computed elsewhere (the device chain, poa_chain.cuh: chain_consensus) installed as the handle's
 * single-cluster result, so that abpoa_output() and the writers treat it like one they generated themselves. */
void poa_cons_install(abpoa_t *ab, int n_seq, int len, const uint8_t *base, const int *cov) {
    abpoa_cons_t *abc = ab->abc;
    poa_cons_clear(abc);
    cons_alloc(abc, len > 0 ? len : 1, n_seq, 1);
    abc->clu_n_seq[0] = n_seq;
    for (int i = 0; i < n_seq; ++i) abc->clu_read_ids[0][i] = i;
    for (int j = 0; j < len; ++j) {
        abc->cons_node_ids[0][j] = -1;                     /* node ids stay on the device */
        abc->cons_base[0][j] = base[j]; abc->cons_cov[0][j] = cov[j];
        abc->cons_phred_score[0][j] = column_phred(cov[j], n_seq);
    }
    abc->cons_len[0] = len;
    ab->abg->is_called_cons = 1;
}

/* RC-MSA rows that were computed elsewhere (the device chain, poa_chain.cuh: chain_msa_rows) installed as the handle's
 * result.  Install a device consensus first (poa_cons_install clears abc).  With no graph on the host,
 * abpoa_generate_rc_msa returns at once; with an imported graph it keeps these rows. */
void poa_msa_install(abpoa_t *ab, int n_seq, int n_rows, int msa_len, const uint8_t *rows) {
    abpoa_cons_t *abc = ab->abc;
    abc->n_seq = n_seq; abc->msa_len = msa_len;
    abc->msa_base = (uint8_t **)poa_xmalloc((size_t)n_rows * sizeof(uint8_t *));
    for (int i = 0; i < n_rows; ++i) {
        abc->msa_base[i] = (uint8_t *)poa_xmalloc((size_t)POA_MAX(msa_len, 1));
        memcpy(abc->msa_base[i], rows + (size_t)i * msa_len, (size_t)msa_len);
    }
    poa_graph_set_msa_installed(ab->abg);
}

/* column of a node = max rank over its aligned group, 1-based */
static int msa_column(const abpoa_graph_t *abg, int id) {
    int r = abg->node_id_to_msa_rank[id];
    for (int a = 0; a < abg->node[id].aligned_node_n; ++a)
        r = POA_MAX(r, abg->node_id_to_msa_rank[abg->node[id].aligned_node_id[a]]);
    return r;
}

void abpoa_generate_rc_msa(abpoa_t *ab, abpoa_para_t *abpt) {
    abpoa_graph_t *abg = ab->abg;
    poa_graph_sync_public(abg);
    if (abg->node_n <= 2 || poa_graph_msa_installed(abg)) return;
    poa_set_msa_rank(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID);
    if (abpt->out_cons) abpoa_generate_consensus(ab, abpt);

    abpoa_cons_t *abc = ab->abc;
    const int n_seq = ab->abs->n_seq, msa_len = abg->node_id_to_msa_rank[ABPOA_SINK_NODE_ID] - 1;
    abc->n_seq = n_seq; abc->msa_len = msa_len;
    abc->msa_base = (uint8_t **)poa_xmalloc((size_t)(n_seq + abc->n_cons) * sizeof(uint8_t *));
    for (int i = 0; i < n_seq + abc->n_cons; ++i) {
        abc->msa_base[i] = (uint8_t *)poa_xmalloc((size_t)POA_MAX(msa_len, 1));
        memset(abc->msa_base[i], abpt->m, (size_t)msa_len);       /* code m prints as '-' */
    }
    /* a read occupies the column of every node whose out-edge carries its id */
    for (int id = 2; id < abg->node_n; ++id) {
        const abpoa_node_t *nd = &abg->node[id];
        const int col = msa_column(abg, id) - 1;
        for (int wd = 0; wd < nd->read_ids_n; ++wd)
            for (int e = 0; e < nd->out_edge_n; ++e) {
                uint64_t bits = nd->read_ids[e][wd];
                while (bits) {
                    int b = __builtin_ctzll(bits);
                    abc->msa_base[wd * 64 + b][col] = nd->base;
                    bits &= bits - 1;
                }
            }
    }
    if (abpt->out_cons)
        for (int c = 0; c < abc->n_cons; ++c)
            for (int i = 0; i < abc->cons_len[c]; ++i)
                abc->msa_base[n_seq + c][msa_column(abg, abc->cons_node_ids[c][i]) - 1] = abc->cons_base[c][i];
}

/* ------------------------------------------------------------------ writers */
static void write_cons_header(const abpoa_cons_t *abc, const abpoa_para_t *abpt, int c, char lead, int with_batch, FILE *fp) {
    fprintf(fp, "%cConsensus_sequence", lead);
    if (with_batch && abpt->batch_index > 0) fprintf(fp, "_%d", abpt->batch_index);
    if (abc->n_cons > 1) {
        fprintf(fp, "_%d ", c + 1);
        for (int j = 0; j < abc->clu_n_seq[c]; ++j) fprintf(fp, j ? ",%d" : "%d", abc->clu_read_ids[c][j]);
    }
    fputc('\n', fp);
}

void abpoa_output_fx_consensus(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp) {
    if (!out_fp) return;
    const abpoa_cons_t *abc = ab->abc;
    for (int c = 0; c < abc->n_cons; ++c) {
        write_cons_header(abc, abpt, c, abpt->out_fq ? '@' : '>', 1, out_fp);
        for (int j = 0; j < abc->cons_len[c]; ++j) fputc(ab_char256_table[abc->cons_base[c][j]], out_fp);
        fputc('\n', out_fp);
        if (abpt->out_fq) {
            write_cons_header(abc, abpt, c, '+', 1, out_fp);
            for (int j = 0; j < abc->cons_len[c]; ++j) fputc(abc->cons_phred_score[c][j], out_fp);
            fputc('\n', out_fp);
        }
    }
}

void abpoa_output_rc_msa(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp) {
    if (!out_fp) return;
    const abpoa_seq_t *abs = ab->abs; const abpoa_cons_t *abc = ab->abc;
    if (abc->msa_len <= 0) return;
    for (int i = 0; i < abs->n_seq; ++i) {
        if (abs->name[i].l > 0) fprintf(out_fp, abs->is_rc[i] ? ">%s_reverse_complement\n" : ">%s\n", abs->name[i].s);
        else fprintf(out_fp, ">Seq_%d\n", i + 1);
        for (int j = 0; j < abc->msa_len; ++j) fputc(ab_char256_table[abc->msa_base[i][j]], out_fp);
        fputc('\n', out_fp);
    }
    if (abpt->out_cons)
        for (int c = 0; c < abc->n_cons; ++c) {
            write_cons_header(abc, abpt, c, '>', 0, out_fp);
            for (int j = 0; j < abc->msa_len; ++j) fputc(ab_char256_table[abc->msa_base[abc->n_seq + c][j]], out_fp);
            fputc('\n', out_fp);
        }
}

void abpoa_generate_gfa(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp) {
    (void)ab; (void)abpt; (void)out_fp;
    poa_die(__func__, "GFA output is outside the scope of the GPU hot-path library.");
}

void abpoa_dump_pog(abpoa_t *ab, abpoa_para_t *abpt) {
    (void)ab; (void)abpt;
    poa_die(__func__, "graph plotting is outside the scope of the GPU hot-path library.");
}

void abpoa_output(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp) {
    poa_graph_sync_public(ab->abg);
    if (abpt->out_gfa) abpoa_generate_gfa(ab, abpt, out_fp);
    else {
        if (abpt->out_msa) abpoa_generate_rc_msa(ab, abpt);
        if (abpt->out_cons) {
            abpoa_generate_consensus(ab, abpt);
            if (ab->abg->is_called_cons == 0) fprintf(stderr, "Warning: no consensus sequence generated.\n");
        }
        if (abpt->out_msa) abpoa_output_rc_msa(ab, abpt, out_fp);
        else if (abpt->out_cons) abpoa_output_fx_consensus(ab, abpt, out_fp);
    }
    if (abpt->out_pog) abpoa_dump_pog(ab, abpt);
}

/* poa_cons.c -- consensus (heaviest bundling) and row-column MSA from the final graph.
 *
 * These run once per read group after the last alignment; they exist on the host so
 * that parity with the reference can be expressed on its own outputs (consensus FASTA,
 * RC-MSA).  Behaviour follows
 *   heaviest bundling   reference src/abpoa_output.c:477-547 (tie rules!), :375-391
 *   most frequent base  reference src/abpoa_output.c:393-451, :549-586 (-a 1)
 *   phred of a column   reference src/abpoa_output.c:296-302
 *   RC-MSA              reference src/abpoa_output.c:105-192
 *   writers             reference src/abpoa_output.c:72-103, :588-627
 *   GFA                 reference src/abpoa_output.c:194-294
 *   abpoa_output        reference src/abpoa_align.c:354-370
 * Out of the hot-path scope and therefore not provided (they abort with a message):
 * multi-consensus clustering (max_n_cons > 1), consensus algorithms other than -a 0 / -a 1, dot.
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

static int msa_column(const abpoa_graph_t *abg, int id);

/* Most frequent base per RC-MSA column, single cluster (device twin: chain_mf_consensus in poa_chain.cuh).  Every node
 * (ascending id) sets weight n_read and node id for its base in its column, a later node overwriting an earlier one.  A
 * column votes with codes 0..m-2 only (code m-1, N or the last amino-acid code, counts as gap): the strictly largest
 * count wins, so the lowest code among equal counts; the column is kept iff that count >= the gap count, n_seq minus
 * the votes (under sub_aln the winner's n_span_read minus the votes). */
static void most_frequent(abpoa_graph_t *abg, const abpoa_para_t *abpt, abpoa_cons_t *abc) {
    const int m = abpt->m, n_seq = abc->n_seq;
    poa_set_msa_rank(abg, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID);
    const int msa_len = abg->node_id_to_msa_rank[ABPOA_SINK_NODE_ID] - 1;
    int *w = (int *)poa_xcalloc((size_t)POA_MAX(msa_len, 1) * m, sizeof(int));
    int *id = (int *)poa_xcalloc((size_t)POA_MAX(msa_len, 1) * m, sizeof(int));
    abc->clu_n_seq[0] = n_seq;
    for (int i = 0; i < n_seq; ++i) abc->clu_read_ids[0][i] = i;
    for (int i = 2; i < abg->node_n; ++i) {
        const int col = msa_column(abg, i) - 1, b = abg->node[i].base;
        w[(size_t)col * m + b] = abg->node[i].n_read;
        id[(size_t)col * m + b] = i;
    }
    int len = 0;
    for (int col = 0; col < msa_len; ++col) {
        const int *cw = w + (size_t)col * m;
        int max_c = 0, max_base = m, total_c = 0;
        for (int b = 0; b < m - 1; ++b) {
            if (cw[b] > max_c) { max_c = cw[b]; max_base = b; }
            total_c += cw[b];
        }
        /* no vote: never kept without sub_aln (gap = n_seq); under sub_aln the reference reads past the column's row */
        if (max_base == m) continue;
        const int node_id = id[(size_t)col * m + max_base];
        const int gap_c = (abpt->sub_aln ? abg->node[node_id].n_span_read : n_seq) - total_c;
        if (max_c < gap_c) continue;
        abc->cons_node_ids[0][len] = node_id;
        abc->cons_base[0][len] = (uint8_t)max_base;
        abc->cons_cov[0][len] = max_c;
        abc->cons_phred_score[0][len] = column_phred(max_c, n_seq);
        ++len;
    }
    abc->cons_len[0] = len;
    free(w); free(id);
}

void abpoa_generate_consensus(abpoa_t *ab, abpoa_para_t *abpt) {
    abpoa_graph_t *abg = ab->abg;
    poa_graph_sync_public(abg);
    if (abg->is_called_cons == 1 || abg->node_n <= 2) return;
    if (abpt->max_n_cons > 1) poa_die(__func__, "multi-consensus clustering (max_n_cons > 1) is outside the scope of the GPU hot-path library.");
    if (abpt->cons_algrm != ABPOA_HB && abpt->cons_algrm != ABPOA_MF)
        poa_die(__func__, "unknown consensus algorithm %d (0: heaviest bundling, 1: most frequent base).", abpt->cons_algrm);
    cons_alloc(ab->abc, abg->node_n, ab->abs->n_seq, 1);
    if (abpt->cons_algrm == ABPOA_HB) heaviest_bundling(abg, ab->abc);
    else most_frequent(abg, abpt, ab->abc);
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

/* ------------------------------------------------------------------ GFA
 * H line, then per segment in FIFO Kahn order from SRC (stopping at SINK) its S line and one L line per in-link, then one
 * P line per read (its segments in that order; reads with is_rc reversed, with '-') and with -r 4 the consensus path.  A
 * path with no segment prints "P\t<name>\t" and nothing else, as the reference does.  A headline group has ~500 k path
 * entries: numbers go through put_int into one buffer, not through stdio. */
typedef struct { char *s; size_t l, m; } gfa_buf;

static inline void gb_need(gfa_buf *b, size_t n) {
    if (b->l + n <= b->m) return;
    b->m = (b->l + n) * 2 + 4096;
    b->s = (char *)poa_xrealloc(b->s, b->m);
}
static inline void put_str(gfa_buf *b, const char *s, size_t n) { gb_need(b, n); memcpy(b->s + b->l, s, n); b->l += n; }
#define PUT_LIT(b, lit) put_str((b), (lit), sizeof(lit) - 1)
static inline void put_int(gfa_buf *b, int v) {
    char t[12]; int k = 0;
    unsigned u = v < 0 ? 0u - (unsigned)v : (unsigned)v;
    do { t[k++] = (char)('0' + u % 10); u /= 10; } while (u);
    gb_need(b, 12);
    if (v < 0) b->s[b->l++] = '-';
    while (k) b->s[b->l++] = t[--k];
}

void poa_gfa_from_record(poa_gfa_t *g, const int32_t *rec) {
    g->n_seg = rec[0]; g->n_link = rec[1]; g->ns = rec[2]; g->nl = rec[3]; g->words = rec[4]; g->cons_len = rec[5];
    const int32_t *p = rec + POA_GFA_HDR;
    g->seg_id = p; p += g->n_seg;
    g->seg_base = p; p += g->n_seg;
    g->link_cnt = p; p += g->n_seg;
    g->link_from = p; p += g->n_link;
    g->cons_id = p; p += POA_MAX(g->cons_len, 0);
    if ((p - rec) & 1) ++p;
    g->read_set = (const uint64_t *)(const void *)p;
}

char *poa_gfa_format(const poa_gfa_t *g, const abpoa_seq_t *abs, int np, size_t *len) {
    gfa_buf b = { NULL, 0, 0 };
    const int n_seq = abs->n_seq;
    PUT_LIT(&b, "H\tVN:Z:1.0\tNS:i:"); put_int(&b, g->ns); PUT_LIT(&b, "\tNL:i:"); put_int(&b, g->nl);
    PUT_LIT(&b, "\tNP:i:"); put_int(&b, np); PUT_LIT(&b, "\n");
    for (int i = 0, k = 0; i < g->n_seg; ++i) {
        const int id = g->seg_id[i] - 1;
        PUT_LIT(&b, "S\t"); put_int(&b, id); gb_need(&b, 3);
        b.s[b.l++] = '\t'; b.s[b.l++] = ab_char256_table[g->seg_base[i]]; b.s[b.l++] = '\n';
        for (int e = 0; e < g->link_cnt[i]; ++e, ++k) {
            PUT_LIT(&b, "L\t"); put_int(&b, g->link_from[k] - 1); PUT_LIT(&b, "\t+\t"); put_int(&b, id); PUT_LIT(&b, "\t+\t0M\n");
        }
    }
    /* read sets -> paths: count, then place every segment into the paths of its reads, in segment order */
    int64_t *off = (int64_t *)poa_xcalloc((size_t)n_seq + 1, sizeof(int64_t));
    for (int i = 0; i < g->n_seg; ++i)
        for (int wd = 0; wd < g->words; ++wd)
            for (uint64_t bits = g->read_set[(size_t)i * g->words + wd]; bits; bits &= bits - 1) {
                const int r = wd * 64 + __builtin_ctzll(bits);
                if (r < n_seq) ++off[r + 1];
            }
    for (int r = 0; r < n_seq; ++r) off[r + 1] += off[r];
    int32_t *path = (int32_t *)poa_xmalloc((size_t)POA_MAX(off[n_seq], 1) * sizeof(int32_t));
    int64_t *fill = (int64_t *)poa_xmalloc((size_t)POA_MAX(n_seq, 1) * sizeof(int64_t));
    memcpy(fill, off, (size_t)n_seq * sizeof(int64_t));
    for (int i = 0; i < g->n_seg; ++i)
        for (int wd = 0; wd < g->words; ++wd)
            for (uint64_t bits = g->read_set[(size_t)i * g->words + wd]; bits; bits &= bits - 1) {
                const int r = wd * 64 + __builtin_ctzll(bits);
                if (r < n_seq) path[fill[r]++] = g->seg_id[i] - 1;
            }
    for (int r = 0; r < n_seq; ++r) {
        PUT_LIT(&b, "P\t");
        if (abs->name[r].l > 0) put_str(&b, abs->name[r].s, (size_t)abs->name[r].l); else put_int(&b, r + 1);
        PUT_LIT(&b, "\t");
        const int32_t *p = path + off[r];
        const int64_t n = off[r + 1] - off[r];
        const int rc = abs->is_rc[r];
        for (int64_t j = 0; j < n; ++j) {
            if (j) PUT_LIT(&b, ",");
            put_int(&b, p[rc ? n - 1 - j : j]);
            gb_need(&b, 1); b.s[b.l++] = rc ? '-' : '+';
        }
        if (n > 0) PUT_LIT(&b, "\t*\n");
    }
    if (g->cons_len >= 0) {
        PUT_LIT(&b, "P\tConsensus_sequence\t");
        for (int j = 0; j < g->cons_len; ++j) {
            if (j) PUT_LIT(&b, ",");
            put_int(&b, g->cons_id[j] - 1); PUT_LIT(&b, "+");
        }
        if (g->cons_len > 0) PUT_LIT(&b, "\t*\n");
    }
    free(off); free(path); free(fill);
    *len = b.l;
    return b.s;
}

/* the description of the host graph (per-edge read sets); arrays in *store, released with free() */
typedef struct { int32_t *ints; uint64_t *sets; } gfa_store;

static void gfa_describe_host(abpoa_t *ab, abpoa_para_t *abpt, poa_gfa_t *g, gfa_store *st) {
    const abpoa_graph_t *abg = ab->abg;
    const abpoa_node_t *node = abg->node;
    const int n = abg->node_n, n_seq = ab->abs->n_seq, words = (n_seq + 63) / 64;
    int64_t n_in = 0;
    for (int v = 0; v < n; ++v) n_in += node[v].in_edge_n;
    /* q | deg | seg_base | link_cnt | link_from | cons_id */
    int32_t *q = (int32_t *)poa_xmalloc(((size_t)5 * n + (size_t)n_in + 1) * sizeof(int32_t));
    int32_t *deg = q + n, *seg_base = deg + n, *link_cnt = seg_base + n, *cons_id = link_cnt + n, *link_from = cons_id + n;
    for (int v = 0; v < n; ++v) deg[v] = node[v].in_edge_n;
    int head = 0, tail = 0, n_link = 0;
    q[tail++] = ABPOA_SRC_NODE_ID;
    while (head < tail) {
        const int cur = q[head++];
        if (cur == ABPOA_SINK_NODE_ID) break;
        if (cur != ABPOA_SRC_NODE_ID) {
            const int i = head - 2;
            seg_base[i] = node[cur].base; link_cnt[i] = 0;
            for (int e = 0; e < node[cur].in_edge_n; ++e)
                if (node[cur].in_id[e] != ABPOA_SRC_NODE_ID) { link_from[n_link++] = node[cur].in_id[e]; ++link_cnt[i]; }
        }
        for (int e = 0; e < node[cur].out_edge_n; ++e)
            if (--deg[node[cur].out_id[e]] == 0) q[tail++] = node[cur].out_id[e];
    }
    g->n_seg = q[head - 1] == ABPOA_SINK_NODE_ID ? head - 2 : head - 1;
    g->n_link = n_link; g->ns = n - 2; g->words = words;
    int nl = 0;
    for (int v = 2; v < n; ++v) nl += node[v].in_edge_n;
    g->nl = nl - node[ABPOA_SRC_NODE_ID].out_edge_n;
    g->seg_id = q + 1; g->seg_base = seg_base; g->link_cnt = link_cnt; g->link_from = link_from;
    /* a read passes through a node iff one of the node's out-edges carries it */
    uint64_t *sets = (uint64_t *)poa_xcalloc((size_t)POA_MAX(g->n_seg, 1) * POA_MAX(words, 1), sizeof(uint64_t));
    for (int i = 0; i < g->n_seg; ++i) {
        const abpoa_node_t *nd = &node[q[1 + i]];
        const int nw = POA_MIN(nd->read_ids_n, words);
        for (int e = 0; e < nd->out_edge_n; ++e)
            for (int wd = 0; wd < nw; ++wd) sets[(size_t)i * words + wd] |= nd->read_ids[e][wd];
    }
    g->read_set = sets;
    g->cons_len = -1; g->cons_id = cons_id;
    if (abpt->out_cons) {
        abpoa_generate_consensus(ab, abpt);
        const abpoa_cons_t *abc = ab->abc;
        g->cons_len = 0;
        if (abc->n_cons > 0) {
            g->cons_len = abc->cons_len[0];
            memcpy(cons_id, abc->cons_node_ids[0], (size_t)g->cons_len * sizeof(int32_t));
        }
    }
    st->ints = q; st->sets = sets;
}

/* FIFO order of the host writer (tests compare the device's with it): segment ids into out, returns their number */
int poa_gfa_host_order(abpoa_t *ab, int32_t *out) {
    abpoa_para_t para; memset(&para, 0, sizeof para);       /* out_cons = 0: no consensus */
    poa_graph_sync_public(ab->abg);
    poa_gfa_t g; gfa_store st;
    gfa_describe_host(ab, &para, &g, &st);
    memcpy(out, g.seg_id, (size_t)g.n_seg * sizeof(int32_t));
    free(st.ints); free(st.sets);
    return g.n_seg;
}

void poa_gfa_install(abpoa_t *ab, const int32_t *rec) { poa_graph_set_gfa_record(ab->abg, rec); }

/* A record text as abpoa_generate_gfa prints it (for tests: the device record through the product's formatter) */
char *poa_gfa_record_text(const int32_t *rec, abpoa_t *ab, abpoa_para_t *abpt, size_t *len) {
    poa_gfa_t g; poa_gfa_from_record(&g, rec);
    return poa_gfa_format(&g, ab->abs, ab->abs->n_seq + abpt->out_cons, len);
}

void abpoa_generate_gfa(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp) {
    if (!out_fp) return;                                   /* nothing printed, nothing computed */
    abpoa_graph_t *abg = ab->abg;
    poa_graph_sync_public(abg);
    const int32_t *rec = poa_graph_gfa_record(abg);
    poa_gfa_t g; gfa_store st = { NULL, NULL };
    if (rec) {
        poa_gfa_from_record(&g, rec);
        /* the consensus fields: installed with the record (poa_cons_install), or computed on an imported graph */
        if (abpt->out_cons) abpoa_generate_consensus(ab, abpt);
    } else {
        if (abg->node_n <= 2) return;
        gfa_describe_host(ab, abpt, &g, &st);
    }
    size_t len = 0;
    char *text = poa_gfa_format(&g, ab->abs, ab->abs->n_seq + abpt->out_cons, &len);
    fwrite(text, 1, len, out_fp);
    free(text); free(st.ints); free(st.sets);
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

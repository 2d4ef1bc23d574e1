/* poa_msa.c -- public alignment entry points and the per-group progressive loop.
 *
 *   abpoa_align_sequence_to_(sub)graph   reference src/abpoa_align.c:194-206
 *   progressive loop (abpoa_poa)         reference src/abpoa_align.c:312-352
 *   abpoa_msa                            reference src/abpoa_align.c:401-471
 *
 * Reads of one group are strictly sequential (read i+1 is aligned to the graph that
 * already contains read i).  One call here therefore drives ONE alignment at a time on
 * the GPU; to fill the device use the batched entry points in abpoa_gpu.h, which run
 * many independent groups concurrently through the same kernels.
 */
#include "poa_internal.h"

int abpoa_align_sequence_to_subgraph(abpoa_t *ab, abpoa_para_t *abpt, int exc_beg_node_id, int exc_end_node_id,
                                     uint8_t *query, int qlen, abpoa_res_t *res) {
    if (ab->abg->node_n <= 2) return -1;
    if (ab->abg->is_topological_sorted == 0) abpoa_topological_sort(ab->abg, abpt);
    poa_cuda_align_sequence_to_subgraph(ab, abpt, exc_beg_node_id, exc_end_node_id, query, qlen, res);
    return 0;
}

int abpoa_align_sequence_to_graph(abpoa_t *ab, abpoa_para_t *abpt, uint8_t *query, int qlen, abpoa_res_t *res) {
    return abpoa_align_sequence_to_subgraph(ab, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, query, qlen, res);
}

static void reverse_complement(const uint8_t *seq, const int *w, int l, uint8_t *rc_seq, int *rc_w) {
    for (int j = 0; j < l; ++j) {
        uint8_t b = seq[l - 1 - j];
        rc_seq[j] = b < 4 ? (uint8_t)(3 - b) : 4;
        rc_w[j] = w[l - 1 - j];
    }
}

/* align read i to the graph built from reads 0..i-1, then fuse it in */
static void progressive_poa(abpoa_t *ab, abpoa_para_t *abpt, uint8_t **seqs, int **weights, int *seq_lens, int exist_n_seq, int n_seq) {
    abpoa_seq_t *abs = ab->abs;
    const int tot_n_seq = exist_n_seq + n_seq;
    for (int i = 0; i < n_seq; ++i) {
        int qlen = seq_lens[i], read_id = exist_n_seq + i;
        uint8_t *qseq = seqs[i]; int *weight = weights[i];
        uint8_t *rc_seq = NULL; int *rc_w = NULL;
        abpoa_res_t res; memset(&res, 0, sizeof res);
        if (abpoa_align_sequence_to_graph(ab, abpt, qseq, qlen, &res) >= 0 && abpt->amb_strand &&
            res.best_score < POA_MIN(qlen, ab->abg->node_n - 2) * abpt->max_mat * .3333) {
            /* weak forward hit: also try the reverse complement, keep the better strand */
            rc_seq = (uint8_t *)poa_xmalloc((size_t)qlen); rc_w = (int *)poa_xmalloc((size_t)qlen * sizeof(int));
            reverse_complement(qseq, weight, qlen, rc_seq, rc_w);
            abpoa_res_t rc; memset(&rc, 0, sizeof rc);
            poa_cuda_align_sequence_to_subgraph(ab, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, rc_seq, qlen, &rc);
            if (rc.best_score > res.best_score) {
                if (res.n_cigar) free(res.graph_cigar);
                res = rc; rc.n_cigar = 0; rc.graph_cigar = NULL;
                qseq = rc_seq; weight = rc_w; abs->is_rc[read_id] = 1;
            }
            if (rc.n_cigar) free(rc.graph_cigar);
        }
        abpoa_add_graph_alignment(ab, abpt, qseq, weight, qlen, NULL, res, read_id, tot_n_seq, 1);
        free(rc_seq); free(rc_w);
        if (res.n_cigar) free(res.graph_cigar);
    }
}

int abpoa_msa(abpoa_t *ab, abpoa_para_t *abpt, int n_seq, char **seq_names, int *seq_lens, uint8_t **seqs, int **qual_weights, FILE *out_fp) {
    if (n_seq <= 0) return 0;
    abpoa_seq_t *abs = ab->abs;
    if (abs->n_seq <= 0) {
        abpoa_reset(ab, abpt, 1024);
        if (abpt->incr_fn) abpoa_restore_graph(ab, abpt);
    } else if (abpt->incr_fn != NULL) {
        fprintf(stderr, "[%s] Graph already exists, but incr_fn is also provided. Not restoring graph from file.\n", __func__);
    }
    if (!((abpt->disable_seeding && abpt->progressive_poa == 0) || abpt->align_mode != ABPOA_GLOBAL_MODE))
        poa_die(__func__, "minimizer seeding / guide-tree partitioning (-S / -p) is outside the scope of the GPU hot-path library.");

    const int exist_n_seq = abs->n_seq;
    abs->n_seq += n_seq; poa_seq_reserve(abs);
    for (int i = 0; i < n_seq; ++i) {
        abpoa_str_t *nm = &abs->name[exist_n_seq + i];
        abs->is_rc[exist_n_seq + i] = 0;
        if (seq_names) poa_str_assign(nm, seq_names[i], (int)strlen(seq_names[i]));
        else nm->l = 0;            /* keep any old buffer for reuse, mark the name empty */
    }
    int **weights = (int **)poa_xmalloc((size_t)n_seq * sizeof(int *));
    for (int i = 0; i < n_seq; ++i) {
        weights[i] = (int *)poa_xmalloc((size_t)POA_MAX(seq_lens[i], 1) * sizeof(int));
        const int use_q = abpt->use_qv && qual_weights != NULL && qual_weights[i] != NULL;
        for (int j = 0; j < seq_lens[i]; ++j) weights[i][j] = use_q ? qual_weights[i][j] : 1;
    }
    progressive_poa(ab, abpt, seqs, weights, seq_lens, exist_n_seq, n_seq);
    abpoa_output(ab, abpt, out_fp);
    for (int i = 0; i < n_seq; ++i) free(weights[i]);
    free(weights);
    return 0;
}

/* One MSA from a FASTA/FASTQ file (reference abpoa_msa1, src/abpoa_align.c:473-539): read, encode with the
 * alphabet table chosen by abpoa_post_set_para, quality weights = phred + 1 when -Q, progressive POA, output. */
extern char ab_char26_table[256];
int abpoa_msa1(abpoa_t *ab, abpoa_para_t *abpt, char *read_fn, FILE *out_fp) {
    if (!abpt->out_msa && !abpt->out_cons && !abpt->out_gfa) return 0;
    if (abpt->sort_input_seq) poa_die(__func__, "sorting the input by length (-L) is outside the scope of the GPU hot-path library.");
    abpoa_reset(ab, abpt, 1024);
    if (abpt->incr_fn) abpoa_restore_graph(ab, abpt);
    abpoa_seq_t *abs = ab->abs;
    const int exist_n_seq = abs->n_seq;
    const int n_seq = poa_read_fastx(read_fn, abs);
    if (n_seq < 0) poa_die(__func__, "fail to open file \'%s\'", read_fn);
    if (n_seq == 0) return 0;
    uint8_t **seqs = (uint8_t **)poa_xmalloc((size_t)n_seq * sizeof(uint8_t *));
    int *lens = (int *)poa_xmalloc((size_t)n_seq * sizeof(int)), **weights = (int **)poa_xmalloc((size_t)n_seq * sizeof(int *));
    char **names = (char **)poa_xmalloc((size_t)n_seq * sizeof(char *));
    for (int i = 0; i < n_seq; ++i) {
        const abpoa_str_t *sq = &abs->seq[exist_n_seq + i], *ql = &abs->qual[exist_n_seq + i];
        lens[i] = sq->l;
        seqs[i] = (uint8_t *)poa_xmalloc((size_t)POA_MAX(sq->l, 1));
        weights[i] = (int *)poa_xmalloc((size_t)POA_MAX(sq->l, 1) * sizeof(int));
        for (int j = 0; j < sq->l; ++j) seqs[i][j] = (uint8_t)ab_char26_table[(int)(unsigned char)sq->s[j]];
        const int use_q = abpt->use_qv && ql->l > 0;
        for (int j = 0; j < sq->l; ++j) weights[i][j] = use_q ? (int)ql->s[j] - 32 : 1;
        names[i] = abs->name[exist_n_seq + i].l > 0 ? strdup(abs->name[exist_n_seq + i].s) : strdup("");
    }
    /* abpoa_msa appends to abs itself: hand the records over instead of keeping them twice */
    abs->n_seq = exist_n_seq;
    abpoa_msa(ab, abpt, n_seq, names, lens, seqs, abpt->use_qv ? weights : NULL, out_fp);
    for (int i = 0; i < n_seq; ++i) { free(seqs[i]); free(weights[i]); free(names[i]); }
    free(seqs); free(weights); free(lens); free(names);
    return 0;
}
abpoa_t *abpoa_restore_graph(abpoa_t *ab, abpoa_para_t *abpt) {
    (void)ab; (void)abpt;
    poa_die(__func__, "restoring a graph from GFA/MSA files is outside the scope of the GPU hot-path library.");
}

/* abpoa.h -- public C ABI of the H100-native POA engine (libabpoa_b200.so).
 *
 * This header is the DROP-IN BOUNDARY: it declares, with identical names, argument
 * order, struct layouts and constants, the C interface that abPOA v1.5.6 exposes in
 * its include/abpoa.h (reference: include/abpoa.h:7-51 constants, :58-147 structs,
 * :150-230 functions).  A program compiled against the reference header links and
 * runs against this library unchanged; the sequence-to-graph dynamic program that
 * the reference runs on SSE/AVX (src/abpoa_align_simd.c) is executed here by
 * hand-written sm_90a CUDA kernels.
 *
 * Differences that are invisible to callers:
 *   - the reference includes simd_instruction.h only to name `SIMDi*` for the opaque
 *     DP-workspace pointer (include/abpoa.h:5,138); here it is `void*` (same size and
 *     alignment) and holds the per-handle device context.
 * Additional (batched / multi-GPU) entry points live in abpoa_gpu.h so that this file
 * stays a pure mirror of the reference interface.
 */
#ifndef ABPOA_H
#define ABPOA_H

#include <stdint.h>
#include <stdio.h>

/* alignment modes (reference include/abpoa.h:7-9) */
#define ABPOA_GLOBAL_MODE 0
#define ABPOA_LOCAL_MODE  1
#define ABPOA_EXTEND_MODE 2

/* gap-cost models (reference include/abpoa.h:13-15) */
#define ABPOA_LINEAR_GAP 0
#define ABPOA_AFFINE_GAP 1
#define ABPOA_CONVEX_GAP 2

/* adaptive band: w = ABPOA_EXTRA_B + ABPOA_EXTRA_F * qlen (reference :17-18) */
#define ABPOA_EXTRA_B 10
#define ABPOA_EXTRA_F 0.01

/* graph-CIGAR operation codes (reference :20-26) */
#define ABPOA_CIGAR_STR "MIDXSH"
#define ABPOA_CMATCH     0
#define ABPOA_CINS       1
#define ABPOA_CDEL       2
#define ABPOA_CDIFF      3
#define ABPOA_CSOFT_CLIP 4
#define ABPOA_CHARD_CLIP 5

#define ABPOA_SRC_NODE_ID  0
#define ABPOA_SINK_NODE_ID 1

/* output selectors (reference :31-36) */
#define ABPOA_OUT_CONS     0
#define ABPOA_OUT_MSA      1
#define ABPOA_OUT_CONS_MSA 2
#define ABPOA_OUT_GFA      3
#define ABPOA_OUT_CONS_GFA 4
#define ABPOA_OUT_CONS_FQ  5

/* consensus algorithms (reference :38-39) */
#define ABPOA_HB 0
#define ABPOA_MF 1

#define ABPOA_NONE_VERBOSE 0
#define ABPOA_INFO_VERBOSE 1
#define ABPOA_DEBUG_VERBOSE 2
#define ABPOA_LONG_DEBUG_VERBOSE 3

/* One graph-CIGAR entry is a packed 64-bit word (reference :46-51):
 *   MATCH / MISMATCH : node_id  << 34 | query_id << 4 | op
 *   INSERTION / CLIP : query_id << 34 | op_len   << 4 | op
 *   DELETION         : node_id  << 34 | op_len   << 4 | op      (op_len is always 1)
 */
#define abpoa_cigar_t uint64_t

#ifdef __cplusplus
extern "C" {
#endif

/* Alignment result (reference :58-65).  graph_cigar is malloc'ed by the library and
 * free()d by the caller when n_cigar > 0. */
typedef struct {
    int n_cigar, m_cigar; abpoa_cigar_t *graph_cigar;
    int node_s, node_e, query_s, query_e;
    int n_aln_bases, n_matched_bases;
    int32_t best_score;
} abpoa_res_t;

/* Parameter block (reference :67-90); field order and bit-field packing are ABI. */
typedef struct {
    int m; int *mat; char *mat_fn;
    int use_score_matrix;
    int match, max_mat, mismatch, min_mis, gap_open1, gap_open2, gap_ext1, gap_ext2; int inf_min;
    int sort_input_seq;
    int inc_path_score;
    int k, w, min_w;
    int wb; float wf;
    int zdrop, end_bonus;
    uint8_t ret_cigar:1, rev_cigar:1, out_msa:1, out_cons:1, out_gfa:1, out_fq:1, use_read_ids:1, amb_strand:1;
    uint8_t sub_aln:1, use_qv:1, disable_seeding:1, progressive_poa:1, put_gap_on_right:1, put_gap_at_end:1;
    char *incr_fn, *out_pog;
    int align_mode, gap_mode, max_n_cons, cons_algrm;
    double min_freq;
    int verbose;
    int batch_index;
} abpoa_para_t;

/* Graph node (reference :92-105). */
typedef struct {
    int node_id;
    int in_edge_n, in_edge_m, *in_id; int *in_edge_weight;
    int out_edge_n, out_edge_m, *out_id; int *out_edge_weight;
    int *read_weight, n_read, m_read, n_span_read;
    uint64_t **read_ids; int read_ids_n;
    int aligned_node_n, aligned_node_m, *aligned_node_id;
    uint8_t base;
} abpoa_node_t;

/* Partial-order graph (reference :107-112). */
typedef struct {
    abpoa_node_t *node; int node_n, node_m, index_rank_m;
    int *index_to_node_id;
    int *node_id_to_index, *node_id_to_max_pos_left, *node_id_to_max_pos_right, *node_id_to_max_remain, *node_id_to_msa_rank;
    uint8_t is_topological_sorted:1, is_called_cons:1, is_set_msa_rank:1;
} abpoa_graph_t;

/* Consensus / RC-MSA results (reference :114-124). */
typedef struct {
    int n_cons, n_seq, msa_len;
    int *clu_n_seq;
    int **clu_read_ids;
    int *cons_len;
    int **cons_node_ids;
    uint8_t **cons_base;
    uint8_t **msa_base;
    int **cons_cov;
    int **cons_phred_score;
} abpoa_cons_t;

typedef struct {
    int l, m; char *s;
} abpoa_str_t;

typedef struct {
    int n_seq, m_seq;
    abpoa_str_t *seq, *name, *comment, *qual;
    uint8_t *is_rc;
} abpoa_seq_t;

/* DP workspace record (reference :137-140).  s_mem is opaque to callers; in this
 * library it owns the per-handle device context (stream, HBM arenas, pinned staging).
 * dp_beg/dp_end hold the band of every DP row of the most recent alignment, exactly
 * as the reference leaves them (used to count DP cells). */
typedef struct {
    void *s_mem; uint64_t s_msize;
    int *dp_beg, *dp_end, *dp_beg_sn, *dp_end_sn, rang_m;
} abpoa_simd_matrix_t;

typedef struct {
    abpoa_graph_t *abg;
    abpoa_seq_t *abs;
    abpoa_simd_matrix_t *abm;
    abpoa_cons_t *abc;
} abpoa_t;

/* ---- parameters (reference src/abpoa_align.c:61-184) ---- */
abpoa_para_t *abpoa_init_para(void);
void abpoa_set_mat_from_file(abpoa_para_t *abpt, char *mat_fn);
void abpoa_post_set_para(abpoa_para_t *abpt);
void abpoa_free_para(abpoa_para_t *abpt);

/* ---- handle life cycle (reference src/abpoa_graph.c:174-189, :783-845) ---- */
abpoa_t *abpoa_init(void);
void abpoa_free(abpoa_t *ab);
void abpoa_reset(abpoa_t *ab, abpoa_para_t *abpt, int qlen);
void abpoa_clean_msa_cons(abpoa_t *ab);

/* ---- MSA drivers (reference src/abpoa_align.c:401-539) ---- */
int abpoa_msa(abpoa_t *ab, abpoa_para_t *abpt, int n_seqs, char **seq_names, int *seq_lens, uint8_t **seqs, int **qual_weights, FILE *out_fp);
int abpoa_msa1(abpoa_t *ab, abpoa_para_t *abpt, char *read_fn, FILE *out_fp);
abpoa_t *abpoa_restore_graph(abpoa_t *ab, abpoa_para_t *abpt);

/* ---- sequence-to-graph alignment: THE HOT PATH (reference src/abpoa_align.c:194-206,
 *      which forwards to src/abpoa_align_simd.c:1235-1338).  Runs on the GPU. ---- */
int abpoa_align_sequence_to_graph(abpoa_t *ab, abpoa_para_t *abpt, uint8_t *query, int qlen, abpoa_res_t *res);
void abpoa_subgraph_nodes(abpoa_t *ab, abpoa_para_t *abpt, int inc_beg, int inc_end, int *exc_beg, int *exc_end);
int abpoa_align_sequence_to_subgraph(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id, uint8_t *query, int qlen, abpoa_res_t *res);

/* ---- graph construction (reference src/abpoa_graph.c:471-778) ---- */
int abpoa_add_graph_node(abpoa_graph_t *abg, uint8_t base);
int abpoa_add_graph_edge(abpoa_graph_t *abg, int from_id, int to_id, int check_edge, int w, uint8_t add_read_id, uint8_t add_read_weight, int read_id, int read_ids_n, int tot_read_n);
int abpoa_add_graph_alignment(abpoa_t *ab, abpoa_para_t *abpt, uint8_t *query, int *weight, int qlen, int *qpos_to_node_id, abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends);
int abpoa_add_subgraph_alignment(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id, uint8_t *query, int *weight, int qlen, int *qpos_to_node_id, abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends);

void abpoa_BFS_set_node_index(abpoa_graph_t *abg, int src_id, int sink_id);
void abpoa_BFS_set_node_remain(abpoa_graph_t *abg, int src_id, int sink_id);
void abpoa_topological_sort(abpoa_graph_t *abg, abpoa_para_t *abpt);

/* ---- consensus / MSA output (reference src/abpoa_output.c) ---- */
void abpoa_generate_consensus(abpoa_t *ab, abpoa_para_t *abpt);
void abpoa_output_fx_consensus(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp);
void abpoa_generate_rc_msa(abpoa_t *ab, abpoa_para_t *abpt);
void abpoa_output_rc_msa(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp);
void abpoa_generate_gfa(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp);
void abpoa_output(abpoa_t *ab, abpoa_para_t *abpt, FILE *out_fp);
void abpoa_dump_pog(abpoa_t *ab, abpoa_para_t *abpt);

#ifdef __cplusplus
}
#endif

#endif

/* poa_internal.h -- private declarations shared by the host-side C sources of
 * libabpoa_b200.  Nothing here is part of the ABI (see include/abpoa.h, abpoa_gpu.h). */
#ifndef POA_INTERNAL_H
#define POA_INTERNAL_H

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "abpoa.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- fatal-on-error helpers: the reference's contract is "message on stderr and
 *      exit(EXIT_FAILURE)" for OOM / invalid input (reference src/utils.c:91-117). ---- */
void poa_die(const char *where, const char *fmt, ...) __attribute__((noreturn, format(printf, 2, 3)));
void *poa_xmalloc(size_t n);
void *poa_xcalloc(size_t n, size_t sz);
void *poa_xrealloc(void *p, size_t n);

static inline int poa_roundup32(int x) {           /* next power of two >= x */
    uint32_t v = (uint32_t)x; if (v == 0) return 0;
    --v; v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16; return (int)(v + 1);
}
#define POA_MIN(a, b) ((a) < (b) ? (a) : (b))
#define POA_MAX(a, b) ((a) > (b) ? (a) : (b))

/* backtrack state bits (reference src/abpoa_align.h:20-27) */
#define POA_OP_M   0x1
#define POA_OP_E1  0x2
#define POA_OP_E2  0x4
#define POA_OP_E   0x6
#define POA_OP_F1  0x8
#define POA_OP_F2  0x10
#define POA_OP_F   0x18
#define POA_OP_ALL 0x1f

/* ---- sequence container (poa_seq.c) ---- */
abpoa_seq_t *poa_seq_new(void);
void poa_seq_free(abpoa_seq_t *abs);
void poa_seq_reserve(abpoa_seq_t *abs);            /* grow arrays so that n_seq entries exist */
void poa_str_assign(abpoa_str_t *dst, const char *s, int l);
void poa_encode_residues(const char *s, int l, uint8_t *out);     /* letters -> codes (alphabet of the last abpoa_post_set_para) */
int poa_read_fastx(const char *fn, abpoa_seq_t *abs);   /* append every FASTA/FASTQ record of a (gz) file; returns the count, -1: cannot open */

/* ---- graph (poa_graph.c) ---- */
abpoa_graph_t *poa_graph_new(void);
void poa_graph_free(abpoa_graph_t *abg);
abpoa_cons_t *poa_cons_new(void);
void poa_cons_clear(abpoa_cons_t *abc);            /* free members, keep the struct */
void poa_cons_free(abpoa_cons_t *abc);
void poa_set_msa_rank(abpoa_graph_t *abg, int src_id, int sink_id);
void poa_cons_install(abpoa_t *ab, int n_seq, int len, const uint8_t *base, const int *cov);   /* a consensus computed on the device */
/* RC-MSA rows computed on the device: n_rows rows of msa_len codes back to back (n_seq reads, then the consensus row) */
void poa_msa_install(abpoa_t *ab, int n_seq, int n_rows, int msa_len, const uint8_t *rows);
int poa_graph_msa_installed(const abpoa_graph_t *abg);  /* abc holds installed rows for the current graph */
void poa_graph_set_msa_installed(abpoa_graph_t *abg);
/* GFA (-r 3 / -r 4).  One formatter prints every GFA this library writes, from a compact description of the graph:
 * the segments (node ids >= 2) in the writer's FIFO Kahn order, the base and in-links of each (SRC excluded, in in-edge
 * order), the set of reads whose path passes through each, and optionally the consensus path.  The host graph
 * (abpoa_generate_gfa) and the device chain's record (poa_chain.cuh: chain_gfa_record) both feed it.
 * A record is int32 words, its start 8-byte aligned:
 *   [0] n_seg  [1] n_link  [2] NS (node_n - 2)  [3] NL  [4] words per read set  [5] consensus length, -1: none
 *   seg_id[n_seg], seg_base[n_seg], link_cnt[n_seg], link_from[n_link], cons_id[max(0, cons_len)], one pad word if
 *   the count so far is odd, then the read sets as uint64 [n_seg][words] */
typedef struct {
    int n_seg, n_link, ns, nl, words, cons_len;
    const int32_t *seg_id, *seg_base, *link_cnt, *link_from, *cons_id;
    const uint64_t *read_set;
} poa_gfa_t;
#define POA_GFA_HDR 6
void poa_gfa_from_record(poa_gfa_t *g, const int32_t *rec);
/* the text for the reads of `abs` (names, is_rc); np = the header's NP; returns a malloc'ed buffer of *len bytes */
char *poa_gfa_format(const poa_gfa_t *g, const abpoa_seq_t *abs, int np, size_t *len);
/* a GFA record computed elsewhere (the device chain) for the handle's current group: abpoa_generate_gfa prints it
 * instead of walking the host graph.  Borrowed: install NULL before the record's memory goes away. */
void poa_gfa_install(abpoa_t *ab, const int32_t *rec);
/* for the tests: the host writer's segment order (returns n_seg), and a record's text as abpoa_generate_gfa prints it */
int poa_gfa_host_order(abpoa_t *ab, int32_t *out);
char *poa_gfa_record_text(const int32_t *rec, abpoa_t *ab, abpoa_para_t *abpt, size_t *len);
const int32_t *poa_graph_gfa_record(const abpoa_graph_t *abg);
void poa_graph_set_gfa_record(abpoa_graph_t *abg, const int32_t *rec);
int poa_edge_path_score(const abpoa_graph_t *abg, int node_id, int in_idx);  /* -G scores */
/* dense, node-id-indexed views kept by poa_graph.c (see poa_graph_x) */
void poa_graph_sync_public(abpoa_graph_t *abg);        /* fold dense n_read / n_span_read into node[] */
/* batch engine, global mode: keep the previous topological order and splice new nodes in instead of
 * a full Kahn pass per read (poa_graph.c, "spliced order"); counters for diagnostics */
void poa_graph_set_fast_order(abpoa_graph_t *abg, int on);
void poa_graph_order_stats(const abpoa_graph_t *abg, int64_t *spliced, int64_t *fallback);
int poa_add_alignment_nosync(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id, uint8_t *seq, int *weight,
                             int seq_l, int *qpos_to_node_id, abpoa_res_t res, int read_id, int tot_read_n, int inc_both_ends);
void poa_graph_import(abpoa_t *ab, abpoa_para_t *abpt, const int32_t *ex);     /* rebuild a device-built graph (poa_chain) */
int64_t poa_graph_edge_count(const abpoa_graph_t *abg);
const uint8_t *poa_graph_bases(const abpoa_graph_t *abg);
const int *poa_graph_in_degrees(const abpoa_graph_t *abg);
const int *poa_graph_in_ids(const abpoa_graph_t *abg, int id);
const int *poa_graph_in_ids_inline(const abpoa_graph_t *abg, int id);

/* log2 / popcount tables the reference exposes as globals (src/abpoa_output.c:13-14) */
void poa_set_65536_table(void);
void poa_set_bit_table16(void);

/* ---- flattened graph handed to the device (poa_flat.c) ----
 * One alignment = one "job blob" (layout: PoaJobHeader in poa_device.cuh): the rows are the
 * topological indices beg_index..end_index of the (sub)graph, restricted to nodes reachable
 * from the begin node (the reference's index_map, src/abpoa_align_simd.c:1257-1269), with
 * predecessor rows in the node's in_id order.  Row r <-> topological index beg_index + r. */
typedef struct {
    int n_rows;            /* end_index - beg_index + 1 (SINK row included, never computed) */
    int n_pred_max;        /* upper bound on predecessor entries                            */
    int qlen, beg_index, whole_graph, w, with_remain, with_score;
    size_t bytes;          /* blob size, multiple of 16                                     */
} poa_blob_plan;

int poa_band_halfwidth(const abpoa_para_t *abpt, int qlen);     /* w of reference :474, <0 = unbanded */
void poa_blob_plan_make(poa_blob_plan *pl, const abpoa_graph_t *abg, const abpoa_para_t *abpt,
                        int beg_node_id, int end_node_id, int qlen);
void poa_blob_fill(uint8_t *dst, const poa_blob_plan *pl, const abpoa_graph_t *abg, const abpoa_para_t *abpt,
                   int beg_node_id, int end_node_id, const uint8_t *query);
/* score width the reference would pick for this alignment (src/abpoa_align_simd.c:1293-1303) */
int poa_score_bits(const abpoa_para_t *abpt, int qlen, int n_rows);
int poa_p16_ok(const abpoa_para_t *abpt, int qlen, int n_rows);

/* ---- CUDA backend (poa_cuda.cu) ---- */
typedef struct poa_dev_ctx poa_dev_ctx;            /* per-handle stream + HBM arenas */
poa_dev_ctx *poa_dev_ctx_new(void);
void poa_dev_ctx_free(poa_dev_ctx *c);

/* The seam the reference fills with cpuid dispatch (src/abpoa_dispatch_simd.c:58-81,
 * prototype src/abpoa_align_simd.h:12).  Always runs on the GPU; there is no CPU path. */
int poa_cuda_align_sequence_to_subgraph(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id,
                                        uint8_t *query, int qlen, abpoa_res_t *res);

#ifdef __cplusplus
}
#endif
#endif

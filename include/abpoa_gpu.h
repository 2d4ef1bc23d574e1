/* abpoa_gpu.h -- ADDITIVE entry points of libabpoa_b200: batched, multi-stream, multi-GPU
 * partial-order alignment.  abpoa.h stays a pure mirror of the reference interface; nothing
 * here exists in the reference (it is single-threaded and has no batch API).
 *
 * Why: reads of one group are strictly sequential, so one abpoa_msa() call can keep only a
 * single warp of the GPU busy.  A batch of independent groups (the reference CLI's `-l`
 * list mode, src/abpoa.c:148-168, one abpoa_msa1 per file) is what fills the device: the
 * engine advances many groups concurrently -- worker threads each own a CUDA stream, launch
 * the DP/backtrace kernels for the current read of a chunk of groups (one warp per
 * alignment) and fuse the returned graph-CIGARs on the host while other chunks compute.
 *
 * Results are identical to calling abpoa_msa() group by group (reference
 * src/abpoa_align.c:401-471) with the same abpoa_para_t.
 *
 * Two engines sit behind abpoa_gpu_msa_batch (DESIGN.md section 5).  The device-resident CHAIN engine keeps
 * the graph of every group in HBM and runs align -> fuse -> re-order -> flatten entirely on the GPU (global,
 * or extend -m 2 with or without z-drop on affine / convex gaps with the reference's Kahn row order built on the device;
 * banded, convex / affine / linear gaps, heaviest-bundling or most-frequent-base consensus, RC-MSA or GFA output, ambiguous
 * strand -s, quality weights -Q of 0..255, path scores -G): two persistent kernels per batch -- one resident warp per group
 * running its alignments back to back, one fuse CTA per SM serving a task queue -- so every group advances at
 * its own pace; reads go up once, consensus bytes, MSA rows and GFA records come back once.  Everything else --
 * local mode, linear-gap extend, -d > 1, -a 1 with sub_aln, a weight outside 0..255, -G groups that could weigh more than 2^20 at a
 * node, groups that outgrow their device slot -- runs on the
 * LAUNCH engine: worker threads flatten and fuse on the host and launch one kernel grid per round, each
 * worker keeping ABPOA_GPU_PIPE_DEPTH sub-chunks in flight.  Same results either way.
 */
#ifndef ABPOA_GPU_H
#define ABPOA_GPU_H

#include <stdint.h>
#include "abpoa.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct abpoa_gpu_batch abpoa_gpu_batch_t;      /* opaque engine */

/* one read group = the arguments of one abpoa_msa() call (reads already encoded 0..m-1) */
typedef struct {
    int n_seq;
    const int *seq_lens;
    const uint8_t *const *seqs;
    const int *const *qual_weights;     /* NULL, or per read NULL / weights (used when abpt->use_qv) */
} abpoa_gpu_group_t;

/* what abpoa_msa() leaves in ab->abc, plus per-group accounting; arrays are malloc'ed by
 * the library and released with abpoa_gpu_group_result_free() */
typedef struct {
    int n_cons; int *cons_len; uint8_t **cons_base; int **cons_cov;
    int msa_len, n_msa_rows; uint8_t **msa_base;      /* filled when abpt->out_msa               */
    int64_t dp_cells;                                  /* DP cells of all alignments of the group */
    int n_aligned;                                     /* alignments performed (n_seq - 1)        */
    /* per-read records, filled when ABPOA_GPU_RECORD_READS is passed (NULL otherwise) */
    int32_t *read_best_score;                          /* [n_seq] (0 for the first read)          */
    int32_t *read_n_cigar;                             /* [n_seq]                                 */
    uint64_t *read_cigar_hash;                         /* [n_seq] FNV-1a over the CIGAR words     */
} abpoa_gpu_group_result_t;

typedef struct {
    double kernel_ms;                   /* sum over streams of CUDA-event time of the alignment kernels */
    double wall_ms;                     /* wall time of the last abpoa_gpu_msa_batch call               */
    int64_t cells, alignments, launches, retries;    /* launches: kernel launches (the resident engine: one per call) */
    uint64_t h2d_bytes, d2h_bytes;
    int n_workers, device;
    int64_t fwd_clk, bt_clk;            /* SM clock cycles inside the forward DP / the backtrace, summed over alignments */
    /* device-resident chain engine: CUDA-event time from "reads resident in HBM" to "last group fused" (summed over
     * waves), the DP cells computed inside it, groups it finished / handed back to the launch engine */
    double chain_device_ms; int64_t chain_cells; int chain_groups, chain_fallback_groups;
    /* per-launch CUDA-event times of its two kernels summed over rounds and over the concurrent cohort streams */
    double chain_dp_ms, chain_fuse_ms; int64_t chain_dp_launches;
    /* free-running chain (the default; ABPOA_GPU_CHAIN_ROUNDS=1 selects lock-step rounds): chain_dp_ms / chain_fuse_ms are then
     * sums over GROUPS of the time spent inside alignments / inside the fuse step, chain_wait_ms of the time alignment warps
     * waited for a fuse worker (queueing + the fuse itself), chain_dp_launches the number of alignments */
    double chain_wait_ms; int chain_free_running;
} abpoa_gpu_stats_t;

#define ABPOA_GPU_RECORD_READS 0x1
#define ABPOA_GPU_CAPTURE_JOBS 0x2      /* keep a copy of every flattened alignment job for abpoa_gpu_replay() */
#define ABPOA_GPU_NO_CHAIN     0x4      /* do not use the device-resident chain engine (launch-per-round engine only) */

int abpoa_gpu_device_count(void);

/* device < 0: the calling thread's current CUDA device.  n_workers <= 0 / groups_per_launch
 * <= 0: choose from the host core count and the device memory. */
abpoa_gpu_batch_t *abpoa_gpu_batch_init(int device, int n_workers, int groups_per_launch);
void abpoa_gpu_batch_free(abpoa_gpu_batch_t *eng);

/* Run n_groups independent MSAs; results[g] is overwritten.  Returns 0. */
int abpoa_gpu_msa_batch(abpoa_gpu_batch_t *eng, abpoa_para_t *abpt, int n_groups, const abpoa_gpu_group_t *groups,
                        abpoa_gpu_group_result_t *results, int flags);
void abpoa_gpu_group_result_free(abpoa_gpu_group_result_t *r);

/* The same, plus the text `abpoa -l` prints: for every group, in group order, what abpoa_output() writes
 * (consensus FASTA / FASTQ, RC-MSA or GFA according to abpt, consensus headers numbered by group as the reference
 * CLI does in list mode, src/abpoa.c:148-168).  names[g][i]: name of read i of group g (names or names[g]
 * may be NULL: rows are called Seq_1 ...).  results may be NULL. */
int abpoa_gpu_msa_batch_write(abpoa_gpu_batch_t *eng, abpoa_para_t *abpt, int n_groups, const abpoa_gpu_group_t *groups,
                              const char *const *const *names, FILE *out_fp, abpoa_gpu_group_result_t *results, int flags);

/* Device-resident measurement of the hot path: the jobs captured by the last
 * abpoa_gpu_msa_batch(..., ABPOA_GPU_CAPTURE_JOBS) call (flattened graphs + reads) are uploaded to
 * HBM once; then `repeats` timed passes launch the DP/backtrace kernels over ALL of them with no
 * host work in between (CUDA events on the launching stream, L2-cold inputs: the job set is far
 * larger than L2).  Results are checked against the captured run (score + CIGAR length). */
typedef struct {
    int64_t n_jobs, cells, rows, preds;     /* totals over the captured jobs                    */
    int64_t jobs16, cells16;                /* of which computed with int16 planes               */
    double kernel_ms;                       /* mean over the timed passes                        */
    double kernel_ms_min;
    int64_t launches;                       /* kernel launches per pass                          */
    int64_t mismatches;                     /* jobs whose replayed result differs from the capture */
    uint64_t input_bytes;                   /* HBM-resident job blobs                            */
} abpoa_gpu_replay_t;
int abpoa_gpu_replay(abpoa_gpu_batch_t *eng, abpoa_para_t *abpt, int warmup, int repeats, abpoa_gpu_replay_t *out);
void abpoa_gpu_capture_clear(abpoa_gpu_batch_t *eng);

void abpoa_gpu_batch_get_stats(abpoa_gpu_batch_t *eng, abpoa_gpu_stats_t *out);
void abpoa_gpu_batch_reset_stats(abpoa_gpu_batch_t *eng);

#ifdef __cplusplus
}
#endif
#endif

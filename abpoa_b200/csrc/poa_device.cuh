/* poa_device.cuh -- device-side data layout shared by the CUDA kernels and their host
 * launchers.  Not part of the ABI. */
#ifndef POA_DEVICE_CUH
#define POA_DEVICE_CUH

#include <stdint.h>
#include <stddef.h>

#define POA_GROUP 8                 /* DP cells handled by one lane per pass (one 16 B int16 vector) */
#define POA_MAX_M 32                /* largest alphabet held in shared memory                         */
#define POA_NEG32 (-(1 << 29))      /* "-inf" of the 32-bit register arithmetic                       */

/* status codes written by the kernel */
#define POA_ST_OK         0
#define POA_ST_PLANE_OVF  1         /* band planes did not fit the slab handed to the job  */
#define POA_ST_BT_ERROR   2         /* backtrack found no valid move (reference: fatal)    */
#define POA_ST_CIGAR_OVF  3
#define POA_ST_RANGE      4         /* packed int16 kernel: scores left the safe window, redo in 32 bits */

/* Input blob of one alignment job (host builds it in pinned memory, one H2D copy).
 * All offsets are in bytes from the start of the blob; every section is 16 B aligned. */
typedef struct PoaJobHeader {
    int32_t n_rows;         /* DP rows incl. the SINK row (which is never computed)            */
    int32_t qlen;
    int32_t w;              /* band half width, < 0: unbanded                                   */
    int32_t node_n;         /* graph->node_n: initial max_pos_left of every row                 */
    int32_t off_rowmeta;    /* int2   [n_rows+1] x = start of the row's predecessor list in pred[]        */
                            /*                   y = (band-centre term << 8) | residue code of the node   */
    int32_t off_pred;       /* int32  [n_pred]  predecessor rows, reference in_id order                  */
    int32_t off_predscore;  /* int32  [n_pred]  -G path scores, or -1                                    */
    int32_t off_live;       /* uint8  [n_rows]  sub-graph row mask, or -1 (all rows live)                */
    int32_t off_qs;         /* uint8  [qlen+1 padded] shifted query: qs[j] = query[j-1], qs[0]=0         */
    int32_t rsv[4];
    int32_t blob_bytes;
    int32_t pn;             /* lanes of the reference's AVX2 vector for ITS score width (16 / 8): beg-clamp rule */
    int32_t pad[2];
} PoaJobHeader;

/* one DP row's band and arg-max, 16 B: the adaptive band of a successor row is derived
 * from (left, right) of its predecessors */
typedef struct PoaRowInfo { int32_t beg, end, left, right; } PoaRowInfo;
/* where a row's planes start (in units of POA_GROUP cells) and the row's first predecessor (-1: none): one 8-byte
 * record, so that the backtrace and its prefetching scout learn "where next" with a single load */
typedef struct __attribute__((aligned(8))) PoaRowOff { uint32_t off; int32_t p0; } PoaRowOff;

typedef struct PoaResultDev {
    int32_t status;
    int32_t best_score, best_i, best_j;
    int32_t n_ops;                      /* cigar words written (in backtrack order)         */
    int32_t start_i, start_j;           /* last (row, j) visited by the backtrack           */
    int32_t n_aln_bases, n_matched_bases;
    int32_t max_band;                   /* widest row (cells)                               */
    int64_t cells;                      /* sum over DP rows of (end - beg + 1)              */
    uint64_t plane_units_used;          /* 8-cell units of plane storage consumed           */
    int64_t fwd_clk, bt_clk;            /* SM clock cycles spent in the forward DP / the backtrace */
    uint64_t t_start_ns, t_end_ns;      /* %globaltimer at entry / exit of the job's warp          */
    int64_t prof[6];                    /* optional per-phase SM cycles (ABPOA kernel built with -DPOA_KPROF) */
    int32_t diag[4];                    /* -DPOA_KPROF: rows on the straight-line path / rows sent to the generic path because of
                                           > 2 predecessors / a predecessor outside the ring / a predecessor band wider than its ring slot */
    int32_t btdiag[5];                  /* -DPOA_KPROF: backtrace steps taken by the speculative shortcut / its rounds / general steps /
                                           k-cycles spent in general steps / rows whose F planes the insertion step recomputed */
} PoaResultDev;

/* Backtrace shortcut record of one DP row, written by the packed forward kernel (64 B, one cache-line half):
 * bit k says "cell c0 + k of this row is explained by the diagonal of the row's FIRST predecessor"
 * (H[i][j] == H[p0][j-1] + s(i,j) (+ path score) with j-1 inside p0's band) -- the test the reference's backtrace makes
 * first whenever a match is allowed (src/abpoa_align_simd.c:211-227), true on ~90 % of its steps.  With the first
 * predecessor and the residue in the same record, such a step needs one small load instead of the generic machinery. */
#define POA_BTREC_BYTES 64
#define POA_BTREC_GROUPS 48
#define POA_BTREC_BITS  (POA_BTREC_GROUPS * 8)
typedef struct __attribute__((aligned(16))) PoaBtRec {
    int32_t c0;                         /* column of bit 0 (first cell of the row's first stored group)   */
    int32_t p0;                         /* first predecessor row, -1: none                                 */
    uint8_t base, valid;                /* residue of the node; valid = 0: the row has no bitmap (too wide) */
    uint16_t ngrp;                      /* 8-cell groups the row stores per plane                           */
    uint32_t off;                       /* start of the row's planes in the job's slab (8-cell units), as PoaRowOff.off */
    uint8_t bits[POA_BTREC_GROUPS];
} PoaBtRec;
#ifdef __cplusplus
/* the kernels read the header as one uint4 (c0, p0, base | valid << 8 | ngrp << 16, off) and the bitmap as words at +16 */
static_assert(sizeof(PoaBtRec) == POA_BTREC_BYTES && offsetof(PoaBtRec, p0) == 4 && offsetof(PoaBtRec, base) == 8 && offsetof(PoaBtRec, valid) == 9 &&
              offsetof(PoaBtRec, ngrp) == 10 && offsetof(PoaBtRec, off) == 12 && offsetof(PoaBtRec, bits) == 16 && POA_BTREC_GROUPS % 4 == 0,
              "PoaBtRec layout is hard-wired in poa_kernels.cu (forward writer and poa_backtrack)");
#endif

/* device pointers of one job */
typedef struct PoaJobDesc {
    const uint8_t *blob;
    void *planes;                       /* score planes slab of this job                    */
    uint64_t plane_cap_units;           /* capacity in units of POA_GROUP cells             */
    PoaRowInfo *rowinfo;                /* [n_rows]                                         */
    PoaRowOff *rowoff;                  /* [n_rows] start of the row's planes (units) + first predecessor row */
    uint64_t *cigar;                    /* [cigar_cap]                                      */
    int32_t cigar_cap;
    int32_t pad;
    PoaResultDev *result;               /* may live in mapped pinned host memory            */
    int32_t *done;                      /* unused (kept for layout)                                        */
    int16_t *qprof;                     /* packed kernel: query profile scratch [m][qstride] in HBM         */
    PoaBtRec *btrec;                    /* packed kernel: [n_rows] backtrace shortcut records, or NULL               */
} PoaJobDesc;

/* alignment parameters, identical for all jobs of a launch */
typedef struct PoaParamsDev {
    int32_t m;
    int32_t align_mode;                 /* ABPOA_GLOBAL/LOCAL/EXTEND_MODE                   */
    int32_t gap_mode;
    int32_t e1, o1, oe1, e2, o2, oe2;
    int32_t zdrop;
    int32_t put_gap_on_right, put_gap_at_end;
    int32_t ret_cigar;
    int32_t zero;                       /* always 0 (see poa_kernels.cu: LOCAL floors) */
    int32_t pn_unused;
    int32_t mat[POA_MAX_M * POA_MAX_M];
} PoaParamsDev;

#endif

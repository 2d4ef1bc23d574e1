/* poa_kernels.cu -- sm_90a kernels for the adaptive-banded sequence-to-POA-graph DP
 * and its backtrace.
 *
 * What is computed (the specification, validated cell-for-cell against the reference):
 *   band + recurrences  reference src/abpoa_align_simd.c:727-815 (linear), :817-933 (affine),
 *                       :935-1074 (convex); first row :582-688; band macros src/abpoa_align.h:34-35
 *   row arg-max / band hints   reference src/abpoa_align_simd.c:1107-1130
 *   end cell                   reference src/abpoa_align_simd.c:1092-1105
 *   backtrace state machine    reference src/abpoa_align_simd.c:116-458
 *
 * How it is mapped to the GPU (nothing of this exists in the reference):
 *   - ONE WARP PER ALIGNMENT, one CTA = one warp, thousands of independent alignments
 *     (one per read group) resident at once.  Rows (graph nodes in topological order) are
 *     sequentially dependent; the cells of a row's band are the parallel axis.
 *   - A lane owns POA_GROUP = 8 consecutive cells (one 16 B int16 vector); a warp covers 256
 *     cells per pass and loops for wider bands.  Rows are stored on an absolute 8-cell grid,
 *     so the predecessor's cells for the same columns are one aligned vector load and the
 *     "j-1" neighbour is one warp shuffle.
 *   - The horizontal gap dependency F[j] = max(T[j-1]-oe, F[j-1]-e) is rewritten as an
 *     exclusive prefix-max of A[k] = T[k]-oe+e*k, resolved by an in-lane chain plus one
 *     5-step warp-shuffle max-scan per plane.
 *   - Row maximum + first/last arg-max use the redux unit and ballots; the adaptive band of
 *     row i is pulled from its predecessors' (left,right) instead of being pushed to
 *     successors (same values, no scattered writes).
 *   - Arithmetic is done in 32-bit registers with the DPX add-max instructions; planes are
 *     stored as int16 when the reference would use int16 (same criterion), else int32.
 *   - The backtrace runs in the same warp right after the forward pass, lanes evaluating the
 *     predecessors of the current cell in parallel and electing the first hit in reference order.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include "poa_device.cuh"
#include "poa_chain.cuh"

#define FULL 0xffffffffu
#define NEG POA_NEG32

enum { LG = 0, AG = 1, CG = 2 };
enum { GLOBAL = 0, LOCAL = 1, EXTEND = 2 };

#define OP_M   0x1
#define OP_E1  0x2
#define OP_E2  0x4
#define OP_E   0x6
#define OP_F1  0x8
#define OP_F2  0x10
#define OP_F   0x18
#define OP_ALL 0x1f

/* ------------------------------------------------------------------ plane vectors */
__device__ __forceinline__ void ld8(const int16_t *p, int v[8]) {
    const uint4 u = *reinterpret_cast<const uint4 *>(p);
    v[0] = (int)(short)(u.x & 0xffff); v[1] = ((int)u.x) >> 16;
    v[2] = (int)(short)(u.y & 0xffff); v[3] = ((int)u.y) >> 16;
    v[4] = (int)(short)(u.z & 0xffff); v[5] = ((int)u.z) >> 16;
    v[6] = (int)(short)(u.w & 0xffff); v[7] = ((int)u.w) >> 16;
}
__device__ __forceinline__ void ld8(const int32_t *p, int v[8]) {
    const int4 a = reinterpret_cast<const int4 *>(p)[0], b = reinterpret_cast<const int4 *>(p)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ unsigned pack16(int lo, int hi) {
    lo = max(lo, -32768); hi = max(hi, -32768);
    return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16);
}
__device__ __forceinline__ void st8(int16_t *p, const int v[8]) {
    uint4 u;
    u.x = pack16(v[0], v[1]); u.y = pack16(v[2], v[3]); u.z = pack16(v[4], v[5]); u.w = pack16(v[6], v[7]);
    *reinterpret_cast<uint4 *>(p) = u;
}
__device__ __forceinline__ void st8(int32_t *p, const int v[8]) {
    int4 a, b;
    a.x = max(v[0], NEG); a.y = max(v[1], NEG); a.z = max(v[2], NEG); a.w = max(v[3], NEG);
    b.x = max(v[4], NEG); b.y = max(v[5], NEG); b.z = max(v[6], NEG); b.w = max(v[7], NEG);
    reinterpret_cast<int4 *>(p)[0] = a; reinterpret_cast<int4 *>(p)[1] = b;
}
__device__ __forceinline__ void fill8(int v[8], int x) {
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = x;
}
/* exclusive max-scan across the warp of one value per lane; returns the exclusive prefix and
 * the warp total (lane 31's inclusive value) */
__device__ __forceinline__ int warp_excl_max(int v, int lane, int &total) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULL, v, d);
        if (lane >= d) v = max(v, t);
    }
    total = __shfl_sync(FULL, v, 31);
    int e = __shfl_up_sync(FULL, v, 1);
    return lane == 0 ? 2 * NEG : e;
}

template <int GAP> struct Planes {
    static constexpr int N = GAP == LG ? 1 : (GAP == AG ? 3 : 5);
    static constexpr int H = 0, E1 = 1, E2 = 2, F1 = (GAP == AG ? 2 : 3), F2 = 4;
};

/* Compact row layout (FB, the chain engine's packed kernel): only H (+E1 (+E2)) as int16 planes, no F planes.  The F
 * planes are read by nothing but the backtrace's insertion step, which recomputes them for the one row it needs them in
 * (fb_recompute) and keeps, per cell, one byte with the outcome of every comparison it makes on them.  For F plane k
 * (bits 3k..3k+2):
 *   FB_A  H[i][j] == F_k[i][j]
 *   FB_B  H[i][j-1] - oe_k == F_k[i][j]     (0 when j-1 is outside the band)
 *   FB_C  F_k[i][j-1] - e_k == F_k[i][j]    (0 when j-1 is outside the band)
 * Cells outside the band are 0.  A row of ngrp 8-cell groups takes ngrp * N16 16-byte units. */
enum { FB_A = 1, FB_B = 2, FB_C = 4 };
template <int GAP, bool FB> struct RowLayout {
    static constexpr int N16 = FB ? (GAP == LG ? 1 : (GAP == AG ? 2 : 3)) : Planes<GAP>::N;   /* int16 planes in HBM */
    static constexpr bool BITS = FB && GAP != LG;                                              /* linear gaps need no F */
    __host__ __device__ static constexpr uint32_t units(uint32_t ngrp) { return ngrp * N16; }
};

/* Blob loads: plain coherent loads (blobs may be produced on the device by an earlier kernel of the
 * same stream; nothing here relies on the read-only path). */
template <typename T> __device__ __forceinline__ T ldb(const T *p) { return *p; }

/* ------------------------------------------------------------------ job view */
struct JobView {
    const int2 *rowmeta; const int32_t *pred, *predscore; const uint8_t *live, *qs;
    int n_rows, qlen, w, node_n, pn;
    __device__ __forceinline__ int predoff(int i) const { return ldb(&rowmeta[i].x); }
    __device__ __forceinline__ int base(int i) const { return ldb(&rowmeta[i].y) & 0xff; }
    __device__ __forceinline__ int remain(int i) const { return ldb(&rowmeta[i].y) >> 8; }
};
__device__ __forceinline__ JobView open_job(const uint8_t *blob) {
    const PoaJobHeader *h = reinterpret_cast<const PoaJobHeader *>(blob);
    JobView v;
    v.n_rows = h->n_rows; v.qlen = h->qlen; v.w = h->w; v.node_n = h->node_n; v.pn = h->pn;
    v.rowmeta = reinterpret_cast<const int2 *>(blob + h->off_rowmeta);
    v.pred = reinterpret_cast<const int32_t *>(blob + h->off_pred);
    v.predscore = h->off_predscore >= 0 ? reinterpret_cast<const int32_t *>(blob + h->off_predscore) : nullptr;
    v.live = h->off_live >= 0 ? blob + h->off_live : nullptr;
    v.qs = blob + h->off_qs;
    return v;
}

/* ================================================================== backtrace */
/* Row record of the backtrace: band, virtual cell-0 pointer of the H plane, predecessor list and the
 * first two predecessors.  `me` (uniform) describes the current row; on lane k a second record
 * describes candidate predecessor k, loaded once per row and valid across insertion steps.  It is
 * LOOK-AHEAD: when the walk moves to a candidate the new row needs no loads at all (its record is
 * broadcast from the winning lane and H[i][j] is the cell that was just compared), so the common
 * diagonal step costs: candidate record (mostly L1/L2 hits) -> one cell -> ballot. */
template <typename ST> struct BtRow {
    int row;                      /* -1: the lane holds no candidate                         */
    int beg, end; uint32_t off;   /* band and slab offset                                    */
    int pb, np, base;             /* predecessor list (start, count) and residue              */
    int p0, p1;                   /* first two predecessors (rows), -1 if absent              */
    const ST *ptr;                /* &H[row][0] (virtual: only cells beg..end exist)          */
    int pstride;                  /* elements between planes of the row                      */
    __device__ __forceinline__ bool has(int j) const { return j >= beg && j <= end; }      /* empty for end < beg (no candidate) */
    /* xs: log2 of the storage granule of a row -- 3 (the 8-cell grid) everywhere except banded linear-gap rows of the
     * generic kernel, which store whole reference vectors (16 / 8 cells) around the band (see "lgx" below) */
    __device__ __forceinline__ void locate(const ST *planes, int xs = 3) {
        const int g0 = ((beg >> xs) << xs) >> 3, g1 = ((((end >> xs) + 1) << xs) - 1) >> 3;
        pstride = (g1 - g0 + 1) * POA_GROUP;
        ptr = planes + ((ptrdiff_t)off - g0) * POA_GROUP;
    }
};
template <typename ST>
__device__ __forceinline__ void bt_load_row(BtRow<ST> &r, const JobView &jv, const ST *planes, const PoaRowInfo *rowinfo, const PoaRowOff *rowoff, int row, int xs = 3) {
    r.row = row;
    const PoaRowInfo pi = rowinfo[row];
    const uint2 ro = *reinterpret_cast<const uint2 *>(rowoff + row);       /* { plane offset, first predecessor } */
    const int2 m0 = ldb(jv.rowmeta + row);
    const int nx = ldb(&jv.rowmeta[row + 1].x);
    r.beg = pi.beg; r.end = pi.end; r.off = ro.x;
    r.pb = m0.x; r.np = nx - m0.x; r.base = m0.y & 0xff;
    r.p0 = r.np > 0 ? (int)ro.y : -1;
    r.p1 = r.np > 1 ? ldb(jv.pred + r.pb + 1) : -1;
    r.locate(planes, xs);
}

struct CigarSink {
    uint64_t *out; int cap; int n; uint64_t pending; int lane; int ovf;
    __device__ __forceinline__ void emit(uint64_t w) {
        if (n < cap) { if (lane == 0) out[n] = w; } else ovf = 1;
        ++n;
    }
    __device__ __forceinline__ void flush() { if (pending) { emit(pending); pending = 0; } }
    __device__ __forceinline__ void ins(int len, int qpos) {           /* consecutive insertions merge */
        if (pending) pending += (uint64_t)len << 4;
        else pending = ((uint64_t)(uint32_t)qpos << 34) | ((uint64_t)len << 4) | 1u;
    }
    __device__ __forceinline__ void match(int node_id, int qpos) { flush(); emit(((uint64_t)node_id << 34) | ((uint64_t)qpos << 4)); }
    __device__ __forceinline__ void del(int node_id) { flush(); emit(((uint64_t)node_id << 34) | (1ull << 4) | 2u); }
};

/* What the backtrace of the compact layout needs to recompute a row's F planes (fb_recompute, after the packed kernel) */
struct P16Consts;
struct FbCtx {
    const P16Consts *kc; const uint4 *cap_lo, *cap_hi;   /* the packed kernel's constants and band-mask tables          */
    uint8_t *buf; int buf_cells;                          /* decision bytes of one row: the shared-memory ring, idle now */
};
/* fb_recompute<..., DUMP = true> (debug export poa_debug_chain_replay only): also stores the recomputed F1 (/ F2) of the
 * kept passes, F1 of group g at f + 8 (g - g0), F2 fstride cells later -- the row's F planes as the five-plane layout holds them */
struct FbDumpCtx : FbCtx { int16_t *f; int fstride; };
template <int GAP, int MODE, bool DUMP = false, bool PS = false>
__device__ int fb_recompute(const JobView &jv, const PoaJobDesc &jd, const PoaParamsDev *prm, const FbCtx &fx,
                            int beg, int end, int pb, int np, int base, int j, int lane);

template <int GAP, typename ST, int MODE, bool FB = false, bool PS = false>
__device__ void poa_backtrack(const JobView &jv, const PoaJobDesc &jd, const PoaParamsDev *prm, const int *mat_s,
                              int lane, int best_i, int best_j, PoaResultDev &res, int xs = 3, const PoaBtRec *btrec = nullptr,
                              const FbCtx *fx = nullptr) {
    typedef Planes<GAP> PL;
    typedef RowLayout<GAP, FB> RL;
    const ST *planes = reinterpret_cast<const ST *>(jd.planes);
    const PoaRowInfo *rowinfo = jd.rowinfo; const PoaRowOff *rowoff = jd.rowoff;
    const int m = prm->m, e1 = prm->e1, oe1 = prm->oe1, e2 = prm->e2, oe2 = prm->oe2;
    const int qlen = jv.qlen;
    const bool has_ps = jv.predscore != nullptr;
    CigarSink cg; cg.out = jd.cigar; cg.cap = jd.cigar_cap; cg.n = 0; cg.pending = 0; cg.lane = lane; cg.ovf = 0;

    int i = best_i, j = best_j, start_i = best_i, start_j = best_j, cur = OP_ALL;
    int fb_row = -1, fb_lo = 0;                 /* FB: fx->buf holds the decision bytes of row fb_row from cell fb_lo on */
#ifdef POA_KPROF
    int bd_steps = 0, bd_rounds = 0, bd_general = 0, bd_fbrows = 0; long long bd_clk = 0;
#endif
    int n_aln = 0, n_match = 0, err = 0;
    int gap_at_end = prm->put_gap_at_end; const int gap_on_right = prm->put_gap_on_right;
    if (best_j < qlen) cg.ins(qlen - best_j, qlen - 1);

    BtRow<ST> me; bt_load_row<ST>(me, jv, planes, rowinfo, rowoff, i, xs);
    BtRow<ST> pc; pc.row = -1; pc.beg = 0; pc.end = -1; pc.ptr = planes; pc.pstride = 0;
    int pc_ps = 0;
    bool cand_loaded = false;
    int h_ij = (j > 0 && me.has(j)) ? (int)me.ptr[j] : NEG;       /* carried from step to step afterwards */
    int qc = j > 0 ? (int)jv.qs[j] : 0;

    /* Scout: the planes were written long ago, so every cell the walk touches is an HBM miss, and
     * the walk is one dependent miss per step.  A scout runs BT_LEAD rows ahead along the
     * first-predecessor chain (heaviest edges first = the path most reads take) and prefetches the
     * H cells the walk will compare there, assuming diagonal moves (a 128-byte line holds 64 cells,
     * so a few indels do not matter).  Lane L remembers the row the scout visited L steps ago; when
     * the walk takes another branch it usually rejoins that chain a row or two later and the scout
     * simply carries on, otherwise (the walk overtook it) it restarts at the walk's row. */
    constexpr int BT_LEAD = 6;
    int s_row = i, s_p0 = me.p0, s_ahead = 0, s_hist = (lane == 0) ? i : -1;
    PoaRowInfo s_info; s_info.beg = 0; s_info.end = -1; s_info.left = s_info.right = 0;
    uint2 s_ro = make_uint2(0u, 0u); bool s_pend = false;      /* metadata of row s_row is in flight (loaded one step ago) */
    auto scout_sync = [&](int new_row) {               /* the walk moved to new_row */
        const unsigned on_chain = __ballot_sync(FULL, s_hist == new_row);
        if (on_chain) s_ahead = __ffs(on_chain) - 1;
        else if (new_row <= s_row) { s_row = new_row; s_p0 = me.p0; s_pend = false; s_ahead = 0; s_hist = (lane == 0) ? new_row : -1; }
        else if (s_ahead > 1) --s_ahead;
    };

    /* the walk moves to the candidate row held by lane `sel` */
    auto move_to = [&](const BtRow<ST> &src, int sel) {
        me.row = __shfl_sync(FULL, src.row, sel); me.beg = __shfl_sync(FULL, src.beg, sel); me.end = __shfl_sync(FULL, src.end, sel);
        me.off = __shfl_sync(FULL, src.off, sel); me.pb = __shfl_sync(FULL, src.pb, sel);
        const int nb = __shfl_sync(FULL, (src.np << 8) | src.base, sel); me.np = nb >> 8; me.base = nb & 0xff;
        me.p0 = __shfl_sync(FULL, src.p0, sel); me.p1 = __shfl_sync(FULL, src.p1, sel);
        me.locate(planes, xs);
        i = me.row; cand_loaded = false;
        scout_sync(i);
    };
    /* candidates 32.. of a row with more than 32 predecessors (practically never) */
    auto load_chunk = [&](BtRow<ST> &px, int &px_ps, int kb) {
        px.row = -1; px.beg = 0; px.end = -1; px.ptr = planes; px.pstride = 0; px_ps = 0;
        if (kb + lane < me.np) {
            bt_load_row<ST>(px, jv, planes, rowinfo, rowoff, ldb(jv.pred + me.pb + kb + lane), xs);
            if (has_ps) px_ps = ldb(jv.predscore + me.pb + kb + lane);
        }
    };

    while (i > 0 && j > 0) {
        /* ---- shortcut: while a match is the first thing the reference would test and the row's bitmap says the first
         *      predecessor's diagonal explains the cell, the step is MATCH -> (p0, j-1) (src/abpoa_align_simd.c:211-227) and
         *      everything it needs sits in one 64-byte record per row (PoaBtRec).  Followed one record at a time this is a
         *      pointer chase through memory written long ago.  Instead every round loads the records of the 32 rows below the
         *      walk at once (lane L: row i-L) and follows the first-predecessor chain INSIDE the warp: the rows on the chain
         *      are found by pointer doubling over the lanes (5 x REDUX.OR + SHFL), a chain row's column is j minus its rank on
         *      the chain, and since that rank is at most L each lane only needs the 32 bitmap bits from column j-L on.  The
         *      walk advances to the first chain row whose bit is clear (or past the window), the confirmed steps' graph-CIGAR
         *      words go out in one store, and the next windows' records are prefetched. ---- */
        if (btrec != nullptr && MODE != LOCAL && !gap_on_right) {
            bool moved = false;
            while (i > 0 && j > 0 && (GAP == LG || (cur & OP_M)) && !gap_at_end) {
                const int ri = i - lane;
                unsigned W = 0;                             /* bit d: cell (ri, j - lane + d) is explained by the first predecessor's diagonal */
                int rp0 = -1, rbase_l = 0, jmp = -1; uint32_t r_off = 0, r_ngrp = 0; int r_c0 = 0; bool has_map = false;
                if (ri > 0) {
                    const uint8_t *rec = reinterpret_cast<const uint8_t *>(btrec + ri);
                    const uint4 hd = *reinterpret_cast<const uint4 *>(rec);        /* c0, p0, base | valid << 8 | ngrp << 16, off */
                    rp0 = (int)hd.y; rbase_l = (int)(hd.z & 0xffu); r_c0 = (int)hd.x; r_off = hd.w; r_ngrp = hd.z >> 16;
                    has_map = ((hd.z >> 8) & 0xffu) != 0;
                    const int kb0 = (j - lane) - r_c0;
                    if (has_map && kb0 > -32 && kb0 < POA_BTREC_BITS) {
                        const int wi = kb0 >> 5;            /* arithmetic shift: -1 for kb0 in [-31, -1] */
                        const uint32_t *wds = reinterpret_cast<const uint32_t *>(rec + 16);
                        const unsigned lo = (wi >= 0) ? wds[wi] : 0u, hi = (wi + 1 < POA_BTREC_GROUPS / 4) ? wds[wi + 1] : 0u;
                        W = __funnelshift_r(lo, hi, (unsigned)kb0 & 31u);
                    }
                    if (rp0 >= 0 && i - rp0 < 32) jmp = i - rp0;        /* the lane that holds the first predecessor's record */
                }
                /* rows on the chain i -> p0(i) -> p0(p0(i)) ... inside the window (chain order = lane order) */
                unsigned M = 1u;
                {
                    int jp = jmp;
#pragma unroll
                    for (int it = 0; it < 5; ++it) {
                        const unsigned add = __reduce_or_sync(FULL, (((M >> lane) & 1u) && jp >= 0) ? (1u << jp) : 0u);
                        M |= add;
                        const int nx = __shfl_sync(FULL, jp, jp & 31);
                        jp = jp >= 0 ? nx : -1;
                    }
                }
                const bool on_chain = (M >> lane) & 1u;
                const int rank = __popc(M & ((1u << lane) - 1u));       /* steps before this row */
                const int col = j - rank;
                const bool ok = on_chain && ri > 0 && col > 0 && ((W >> (lane - rank)) & 1u);
                const unsigned fail = __ballot_sync(FULL, on_chain && !ok);
                const unsigned E = fail ? (M & ((fail & (0u - fail)) - 1u)) : M;     /* executed steps: chain rows before the first failure */
                const int r = __popc(E);
#ifdef POA_KPROF
                ++bd_rounds; bd_steps += r;
#endif
                /* the general step at the row where the run stops (and its candidates, the next chain rows) reads the cells around
                 * (row, column) of every plane: request them now */
                if (on_chain && !((E >> lane) & 1u) && ri > 0 && has_map) {
                    const int kb = col - r_c0;
                    if (kb >= 0 && kb < (int)r_ngrp * POA_GROUP) {
                        const ST *cell = planes + (size_t)r_off * POA_GROUP + kb;
                        const size_t gplane = (size_t)r_ngrp * POA_GROUP;
#pragma unroll
                        for (int pl = 0; pl < RL::N16; ++pl) asm volatile("prefetch.global.L1 [%0];" :: "l"(cell + pl * gplane));
                    }
                }
                if (r == 0) break;
                const bool exec = (E >> lane) & 1u;
                cg.flush();
                if (exec && cg.n + rank < cg.cap) cg.out[cg.n + rank] = ((uint64_t)ri << 34) | ((uint64_t)(col - 1) << 4);
                if (cg.n + r > cg.cap) cg.ovf = 1;
                cg.n += r;
                n_aln += r; n_match += __popc(__ballot_sync(FULL, exec && rbase_l == (int)jv.qs[exec ? col : 0]));
                const int last = 31 - __clz(E);                         /* lane of the last executed step */
                start_i = i - last; start_j = j - (r - 1);
                i = __shfl_sync(FULL, rp0, last); j -= r; cur = OP_ALL; moved = true;
                /* records of the coming windows (a round advances 9 rows on average and lasts well under one HBM round trip:
                 * the frontier runs three windows ahead, the far ones into L2 only), and the row records a general step needs where a run stops */
                if (i - 32 - lane > 0) asm volatile("prefetch.global.L1 [%0];" :: "l"(btrec + (i - 32 - lane)));
                if (i - 64 - lane > 0) asm volatile("prefetch.global.L2 [%0];" :: "l"(btrec + (i - 64 - lane)));       /* L1 is 28 KB for 7 warps */
                if (i - 96 - lane > 0) asm volatile("prefetch.global.L2 [%0];" :: "l"(btrec + (i - 96 - lane)));
#pragma unroll
                for (int wnd = 0; wnd < 64; wnd += 32)
                    if (i - wnd - lane > 0) {
                        asm volatile("prefetch.global.L1 [%0];" :: "l"(rowinfo + (i - wnd - lane)));
                        asm volatile("prefetch.global.L1 [%0];" :: "l"(rowoff + (i - wnd - lane)));
                        asm volatile("prefetch.global.L1 [%0];" :: "l"(jv.rowmeta + (i - wnd - lane)));
                    }
            }
            if (moved) {                               /* back to the general step: rebuild its view of (i, j) */
                if (!(i > 0 && j > 0)) break;
                bt_load_row<ST>(me, jv, planes, rowinfo, rowoff, i, xs);
                h_ij = me.has(j) ? (int)me.ptr[j] : NEG;
                qc = (int)jv.qs[j];
                cand_loaded = false;
                s_row = i; s_p0 = me.p0; s_pend = false; s_ahead = 0; s_hist = (lane == 0) ? i : -1;
            }
        }
        if (MODE == LOCAL && h_ij == 0) break;
#ifdef POA_KPROF
        ++bd_general; const long long bd_t0 = clock64();
#endif
        start_i = i; start_j = j;
        const int id = i;                       /* the host maps DP rows back to node ids */
        const int rb = me.base, np = me.np;
        const int qprev = (int)jv.qs[j - 1];    /* next column's residue: off the critical path */
        const int s = mat_s[rb * m + qc];
        if (!cand_loaded) {                     /* new row: lane k learns about candidate k (lanes 0/1 already know which row) */
            pc.row = -1; pc.beg = 0; pc.end = -1; pc_ps = 0;
            if (lane < np) {
                const int prow = lane == 0 ? me.p0 : (lane == 1 ? me.p1 : ldb(jv.pred + me.pb + lane));
                bt_load_row<ST>(pc, jv, planes, rowinfo, rowoff, prow, xs);
                if (has_ps) pc_ps = ldb(jv.predscore + me.pb + lane);
            }
            cand_loaded = true;
        }
        /* every cell the tests below may look at is requested now, together: the planes were written long ago (one HBM
         * round trip each) and the tests are sequential (match, then E planes of the candidates, then F planes of this row) */
        {
            if (pc.has(j - 1)) asm volatile("prefetch.global.L1 [%0];" :: "l"(pc.ptr + (j - 1)));
            if (GAP != LG && pc.has(j)) {
                asm volatile("prefetch.global.L1 [%0];" :: "l"(pc.ptr + PL::E1 * pc.pstride + j));
                if (GAP == CG) asm volatile("prefetch.global.L1 [%0];" :: "l"(pc.ptr + PL::E2 * pc.pstride + j));
            }
            if (lane < RL::N16 && me.has(j)) asm volatile("prefetch.global.L1 [%0];" :: "l"(me.ptr + lane * me.pstride + j));
        }
        const bool c_in_m = pc.has(j - 1);
        const int c_hm1 = c_in_m ? (int)pc.ptr[j - 1] : NEG;
        int hit = 0;
        /* One scout row per step, software-pipelined: the row record requested in the previous step (band + plane offset +
         * ITS first predecessor, 24 bytes in two loads) is consumed now -- prefetch the cells the walk will look at there,
         * learn the next row of the chain -- and the next row's record is requested.  Nothing the scout loads is needed
         * in the step that loads it (ncu, round-2 pass B: the unpipelined scout cost 8.6 % of all stall samples). */
        if (s_pend) {
            s_pend = false;
            s_p0 = (int)s_ro.y;
            const int jp = j - s_ahead - 1;
            if (s_info.end >= s_info.beg) {
                const ST *sp = planes + ((ptrdiff_t)s_ro.x - (((s_info.beg >> xs) << xs) >> 3)) * POA_GROUP;
                const int ja = min(max(jp - 16, s_info.beg), s_info.end), jb = min(max(jp + 8, s_info.beg), s_info.end);
                asm volatile("prefetch.global.L1 [%0];" :: "l"(sp + ja));
                asm volatile("prefetch.global.L1 [%0];" :: "l"(sp + jb));
            }
        }
        if (s_ahead < BT_LEAD && s_p0 > 0) {
            s_row = s_p0; ++s_ahead; s_p0 = -1;
            const int up = __shfl_up_sync(FULL, s_hist, 1); s_hist = lane == 0 ? s_row : up;
            s_info = rowinfo[s_row];
            s_ro = *reinterpret_cast<const uint2 *>(rowoff + s_row);
            s_pend = true;
        }

        /* first predecessor (reference order) whose diagonal cell explains H[i][j] */
        auto try_match = [&]() {
            unsigned b = __ballot_sync(FULL, c_in_m && (c_hm1 + s + pc_ps == h_ij));
            BtRow<ST> sx = pc; int hv = c_hm1;
            if (!b && np > 32) {
                for (int kb = 32; kb < np && !b; kb += 32) {
                    int x_ps; load_chunk(sx, x_ps, kb);
                    const bool in = sx.has(j - 1);
                    hv = in ? (int)sx.ptr[j - 1] : NEG;
                    b = __ballot_sync(FULL, in && (hv + s + x_ps == h_ij));
                }
            }
            if (!b) return;
            const int sel = __ffs(b) - 1;
            cg.match(id, j - 1);
            h_ij = __shfl_sync(FULL, hv, sel);
            move_to(sx, sel);
            ++n_aln; n_match += (rb == qc);
            --j; qc = qprev; cur = OP_ALL; hit = 1;
        };

        if (!gap_on_right && !gap_at_end && (GAP == LG || (cur & OP_M))) try_match();

        if (!hit && (GAP == LG || (cur & OP_E))) {                      /* deletion: come from (p, j) */
            int e1_ij = NEG, e2_ij = NEG;
            if (GAP != LG && me.has(j)) {
                e1_ij = (int)me.ptr[PL::E1 * me.pstride + j];
                if (GAP == CG) e2_ij = (int)me.ptr[PL::E2 * me.pstride + j];
            }
            BtRow<ST> sx = pc; int x_ps = pc_ps;
            for (int kb = 0; kb < np && !hit; kb += 32) {
                if (kb > 0) load_chunk(sx, x_ps, kb);
                int code = 0, c_hj = NEG;                               /* 1: via E1, 2: via E2; +4: gap opened at p */
                if (sx.has(j)) {
                    c_hj = (int)sx.ptr[j];
                    if (GAP == LG) {
                        if (c_hj - e1 + x_ps == h_ij) code = 1;
                    } else {
                        const int c_e1 = (int)sx.ptr[PL::E1 * sx.pstride + j];
                        if (cur & OP_E1) {
                            const bool ok = (cur & OP_M) ? (h_ij == c_e1 + x_ps) : (e1_ij == c_e1 - e1 + x_ps);
                            if (ok) code = 1 | ((c_hj - oe1 == c_e1) ? 4 : 0);
                        }
                        if (GAP == CG && code == 0 && (cur & OP_E2)) {
                            const int c_e2 = (int)sx.ptr[PL::E2 * sx.pstride + j];
                            const bool ok = (cur & OP_M) ? (h_ij == c_e2 + x_ps) : (e2_ij == c_e2 - e2 + x_ps);
                            if (ok) code = 2 | ((c_hj - oe2 == c_e2) ? 4 : 0);
                        }
                    }
                }
                const unsigned b = __ballot_sync(FULL, code != 0);
                if (b) {
                    const int sel = __ffs(b) - 1;
                    const int c = __shfl_sync(FULL, code, sel);
                    if (GAP != LG) cur = (c & 4) ? (OP_M | OP_F) : ((c & 3) == 1 ? OP_E1 : OP_E2);
                    cg.del(id);
                    h_ij = __shfl_sync(FULL, c_hj, sel);
                    move_to(sx, sel);
                    hit = 1; gap_at_end = 0;
                }
            }
        }

        if (!hit && (GAP == LG || (cur & OP_F))) {                      /* insertion: come from (i, j-1) */
            const bool in_j = me.has(j), in_jm1 = me.has(j - 1);
            const int h_jm1 = in_jm1 ? (int)me.ptr[j - 1] : NEG;
            if (GAP == LG) {
                if (h_jm1 - e1 == h_ij) hit = 1;
            } else if constexpr (RL::BITS) {                            /* the comparisons below, on the recomputed F planes */
                if (in_j && (i != fb_row || j < fb_lo)) {               /* first insertion step of this row (or left of the window) */
                    fb_lo = fb_recompute<GAP, MODE, false, PS>(jv, jd, prm, *fx, me.beg, me.end, me.pb, me.np, me.base, j, lane);
                    fb_row = i;
#ifdef POA_KPROF
                    ++bd_fbrows;
#endif
                }
                const int fb = in_j ? (int)fx->buf[j - fb_lo] : 0;
                if (GAP == AG || (cur & OP_F1)) {
                    if (!(cur & OP_M) || (fb & FB_A)) {
                        if (fb & FB_B) { cur = OP_M | OP_E; hit = 1; }
                        else if (fb & FB_C) { cur = OP_F1; hit = 1; }
                    }
                }
                if (GAP == CG && !hit && (cur & OP_F2)) {
                    if (!(cur & OP_M) || (fb & (FB_A << 3))) {
                        if (fb & (FB_B << 3)) { cur = OP_M | OP_E; hit = 1; }
                        else if (fb & (FB_C << 3)) { cur = OP_F2; hit = 1; }
                    }
                }
            } else {
                if (GAP == AG || (cur & OP_F1)) {
                    const int f_ij = in_j ? (int)me.ptr[PL::F1 * me.pstride + j] : NEG;
                    const int f_jm1 = in_jm1 ? (int)me.ptr[PL::F1 * me.pstride + j - 1] : NEG;
                    if (!(cur & OP_M) || h_ij == f_ij) {
                        if (h_jm1 - oe1 == f_ij) { cur = OP_M | OP_E; hit = 1; }
                        else if (f_jm1 - e1 == f_ij) { cur = OP_F1; hit = 1; }
                    }
                }
                if (GAP == CG && !hit && (cur & OP_F2)) {
                    const int f_ij = in_j ? (int)me.ptr[PL::F2 * me.pstride + j] : NEG;
                    const int f_jm1 = in_jm1 ? (int)me.ptr[PL::F2 * me.pstride + j - 1] : NEG;
                    if (!(cur & OP_M) || h_ij == f_ij) {
                        if (h_jm1 - oe2 == f_ij) { cur = OP_M | OP_E; hit = 1; }
                        else if (f_jm1 - e2 == f_ij) { cur = OP_F2; hit = 1; }
                    }
                }
            }
            if (hit) { cg.ins(1, j - 1); h_ij = h_jm1; --j; qc = qprev; gap_at_end = 0; ++n_aln; }   /* same row: candidates stay valid */
        }

        if (!hit && (GAP == LG || (cur & OP_M))) { try_match(); if (hit) gap_at_end = 0; }
#ifdef POA_KPROF
        bd_clk += clock64() - bd_t0;
#endif
        if (!hit) { err = 1; break; }
    }
    if (!err && j > 0) cg.ins(j, j - 1);
    cg.flush();
    if (lane == 0) {
        res.n_ops = cg.n; res.start_i = start_i; res.start_j = start_j;
        res.n_aln_bases = n_aln; res.n_matched_bases = n_match;
        if (err) res.status = POA_ST_BT_ERROR; else if (cg.ovf) res.status = POA_ST_CIGAR_OVF;
#ifdef POA_KPROF
        res.btdiag[0] = bd_steps; res.btdiag[1] = bd_rounds; res.btdiag[2] = bd_general; res.btdiag[3] = (int)(bd_clk >> 10); res.btdiag[4] = bd_fbrows;
#endif
    }
}

/* ================================================================== forward DP + backtrace */
/* Tell the host this job is finished: results (possibly in mapped host memory) are made
 * visible system-wide, then its t_end_ns field turns non-zero (a plain store: no PCIe atomics
 * needed).  The host sleeps on those fields instead of on a stream event, so nothing that waits for the kernel is ever
 * queued behind it in a hardware channel shared with other streams. */
__device__ __forceinline__ void signal_done(const PoaJobDesc &jd) {
    uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    __threadfence_system();
    *reinterpret_cast<volatile uint64_t *>(&jd.result->t_end_ns) = t | 1ull;      /* non-zero == finished */
}

/* planes a successor row reads from its predecessors: H (+E1 (+E2)) */
template <int GAP> struct RingPlanes { static constexpr int N = GAP == LG ? 1 : (GAP == AG ? 2 : 3); };

template <int GAP, typename ST, int MODE>
__global__ void __launch_bounds__(32) poa_align_kernel(const PoaJobDesc *__restrict__ jobs, const PoaParamsDev *__restrict__ prm,
                                                       int n_jobs, int ring_rows, int ring_cells) {
    typedef Planes<GAP> PL;
    constexpr int RN = RingPlanes<GAP>::N;
    /* shared memory: substitution matrix | ring of the last `ring_rows` rows' (band, arg-max, slab offset)
     * | ring of their H/E planes.  Predecessors are almost always within a few rows (BFS order), so the
     * row recurrence is fed from shared memory; HBM only receives the planes the backtrace will need. */
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    int *mat_s = reinterpret_cast<int *>(dyn_smem);
    PoaRowInfo *ring_info = reinterpret_cast<PoaRowInfo *>(dyn_smem + POA_MAX_M * POA_MAX_M * sizeof(int));
    uint32_t *ring_off = reinterpret_cast<uint32_t *>(ring_info + ring_rows);
    ST *ring_data = reinterpret_cast<ST *>(reinterpret_cast<uint8_t *>(ring_off) + (((size_t)ring_rows * 4 + 15) & ~(size_t)15));
    const int rmask = ring_rows - 1, ring_groups = ring_cells >> 3;

    const int lane = threadIdx.x;
    const int job = blockIdx.x;
    if (job >= n_jobs) return;
    const long long clk0 = clock64();
    uint64_t t_start_ns; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start_ns));
    const int m = prm->m;
    for (int t = lane; t < m * m; t += 32) mat_s[t] = prm->mat[t];
    __syncwarp();

    const PoaJobDesc jd = jobs[job];
    const JobView jv = open_job(jd.blob);
    ST *planes = reinterpret_cast<ST *>(jd.planes);
    PoaRowInfo *rowinfo = jd.rowinfo; PoaRowOff *rowoff = jd.rowoff;
    const int qlen = jv.qlen, n_rows = jv.n_rows, w = jv.w;
    const bool banded = w >= 0;
    const int e1 = prm->e1, o1 = prm->o1, oe1 = prm->oe1, e2 = prm->e2, o2 = prm->o2, oe2 = prm->oe2;
    const int pnv = jv.pn;
    const int zr = prm->zero;            /* run-time 0: keeps ptxas from fusing the LOCAL floors into VIMNMX.RELU */
    /* "lgx": banded linear gaps outside local mode.  There the specification is the reference's VECTOR procedure
     * (simd_abpoa_lg_dp, src/abpoa_align_simd.c:727-815; SURVEY 8a row a7), whose band edges depend on the vector width
     * pn (16 lanes for int16 scores, 8 for int32):
     *   - a row is stored in whole vectors around its band, xbeg = beg/pn*pn .. xend = (end/pn+1)*pn-1;
     *   - the cells end+1 .. xend are not re-masked after the scan, they hold H[end] - k*E1 and successors see them;
     *   - predecessor p contributes to the cells of vectors <= (p.end+1)/pn only;
     *   - vectors beyond V1 = max_p(p.end/pn) + 1 are scanned incompletely (SIMD_SET_F with set_num 0): in vector
     *     V1 + 1 only the even lanes receive the running value, later vectors nothing.
     * The scalar oracle (oracle/poa_oracle.c: lg_vector_row, lg_set_f) restates that procedure lane by lane; the closed
     * form used here is pinned against it and against the live reference by the banded linear-gap sweeps in tests/. */
    const bool lgx = GAP == LG && MODE != LOCAL && banded;
    const int xs = lgx ? (pnv == 16 ? 4 : 3) : 3;         /* log2 of a row's storage granule */

    PoaResultDev res;
    res.status = POA_ST_OK; res.best_score = NEG; res.best_i = 0; res.best_j = 0; res.n_ops = 0;
    res.start_i = res.start_j = 0; res.n_aln_bases = res.n_matched_bases = 0; res.max_band = 0; res.cells = 0; res.plane_units_used = 0;
    res.fwd_clk = 0; res.bt_clk = 0; res.t_start_ns = t_start_ns; res.t_end_ns = 0;

    uint64_t cursor = 0;                 /* bump allocator over the job's plane slab, in 8-cell units */
    int64_t cells = 0; int max_band = 0;
    int best_score = NEG, best_i = 0, best_j = 0, best_row = 0;
    bool stop = false;

    /* ---------------- row 0 (the begin node): reference first_dp, :582-688 ---------------- */
    {
        int end0 = qlen;
        if (banded) end0 = min(qlen, max(0, qlen - jv.remain(0)) + w);
        const int g1 = ((((end0 >> xs) + 1) << xs) - 1) >> 3, ngrp = g1 + 1;
        if ((uint64_t)ngrp * PL::N > jd.plane_cap_units) { if (lane == 0) { res.status = POA_ST_PLANE_OVF; *jd.result = res; signal_done(jd); } return; }
        for (int gp = 0; gp <= g1; gp += 32) {
            const int g = gp + lane;
            if (g <= g1) {
                int h[8], ea[8], eb[8], fa[8], fb[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int j = g * 8 + c;
                    if (MODE == LOCAL) { h[c] = ea[c] = eb[c] = fa[c] = fb[c] = (j <= end0) ? 0 : NEG; }
                    else if (j > end0) { h[c] = ea[c] = eb[c] = fa[c] = fb[c] = NEG; }
                    else if (GAP == LG) { h[c] = -e1 * j; }
                    else if (j == 0) { h[c] = 0; ea[c] = -oe1; eb[c] = -oe2; fa[c] = fb[c] = NEG; }
                    else {
                        fa[c] = -o1 - e1 * j; fb[c] = -o2 - e2 * j; ea[c] = eb[c] = NEG;
                        h[c] = (GAP == CG) ? max(fa[c], fb[c]) : fa[c];
                    }
                }
                ST *rp = planes + (size_t)g * POA_GROUP;
                st8(rp, h);
                if (GAP != LG) { st8(rp + (size_t)PL::E1 * ngrp * POA_GROUP, ea); st8(rp + (size_t)PL::F1 * ngrp * POA_GROUP, fa); }
                if (GAP == CG) { st8(rp + (size_t)PL::E2 * ngrp * POA_GROUP, eb); st8(rp + (size_t)PL::F2 * ngrp * POA_GROUP, fb); }
                if (g < ring_groups) {
                    ST *rq = ring_data + (size_t)g * POA_GROUP;               /* slot 0 */
                    st8(rq, h);
                    if (GAP != LG) st8(rq + ring_cells, ea);
                    if (GAP == CG) st8(rq + 2 * ring_cells, eb);
                }
            }
        }
        if (lane == 0) {
            PoaRowInfo r0; r0.beg = 0; r0.end = end0; r0.left = 0; r0.right = 0;
            rowinfo[0] = r0; { PoaRowOff z; z.off = 0; z.p0 = -1; rowoff[0] = z; } ring_info[0] = r0; ring_off[0] = 0;
        }
        cursor = (uint64_t)ngrp * PL::N;
        cells += end0 + 1; max_band = end0 + 1;
        __syncwarp();
    }

    /* ---------------- rows 1 .. n_rows-2 in topological order ----------------
     * The graph side of a row (predecessor list, residue, band centre) is static: it is fetched
     * one row ahead so that its latency never sits on the row-to-row dependency chain. */
    int pb = 0, pe = 0, rbase = 0, rem = 0, mypred = -1, myps = 0;
    if (n_rows > 2) {
        { const int2 m1 = ldb(jv.rowmeta + 1); pb = m1.x; pe = jv.predoff(2); rbase = m1.y & 0xff; rem = m1.y >> 8; }
        if (lane < pe - pb) { mypred = ldb(jv.pred + pb + lane); if (jv.predscore) myps = ldb(jv.predscore + pb + lane); }
    }
    int nx_y = n_rows > 3 ? ldb(&jv.rowmeta[2].y) : 0;          /* packed (remain, residue) of row i+1 */
    for (int i = 1; i < n_rows - 1 && !stop; ++i) {
        int n_pe = pe, n_rbase = 0, n_rem = 0, n_mypred = -1, n_myps = 0;
        if (i + 1 < n_rows - 1) {
            { const int2 m2 = ldb(jv.rowmeta + i + 2); n_pe = m2.x; n_rbase = nx_y & 0xff; n_rem = nx_y >> 8; nx_y = m2.y; }
            if (lane < n_pe - pe) { n_mypred = ldb(jv.pred + pe + lane); if (jv.predscore) n_myps = ldb(jv.predscore + pe + lane); }
        }
        const int np = pe - pb;
        if (!(jv.live && !ldb(jv.live + i))) {

        /* lane k holds predecessor k (chunk 0); band hints are reductions over all of them */
        int pk_row = -1, pk_beg = 0, pk_end = -1, pk_ps = 0; uint32_t pk_off = 0;
        int ml = jv.node_n, mr = 0, min_pre_beg = INT32_MAX, max_pre_end = -1;
        for (int kb = 0; kb < np; kb += 32) {
            const int k = kb + lane;
            int l1 = INT32_MAX, r1 = INT32_MIN, b1 = INT32_MAX, e1x = -1;
            if (k < np) {
                const int prow = kb == 0 ? mypred : ldb(jv.pred + pb + k);
                const bool near = (i - prow) <= rmask;
                const PoaRowInfo pi = near ? ring_info[prow & rmask] : rowinfo[prow];
                l1 = pi.left + 1; r1 = pi.right + 1; b1 = pi.beg; e1x = pi.end;
                if (kb == 0) {
                    pk_row = prow; pk_beg = pi.beg; pk_end = pi.end; pk_ps = myps;
                    pk_off = near ? ring_off[prow & rmask] : rowoff[prow].off;
                }
            }
            if (banded) {
                ml = min(ml, __reduce_min_sync(FULL, l1));
                mr = max(mr, __reduce_max_sync(FULL, r1));
                min_pre_beg = min(min_pre_beg, __reduce_min_sync(FULL, b1));
                if (lgx) max_pre_end = max(max_pre_end, __reduce_max_sync(FULL, e1x));
            }
        }
        int beg = 0, end = qlen;
        if (banded) {
            const int r = qlen - rem;
            beg = max(0, min(ml, r) - w);
            end = min(qlen, max(mr, r) + w);
            if (np > 0 && beg / pnv < min_pre_beg / pnv) beg = min_pre_beg;      /* reference's vector-granular clamp */
        }
        const int g0 = ((beg >> xs) << xs) >> 3, g1 = ((((end >> xs) + 1) << xs) - 1) >> 3, ngrp = g1 - g0 + 1;
        const int lgx_v1 = lgx ? (max_pre_end >> xs) + 1 : 0;                 /* last vector with a complete scan */
        if (cursor + (uint64_t)ngrp * PL::N > jd.plane_cap_units || cursor + (uint64_t)ngrp * PL::N > 0xffffffffull) {
            if (lane == 0) { res.status = POA_ST_PLANE_OVF; res.plane_units_used = cursor; *jd.result = res; signal_done(jd); }
            return;
        }
        const uint32_t my_off = (uint32_t)cursor;
        cursor += (uint64_t)ngrp * PL::N;
        ST *rowp = planes + (size_t)my_off * POA_GROUP;
        ST *ringp = ring_data + (size_t)(i & rmask) * RN * ring_cells;
        cells += (end >= beg) ? (end - beg + 1) : 0;
        max_band = max(max_band, end - beg + 1);

        int carry1 = 2 * NEG, carry2 = 2 * NEG;            /* prefix-max of A over finished passes */
        int row_max = NEG, row_left = -1, row_right = -1;
        const int jbase = g0 * 8;

        for (int gp = g0; gp <= g1; gp += 32) {
            const int g = gp + lane;
            const bool active = g <= g1;
            /* this lane's 8 query residues; independent of the predecessors, so issued first */
            uint2 qv = make_uint2(0u, 0u);
            if (active) qv = ldb(reinterpret_cast<const uint2 *>(jv.qs + (size_t)g * 8));
            int M[8], X1[8], X2[8];                         /* M: diagonal term; X1/X2: E1/E2 inputs (LG: X1 = vertical term) */
            fill8(M, NEG); fill8(X1, NEG); if (GAP == CG) fill8(X2, NEG);

            for (int kb = 0; kb < np; kb += 32) {
                int c_row = pk_row, c_beg = pk_beg, c_end = pk_end, c_ps = pk_ps; uint32_t c_off = pk_off;
                if (kb > 0) {                               /* rare: more than 32 predecessors */
                    const int k = kb + lane; c_row = -1;
                    if (k < np) {
                        c_row = ldb(jv.pred + pb + k); const PoaRowInfo pi = rowinfo[c_row];
                        c_beg = pi.beg; c_end = pi.end; c_off = rowoff[c_row].off; c_ps = jv.predscore ? ldb(jv.predscore + pb + k) : 0;
                    }
                }
                const int nk = min(32, np - kb);
                for (int k = 0; k < nk; ++k) {
                    const int p_row = __shfl_sync(FULL, c_row, k);
                    const int p_beg = __shfl_sync(FULL, c_beg, k), p_end = __shfl_sync(FULL, c_end, k);
                    const uint32_t p_off = __shfl_sync(FULL, c_off, k);
                    const int ps = jv.predscore ? __shfl_sync(FULL, c_ps, k) : 0;
                    const int pg0 = ((p_beg >> xs) << xs) >> 3, pg1 = ((((p_end >> xs) + 1) << xs) - 1) >> 3, png = pg1 - pg0 + 1;
                    const int p_vlim = lgx ? ((((p_end + 1) >> xs) + 1) << xs) : INT32_MAX;      /* lgx: p feeds cells j < p_vlim only */
                    const bool near = (i - p_row) <= rmask;
                    const ST *ph = planes + (size_t)p_off * POA_GROUP;                       /* HBM copy   */
                    const ST *rh = ring_data + (size_t)(p_row & rmask) * RN * ring_cells;    /* smem copy  */
                    int hp[8], ep1[8], ep2[8];
                    const bool inr = active && g >= pg0 && g <= pg1;
                    const int rel = g - pg0;
                    if (inr && near && rel < ring_groups) {
                        const ST *q = rh + (size_t)rel * POA_GROUP;
                        ld8(q, hp);
                        if (GAP != LG) ld8(q + ring_cells, ep1);
                        if (GAP == CG) ld8(q + 2 * ring_cells, ep2);
                    } else if (inr) {
                        const ST *q = ph + (size_t)rel * POA_GROUP;
                        ld8(q, hp);
                        if (GAP != LG) ld8(q + (size_t)PL::E1 * png * POA_GROUP, ep1);
                        if (GAP == CG) ld8(q + (size_t)PL::E2 * png * POA_GROUP, ep2);
                    } else { fill8(hp, NEG); if (GAP != LG) fill8(ep1, NEG); if (GAP == CG) fill8(ep2, NEG); }
                    int hm1 = __shfl_up_sync(FULL, hp[7], 1);
                    if (lane == 0) {
                        const int relm = rel - 1;
                        hm1 = NEG;
                        if (relm >= 0 && relm < png) hm1 = (near && relm < ring_groups) ? (int)rh[(size_t)relm * POA_GROUP + 7] : (int)ph[(size_t)relm * POA_GROUP + 7];
                        if (MODE == LOCAL && g == 0) hm1 = 0;
                    }
                    if (GAP == LG && lgx) {
#pragma unroll
                        for (int c = 0; c < 8; ++c) {
                            if (g * 8 + c < p_vlim) { M[c] = max(M[c], (c == 0 ? hm1 : hp[c - 1]) + ps); X1[c] = max(X1[c], hp[c] - e1 + ps); }
                        }
                    } else {
                    M[0] = max(M[0], hm1 + ps);
#pragma unroll
                    for (int c = 1; c < 8; ++c) M[c] = max(M[c], hp[c - 1] + ps);
                    }
                    if (GAP == LG) {
                        if (!lgx) {
#pragma unroll
                        for (int c = 0; c < 8; ++c) X1[c] = max(X1[c], hp[c] - e1 + ps);
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < 8; ++c) X1[c] = max(X1[c], ep1[c] + ps);
                        if (GAP == CG) {
#pragma unroll
                            for (int c = 0; c < 8; ++c) X2[c] = max(X2[c], ep2[c] + ps);
                        }
                    }
                }
            }

            /* substitution scores of this row's residue against the lane's 8 query bases */
            const int *mrow = mat_s + rbase * m;
            int T[8], H[8], Fa[8], Fb[8];
            bool inb[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int j = g * 8 + c;
                inb[c] = active && j >= beg && j <= end;
                const unsigned code = ((c < 4 ? qv.x : qv.y) >> (8 * (c & 3))) & 0xffu;
                int s = mrow[code];
                if (j == 0) s = 0;
                const int hm = inb[c] ? M[c] + s : NEG;
                if (!inb[c]) { X1[c] = NEG; if (GAP == CG) X2[c] = NEG; }
                M[c] = hm;
                if (GAP == LG) T[c] = max(hm, X1[c]);
                else if (GAP == AG) T[c] = hm;               /* affine: F opens from the M-only value (reference :916) */
                else T[c] = max(hm, max(X1[c], X2[c]));
            }

            /* horizontal dependency as prefix-max of A[k] = T[k] - oe + e*jr */
            int a1[8], a2[8], l1 = 2 * NEG, l2 = 2 * NEG;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int jr = g * 8 + c - jbase;
                a1[c] = T[c] + ((GAP == LG ? 0 : -oe1) + e1 * jr);
                l1 = max(l1, a1[c]);
                if (GAP == CG) { a2[c] = T[c] + (-oe2 + e2 * jr); l2 = max(l2, a2[c]); }
            }
            int tot1, tot2 = 0;
            int x1 = max(warp_excl_max(l1, lane, tot1), carry1);
            carry1 = max(carry1, tot1);
            int x2 = 2 * NEG;
            if (GAP == CG) { x2 = max(warp_excl_max(l2, lane, tot2), carry2); carry2 = max(carry2, tot2); }

            int E1o[8], E2o[8];
            int lmax = NEG, lfirst = -1, llast = -1;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int j = g * 8 + c, jr = j - jbase;
                if (GAP == LG) {
                    x1 = max(x1, a1[c]);                    /* inclusive: H[j] = max(H0[j], H[j-1]-e) */
                    int h = max(x1 - e1 * jr, NEG);
                    if (MODE == LOCAL) h = max(h, zr);
                    if (lgx) {                              /* stored cell of the row's vectors: the running value survives to the right of
                                                               `end`; beyond the last completely scanned vector only even lanes of the next one */
                        const int v = j >> xs;
                        const bool keep = active && j >= beg && j <= ((((end >> xs) + 1) << xs) - 1) &&
                                          (v <= lgx_v1 || (v == lgx_v1 + 1 && !(j & 1)));
                        H[c] = keep ? h : NEG;
                    } else
                    H[c] = inb[c] ? h : NEG;
                } else {
                    const int f1 = max(x1 - e1 * (jr - 1), NEG);
                    x1 = max(x1, a1[c]);
                    Fa[c] = f1;
                    if (GAP == AG) {
                        const int t = max(M[c], X1[c]);
                        int h = max(t, f1);
                        if (MODE == LOCAL) h = max(h, zr);
                        /* NOTE (ptxas 12.9, sm_100a): with a literal 0 floor, "max(max(t,f),0) == t" was
                         * fused into VIMNMX.RELU's predicate output and evaluated false for equal
                         * operands (seen on B200: the LOCAL affine kernel stored E = 0 everywhere).
                         * The floor therefore comes from a run-time zero (prm->zero), see `zr`. */
                        const bool from_t = (h == t);
                        E1o[c] = from_t ? max(X1[c] - e1, h - oe1) : (MODE == LOCAL ? 0 : NEG);
                        H[c] = h;
                    } else {
                        const int f2 = max(x2 - e2 * (jr - 1), NEG);
                        x2 = max(x2, a2[c]);
                        Fb[c] = f2;
                        int h = max(T[c], max(f1, f2));
                        if (MODE == LOCAL) h = max(h, zr);
                        int eo1 = max(X1[c] - e1, h - oe1), eo2 = max(X2[c] - e2, h - oe2);
                        if (MODE == LOCAL) { eo1 = max(eo1, zr); eo2 = max(eo2, zr); }
                        E1o[c] = eo1; E2o[c] = eo2; H[c] = h;
                    }
                    if (!inb[c]) { H[c] = NEG; E1o[c] = NEG; if (GAP == CG) E2o[c] = NEG; }
                }
                if (inb[c]) {
                    if (H[c] > lmax) { lmax = H[c]; lfirst = llast = j; }
                    else if (H[c] == lmax) llast = j;
                }
            }

            if (active) {
                const int rel = g - g0;
                if (rel < ring_groups) {                    /* what successors read: shared memory */
                    ST *rq = ringp + (size_t)rel * POA_GROUP;
                    st8(rq, H);
                    if (GAP != LG) st8(rq + ring_cells, E1o);
                    if (GAP == CG) st8(rq + 2 * ring_cells, E2o);
                }
                ST *q = rowp + (size_t)rel * POA_GROUP;    /* what the backtrace reads: HBM */
                st8(q, H);
                if (GAP != LG) { st8(q + (size_t)PL::E1 * ngrp * POA_GROUP, E1o); st8(q + (size_t)PL::F1 * ngrp * POA_GROUP, Fa); }
                if (GAP == CG) { st8(q + (size_t)PL::E2 * ngrp * POA_GROUP, E2o); st8(q + (size_t)PL::F2 * ngrp * POA_GROUP, Fb); }
            }

            /* row maximum with first / last arg-max (reference :1107-1119) */
            if (banded || MODE != GLOBAL) {
                const int pm = __reduce_max_sync(FULL, lmax);
                const unsigned bm = __ballot_sync(FULL, lmax == pm && lfirst >= 0);
                if (bm) {
                    const int pl = __shfl_sync(FULL, lfirst, __ffs(bm) - 1);
                    const int pr = __shfl_sync(FULL, llast, 31 - __clz(bm));
                    if (pm > row_max) { row_max = pm; row_left = pl; row_right = pr; }
                    else if (pm == row_max) row_right = pr;
                }
            }
        }
        if (lane == 0) {
            PoaRowInfo ri; ri.beg = beg; ri.end = end; ri.left = row_left; ri.right = row_right;
            ring_info[i & rmask] = ri; ring_off[i & rmask] = my_off;
            rowinfo[i] = ri; { PoaRowOff z; z.off = my_off; z.p0 = mypred; *reinterpret_cast<uint2 *>(rowoff + i) = make_uint2(z.off, (unsigned)z.p0); }
        }
        if (MODE == LOCAL) {
            if (row_max > best_score) { best_score = row_max; best_i = i; best_j = row_left; }
        } else if (MODE == EXTEND) {
            if (row_max > best_score) { best_score = row_max; best_i = i; best_j = row_right; best_row = i; }
            else if (prm->zdrop > 0) {
                const int delta = jv.remain(best_row) - rem;
                if (best_score - row_max > prm->zdrop + e1 * abs(delta - (row_right - best_j))) stop = true;
            }
        }
        __syncwarp();
        }   /* live row */
        pb = pe; pe = n_pe; rbase = n_rbase; rem = n_rem; mypred = n_mypred; myps = n_myps;
    }

    /* ---------------- global mode: best end cell among the SINK's predecessors ---------------- */
    if (MODE == GLOBAL) {
        const int sb = jv.predoff(n_rows - 1), sn = jv.predoff(n_rows) - sb;
        for (int k = 0; k < sn; ++k) {
            const int prow = jv.pred[sb + k];
            const PoaRowInfo pi = rowinfo[prow];
            const int endc = qlen > pi.end ? pi.end : qlen;
            const int pg0 = ((pi.beg >> xs) << xs) >> 3;
            const int v = (endc >= pi.beg) ? (int)planes[(size_t)rowoff[prow].off * POA_GROUP + (endc - pg0 * 8)] : NEG;
            if (v > best_score) { best_score = v; best_i = prow; best_j = endc; }
        }
    }
    res.best_score = best_score; res.best_i = best_i; res.best_j = best_j;
    res.cells = cells; res.max_band = max_band; res.plane_units_used = cursor;
    const long long clk1 = clock64();
    res.fwd_clk = clk1 - clk0;
    if (lane == 0) *jd.result = res;
    __syncwarp();
    if (prm->ret_cigar) {
        poa_backtrack<GAP, ST, MODE>(jv, jd, prm, mat_s, lane, best_i, best_j, *jd.result, xs);
        if (lane == 0) jd.result->bt_clk = clock64() - clk1;
    }
    if (lane == 0) signal_done(jd);
}

/* ================================================================== packed int16x2 forward DP
 * Same algorithm, same int16 plane layout and the same backtrace as poa_align_kernel<.., int16_t, ..>,
 * but the row arithmetic works on PAIRS of cells with the DPX packed instructions
 * (VIMNMX.S16x2 / VIMNMX3.S16x2 / VIADDMNMX.S16x2 / VIADD.16x2): a lane's 8 cells are 4 registers
 * per plane, loaded and stored as one 16-byte vector without unpacking.
 *   - "minus infinity" is NEGP = -30000: far below any real score the launcher admits to this
 *     kernel, and far enough from -32768 that adding one penalty cannot wrap; every addition that
 *     can go down is a VIADDMNMX clamped at NEGP.
 *   - substitution scores come from a per-job query profile qp[residue][j] (int16, built by the
 *     warp itself at kernel start) as one 16-byte load per row.
 *   - the lane-local part of the F prefix-max runs on packed values; the cross-lane scan runs on
 *     32-bit lane aggregates, so e*jr never has to fit 16 bits.
 *   - band edges are applied with two 16-byte mask vectors from shared-memory tables.
 * The launcher uses this kernel whenever scores provably fit (see poa_p16_ok); a run-time guard
 * (row maxima drifting towards the rails) makes the job fall back to the 32-bit kernel. */
#ifdef POA_KPROF
#define KP_DECL long long kp[6] = {0,0,0,0,0,0}; long long kp_t = clock64(); int kdiag[4] = {0,0,0,0};
#define KP(n) { const long long t_ = clock64(); kp[n] += t_ - kp_t; kp_t = t_; }
#define KP_OUT(res) { for (int z_ = 0; z_ < 6; ++z_) (res).prof[z_] = kp[z_]; for (int z_ = 0; z_ < 4; ++z_) (res).diag[z_] = kdiag[z_]; }
#else
#define KP_DECL
#define KP(n)
#define KP_OUT(res)
#endif
#define NEGP (-30000)
#define NEGP2 0x8AD08AD0u

__device__ __forceinline__ unsigned pk(int lo, int hi) { return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16); }
__device__ __forceinline__ int lo16(unsigned v) { return (int)(short)(v & 0xffffu); }
__device__ __forceinline__ int hi16(unsigned v) { return ((int)v) >> 16; }
__device__ __forceinline__ unsigned bc_hi(unsigned v) { return __byte_perm(v, v, 0x3232); }      /* [hi, hi] */
/* cells shifted by one towards higher j: [prev.hi, cur.lo] */
__device__ __forceinline__ unsigned sh1(unsigned prev, unsigned cur) { return __byte_perm(prev, cur, 0x5432); }

/* lane-local exclusive prefix max: P[c] = max(x, a[0..c-1]) for the 8 packed cells a[0..3], x broadcast in xb */
__device__ __forceinline__ void lane_excl_prefix(const unsigned a[4], unsigned xb, unsigned P[4]) {
    unsigned inc[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) inc[k] = __vmaxs2(a[k], __byte_perm(a[k], NEGP2, 0x1054));   /* [lo, max(lo,hi)] */
    inc[1] = __vmaxs2(inc[1], bc_hi(inc[0]));
    inc[2] = __vmaxs2(inc[2], bc_hi(inc[1]));
    inc[3] = __vmaxs2(inc[3], bc_hi(inc[2]));
    P[0] = __vmaxs2(sh1(xb, inc[0]), xb);
    P[1] = __vmaxs2(sh1(inc[0], inc[1]), xb);
    P[2] = __vmaxs2(sh1(inc[1], inc[2]), xb);
    P[3] = __vmaxs2(sh1(inc[2], inc[3]), xb);
}
/* max over the 8 packed cells as a 32-bit int */
__device__ __forceinline__ int lane_max8(const unsigned a[4]) {
    const unsigned m = __vmaxs2(__vmaxs2(a[0], a[1]), __vmaxs2(a[2], a[3]));
    return max(lo16(m), hi16(m));
}

/* Lane-independent packed constants of the row arithmetic.  Passed to the kernels BY VALUE (__grid_constant__): they
 * then live in the constant bank and are used as instruction operands directly -- kept in registers they were
 * rematerialised by ~30 integer instructions every row (register pressure), see profiles/r02_sass_*.txt. */
struct P16Consts {
    unsigned K1[4], K2[4];          /* e * (2k), e * (2k+1): A[c] = T[c] + e*c                     */
    unsigned KF1[4], KF2[4];        /* -(oe + e*(2k-1)), -(oe + e*2k): F from the exclusive prefix  */
    unsigned KLG[4];                /* -e1*(2k), -e1*(2k+1): linear-gap H from the inclusive prefix */
    unsigned NE1, NOE1, NE2, NOE2;  /* -e, -oe in both halves                                       */
};
static inline unsigned pk_host(int lo, int hi) { return ((unsigned)lo & 0xffffu) | ((unsigned)hi << 16); }
static P16Consts make_p16_consts(int e1, int oe1, int e2, int oe2) {
    P16Consts c;
    for (int k = 0; k < 4; ++k) {
        c.K1[k] = pk_host(e1 * (2 * k), e1 * (2 * k + 1)); c.K2[k] = pk_host(e2 * (2 * k), e2 * (2 * k + 1));
        c.KF1[k] = pk_host(-(oe1 + e1 * (2 * k - 1)), -(oe1 + e1 * (2 * k))); c.KF2[k] = pk_host(-(oe2 + e2 * (2 * k - 1)), -(oe2 + e2 * (2 * k)));
        c.KLG[k] = pk_host(-e1 * (2 * k), -e1 * (2 * k + 1));
    }
    c.NE1 = pk_host(-e1, -e1); c.NOE1 = pk_host(-oe1, -oe1); c.NE2 = pk_host(-e2, -e2); c.NOE2 = pk_host(-oe2, -oe2);
    return c;
}

/* shared-memory layout of one packed-kernel CTA (one warp) */
struct P16Smem {
    int *mat_s; uint4 *cap_lo, *cap_hi, *ring_meta; int16_t *ring_data;
};
__device__ __forceinline__ P16Smem p16_smem_init(uint8_t *dyn_smem, const PoaParamsDev *prm, int ring_rows, int lane) {
    P16Smem sm;
    sm.mat_s = reinterpret_cast<int *>(dyn_smem);
    sm.cap_lo = reinterpret_cast<uint4 *>(dyn_smem + POA_MAX_M * POA_MAX_M * sizeof(int));   /* [9]: first n cells masked */
    sm.cap_hi = sm.cap_lo + 9;                                                                 /* [9]: last n cells masked  */
    sm.ring_meta = sm.cap_hi + 9;                    /* [ring_rows] {beg, end, (left+1)|(right+1)<<16, plane offset} */
    sm.ring_data = reinterpret_cast<int16_t *>(sm.ring_meta + ring_rows);
    const int m = prm->m;
    for (int t = lane; t < m * m; t += 32) sm.mat_s[t] = prm->mat[t];
    if (lane < 9) {
        unsigned lo[4], hi[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            lo[k] = pk(2 * k < lane ? NEGP : 32767, 2 * k + 1 < lane ? NEGP : 32767);
            hi[k] = pk(2 * k >= 8 - lane ? NEGP : 32767, 2 * k + 1 >= 8 - lane ? NEGP : 32767);
        }
        sm.cap_lo[lane] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        sm.cap_hi[lane] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    }
    __syncwarp();
    return sm;
}

/* The row arithmetic of one lane's 8 cells (group g, jr0 = 8 (g - g0)), shared by the forward pass and the backtrace's F
 * recompute so that both give the same bits: from the folded predecessor terms (M: diagonal, X1 / X2: vertical), the query
 * profile S and the band masks to H, the F planes and the outgoing E planes.  carry1 / carry2 carry the F scans from one
 * 256-cell pass to the next; M is left holding Hm, -inf left of the band. */
template <int GAP, int MODE>
__device__ __forceinline__ void p16_cells(const P16Consts &kc, const unsigned CLO[4], const unsigned CAP[4], const unsigned S[4],
                                          unsigned M[4], const unsigned X1[4], const unsigned X2[4], int jr0, int e1, int oe1, int e2, int oe2,
                                          unsigned zr2, int lane, int &carry1, int &carry2,
                                          unsigned H[4], unsigned F1[4], unsigned F2[4], unsigned E1o[4], unsigned E2o[4]) {
    unsigned T[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned hm = __viaddmax_s16x2(M[k], S[k], NEGP2);
        M[k] = __vmins2(hm, CLO[k]);                                 /* Hm, -inf left of the band */
        if (GAP == LG) T[k] = __vmins2(__vmaxs2(hm, X1[k]), CLO[k]);
        else if (GAP == AG) T[k] = M[k];                              /* affine F opens from the M-only value */
        else T[k] = __vmins2(__vimax3_s16x2(hm, X1[k], X2[k]), CLO[k]);
    }
    /* lane-local A = T + e*c ; lane aggregate in 32 bits ; warp scan ; back to lane-local */
    unsigned a1[4], a2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { a1[k] = __vadd2(T[k], kc.K1[k]); if (GAP == CG) a2[k] = __vadd2(T[k], kc.K2[k]); }
    const int off1 = e1 * jr0 - (GAP == LG ? 0 : oe1), off2 = e2 * jr0 - oe2;
    int tot1, tot2 = 0;
    int x1 = max(warp_excl_max(lane_max8(a1) + off1, lane, tot1), carry1);
    carry1 = max(carry1, tot1);
    const int xl1 = min(max(x1 - off1, NEGP), 32767);
    unsigned P1[4], P2[4];
    lane_excl_prefix(a1, pk(xl1, xl1), P1);
    if (GAP == CG) {
        int x2 = max(warp_excl_max(lane_max8(a2) + off2, lane, tot2), carry2);
        carry2 = max(carry2, tot2);
        const int xl2 = min(max(x2 - off2, NEGP), 32767);
        lane_excl_prefix(a2, pk(xl2, xl2), P2);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (GAP == LG) {
            /* inclusive: H[c] = max(P[c], a[c]) - e1*c */
            unsigned h = __viaddmax_s16x2(__vmaxs2(P1[k], a1[k]), kc.KLG[k], NEGP2);
            if (MODE == LOCAL) h = __vmaxs2(h, zr2);
            H[k] = __vmins2(h, CAP[k]);
        } else {
            F1[k] = __viaddmax_s16x2(P1[k], kc.KF1[k], NEGP2);
            if (GAP == AG) {
                const unsigned t = __vmaxs2(M[k], X1[k]);
                unsigned fz = F1[k];
                if (MODE == LOCAL) fz = __vmaxs2(fz, zr2);
                const unsigned h = __vmaxs2(t, fz);
                const unsigned from_t = __vcmpges2(t, fz);            /* h == t, per cell */
                const unsigned ev = __viaddmax_s16x2(X1[k], kc.NE1, __viaddmax_s16x2(h, kc.NOE1, NEGP2));
                const unsigned alt = (MODE == LOCAL) ? zr2 : NEGP2;
                E1o[k] = __vmins2((ev & from_t) | (alt & ~from_t), CAP[k]);
                H[k] = __vmins2(h, CAP[k]);
            } else {
                F2[k] = __viaddmax_s16x2(P2[k], kc.KF2[k], NEGP2);
                unsigned h = __vimax3_s16x2(T[k], F1[k], F2[k]);
                if (MODE == LOCAL) h = __vmaxs2(h, zr2);
                unsigned eo1 = __viaddmax_s16x2(X1[k], kc.NE1, __viaddmax_s16x2(h, kc.NOE1, NEGP2));
                unsigned eo2 = __viaddmax_s16x2(X2[k], kc.NE2, __viaddmax_s16x2(h, kc.NOE2, NEGP2));
                if (MODE == LOCAL) { eo1 = __vmaxs2(eo1, zr2); eo2 = __vmaxs2(eo2, zr2); }
                H[k] = __vmins2(h, CAP[k]); E1o[k] = __vmins2(eo1, CAP[k]); E2o[k] = __vmins2(eo2, CAP[k]);
            }
        }
    }
}

/* The insertion-step decision bytes (FB_A / FB_B / FB_C, see RowLayout) of one lane's 8 cells from the values p16_cells gave
 * (exact: every value is >= NEGP and every penalty <= 1000 (poa_p16_ok), so the packed additions cannot wrap).  left_in:
 * cell 8g-1 is inside the band (g > g0, as beg lies in group g0).  lh / lf1 / lf2 hold H / F of the cell left of lane 0 (high
 * halves, from the previous pass); more: another pass follows, so they are set to lane 31's last cell. */
template <int GAP>
__device__ __forceinline__ uint2 p16_fbits(const P16Consts &kc, const unsigned H[4], const unsigned F1[4], const unsigned F2[4],
                                           const unsigned CLO[4], const unsigned CAP[4], bool left_in, int lane, bool more,
                                           unsigned &lh, unsigned &lf1, unsigned &lf2) {
    const unsigned hl = __shfl_up_sync(FULL, H[3], 1), f1l = __shfl_up_sync(FULL, F1[3], 1);
    unsigned f2l = 0u;
    if (GAP == CG) f2l = __shfl_up_sync(FULL, F2[3], 1);
    const unsigned hp = lane == 0 ? lh : hl, f1p = lane == 0 ? lf1 : f1l, f2p = lane == 0 ? lf2 : f2l;
    const unsigned clp = left_in ? 0x7fff0000u : 0u;
    unsigned v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned inb = __vcmpeq2(CAP[k], 0x7fff7fffu);                          /* j in the band   */
        const unsigned inl = inb & __vcmpeq2(sh1(k ? CLO[k - 1] : clp, CLO[k]), 0x7fff7fffu);   /* and j-1 too */
        const unsigned hs = sh1(k ? H[k - 1] : hp, H[k]), fs1 = sh1(k ? F1[k - 1] : f1p, F1[k]);
        unsigned x = (__vcmpeq2(H[k], F1[k]) & inb & (FB_A * 0x10001u))
                   | (__vcmpeq2(__vadd2(hs, kc.NOE1), F1[k]) & inl & (FB_B * 0x10001u))
                   | (__vcmpeq2(__vadd2(fs1, kc.NE1), F1[k]) & inl & (FB_C * 0x10001u));
        if (GAP == CG) {
            const unsigned fs2 = sh1(k ? F2[k - 1] : f2p, F2[k]);
            x |= (__vcmpeq2(H[k], F2[k]) & inb & ((FB_A << 3) * 0x10001u))
               | (__vcmpeq2(__vadd2(hs, kc.NOE2), F2[k]) & inl & ((FB_B << 3) * 0x10001u))
               | (__vcmpeq2(__vadd2(fs2, kc.NE2), F2[k]) & inl & ((FB_C << 3) * 0x10001u));
        }
        v[k] = x;
    }
    if (more) {
        lh = __shfl_sync(FULL, H[3], 31); lf1 = __shfl_sync(FULL, F1[3], 31);
        if (GAP == CG) lf2 = __shfl_sync(FULL, F2[3], 31);
    }
    return make_uint2(__byte_perm(v[0], v[1], 0x6420), __byte_perm(v[2], v[3], 0x6420));
}

/* Recompute row `row`'s F planes for the backtrace's insertion step (compact layout): the row arithmetic of the forward pass
 * (p16_cells), fed from the predecessors' H / E planes in HBM, the query profile and the band-mask tables, pass by pass from
 * the band's first cell to cell j.  The decision bytes of the last fx.buf_cells / 256 passes up to j's go to fx.buf, from the
 * returned cell on.  PS (-G jobs of the chain): predecessor k's path score is added to its diagonal term and its E planes,
 * as the forward pass adds it, so the recomputed planes match the forward pass bit for bit. */
template <int GAP, int MODE, bool DUMP, bool PS>
__device__ int fb_recompute(const JobView &jv, const PoaJobDesc &jd, const PoaParamsDev *prm, const FbCtx &fx,
                            int beg, int end, int pb, int np, int base, int j, int lane) {
    const P16Consts &kc = *fx.kc;
    const int16_t *planes = reinterpret_cast<const int16_t *>(jd.planes);
    const int e1 = prm->e1, oe1 = prm->oe1, e2 = prm->e2, oe2 = prm->oe2;
    const unsigned zr2 = (unsigned)prm->zero;
    const int qstride = ((jv.qlen + 1 + 7) & ~7) + 8;
    const int16_t *qrow = jd.qprof + (size_t)base * qstride;
    const int g0 = beg >> 3, g1 = end >> 3;
    const int pj = ((j >> 3) - g0) >> 5;                              /* j's pass */
    const int p_lo = max(0, pj - max(fx.buf_cells >> 8, 1) + 1);      /* first pass kept in the buffer */
    const int lo = (g0 + 32 * p_lo) * 8;
    int carry1 = 2 * NEG, carry2 = 2 * NEG;
    unsigned lh = 0u, lf1 = 0u, lf2 = 0u;
    for (int p = 0; p <= pj; ++p) {
        const int gp = g0 + 32 * p, g = gp + lane;
        const bool active = g <= g1;
        uint4 sv = make_uint4(0u, 0u, 0u, 0u);
        if (active) sv = *reinterpret_cast<const uint4 *>(qrow + (size_t)g * 8);
        unsigned M[4], X1[4], X2[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { M[k] = NEGP2; X1[k] = NEGP2; X2[k] = NEGP2; }
        const bool fix_left = (gp > g0) || ((beg & 7) == 0);
        for (int kb = 0; kb < np; kb += 32) {
            int c_g0 = 0, c_ng = 0, c_ps = 0; uint32_t c_off = 0;      /* predecessor kb + lane: first group, groups, path score, slab offset */
            if (kb + lane < np) {
                const int prow = ldb(jv.pred + pb + kb + lane);
                const PoaRowInfo pi = jd.rowinfo[prow];
                c_g0 = pi.beg >> 3; c_ng = (pi.end >> 3) - c_g0 + 1; c_off = jd.rowoff[prow].off;
                if (PS) c_ps = ldb(jv.predscore + pb + kb + lane);
            }
            const int nk = min(32, np - kb);
            for (int k = 0; k < nk; ++k) {
                const int pg0 = __shfl_sync(FULL, c_g0, k), png = __shfl_sync(FULL, c_ng, k);
                const uint32_t off = __shfl_sync(FULL, c_off, k);
                const int16_t *ph = planes + (size_t)off * POA_GROUP;
                const size_t pp = (size_t)png * POA_GROUP;
                const int rel = g - pg0;
                uint4 hp = make_uint4(NEGP2, NEGP2, NEGP2, NEGP2), ep1 = hp, ep2 = hp;
                if (active && (unsigned)rel < (unsigned)png) {
                    const int16_t *q = ph + (size_t)rel * POA_GROUP;
                    hp = *reinterpret_cast<const uint4 *>(q);
                    if (GAP != LG) ep1 = *reinterpret_cast<const uint4 *>(q + (size_t)Planes<GAP>::E1 * pp);
                    if (GAP == CG) ep2 = *reinterpret_cast<const uint4 *>(q + (size_t)Planes<GAP>::E2 * pp);
                }
                unsigned prev = __shfl_up_sync(FULL, hp.w, 1);
                if (lane == 0) {
                    int hm1 = NEGP;
                    if (fix_left && (unsigned)(rel - 1) < (unsigned)png) hm1 = (int)ph[(size_t)(rel - 1) * POA_GROUP + 7];
                    if (MODE == LOCAL && g == 0) hm1 = 0;
                    prev = (unsigned)hm1 << 16;
                }
                unsigned d0 = sh1(prev, hp.x), d1 = sh1(hp.x, hp.y), d2 = sh1(hp.y, hp.z), d3 = sh1(hp.z, hp.w);
                if (PS) {
                    const int ps = __shfl_sync(FULL, c_ps, k);
                    const unsigned ps2 = pk(ps, ps);
                    d0 = __viaddmax_s16x2(d0, ps2, NEGP2); d1 = __viaddmax_s16x2(d1, ps2, NEGP2);
                    d2 = __viaddmax_s16x2(d2, ps2, NEGP2); d3 = __viaddmax_s16x2(d3, ps2, NEGP2);
                    ep1.x = __viaddmax_s16x2(ep1.x, ps2, NEGP2); ep1.y = __viaddmax_s16x2(ep1.y, ps2, NEGP2);
                    ep1.z = __viaddmax_s16x2(ep1.z, ps2, NEGP2); ep1.w = __viaddmax_s16x2(ep1.w, ps2, NEGP2);
                    if (GAP == CG) {
                        ep2.x = __viaddmax_s16x2(ep2.x, ps2, NEGP2); ep2.y = __viaddmax_s16x2(ep2.y, ps2, NEGP2);
                        ep2.z = __viaddmax_s16x2(ep2.z, ps2, NEGP2); ep2.w = __viaddmax_s16x2(ep2.w, ps2, NEGP2);
                    }
                }
                M[0] = __vmaxs2(M[0], d0); M[1] = __vmaxs2(M[1], d1); M[2] = __vmaxs2(M[2], d2); M[3] = __vmaxs2(M[3], d3);
                X1[0] = __vmaxs2(X1[0], ep1.x); X1[1] = __vmaxs2(X1[1], ep1.y); X1[2] = __vmaxs2(X1[2], ep1.z); X1[3] = __vmaxs2(X1[3], ep1.w);
                if (GAP == CG) { X2[0] = __vmaxs2(X2[0], ep2.x); X2[1] = __vmaxs2(X2[1], ep2.y); X2[2] = __vmaxs2(X2[2], ep2.z); X2[3] = __vmaxs2(X2[3], ep2.w); }
            }
        }
        const int nlo = min(max(beg - g * 8, 0), 8), nhi = min(max(g * 8 + 7 - end, 0), 8);
        const uint4 clo = fx.cap_lo[nlo], chi = fx.cap_hi[nhi];
        const unsigned CLO[4] = { clo.x, clo.y, clo.z, clo.w };
        const unsigned CAP[4] = { __vmins2(clo.x, chi.x), __vmins2(clo.y, chi.y), __vmins2(clo.z, chi.z), __vmins2(clo.w, chi.w) };
        const unsigned S[4] = { sv.x, sv.y, sv.z, sv.w };
        unsigned H[4], F1[4], F2[4], E1o[4], E2o[4];
        p16_cells<GAP, MODE>(kc, CLO, CAP, S, M, X1, X2, (g - g0) * 8, e1, oe1, e2, oe2, zr2, lane, carry1, carry2, H, F1, F2, E1o, E2o);
        const uint2 bits = p16_fbits<GAP>(kc, H, F1, F2, CLO, CAP, g > g0, lane, p < pj, lh, lf1, lf2);
        if (p >= p_lo && active) *reinterpret_cast<uint2 *>(fx.buf + (g * 8 - lo)) = bits;
        if constexpr (DUMP) {
            if (p >= p_lo && active) {
                const FbDumpCtx &dx = static_cast<const FbDumpCtx &>(fx);
                int16_t *q = dx.f + (size_t)(g - g0) * POA_GROUP;
                *reinterpret_cast<uint4 *>(q) = make_uint4(F1[0], F1[1], F1[2], F1[3]);
                if (GAP == CG) *reinterpret_cast<uint4 *>(q + dx.fstride) = make_uint4(F2[0], F2[1], F2[2], F2[3]);
            }
        }
    }
    __syncwarp();
    return lo;
}

/* LGX rows of p16_run_job (see there).  xs: log2 of the storage granule, one reference vector of pn = 2^xs cells.
 * First / last stored group of a band [b, e] of a row stored in whole vectors of 2^xs cells */
__device__ __forceinline__ int p16_xg0(int xs, int b) { return ((b >> xs) << xs) >> 3; }
__device__ __forceinline__ int p16_xg1(int xs, int e) { return ((((e >> xs) + 1) << xs) - 1) >> 3; }
/* Predecessor p (band end p_end) feeds the cells j < p_vlim = ((p_end + 1) / pn + 1) * pn only: for group g all of its cells or
 * none, as p_vlim is a multiple of 8.  For the first predecessor the backtrace shortcut bits (D0) also need j - 1 <= p_end: the
 * general step takes a diagonal from a cell of the predecessor's band only, never from a leaked cell. */
__device__ __forceinline__ void p16_lgx_reach(const uint4 *cap_hi, int xs, int g, int p_end, bool first, unsigned &d0, unsigned &d1, unsigned &d2,
                                              unsigned &d3, uint4 &hp, unsigned (&D0)[4]) {
    if (first) {
        const uint4 c = cap_hi[min(max(g * 8 + 7 - (p_end + 1), 0), 8)];
        D0[0] = __vmins2(d0, c.x); D0[1] = __vmins2(d1, c.y); D0[2] = __vmins2(d2, c.z); D0[3] = __vmins2(d3, c.w);
    }
    if (g >= (((((p_end + 1) >> xs) + 1) << xs) >> 3)) { d0 = d1 = d2 = d3 = NEGP2; hp = make_uint4(NEGP2, NEGP2, NEGP2, NEGP2); }
}

/* One alignment job on one warp: forward DP + backtrace.  Writes *jd.result (every status) but does
 * NOT publish completion -- the caller does (signal_done), after whatever it still has to move. */
/* LEAN (whole-graph jobs without -G path scores): rows with one or two predecessors that are still in the
 * shared-memory ring -- practically every row -- take a straight-line path: every lane reads the predecessors'
 * ring records itself (uniform-address shared loads) instead of lane k owning predecessor k and publishing it
 * through reductions and shuffles, and the predecessor planes are folded in without a loop. */
/* TMA (with LEAN): the finished row is staged with ALL its planes in the row's ring slot and drained to HBM by the
 * bulk-copy engine (cp.async.bulk shared -> global, one copy per plane, issued by one lane) instead of five 16-byte
 * stores per lane; a slot is reused ring_rows rows later, after cp.async.bulk.wait_group.read says the engine has
 * finished reading it.  Rows wider than a ring slot keep the plain stores. */
/* FB: the compact row layout (RowLayout): no F planes; the backtrace recomputes them where it needs them (fb_recompute). */
/* PS (with LEAN; the chain's -G jobs): the job carries path scores.  The straight-line rows add predecessor k's score to its
 * diagonal term and its E planes (linear gaps: to H before - e1), the arithmetic of the general rows, with the scores of the
 * row's first LP predecessors broadcast one row ahead next to their rows.  Without PS a LEAN job carries none. */
/* LGX (with LEAN; the chain's linear-gap jobs, which are always banded: poa_chain_eligible refuses wb < 0): the rows follow
 * the reference's vector procedure, as the "lgx" rows of
 * poa_align_kernel do: a row is stored in whole pn-lane vectors around its band (groups p16_xg0 .. p16_xg1), the cells
 * end+1 .. xend keep the running value H[end] - k*e1, predecessor p feeds the cells j < p_vlim only (p16_lgx_reach), and
 * beyond vector V1 = max_p(p.end / pn) + 1 only the even lanes of vector V1 + 1 keep the running value.  In packed form T is
 * masked on both sides of the band and the stored H by CLO and the group's vector rule (KEEP).  The band (beg / end), the row
 * maximum and the cell count stay those of the band itself. */
template <int GAP, int MODE, bool LEAN = false, bool TMA = false, bool FB = false, bool PS = false, bool LGX = false>
__device__ __forceinline__ void p16_run_job(const PoaJobDesc &jd, const PoaParamsDev *__restrict__ prm, const P16Consts &kc, const P16Smem &sm,
                                            int ring_rows, int ring_cells, int lane) {
    static_assert(!(TMA && FB), "the TMA row drain stages the five-plane layout");
    static_assert(!LGX || (GAP == LG && MODE == GLOBAL && LEAN && !TMA), "lgx rows: linear gaps, global mode, the chain's job function");
    typedef int16_t ST;
    typedef Planes<GAP> PL;
    typedef RowLayout<GAP, FB> RL;
    constexpr int RN = RingPlanes<GAP>::N;
    int *mat_s = sm.mat_s; uint4 *cap_lo = sm.cap_lo, *cap_hi = sm.cap_hi, *ring_meta = sm.ring_meta; ST *ring_data = sm.ring_data;
    const int rmask = ring_rows - 1, ring_groups = ring_cells >> 3;
    const long long clk0 = clock64();
    uint64_t t_start_ns; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start_ns));
    const int m = prm->m;
    const JobView jv = open_job(jd.blob);
    ST *planes = reinterpret_cast<ST *>(jd.planes);
    PoaRowInfo *rowinfo = jd.rowinfo; PoaRowOff *rowoff = jd.rowoff;
    const int qlen = jv.qlen, n_rows = jv.n_rows, w = jv.w;
    const bool banded = w >= 0;
    const int e1 = prm->e1, o1 = prm->o1, oe1 = prm->oe1, e2 = prm->e2, o2 = prm->o2, oe2 = prm->oe2;
    const int pnv = jv.pn;
    const unsigned zr2 = (unsigned)prm->zero;     /* run-time packed zero (see the RELU note in poa_align_kernel) */

    PoaResultDev res;
    res.status = POA_ST_OK; res.best_score = NEG; res.best_i = 0; res.best_j = 0; res.n_ops = 0;
    res.start_i = res.start_j = 0; res.n_aln_bases = res.n_matched_bases = 0; res.max_band = 0; res.cells = 0; res.plane_units_used = 0;
    res.fwd_clk = 0; res.bt_clk = 0; res.t_start_ns = t_start_ns; res.t_end_ns = 0;

    /* ---- query profile: qp[r][j] = mat[r][query[j-1]], qp[r][0] = 0 (reference :533-539) ---- */
    int16_t *qp = jd.qprof;
    const int qstride = ((qlen + 1 + 7) & ~7) + 8;
    for (int r = 0; r < m; ++r)
        for (int j = lane; j < qstride; j += 32)
            qp[(size_t)r * qstride + j] = (j == 0 || j > qlen) ? (int16_t)0 : (int16_t)mat_s[r * m + jv.qs[j]];
    __syncwarp();

    uint64_t cursor = 0;
    int64_t cells = 0; int max_band = 0;
    int best_score = NEG, best_i = 0, best_j = 0, best_row = 0;
    int guard_lo = 0, guard_hi = 0;
    bool stop = false;

    /* ---------------- row 0 ---------------- */
    if constexpr (LGX) {                                     /* stored up to the end of end0's vector; cells past end0 are -inf */
        const int xs = pnv == 16 ? 4 : 3;
        int end0 = qlen;
        if (banded) end0 = min(qlen, max(0, qlen - jv.remain(0)) + w);
        const int g1 = p16_xg1(xs, end0), ngrp = g1 + 1;
        if ((uint64_t)RL::units(ngrp) > jd.plane_cap_units) { if (lane == 0) { res.status = POA_ST_PLANE_OVF; *jd.result = res; } return; }
        for (int gp = 0; gp <= g1; gp += 32) {
            const int g = gp + lane;
            if (g <= g1) {
                int h[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) { const int j = g * 8 + c; h[c] = j > end0 ? NEGP : max(-e1 * j, NEGP); }
                st8(planes + (size_t)g * POA_GROUP, h);
                if (g < ring_groups) st8(ring_data + (size_t)g * POA_GROUP, h);
            }
        }
        if (lane == 0) {
            PoaRowInfo r0; r0.beg = 0; r0.end = end0; r0.left = 0; r0.right = 0;
            rowinfo[0] = r0; { PoaRowOff z; z.off = 0; z.p0 = -1; rowoff[0] = z; } ring_meta[0] = make_uint4(0u, (unsigned)end0, 1u | (1u << 16), 0u);
        }
        cursor = RL::units(ngrp);
        cells += end0 + 1; max_band = end0 + 1;
        __syncwarp();
    } else {
        int end0 = qlen;
        if (banded) end0 = min(qlen, max(0, qlen - jv.remain(0)) + w);
        const int g1 = end0 >> 3, ngrp = g1 + 1;
        if ((uint64_t)RL::units(ngrp) > jd.plane_cap_units) { if (lane == 0) { res.status = POA_ST_PLANE_OVF; *jd.result = res; } return; }
        for (int gp = 0; gp <= g1; gp += 32) {
            const int g = gp + lane;
            if (g <= g1) {
                int h[8], ea[8], eb[8], fa[8], fb[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int j = g * 8 + c;
                    if (MODE == LOCAL) { h[c] = ea[c] = eb[c] = fa[c] = fb[c] = (j <= end0) ? 0 : NEGP; }
                    else if (j > end0) { h[c] = ea[c] = eb[c] = fa[c] = fb[c] = NEGP; }
                    else if (GAP == LG) { h[c] = max(-e1 * j, NEGP); }
                    else if (j == 0) { h[c] = 0; ea[c] = -oe1; eb[c] = -oe2; fa[c] = fb[c] = NEGP; }
                    else {
                        fa[c] = max(-o1 - e1 * j, NEGP); fb[c] = max(-o2 - e2 * j, NEGP); ea[c] = eb[c] = NEGP;
                        h[c] = (GAP == CG) ? max(fa[c], fb[c]) : fa[c];
                    }
                }
                ST *rp = planes + (size_t)g * POA_GROUP;
                st8(rp, h);
                if (GAP != LG) st8(rp + (size_t)PL::E1 * ngrp * POA_GROUP, ea);
                if (GAP == CG) st8(rp + (size_t)PL::E2 * ngrp * POA_GROUP, eb);
                if (!FB && GAP != LG) st8(rp + (size_t)PL::F1 * ngrp * POA_GROUP, fa);
                if (!FB && GAP == CG) st8(rp + (size_t)PL::F2 * ngrp * POA_GROUP, fb);
                if (g < ring_groups) {
                    ST *rq = ring_data + (size_t)g * POA_GROUP;
                    st8(rq, h);
                    if (GAP != LG) st8(rq + ring_cells, ea);
                    if (GAP == CG) st8(rq + 2 * ring_cells, eb);
                }
            }
        }
        if (lane == 0) {
            PoaRowInfo r0; r0.beg = 0; r0.end = end0; r0.left = 0; r0.right = 0;
            rowinfo[0] = r0; { PoaRowOff z; z.off = 0; z.p0 = -1; rowoff[0] = z; } ring_meta[0] = make_uint4(0u, (unsigned)end0, 1u | (1u << 16), 0u);
        }
        cursor = RL::units(ngrp);
        cells += end0 + 1; max_band = end0 + 1;
        __syncwarp();
    }

    /* ---------------- rows 1 .. n_rows-2 ----------------
     * Lean row loop: per-row graph metadata arrives one row ahead as a single 8-byte load; lane k
     * owns predecessor k and publishes what the other lanes need about it in two packed words
     * (two shuffles per predecessor); the ring is addressed with 32-bit shared-memory offsets. */
    const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring_data);
    constexpr int RS = TMA ? PL::N : RN;                  /* planes kept per ring row: what successors read, or (TMA) everything */
    const uint32_t ring_row_bytes = (uint32_t)(RS * ring_cells * 2), ring_plane_bytes = (uint32_t)(ring_cells * 2);
    const int pn_shift = pnv == 16 ? 4 : 3;
    const uint32_t cap32 = jd.plane_cap_units > 0xffffffffull ? 0xffffffffu : (uint32_t)jd.plane_cap_units;
    uint32_t cur32 = (uint32_t)cursor;
    const bool has_ps = LEAN ? PS : (jv.predscore != nullptr);

    /* Graph metadata runs one full row ahead of its use: what iteration i loads (row i+1's list end, residue / band centre
     * and -- unconditionally, clamped to the list -- its per-lane predecessor entries) is first touched at the top of
     * iteration i+1.  (ncu: with the loads consumed in the same iteration -- the list length as the predicate of the
     * predecessor load, the loaded predecessors by the LEAN broadcast -- 10 % of all stall samples sat on these two.) */
    const int npred_tot = ldb(&jv.rowmeta[n_rows].x);
    int pb = 0, pe = 0, rbase = 0, rem = 0, raw_pred = -1, raw_ps = 0;
    if (n_rows > 2) {
        { const int2 m1 = ldb(jv.rowmeta + 1); pb = m1.x; pe = jv.predoff(2); rbase = m1.y & 0xff; rem = m1.y >> 8; }
        { const int k = max(min(pb + lane, npred_tot - 1), 0); raw_pred = ldb(jv.pred + k); if (has_ps) raw_ps = ldb(jv.predscore + k); }
    }
    int nx_y = n_rows > 3 ? ldb(&jv.rowmeta[2].y) : 0;          /* packed (remain, residue) of row i+1 */
    constexpr int LP = 4;                                     /* LEAN: up to LP predecessors per row on the straight-line path (> 2: 14 % of the rows at 10 kbp x 50) */
    int lp_c[LP], lps_c[LP];                                  /* the coming row's first LP predecessors (and -G scores), broadcast off the row-to-row chain */
#pragma unroll
    for (int k = 0; k < LP; ++k) {
        lp_c[k] = LEAN ? __shfl_sync(FULL, lane < pe - pb ? raw_pred : -1, k) : -1;
        lps_c[k] = PS ? __shfl_sync(FULL, lane < pe - pb ? raw_ps : 0, k) : 0;
    }
    KP_DECL
    for (int i = 1; i < n_rows - 1 && !stop; ++i) {
        KP(5)
        const int np = pe - pb;
        const int mypred = lane < np ? raw_pred : -1, myps = lane < np ? raw_ps : 0;
        int lp[LP], lps[LP];                                  /* the row's first LP predecessors and scores, known to every lane (broadcast at the end of the previous iteration) */
#pragma unroll
        for (int k = 0; k < LP; ++k) { lp[k] = lp_c[k]; lps[k] = lps_c[k]; }
        /* unconditional: rowmeta has n_rows + 1 entries and i + 2 <= n_rows; the predecessor index is clamped (a predicated
         * load would need a select on its result, which the compiler schedules right behind the load) */
        int2 m2;                                              /* two 32-bit loads: a 64-bit one ties up an aligned register pair that ptxas frees by
                                                                 copying the result out right behind the load, i.e. by waiting for it */
        m2.x = ldb(&jv.rowmeta[i + 2].x); m2.y = ldb(&jv.rowmeta[i + 2].y);
        const int n_rbase = nx_y & 0xff, n_rem = nx_y >> 8;
        int n_raw_pred, n_raw_ps = 0;
        { const int k = max(min(pe + lane, npred_tot - 1), 0); n_raw_pred = ldb(jv.pred + k); if (has_ps) n_raw_ps = ldb(jv.predscore + k); }
        if (LEAN || !(jv.live && !ldb(jv.live + i))) {

        /* ---- LEAN fast row: <= 2 predecessors, all in the ring, their whole bands cached there ---- */
        bool lean_row = false;
        uint4 lm[LP];
#pragma unroll
        for (int k = 0; k < LP; ++k) lm[k] = make_uint4(0u, 0u, 0u, 0u);
        if (LEAN) {
            lean_row = np >= 1 && np <= LP;
#pragma unroll
            for (int k = 0; k < LP; ++k) if (k < np && (i - lp[k]) > rmask) lean_row = false;       /* every predecessor still in the ring */
#ifdef POA_KPROF
            if (!lean_row) { if (np > LP || np < 1) ++kdiag[1]; else ++kdiag[2]; }
#endif
            if (lean_row) {
                lm[0] = ring_meta[lp[0] & rmask];
                int wide = (int)(lm[0].y >> 3) - (int)(lm[0].x >> 3) + 1;
                if constexpr (LGX) wide = p16_xg1(pn_shift, (int)lm[0].y) - p16_xg0(pn_shift, (int)lm[0].x) + 1;
#pragma unroll
                for (int k = 1; k < LP; ++k) {
                    lm[k] = k < np ? ring_meta[lp[k] & rmask] : lm[0];
                    if constexpr (LGX) wide = max(wide, p16_xg1(pn_shift, (int)lm[k].y) - p16_xg0(pn_shift, (int)lm[k].x) + 1);
                    else wide = max(wide, (int)(lm[k].y >> 3) - (int)(lm[k].x >> 3) + 1);
                }
                if (wide > ring_groups) lean_row = false;            /* a row wider than its ring slot: only a prefix is cached */
#ifdef POA_KPROF
                if (lean_row) ++kdiag[0]; else ++kdiag[3];
#endif
            }
        }
        /* ---- predecessor k on lane k: band hints + the two broadcast words ---- */
        unsigned wA = 0, wB = 0;                      /* A: pg0 | png<<12 | near<<25 | slot<<26 ; B: plane offset (8-cell units) */
        int l1 = INT32_MAX, r1 = INT32_MIN, b1 = INT32_MAX;
        int e1x = -1;                                 /* LGX: the predecessor's band end (its reach) */
        if (!lean_row && lane < np) {
            const int prow = mypred;
            const bool near = (i - prow) <= rmask;
            uint4 mi;
            if (near) mi = ring_meta[prow & rmask];
            else { const PoaRowInfo pi = rowinfo[prow]; mi = make_uint4((unsigned)pi.beg, (unsigned)pi.end, (unsigned)(pi.left + 1) | ((unsigned)(pi.right + 1) << 16), rowoff[prow].off); }
            l1 = (int)(mi.z & 0xffffu); r1 = (int)(mi.z >> 16); b1 = (int)mi.x;
            const unsigned pg0 = mi.x >> 3, png = (mi.y >> 3) - pg0 + 1;
            wA = pg0 | (png << 12) | ((unsigned)near << 25) | ((unsigned)(prow & rmask) << 26);
            if constexpr (LGX) {
                e1x = (int)mi.y;
                const unsigned xg0 = (unsigned)p16_xg0(pn_shift, (int)mi.x), xng = (unsigned)p16_xg1(pn_shift, (int)mi.y) - xg0 + 1;
                wA = xg0 | (xng << 12) | ((unsigned)near << 25) | ((unsigned)(prow & rmask) << 26);
            }
            wB = mi.w;
        }
        int ml = jv.node_n, mr = 0, min_pre_beg = INT32_MAX;
        int max_pre_end = -1;                         /* LGX */
        if (lean_row) {
#pragma unroll
            for (int k = 0; k < LP; ++k) {                   /* lm[k >= np] repeats lm[0]: harmless for min / max */
                ml = min(ml, (int)(lm[k].z & 0xffffu)); mr = max(mr, (int)(lm[k].z >> 16)); min_pre_beg = min(min_pre_beg, (int)lm[k].x);
                if constexpr (LGX) max_pre_end = max(max_pre_end, (int)lm[k].y);
            }
        } else if (banded) {
            ml = min(ml, __reduce_min_sync(FULL, l1));
            mr = max(mr, __reduce_max_sync(FULL, r1));
            min_pre_beg = __reduce_min_sync(FULL, b1);
            if constexpr (LGX) max_pre_end = __reduce_max_sync(FULL, e1x);
            for (int kb = 32; kb < np; kb += 32) {          /* more than 32 predecessors: practically never */
                const int k = kb + lane;
                int l2 = INT32_MAX, r2 = INT32_MIN, b2 = INT32_MAX;
                if (k < np) { const PoaRowInfo pi = rowinfo[ldb(jv.pred + pb + k)]; l2 = pi.left + 1; r2 = pi.right + 1; b2 = pi.beg; }
                ml = min(ml, __reduce_min_sync(FULL, l2)); mr = max(mr, __reduce_max_sync(FULL, r2)); min_pre_beg = min(min_pre_beg, __reduce_min_sync(FULL, b2));
                if constexpr (LGX) {
                    const int e2x = k < np ? rowinfo[ldb(jv.pred + pb + k)].end : -1;
                    max_pre_end = max(max_pre_end, __reduce_max_sync(FULL, e2x));
                }
            }
        }
        int beg = 0, end = qlen;
        if (banded) {
            const int r = qlen - rem;
            beg = max(0, min(ml, r) - w);
            end = min(qlen, max(mr, r) + w);
            if (np > 0 && (beg >> pn_shift) < (min_pre_beg >> pn_shift)) beg = min_pre_beg;   /* reference's vector-granular clamp */
        }
        int g0 = beg >> 3, g1 = end >> 3;
        if constexpr (LGX) { g0 = p16_xg0(pn_shift, beg); g1 = p16_xg1(pn_shift, end); }
        const int ngrp = g1 - g0 + 1;
        const uint32_t need = RL::units((uint32_t)ngrp);
        if (need > cap32 - cur32) {
            if (TMA) { if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); __syncwarp(); }     /* nothing may still read this CTA's smem */
            if (lane == 0) { res.status = POA_ST_PLANE_OVF; res.plane_units_used = cur32; *jd.result = res; }
            return;
        }
        const bool tma_row = TMA && ngrp <= ring_groups;
        const uint32_t my_off = cur32;
        cur32 += need;
        ST *rowp = planes + (size_t)my_off * POA_GROUP;
        const size_t gplane = (size_t)ngrp * POA_GROUP;                 /* elements between planes in HBM */
        const uint32_t my_ring_s = ring_s + (uint32_t)(i & rmask) * ring_row_bytes;
        cells += (end >= beg) ? (end - beg + 1) : 0;
        max_band = max(max_band, end - beg + 1);
        const int16_t *qrow = qp + (size_t)rbase * qstride;
        /* The query profile of a job (m x qlen x 2 B, ~100 KB at 10 kbp) does not stay in L1 with several jobs per SM, so a
         * row's 16-byte profile load used to be an L2 round trip on the row-to-row chain (ncu: long-scoreboard stall 1.7 per
         * issue).  The NEXT row's residue is known already: pull its profile lines into L1 one row ahead.  Its band starts at
         * this row's g0 or one group later, which the 16-byte-per-lane footprint plus one extra line covers. */
        if (i + 1 < n_rows - 1) {
            const int16_t *nrow = qp + (size_t)n_rbase * qstride;
            const int c0 = min((g0 + lane) * 8, qstride - 8);
            asm volatile("prefetch.global.L1 [%0];" :: "l"(nrow + c0));
            if (lane >= 24) asm volatile("prefetch.global.L1 [%0];" :: "l"(nrow + min(c0 + 64, qstride - 8)));
        }

        int carry1 = 2 * NEG, carry2 = 2 * NEG;
        int row_max = NEG, row_left = -1, row_right = -1;
        KP(0)

        for (int gp = g0; gp <= g1; gp += 32) {
            const int g = gp + lane;
            const bool active = g <= g1;
            uint4 sv = make_uint4(0u, 0u, 0u, 0u);
            if (active) sv = *reinterpret_cast<const uint4 *>(qrow + (size_t)g * 8);
            unsigned M[4], X1[4], X2[4];
            unsigned D0[4];                                   /* diagonal term of the FIRST predecessor alone (backtrace shortcut bits) */
#pragma unroll
            for (int k = 0; k < 4; ++k) { M[k] = NEGP2; X1[k] = NEGP2; X2[k] = NEGP2; D0[k] = NEGP2; }
            /* lane 0's left neighbour (cell 8g-1) lives in the previous group: only needed when that
             * cell is inside the band, i.e. on later passes or when the band starts on a group boundary */
            const bool fix_left = (gp > g0) || ((beg & 7) == 0);

            if (lean_row) {
#pragma unroll
                for (int k = 0; k < LP; ++k) {
                    if (k >= np) break;
                    const uint4 mi = lm[k];
                    int pg0 = (int)(mi.x >> 3), png = (int)(mi.y >> 3) - pg0 + 1;
                    if constexpr (LGX) { pg0 = p16_xg0(pn_shift, (int)mi.x); png = p16_xg1(pn_shift, (int)mi.y) - pg0 + 1; }
                    const int rel = g - pg0;
                    const bool inr = active && (unsigned)rel < (unsigned)png;
                    const uint32_t prs = ring_s + (uint32_t)(lp[k] & rmask) * ring_row_bytes;
                    uint4 hp = make_uint4(NEGP2, NEGP2, NEGP2, NEGP2), ep1 = hp, ep2 = hp;
                    if (inr) {
                        const uint32_t a = prs + (uint32_t)rel * 16u;
                        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(hp.x), "=r"(hp.y), "=r"(hp.z), "=r"(hp.w) : "r"(a));
                        if (GAP != LG) asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(ep1.x), "=r"(ep1.y), "=r"(ep1.z), "=r"(ep1.w) : "r"(a + ring_plane_bytes));
                        if (GAP == CG) asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(ep2.x), "=r"(ep2.y), "=r"(ep2.z), "=r"(ep2.w) : "r"(a + 2 * ring_plane_bytes));
                    }
                    unsigned prev = __shfl_up_sync(FULL, hp.w, 1);
                    if (fix_left) {                          /* uniform: the cell left of lane 0's group is inside the band */
                        if (lane == 0) {
                            int hm1 = NEGP;
                            const int relm = rel - 1;
                            if ((unsigned)relm < (unsigned)png) { unsigned short v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(prs + (uint32_t)relm * 16u + 14u)); hm1 = (int)(short)v; }
                            if (MODE == LOCAL && g == 0) hm1 = 0;
                            prev = (unsigned)hm1 << 16;
                        }
                    } else if (lane == 0) prev = (MODE == LOCAL && g == 0) ? 0u : ((unsigned)NEGP << 16);
                    unsigned d0 = sh1(prev, hp.x), d1 = sh1(hp.x, hp.y), d2 = sh1(hp.y, hp.z), d3 = sh1(hp.z, hp.w);
                    if (PS) {
                        const unsigned ps2 = pk(lps[k], lps[k]);
                        d0 = __viaddmax_s16x2(d0, ps2, NEGP2); d1 = __viaddmax_s16x2(d1, ps2, NEGP2);
                        d2 = __viaddmax_s16x2(d2, ps2, NEGP2); d3 = __viaddmax_s16x2(d3, ps2, NEGP2);
                        if (GAP == LG) {
                            hp.x = __viaddmax_s16x2(hp.x, ps2, NEGP2); hp.y = __viaddmax_s16x2(hp.y, ps2, NEGP2);
                            hp.z = __viaddmax_s16x2(hp.z, ps2, NEGP2); hp.w = __viaddmax_s16x2(hp.w, ps2, NEGP2);
                        } else {
                            ep1.x = __viaddmax_s16x2(ep1.x, ps2, NEGP2); ep1.y = __viaddmax_s16x2(ep1.y, ps2, NEGP2);
                            ep1.z = __viaddmax_s16x2(ep1.z, ps2, NEGP2); ep1.w = __viaddmax_s16x2(ep1.w, ps2, NEGP2);
                            if (GAP == CG) {
                                ep2.x = __viaddmax_s16x2(ep2.x, ps2, NEGP2); ep2.y = __viaddmax_s16x2(ep2.y, ps2, NEGP2);
                                ep2.z = __viaddmax_s16x2(ep2.z, ps2, NEGP2); ep2.w = __viaddmax_s16x2(ep2.w, ps2, NEGP2);
                            }
                        }
                    }
                    if (GAP == LG) {
                        hp.x = __viaddmax_s16x2(hp.x, kc.NE1, NEGP2); hp.y = __viaddmax_s16x2(hp.y, kc.NE1, NEGP2); hp.z = __viaddmax_s16x2(hp.z, kc.NE1, NEGP2); hp.w = __viaddmax_s16x2(hp.w, kc.NE1, NEGP2);
                    }
                    if constexpr (LGX) p16_lgx_reach(cap_hi, pn_shift, g, (int)mi.y, k == 0, d0, d1, d2, d3, hp, D0);
                    const uint4 x1 = GAP == LG ? hp : ep1;
                    if (k == 0) {
                        if constexpr (!LGX) { D0[0] = d0; D0[1] = d1; D0[2] = d2; D0[3] = d3; }
                        M[0] = d0; M[1] = d1; M[2] = d2; M[3] = d3;
                        X1[0] = x1.x; X1[1] = x1.y; X1[2] = x1.z; X1[3] = x1.w;
                        if (GAP == CG) { X2[0] = ep2.x; X2[1] = ep2.y; X2[2] = ep2.z; X2[3] = ep2.w; }
                    } else {
                        M[0] = __vmaxs2(M[0], d0); M[1] = __vmaxs2(M[1], d1); M[2] = __vmaxs2(M[2], d2); M[3] = __vmaxs2(M[3], d3);
                        X1[0] = __vmaxs2(X1[0], x1.x); X1[1] = __vmaxs2(X1[1], x1.y); X1[2] = __vmaxs2(X1[2], x1.z); X1[3] = __vmaxs2(X1[3], x1.w);
                        if (GAP == CG) { X2[0] = __vmaxs2(X2[0], ep2.x); X2[1] = __vmaxs2(X2[1], ep2.y); X2[2] = __vmaxs2(X2[2], ep2.z); X2[3] = __vmaxs2(X2[3], ep2.w); }
                    }
                }
            } else
            for (int kb = 0; kb < np; kb += 32) {
                unsigned cA = wA, cB = wB; int c_ps = myps;
                int c_end = e1x;
                if (kb > 0) {
                    const int k = kb + lane; cA = 0; cB = 0; c_ps = 0;
                    if (k < np) {
                        const int prow = ldb(jv.pred + pb + k); const PoaRowInfo pi = rowinfo[prow];
                        const unsigned pg0 = (unsigned)pi.beg >> 3, png = ((unsigned)pi.end >> 3) - pg0 + 1;
                        cA = pg0 | (png << 12); cB = rowoff[prow].off; if (has_ps) c_ps = ldb(jv.predscore + pb + k);
                        if constexpr (LGX) {
                            c_end = pi.end;
                            const unsigned xg0 = (unsigned)p16_xg0(pn_shift, pi.beg), xng = (unsigned)p16_xg1(pn_shift, pi.end) - xg0 + 1;
                            cA = xg0 | (xng << 12);
                        }
                    }
                }
                const int nk = min(32, np - kb);
                for (int k = 0; k < nk; ++k) {
                    const unsigned A = __shfl_sync(FULL, cA, k), B = __shfl_sync(FULL, cB, k);
                    const int pg0 = (int)(A & 0xfffu), png = (int)((A >> 12) & 0x1fffu);
                    const bool near = (A >> 25) & 1u;
                    const int rel = g - pg0;
                    const bool inr = active && (unsigned)rel < (unsigned)png;
                    uint4 hp = make_uint4(NEGP2, NEGP2, NEGP2, NEGP2), ep1 = hp, ep2 = hp;
                    const uint32_t prs = ring_s + (A >> 26) * ring_row_bytes;        /* predecessor's ring row */
                    const ST *ph = planes + (size_t)B * POA_GROUP;                     /* predecessor's HBM row  */
                    if (inr) {
                        if (near && rel < ring_groups) {
                            const uint32_t a = prs + (uint32_t)rel * 16u;
                            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(hp.x), "=r"(hp.y), "=r"(hp.z), "=r"(hp.w) : "r"(a));
                            if (GAP != LG) asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(ep1.x), "=r"(ep1.y), "=r"(ep1.z), "=r"(ep1.w) : "r"(a + ring_plane_bytes));
                            if (GAP == CG) asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(ep2.x), "=r"(ep2.y), "=r"(ep2.z), "=r"(ep2.w) : "r"(a + 2 * ring_plane_bytes));
                        } else {
                            const ST *q = ph + (size_t)rel * POA_GROUP;
                            const size_t pp = (size_t)png * POA_GROUP;
                            hp = *reinterpret_cast<const uint4 *>(q);
                            if (GAP != LG) ep1 = *reinterpret_cast<const uint4 *>(q + (size_t)PL::E1 * pp);
                            if (GAP == CG) ep2 = *reinterpret_cast<const uint4 *>(q + (size_t)PL::E2 * pp);
                        }
                    }
                    unsigned prev = __shfl_up_sync(FULL, hp.w, 1);
                    if (lane == 0) {
                        int hm1 = NEGP;
                        if (fix_left) {
                            const int relm = rel - 1;
                            if ((unsigned)relm < (unsigned)png) {
                                if (near && relm < ring_groups) { unsigned short v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(prs + (uint32_t)relm * 16u + 14u)); hm1 = (int)(short)v; }
                                else hm1 = (int)ph[(size_t)relm * POA_GROUP + 7];
                            }
                        }
                        if (MODE == LOCAL && g == 0) hm1 = 0;
                        prev = (unsigned)hm1 << 16;
                    }
                    unsigned d0 = sh1(prev, hp.x), d1 = sh1(hp.x, hp.y), d2 = sh1(hp.y, hp.z), d3 = sh1(hp.z, hp.w);
                    if (has_ps) {
                        const int ps = __shfl_sync(FULL, c_ps, k);
                        const unsigned ps2 = pk(ps, ps);
                        d0 = __viaddmax_s16x2(d0, ps2, NEGP2); d1 = __viaddmax_s16x2(d1, ps2, NEGP2);
                        d2 = __viaddmax_s16x2(d2, ps2, NEGP2); d3 = __viaddmax_s16x2(d3, ps2, NEGP2);
                        if (GAP == LG) {
                            hp.x = __viaddmax_s16x2(hp.x, ps2, NEGP2); hp.y = __viaddmax_s16x2(hp.y, ps2, NEGP2);
                            hp.z = __viaddmax_s16x2(hp.z, ps2, NEGP2); hp.w = __viaddmax_s16x2(hp.w, ps2, NEGP2);
                        } else {
                            ep1.x = __viaddmax_s16x2(ep1.x, ps2, NEGP2); ep1.y = __viaddmax_s16x2(ep1.y, ps2, NEGP2);
                            ep1.z = __viaddmax_s16x2(ep1.z, ps2, NEGP2); ep1.w = __viaddmax_s16x2(ep1.w, ps2, NEGP2);
                            if (GAP == CG) {
                                ep2.x = __viaddmax_s16x2(ep2.x, ps2, NEGP2); ep2.y = __viaddmax_s16x2(ep2.y, ps2, NEGP2);
                                ep2.z = __viaddmax_s16x2(ep2.z, ps2, NEGP2); ep2.w = __viaddmax_s16x2(ep2.w, ps2, NEGP2);
                            }
                        }
                    }
                    if constexpr (LGX) p16_lgx_reach(cap_hi, pn_shift, g, __shfl_sync(FULL, c_end, k), kb == 0 && k == 0, d0, d1, d2, d3, hp, D0);
                    else if (kb == 0 && k == 0) { D0[0] = d0; D0[1] = d1; D0[2] = d2; D0[3] = d3; }
                    M[0] = __vmaxs2(M[0], d0); M[1] = __vmaxs2(M[1], d1); M[2] = __vmaxs2(M[2], d2); M[3] = __vmaxs2(M[3], d3);
                    if (GAP == LG) {        /* vertical term H[p][j] - e1 */
                        X1[0] = __vmaxs2(X1[0], __viaddmax_s16x2(hp.x, kc.NE1, NEGP2)); X1[1] = __vmaxs2(X1[1], __viaddmax_s16x2(hp.y, kc.NE1, NEGP2));
                        X1[2] = __vmaxs2(X1[2], __viaddmax_s16x2(hp.z, kc.NE1, NEGP2)); X1[3] = __vmaxs2(X1[3], __viaddmax_s16x2(hp.w, kc.NE1, NEGP2));
                    } else {
                        X1[0] = __vmaxs2(X1[0], ep1.x); X1[1] = __vmaxs2(X1[1], ep1.y); X1[2] = __vmaxs2(X1[2], ep1.z); X1[3] = __vmaxs2(X1[3], ep1.w);
                        if (GAP == CG) { X2[0] = __vmaxs2(X2[0], ep2.x); X2[1] = __vmaxs2(X2[1], ep2.y); X2[2] = __vmaxs2(X2[2], ep2.z); X2[3] = __vmaxs2(X2[3], ep2.w); }
                    }
                }
            }

            KP(1)
            /* band-edge masks of this lane's 8 cells */
            const int nlo = min(max(beg - g * 8, 0), 8), nhi = min(max(g * 8 + 7 - end, 0), 8);
            const uint4 clo = cap_lo[nlo], chi = cap_hi[nhi];
            const unsigned CLO[4] = { clo.x, clo.y, clo.z, clo.w };
            const unsigned CAP[4] = { __vmins2(clo.x, chi.x), __vmins2(clo.y, chi.y), __vmins2(clo.z, chi.z), __vmins2(clo.w, chi.w) };
            const unsigned S[4] = { sv.x, sv.y, sv.z, sv.w };

            unsigned H[4], F1[4], F2[4], E1o[4], E2o[4];
            if constexpr (LGX) {                              /* T inside the band only; H stored from beg to the vector end by KEEP */
                const int v = (g * 8) >> pn_shift, v1 = (max_pre_end >> pn_shift) + 1;
                const unsigned keep = v <= v1 ? 0x7fff7fffu : (v == v1 + 1 ? 0x8AD07FFFu : NEGP2);      /* V1 + 1: the even lanes (low halves) */
                const unsigned HK[4] = { __vmins2(CLO[0], keep), __vmins2(CLO[1], keep), __vmins2(CLO[2], keep), __vmins2(CLO[3], keep) };
                p16_cells<GAP, MODE>(kc, CAP, HK, S, M, X1, X2, (g - g0) * 8, e1, oe1, e2, oe2, zr2, lane, carry1, carry2, H, F1, F2, E1o, E2o);
            } else
            p16_cells<GAP, MODE>(kc, CLO, CAP, S, M, X1, X2, (g - g0) * 8, e1, oe1, e2, oe2, zr2, lane, carry1, carry2, H, F1, F2, E1o, E2o);

            /* backtrace shortcut record (PoaBtRec): one bit per cell -- is H explained by the first predecessor's diagonal? */
            if (jd.btrec != nullptr) {
                unsigned t = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    t |= __vcmpeq2(__viaddmax_s16x2(D0[k], S[k], NEGP2), H[k]) & (0x00020001u << (2 * k));
                const unsigned byte = (t | (t >> 16)) & 0xffu;
                uint8_t *rec = reinterpret_cast<uint8_t *>(jd.btrec + i);
                const int rel = g - g0;
                if (active && rel < POA_BTREC_GROUPS) rec[16 + rel] = (uint8_t)byte;
                if (lane == 0 && gp == g0)
                    *reinterpret_cast<uint4 *>(rec) = make_uint4((unsigned)(g0 * 8), (unsigned)mypred,
                                                                 (unsigned)rbase | (ngrp <= POA_BTREC_GROUPS ? 0x100u : 0u) | ((unsigned)min(ngrp, 0xffff) << 16), (unsigned)my_off);
            }
            KP(2)
            if (TMA && tma_row) {
                if (gp == g0) {                              /* the slot's previous tenant (ring_rows rows ago) must have been read out */
                    if (lane == 0) { if (ring_rows >= 8) asm volatile("cp.async.bulk.wait_group.read 7;" ::: "memory"); else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
                    __syncwarp();
                }
                if (active) {
                    const uint32_t a = my_ring_s + (uint32_t)(g - g0) * 16u;
                    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a), "r"(H[0]), "r"(H[1]), "r"(H[2]), "r"(H[3]) : "memory");
                    if (GAP != LG) {
                        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + (uint32_t)PL::E1 * ring_plane_bytes), "r"(E1o[0]), "r"(E1o[1]), "r"(E1o[2]), "r"(E1o[3]) : "memory");
                        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + (uint32_t)PL::F1 * ring_plane_bytes), "r"(F1[0]), "r"(F1[1]), "r"(F1[2]), "r"(F1[3]) : "memory");
                    }
                    if (GAP == CG) {
                        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + (uint32_t)PL::E2 * ring_plane_bytes), "r"(E2o[0]), "r"(E2o[1]), "r"(E2o[2]), "r"(E2o[3]) : "memory");
                        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + (uint32_t)PL::F2 * ring_plane_bytes), "r"(F2[0]), "r"(F2[1]), "r"(F2[2]), "r"(F2[3]) : "memory");
                    }
                }
            } else
            if (active) {
                const int rel = g - g0;
                if (rel < ring_groups) {
                    const uint32_t a = my_ring_s + (uint32_t)rel * 16u;
                    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a), "r"(H[0]), "r"(H[1]), "r"(H[2]), "r"(H[3]) : "memory");
                    if (GAP != LG) asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + ring_plane_bytes), "r"(E1o[0]), "r"(E1o[1]), "r"(E1o[2]), "r"(E1o[3]) : "memory");
                    if (GAP == CG) asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a + 2 * ring_plane_bytes), "r"(E2o[0]), "r"(E2o[1]), "r"(E2o[2]), "r"(E2o[3]) : "memory");
                }
                ST *q = rowp + (size_t)rel * POA_GROUP;
                *reinterpret_cast<uint4 *>(q) = make_uint4(H[0], H[1], H[2], H[3]);
                if (GAP != LG) *reinterpret_cast<uint4 *>(q + (size_t)PL::E1 * gplane) = make_uint4(E1o[0], E1o[1], E1o[2], E1o[3]);
                if (GAP == CG) *reinterpret_cast<uint4 *>(q + (size_t)PL::E2 * gplane) = make_uint4(E2o[0], E2o[1], E2o[2], E2o[3]);
                if (!FB && GAP != LG) *reinterpret_cast<uint4 *>(q + (size_t)PL::F1 * gplane) = make_uint4(F1[0], F1[1], F1[2], F1[3]);
                if (!FB && GAP == CG) *reinterpret_cast<uint4 *>(q + (size_t)PL::F2 * gplane) = make_uint4(F2[0], F2[1], F2[2], F2[3]);
            }

            KP(3)
            if constexpr (LGX) {                              /* the row maximum is taken over the band, not the leaked cells */
#pragma unroll
                for (int k = 0; k < 4; ++k) H[k] = __vmins2(H[k], CAP[k]);
            }
            /* row maximum with first / last arg-max; masked cells hold NEGP and never win against a real cell */
            {
                const int lmax = active ? lane_max8(H) : NEGP;
                /* one bit per cell that equals the LANE's maximum: where the row maximum sits inside the lanes that hold it,
                 * computed while the warp-wide reduction is in flight */
                unsigned eq = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) { eq |= (unsigned)(lo16(H[k]) == lmax) << (2 * k); eq |= (unsigned)(hi16(H[k]) == lmax) << (2 * k + 1); }
                const int lfirst = g * 8 + __ffs(eq) - 1, llast = g * 8 + 31 - __clz(eq);
                const int pm = __reduce_max_sync(FULL, lmax);
                const unsigned bm = __ballot_sync(FULL, lmax == pm && pm > NEGP);
                if (bm) {
                    const int pl = __shfl_sync(FULL, lfirst, __ffs(bm) - 1);
                    const int pr = __shfl_sync(FULL, llast, 31 - __clz(bm));
                    if (pm > row_max) { row_max = pm; row_left = pl; row_right = pr; }
                    else if (pm == row_max) row_right = pr;
                }
            }
        }
        KP(4)
        if (TMA && tma_row) {                                /* drain the row: one bulk copy per plane, shared -> global */
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                const uint32_t bytes = (uint32_t)ngrp * 16u;
#pragma unroll
                for (int pl = 0; pl < PL::N; ++pl)
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                                 :: "l"(rowp + (size_t)pl * gplane), "r"(my_ring_s + (uint32_t)pl * ring_plane_bytes), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
        if (lane == 0) {
            ring_meta[i & rmask] = make_uint4((unsigned)beg, (unsigned)end, (unsigned)(row_left + 1) | ((unsigned)(row_right + 1) << 16), my_off);
            PoaRowInfo ri; ri.beg = beg; ri.end = end; ri.left = row_left; ri.right = row_right;
            rowinfo[i] = ri; { PoaRowOff z; z.off = my_off; z.p0 = mypred; *reinterpret_cast<uint2 *>(rowoff + i) = make_uint2(z.off, (unsigned)z.p0); }
        }
        guard_lo |= (row_max < -14000); guard_hi |= (row_max > 29000);
        if (MODE == LOCAL) {
            if (row_max > best_score) { best_score = row_max; best_i = i; best_j = row_left; }
        } else if (MODE == EXTEND) {
            if (row_max > best_score) { best_score = row_max; best_i = i; best_j = row_right; best_row = i; }
            else if (prm->zdrop > 0) {
                const int delta = jv.remain(best_row) - rem;
                if (best_score - row_max > prm->zdrop + e1 * abs(delta - (row_right - best_j))) stop = true;
            }
        }
        __syncwarp();
        }   /* live row */
        /* The compiler must not pull this rotation up to the loads at the top of the iteration (it did: the copy of m2.x then
         * waited for the load in the very iteration that issued it).  An empty volatile asm pins "first use" here, after the
         * row's volatile shared-memory stores, a whole row later. */
        asm volatile("" : "+r"(m2.x), "+r"(m2.y), "+r"(n_raw_pred), "+r"(n_raw_ps));
        pb = pe; pe = m2.x; rbase = n_rbase; rem = n_rem; nx_y = m2.y; raw_pred = n_raw_pred; raw_ps = n_raw_ps;
#pragma unroll
        for (int k = 0; k < LP; ++k) {
            lp_c[k] = LEAN ? __shfl_sync(FULL, lane < pe - pb ? raw_pred : -1, k) : -1;
            lps_c[k] = PS ? __shfl_sync(FULL, lane < pe - pb ? raw_ps : 0, k) : 0;
        }
    }
    cursor = cur32;
    KP_OUT(res)
    if (TMA) {                                               /* the end-cell lookup and the backtrace read the planes from HBM */
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        __syncwarp();
    }

    if (MODE == GLOBAL) {
        const int sb = jv.predoff(n_rows - 1), sn = jv.predoff(n_rows) - sb;
        for (int k = 0; k < sn; ++k) {
            const int prow = jv.pred[sb + k];
            const PoaRowInfo pi = rowinfo[prow];
            const int endc = qlen > pi.end ? pi.end : qlen;
            int pg0 = pi.beg >> 3;
            if constexpr (LGX) pg0 = p16_xg0(pn_shift, pi.beg);
            const int v = (endc >= pi.beg) ? (int)planes[(size_t)rowoff[prow].off * POA_GROUP + (endc - pg0 * 8)] : NEG;
            if (v > best_score) { best_score = v; best_i = prow; best_j = endc; }
        }
    }
    res.best_score = best_score; res.best_i = best_i; res.best_j = best_j;
    res.cells = cells; res.max_band = max_band; res.plane_units_used = cursor;
    /* Scores left the safe int16 window: redo in 32 bits.  Besides the row maxima, the widest band is
     * watched: beg/end follow min(ml, r) - w / max(mr, r) + w, so when the arg-max drifts away from the
     * remain-centre a row can be far wider than 2w and a cell far from the row's maximum could reach the
     * NEGP clamp without the maxima ever leaving [-14000, 29000]. */
    if (guard_lo || guard_hi || best_score <= NEGP + 2000) res.status = POA_ST_RANGE;
    if (banded && MODE != LOCAL && (int64_t)max_band * max(e1, e2) + max(oe1, oe2) > 15000) res.status = POA_ST_RANGE;
    const long long clk1 = clock64();
    res.fwd_clk = clk1 - clk0;
#ifndef POA_KPROF
    { unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid)); res.prof[5] = (int64_t)smid; }   /* which SM served the job (diagnostics) */
#endif
    if (lane == 0) *jd.result = res;
    __syncwarp();
    if (prm->ret_cigar && res.status == POA_ST_OK) {
        FbCtx fx;                                            /* FB: the ring is free now and holds the recomputed decision bytes */
        fx.kc = &kc; fx.cap_lo = cap_lo; fx.cap_hi = cap_hi;
        fx.buf = reinterpret_cast<uint8_t *>(ring_data); fx.buf_cells = (int)ring_row_bytes * ring_rows;
        if constexpr (LGX) poa_backtrack<GAP, ST, MODE, FB, PS>(jv, jd, prm, mat_s, lane, best_i, best_j, *jd.result, pn_shift, jd.btrec, &fx);
        else poa_backtrack<GAP, ST, MODE, FB, PS>(jv, jd, prm, mat_s, lane, best_i, best_j, *jd.result, 3, jd.btrec, &fx);
        if (lane == 0) jd.result->bt_clk = clock64() - clk1;
    }
}


/* POA_P16_MINB (build-time, experiments): minimum resident CTAs per SM the compiler must allow for, i.e. a
 * register cap of 65536 / (32 * POA_P16_MINB) per thread */
#ifndef POA_P16_MINB
#define POA_P16_MINB 10      /* register budget 65536 / (32 * 10) = 204 per thread: without a budget ptxas settles on 128 and spills */
#endif
#define POA_P16_BOUNDS __launch_bounds__(32, POA_P16_MINB)
template <int GAP, int MODE, bool LEAN, bool TMA>
__global__ void POA_P16_BOUNDS poa_align_kernel_p16(const PoaJobDesc *__restrict__ jobs, const PoaParamsDev *__restrict__ prm,
                                                           int n_jobs, int ring_rows, int ring_cells, const __grid_constant__ P16Consts kc) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const int lane = threadIdx.x;
    const int job = blockIdx.x;
    if (job >= n_jobs) return;
    const P16Smem sm = p16_smem_init(dyn_smem, prm, ring_rows, lane);
    const PoaJobDesc jd = jobs[job];
    p16_run_job<GAP, MODE, LEAN, TMA>(jd, prm, kc, sm, ring_rows, ring_cells, lane);
    __syncwarp();
    if (lane == 0) signal_done(jd);
}

static inline size_t ring_smem_bytes(int gap, int bits, int ring_rows, int ring_cells, int all_planes = 0);

/* ------------------------------------------------------------------ one read of a chain group
 * The job the fuse left in the slot (read sl->fused), on one warp.  STRAND (-s, PoaChainParams::amb_strand; the host
 * picks the instantiation, so a run without -s compiles to the bare job): a weak forward hit (chain_weak_hit) is aligned
 * again as the reverse complement, the reference's strand retry (src/abpoa_align.c:322-344).  The second pass writes the
 * complemented bases over the blob's query and runs into rc_cigar / rc_result; it may overwrite qs, qprof, rowinfo, rowoff
 * and btrec, which only the next flatten reads, and it rewrites them.  The reverse complement wins only if it scores
 * strictly more; its CIGAR words and result are then copied over the primary ones, so the fuse reads one place either
 * way.  The primary result carries the DP cells and cycles of both passes and the first status that is not OK (a failed
 * pair is re-run or handed back like a failed alignment); read_rc[r] records the strand (bit 0) and whether the retry
 * ran (bit 1).  PS (-G; the host picks the instantiation): the job blob carries path scores (p16_run_job).  EXT (extend
 * runs, -m 2; the host picks the instantiation): the EXTEND rows -- the same straight-line LEAN rows and compact layout,
 * then the best cell of the first row that holds the maximum and the z-drop stop (prm->zdrop); the job's rows follow the
 * reference's Kahn order (chain_fuse's KO). */
template <int GAP, bool STRAND, bool PS, bool EXT = false>
__device__ __forceinline__ void chain_align_read(const PoaJobDesc &jd, const PoaChainSlot *sl, const PoaChainParams *__restrict__ cp,
                                                 const PoaParamsDev *__restrict__ prm, const P16Consts &kc, const P16Smem &sm, int ring_rows, int ring_cells,
                                                 int lane) {
    PoaJobDesc jp = jd;
    bool second = false;
    for (int pass = 0; pass < (STRAND ? 2 : 1); ++pass) {
        p16_run_job<GAP, EXT ? EXTEND : GLOBAL, true, false, true, PS, GAP == LG && !EXT>(jp, prm, kc, sm, ring_rows, ring_cells, lane);
        __syncwarp();
        if (!STRAND || pass) break;
        const PoaJobHeader *h = reinterpret_cast<const PoaJobHeader *>(jd.blob);
        const int qlen = h->qlen;
        if (jd.result->status != POA_ST_OK || !chain_weak_hit(jd.result->best_score, qlen, h->n_rows, cp->max_mat)) break;
        const uint8_t *q = sl->reads + sl->read_off[sl->fused];
        uint8_t *qs = const_cast<uint8_t *>(jd.blob) + h->off_qs;
        for (int k = lane; k < qlen; k += 32) qs[1 + k] = chain_comp(q[qlen - 1 - k]);
        __syncwarp();
        jp.cigar = sl->rc_cigar; jp.result = sl->rc_result;
        second = true;
    }
    if (!STRAND) return;
    int rc = 0;
    if (second) {
        const PoaResultDev *f = jd.result, *b = sl->rc_result;
        rc = b->status == POA_ST_OK && b->best_score > f->best_score;
        if (rc) for (int t = lane; t < b->n_ops; t += 32) jd.cigar[t] = sl->rc_cigar[t];
        __syncwarp();
        if (lane == 0) {
            PoaResultDev out = rc ? *b : *f;
            out.status = f->status != POA_ST_OK ? f->status : b->status;
            out.cells = f->cells + b->cells; out.fwd_clk = f->fwd_clk + b->fwd_clk; out.bt_clk = f->bt_clk + b->bt_clk;
            *jd.result = out;
        }
    }
    if (lane == 0) sl->read_rc[sl->fused] = (uint8_t)(rc | (second ? 2 : 0));
    __syncwarp();
}

/* ------------------------------------------------------------------ chain engine entry
 * The same job function, fed from device-resident slots (poa_chain.cuh): the job blob of a slot is written
 * by the fuse kernel of the previous round, nothing comes from the host.  Block 0 also zeroes the plane-pool
 * cursor the coming fuse kernel will fill (see PoaChainSlot). */
template <int GAP, bool STRAND, bool PS, bool EXT = false>
__global__ void POA_P16_BOUNDS poa_chain_align_kernel_p16(const PoaChainSlot *__restrict__ slots, const int32_t *__restrict__ idx,
                                                           const PoaChainParams *__restrict__ cp, const PoaParamsDev *__restrict__ prm, int n_jobs,
                                                           int round, int ring_rows, int ring_cells, const __grid_constant__ P16Consts kc) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const int lane = threadIdx.x;
    const int job = blockIdx.x;
    if (job >= n_jobs) return;
    const PoaChainSlot *sl = &slots[idx[job]];
    if (job == 0 && lane == 0 && sl->pool_cursor) sl->pool_cursor[(round + 1) & 1] = 0ull;
    const PoaJobDesc jd = sl->jd;
    const int n_rows = reinterpret_cast<const PoaJobHeader *>(jd.blob)->n_rows;
    if (sl->failed || sl->fused >= sl->n_reads || n_rows < 3) { if (lane == 0) jd.result->status = POA_ST_SKIP; return; }
    const P16Smem sm = p16_smem_init(dyn_smem, prm, ring_rows, lane);
    chain_align_read<GAP, STRAND, PS, EXT>(jd, sl, cp, prm, kc, sm, ring_rows, ring_cells, lane);
}

/* Free-running chain (PoaChainSync in poa_chain.cuh): one resident warp per group runs the group's alignments back to
 * back.  Between two alignments the slot belongs to a fuse worker (poa_chain_fuse_worker_kernel); the hand-over is a
 * release store / relaxed poll + acquire fence pair on slot->turn, so nothing read here is stale in this SM's L1. */
__device__ __forceinline__ int chain_ld_relaxed(const int32_t *p) { int v; asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void chain_st_relaxed(int32_t *p, int v) { asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned long long chain_now_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

template <int GAP, bool STRAND, bool PS, bool EXT = false>
__global__ void POA_P16_BOUNDS poa_chain_dp_worker_kernel(PoaChainSlot *slots, PoaChainSync *sync, const PoaChainParams *__restrict__ cp,
                                                          const PoaParamsDev *__restrict__ prm, int n_groups, int ring_rows, int ring_cells, int dbg,
                                                          const __grid_constant__ P16Consts kc) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const int lane = threadIdx.x;
    const int g = blockIdx.x;
    if (g >= n_groups) return;
    PoaChainSlot *sl = &slots[g];
    const P16Smem sm = p16_smem_init(dyn_smem, prm, ring_rows, lane);
    const unsigned long long limit = sync->watchdog_ns;
    int pushed = 0;
    unsigned long long waited = 0;
    for (;;) {
        /* ---- wait for the slot.  The loop is warp-uniform on purpose (every lane polls, lane 0's view decides): a spin
         *      loop that only lane 0 runs left the warp in a state where every later warp-collective (SHFL / VOTE / REDUX) took
         *      its slow path -- measured 4x longer alignments.  Poll the slot's own word, gently (a fuse takes a millisecond
         *      or more; a thousand warps wait like this at once); the shared abort flag and the clock every 64th poll. ---- */
        int state = 0;                                         /* 0 go, 2 stop */
        {
            const unsigned long long t0 = chain_now_ns();
            unsigned ns = 500, polls = 0;
            for (;;) {
                const int v = __shfl_sync(0xffffffffu, chain_ld_relaxed(&sl->turn), 0);
                if (v == 0) break;
                __nanosleep(ns); if (ns < 8000) ns <<= 1;
                if ((++polls & 63u) == 0) {
                    const int a = __shfl_sync(0xffffffffu, chain_ld_relaxed(&sync->abort), 0);
                    const unsigned late = __shfl_sync(0xffffffffu, (unsigned)(chain_now_ns() - t0 > limit), 0);
                    if (a) { state = 2; break; }
                    if (late) { if (lane == 0) chain_st_relaxed(&sync->abort, 1); state = 2; break; }
                }
            }
            waited += chain_now_ns() - t0;
        }
        if (state) break;
        if (!(dbg & 1)) __threadfence();                       /* acquire side: also drops this SM's L1 lines of the slot / job blob */
        const PoaJobDesc jd = sl->jd;
        const int n_rows = reinterpret_cast<const PoaJobHeader *>(jd.blob)->n_rows;
        if (sl->failed || sl->fused >= sl->n_reads || n_rows < 3) break;
        chain_align_read<GAP, STRAND, PS, EXT>(jd, sl, cp, prm, kc, sm, ring_rows, ring_cells, lane);
        __syncwarp();
        if (!(dbg & 1)) __threadfence();                       /* release side: CIGAR + result are out before the task is */
        if (lane == 0) {
            chain_st_relaxed(&sl->turn, 1);
            const unsigned slot = atomicAdd(&sync->q_tail, 1u);
            chain_st_relaxed(&sync->tasks[slot], g);
        }
        ++pushed;
        __syncwarp();
    }
    /* the group is finished, failed or the run was aborted: fuse tasks it will never append leave the count */
    if (lane == 0) {
        const int never = sl->n_reads - 1 - pushed;
        if (never > 0) atomicSub(&sync->total, never);
        sl->wait_ns = waited;
    }
}

template <int GAP, bool STRAND, bool PS, bool EXT>
static cudaError_t launch_chain_worker_one(PoaChainSlot *slots, PoaChainSync *sync, int n_groups, const PoaChainParams *cp, const PoaParamsDev *prm,
                                           int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    /* at least 23 KB: at most 9 of these CTAs fit one SM, which leaves registers (9 x 160 x 32 of 64 K) and shared memory for a
     * 256-thread fuse worker next to them even if the alignment warps were dispatched first -- they wait for fuse workers */
    /* experiment hooks (timing only): ABPOA_GPU_CHAIN_DBG bit 0 = no fences (UNSAFE), bit 1 = no shared-memory padding; ABPOA_GPU_CHAIN_CARVEOUT */
    static const int dbg = [] { const char *e = getenv("ABPOA_GPU_CHAIN_DBG"); return e && *e ? atoi(e) : 0; }();
    const size_t smem0 = ring_smem_bytes(GAP, 16, ring_rows, ring_cells) + 18 * sizeof(uint4);
    const size_t smem = (dbg & 2) ? smem0 : std::max<size_t>(smem0, (size_t)23 * 1024);
    cudaError_t e = cudaFuncSetAttribute(poa_chain_dp_worker_kernel<GAP, STRAND, PS, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return e;
    /* the same L1/shared split as the fuse workers ask for (poa_chain.cu): CTAs of both kernels share SMs for the whole run */
    { const char *cv = getenv("ABPOA_GPU_CHAIN_CARVEOUT");
      e = cudaFuncSetAttribute(poa_chain_dp_worker_kernel<GAP, STRAND, PS, EXT>, cudaFuncAttributePreferredSharedMemoryCarveout, cv && *cv ? atoi(cv) : (int)cudaSharedmemCarveoutMaxShared);
      if (e != cudaSuccess) return e; }
    poa_chain_dp_worker_kernel<GAP, STRAND, PS, EXT><<<n_groups, 32, smem, st>>>(slots, sync, cp, prm, n_groups, ring_rows, ring_cells, dbg, kc);
    return cudaGetLastError();
}
template <bool STRAND, bool PS, bool EXT>
static cudaError_t launch_chain_worker_gap(int gap_mode, PoaChainSlot *slots, PoaChainSync *sync, int n_groups, const PoaChainParams *cp,
                                           const PoaParamsDev *prm, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    if constexpr (EXT) { if (gap_mode == LG) return cudaErrorInvalidValue; }          /* linear-gap extend: not on the chain */
    else if (gap_mode == LG) return launch_chain_worker_one<LG, STRAND, PS, false>(slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st);
    if (gap_mode == AG) return launch_chain_worker_one<AG, STRAND, PS, EXT>(slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st);
    return launch_chain_worker_one<CG, STRAND, PS, EXT>(slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st);
}
template <bool EXT>
static cudaError_t launch_chain_worker_ext(int gap_mode, PoaChainSlot *slots, PoaChainSync *sync, int n_groups, const PoaChainParams *cp, int strand,
                                           int ps, const PoaParamsDev *prm, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    if (strand) return ps ? launch_chain_worker_gap<true, true, EXT>(gap_mode, slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st)
                          : launch_chain_worker_gap<true, false, EXT>(gap_mode, slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st);
    return ps ? launch_chain_worker_gap<false, true, EXT>(gap_mode, slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st)
              : launch_chain_worker_gap<false, false, EXT>(gap_mode, slots, sync, n_groups, cp, prm, ring_rows, ring_cells, kc, st);
}
/* strand / ps / ext: the host's PoaChainParams::amb_strand (-s), whether the run has -G path scores and whether it is an extend
 * run (-m 2), which pick the kernel instantiation */
extern "C" cudaError_t poa_launch_chain_dp_worker(int gap_mode, const int *gaps, PoaChainSlot *slots, PoaChainSync *sync, int n_groups,
                                                  const PoaChainParams *cp, int strand, int ps, int ext, const PoaParamsDev *prm, int ring_rows,
                                                  int ring_cells, cudaStream_t st) {
    if (n_groups <= 0) return cudaSuccess;
    const P16Consts kc = make_p16_consts(gaps[0], gaps[1], gaps[2], gaps[3]);
    return ext ? launch_chain_worker_ext<true>(gap_mode, slots, sync, n_groups, cp, strand, ps, prm, ring_rows, ring_cells, kc, st)
               : launch_chain_worker_ext<false>(gap_mode, slots, sync, n_groups, cp, strand, ps, prm, ring_rows, ring_cells, kc, st);
}

template <int GAP, bool STRAND, bool PS, bool EXT>
static cudaError_t launch_chain_one(const PoaChainSlot *slots, const int32_t *idx, int n_jobs, int round, const PoaChainParams *cp, const PoaParamsDev *prm,
                                    int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    const size_t smem = ring_smem_bytes(GAP, 16, ring_rows, ring_cells) + 18 * sizeof(uint4);
    cudaError_t e = cudaFuncSetAttribute(poa_chain_align_kernel_p16<GAP, STRAND, PS, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return e;
    poa_chain_align_kernel_p16<GAP, STRAND, PS, EXT><<<n_jobs, 32, smem, st>>>(slots, idx, cp, prm, n_jobs, round, ring_rows, ring_cells, kc);
    return cudaGetLastError();
}
template <bool STRAND, bool PS, bool EXT>
static cudaError_t launch_chain_gap(int gap_mode, const PoaChainSlot *slots, const int32_t *idx, int n_jobs, int round, const PoaChainParams *cp,
                                    const PoaParamsDev *prm, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    if constexpr (EXT) { if (gap_mode == LG) return cudaErrorInvalidValue; }          /* linear-gap extend: not on the chain */
    else if (gap_mode == LG) return launch_chain_one<LG, STRAND, PS, false>(slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st);
    if (gap_mode == AG) return launch_chain_one<AG, STRAND, PS, EXT>(slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st);
    return launch_chain_one<CG, STRAND, PS, EXT>(slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st);
}
template <bool EXT>
static cudaError_t launch_chain_ext(int gap_mode, const PoaChainSlot *slots, const int32_t *idx, int n_jobs, int round, const PoaChainParams *cp,
                                    int strand, int ps, const PoaParamsDev *prm, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    if (strand) return ps ? launch_chain_gap<true, true, EXT>(gap_mode, slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st)
                          : launch_chain_gap<true, false, EXT>(gap_mode, slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st);
    return ps ? launch_chain_gap<false, true, EXT>(gap_mode, slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st)
              : launch_chain_gap<false, false, EXT>(gap_mode, slots, idx, n_jobs, round, cp, prm, ring_rows, ring_cells, kc, st);
}
/* gaps[4] = { e1, oe1, e2, oe2 } (host copy of what prm holds on the device) */
extern "C" cudaError_t poa_launch_chain_align_p16(int gap_mode, const int *gaps, const PoaChainSlot *slots, const int32_t *idx, int n_jobs, int round,
                                                  const PoaChainParams *cp, int strand, int ps, int ext, const PoaParamsDev *prm, int ring_rows,
                                                  int ring_cells, cudaStream_t st) {
    if (n_jobs <= 0) return cudaSuccess;
    const P16Consts kc = make_p16_consts(gaps[0], gaps[1], gaps[2], gaps[3]);
    return ext ? launch_chain_ext<true>(gap_mode, slots, idx, n_jobs, round, cp, strand, ps, prm, ring_rows, ring_cells, kc, st)
               : launch_chain_ext<false>(gap_mode, slots, idx, n_jobs, round, cp, strand, ps, prm, ring_rows, ring_cells, kc, st);
}

/* ------------------------------------------------------------------ debug: the chain's job function on one job
 * (poa_debug_chain_replay in poa_cuda.cu, for the tests).  The replay kernel makes the call poa_chain_dp_worker_kernel
 * makes, on a job the host hands over with fresh output buffers.  The dump kernel (one warp per row 1 .. n_rows - 2)
 * then rebuilds every row's F planes with the backtrace's fb_recompute, right to left the way the insertion steps walk: at
 * the row's last cell first, then at the cell left of the previous window, down to the band's first cell.  It keeps the
 * decision bytes as the backtrace reads them back from the buffer, bits[off * 8 + (j - 8 g0)] for a row stored at
 * plane offset off, and the F values at the same offsets in an int16 slab (F1, then F2, ngrp * 8 cells each). */
template <int GAP, bool PS, bool EXT = false>
__global__ void POA_P16_BOUNDS poa_chain_replay_kernel(const __grid_constant__ PoaJobDesc jd, const PoaParamsDev *__restrict__ prm,
                                                       int ring_rows, int ring_cells, const __grid_constant__ P16Consts kc) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const int lane = threadIdx.x;
    const P16Smem sm = p16_smem_init(dyn_smem, prm, ring_rows, lane);
    p16_run_job<GAP, EXT ? EXTEND : GLOBAL, true, false, true, PS, GAP == LG && !EXT>(jd, prm, kc, sm, ring_rows, ring_cells, lane);
}

template <int GAP, bool PS>
__global__ void __launch_bounds__(32) poa_fb_dump_kernel(const __grid_constant__ PoaJobDesc jd, const PoaParamsDev *__restrict__ prm, int buf_cells,
                                                         int16_t *fslab, uint8_t *fbits, int32_t *windows, const __grid_constant__ P16Consts kc) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const int lane = threadIdx.x, i = blockIdx.x + 1;
    const JobView jv = open_job(jd.blob);
    if (i >= jv.n_rows - 1) return;
    const P16Smem sm = p16_smem_init(dyn_smem, prm, 0, lane);            /* no ring: the byte buffer follows the mask tables */
    const PoaRowInfo ri = jd.rowinfo[i];
    int n = 0;
    if (ri.end >= ri.beg) {
        const uint32_t off = jd.rowoff[i].off;
        const int g0 = ri.beg >> 3, ngrp = (ri.end >> 3) - g0 + 1;
        FbDumpCtx fx;
        fx.kc = &kc; fx.cap_lo = sm.cap_lo; fx.cap_hi = sm.cap_hi;
        fx.buf = reinterpret_cast<uint8_t *>(sm.ring_data); fx.buf_cells = buf_cells;
        fx.f = fslab + (size_t)off * POA_GROUP; fx.fstride = ngrp * POA_GROUP;
        const int2 m0 = ldb(jv.rowmeta + i);
        const int np = ldb(&jv.rowmeta[i + 1].x) - m0.x;
        uint8_t *ob = fbits + (size_t)off * POA_GROUP;
        for (int j = ri.end; j >= ri.beg; ++n) {
            const int lo = fb_recompute<GAP, GLOBAL, true, PS>(jv, jd, prm, fx, ri.beg, ri.end, m0.x, np, m0.y & 0xff, j, lane);
            for (int c = lo + lane; c <= j; c += 32) ob[c - g0 * 8] = fx.buf[c - lo];
            __syncwarp();
            j = lo - 1;
        }
    }
    if (lane == 0) windows[i] = n;
}

/* largest dynamic shared memory of one CTA (sm_90) */
#define POA_SMEM_MAX (227 * 1024)
template <int GAP, bool PS, bool EXT = false>
static cudaError_t launch_chain_replay_one(const PoaJobDesc &jd, const PoaParamsDev *prm, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    const size_t smem = ring_smem_bytes(GAP, 16, ring_rows, ring_cells) + 18 * sizeof(uint4);
    if (smem > POA_SMEM_MAX) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(poa_chain_replay_kernel<GAP, PS, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, POA_SMEM_MAX);
    if (e != cudaSuccess) return e;
    poa_chain_replay_kernel<GAP, PS, EXT><<<1, 32, smem, st>>>(jd, prm, ring_rows, ring_cells, kc);
    return cudaGetLastError();
}
/* ring_rows: a power of two >= 2; ring_cells: a positive multiple of 8 (poa_pick_ring gives no less); their ring must fit one CTA.
 * ps: the job carries -G path scores (the path-score instantiation of the chain's job function); ext: an extend job (the
 * chain's EXTEND instantiation; affine or convex gaps) */
extern "C" cudaError_t poa_launch_chain_replay(int gap_mode, const int *gaps, const PoaJobDesc *jd, const PoaParamsDev *prm, int ring_rows, int ring_cells,
                                               int ps, int ext, cudaStream_t st) {
    if (ring_rows < 2 || (ring_rows & (ring_rows - 1)) || ring_cells < 8 || (ring_cells & 7)) return cudaErrorInvalidValue;
    const P16Consts kc = make_p16_consts(gaps[0], gaps[1], gaps[2], gaps[3]);
    if (ext) {
        if (gap_mode == LG) return cudaErrorInvalidValue;
        if (gap_mode == AG) return ps ? launch_chain_replay_one<AG, true, true>(*jd, prm, ring_rows, ring_cells, kc, st) : launch_chain_replay_one<AG, false, true>(*jd, prm, ring_rows, ring_cells, kc, st);
        return ps ? launch_chain_replay_one<CG, true, true>(*jd, prm, ring_rows, ring_cells, kc, st) : launch_chain_replay_one<CG, false, true>(*jd, prm, ring_rows, ring_cells, kc, st);
    }
    if (gap_mode == LG) return ps ? launch_chain_replay_one<LG, true>(*jd, prm, ring_rows, ring_cells, kc, st) : launch_chain_replay_one<LG, false>(*jd, prm, ring_rows, ring_cells, kc, st);
    if (gap_mode == AG) return ps ? launch_chain_replay_one<AG, true>(*jd, prm, ring_rows, ring_cells, kc, st) : launch_chain_replay_one<AG, false>(*jd, prm, ring_rows, ring_cells, kc, st);
    return ps ? launch_chain_replay_one<CG, true>(*jd, prm, ring_rows, ring_cells, kc, st) : launch_chain_replay_one<CG, false>(*jd, prm, ring_rows, ring_cells, kc, st);
}
/* the bytes of the chain's backtrace buffer for a ring geometry (fx.buf_cells in p16_run_job) */
extern "C" int poa_chain_fb_buf_cells(int gap_mode, int ring_rows, int ring_cells) {
    const int rn = gap_mode == LG ? RingPlanes<LG>::N : (gap_mode == AG ? RingPlanes<AG>::N : RingPlanes<CG>::N);
    return rn * ring_cells * 2 * ring_rows;
}
template <int GAP, bool PS>
static cudaError_t launch_fb_dump_one(const PoaJobDesc &jd, const PoaParamsDev *prm, int n_rows, int buf_cells, int16_t *fslab, uint8_t *fbits,
                                      int32_t *windows, const P16Consts &kc, cudaStream_t st) {
    const size_t smem = (size_t)POA_MAX_M * POA_MAX_M * sizeof(int) + 18 * sizeof(uint4) + (size_t)std::max(buf_cells >> 8, 1) * 256;
    if (smem > POA_SMEM_MAX) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(poa_fb_dump_kernel<GAP, PS>, cudaFuncAttributeMaxDynamicSharedMemorySize, POA_SMEM_MAX);
    if (e != cudaSuccess) return e;
    if (n_rows > 2) poa_fb_dump_kernel<GAP, PS><<<n_rows - 2, 32, smem, st>>>(jd, prm, buf_cells, fslab, fbits, windows, kc);
    return cudaGetLastError();
}
extern "C" cudaError_t poa_launch_fb_dump(int gap_mode, const int *gaps, const PoaJobDesc *jd, const PoaParamsDev *prm, int n_rows, int buf_cells,
                                          int16_t *fslab, uint8_t *fbits, int32_t *windows, int ps, cudaStream_t st) {
    if (gap_mode == LG) return cudaErrorInvalidValue;
    const P16Consts kc = make_p16_consts(gaps[0], gaps[1], gaps[2], gaps[3]);
    if (gap_mode == AG) return ps ? launch_fb_dump_one<AG, true>(*jd, prm, n_rows, buf_cells, fslab, fbits, windows, kc, st)
                                  : launch_fb_dump_one<AG, false>(*jd, prm, n_rows, buf_cells, fslab, fbits, windows, kc, st);
    return ps ? launch_fb_dump_one<CG, true>(*jd, prm, n_rows, buf_cells, fslab, fbits, windows, kc, st)
              : launch_fb_dump_one<CG, false>(*jd, prm, n_rows, buf_cells, fslab, fbits, windows, kc, st);
}

/* ------------------------------------------------------------------ launcher */
/* all_planes: the TMA variant stages every plane of a row in its ring slot, not only the ones successors read */
static inline size_t ring_smem_bytes(int gap, int bits, int ring_rows, int ring_cells, int all_planes) {
    const int rn = all_planes ? (gap == LG ? 1 : (gap == AG ? 3 : 5)) : (gap == LG ? 1 : (gap == AG ? 2 : 3));
    return (size_t)POA_MAX_M * POA_MAX_M * sizeof(int) + (size_t)ring_rows * sizeof(PoaRowInfo) + (((size_t)ring_rows * 4 + 15) & ~(size_t)15)
           + (size_t)ring_rows * rn * ring_cells * (bits / 8);
}

template <int GAP, typename ST, int MODE>
static cudaError_t launch_one(const PoaJobDesc *jobs, const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, cudaStream_t st) {
    const size_t smem = ring_smem_bytes(GAP, (int)sizeof(ST) * 8, ring_rows, ring_cells);
    cudaError_t e = cudaFuncSetAttribute(poa_align_kernel<GAP, ST, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return e;
    const char *cv = getenv("ABPOA_GPU_CARVEOUT");
    if (cv && *cv) cudaFuncSetAttribute(poa_align_kernel<GAP, ST, MODE>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv));
    poa_align_kernel<GAP, ST, MODE><<<n_jobs, 32, smem, st>>>(jobs, prm, n_jobs, ring_rows, ring_cells);
    return cudaGetLastError();
}

template <int GAP, typename ST>
static cudaError_t launch_mode(int mode, const PoaJobDesc *jobs, const PoaParamsDev *prm, int n_jobs, int rr, int rc, cudaStream_t st) {
    switch (mode) {
    case GLOBAL: return launch_one<GAP, ST, GLOBAL>(jobs, prm, n_jobs, rr, rc, st);
    case LOCAL:  return launch_one<GAP, ST, LOCAL>(jobs, prm, n_jobs, rr, rc, st);
    default:     return launch_one<GAP, ST, EXTEND>(jobs, prm, n_jobs, rr, rc, st);
    }
}

/* Pick the shared-memory ring geometry for a launch: slots wide enough for the expected band
 * (`band_cells`, already a multiple of 8) and as many rows as fit the per-CTA budget. */
extern "C" int poa_tma_enabled(void) { static const int on = [] { const char *e = getenv("ABPOA_GPU_TMA"); return e && *e == '1'; }(); return on; }
/* ABPOA_GPU_NO_LEAN=1: whole-graph global jobs of the packed kernel take the general predecessor loop too */
extern "C" int poa_lean_disabled(void) { static const int off = [] { const char *e = getenv("ABPOA_GPU_NO_LEAN"); return e && *e == '1'; }(); return off; }
extern "C" void poa_pick_ring(int gap_mode, int bits, int band_cells, size_t smem_budget, int *ring_rows, int *ring_cells) {
    int rc = band_cells < 64 ? 64 : band_cells;
    int rr = 64;
    const int all = bits == 16 && poa_tma_enabled();
    if (all) smem_budget += 12 * 1024;                                        /* two more planes per ring row */
    smem_budget = smem_budget > 512 ? smem_budget - 512 : smem_budget;      /* mask tables of the packed kernel */
    while (rr > 2 && ring_smem_bytes(gap_mode, bits, rr, rc, all) > smem_budget) rr >>= 1;
    while (rc > 64 && ring_smem_bytes(gap_mode, bits, rr, rc, all) > smem_budget) rc -= 64;   /* very wide rows: cache a prefix */
    *ring_rows = rr; *ring_cells = rc;
}

template <int GAP, int MODE, bool LEAN, bool TMA>
static cudaError_t launch_p16_one(const PoaJobDesc *jobs, const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, const P16Consts &kc, cudaStream_t st) {
    const size_t smem = ring_smem_bytes(GAP, 16, ring_rows, ring_cells, TMA) + 18 * sizeof(uint4);
    /* per device and instantiation; cudaFuncSetAttribute is cheap and idempotent, so no process-wide cache (a second
     * GPU in the same process needs its own call) */
    cudaError_t e = cudaFuncSetAttribute(poa_align_kernel_p16<GAP, MODE, LEAN, TMA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e != cudaSuccess) return e;
    const char *cv = getenv("ABPOA_GPU_CARVEOUT");          /* shared-memory share of the L1/shared array, percent */
    if (cv && *cv) cudaFuncSetAttribute(poa_align_kernel_p16<GAP, MODE, LEAN, TMA>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv));
    poa_align_kernel_p16<GAP, MODE, LEAN, TMA><<<n_jobs, 32, smem, st>>>(jobs, prm, n_jobs, ring_rows, ring_cells, kc);
    return cudaGetLastError();
}
template <int GAP>
static cudaError_t launch_p16_mode(int mode, int lean, const PoaJobDesc *jobs, const PoaParamsDev *prm, int n_jobs, int rr, int rc, const P16Consts &kc, cudaStream_t st) {
    switch (mode) {
    case GLOBAL:
        if (lean && poa_tma_enabled()) return launch_p16_one<GAP, GLOBAL, true, true>(jobs, prm, n_jobs, rr, rc, kc, st);
        return lean ? launch_p16_one<GAP, GLOBAL, true, false>(jobs, prm, n_jobs, rr, rc, kc, st) : launch_p16_one<GAP, GLOBAL, false, false>(jobs, prm, n_jobs, rr, rc, kc, st);
    case LOCAL:  return launch_p16_one<GAP, LOCAL, false, false>(jobs, prm, n_jobs, rr, rc, kc, st);
    default:     return launch_p16_one<GAP, EXTEND, false, false>(jobs, prm, n_jobs, rr, rc, kc, st);
    }
}
/* the packed int16x2 kernel (int16 planes, DPX pair arithmetic).  lean != 0: every job aligns to the whole graph and
 * carries no -G path scores (the straight-line predecessor path of p16_run_job may be used; global mode only) */
extern "C" cudaError_t poa_launch_align_p16(int gap_mode, int align_mode, int lean, const int *gaps, const PoaJobDesc *jobs,
                                            const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, cudaStream_t st) {
    if (n_jobs <= 0) return cudaSuccess;
    const P16Consts kc = make_p16_consts(gaps[0], gaps[1], gaps[2], gaps[3]);
    if (poa_lean_disabled()) lean = 0;
    if (gap_mode == LG) return launch_p16_mode<LG>(align_mode, lean, jobs, prm, n_jobs, ring_rows, ring_cells, kc, st);
    if (gap_mode == AG) return launch_p16_mode<AG>(align_mode, lean, jobs, prm, n_jobs, ring_rows, ring_cells, kc, st);
    return launch_p16_mode<CG>(align_mode, lean, jobs, prm, n_jobs, ring_rows, ring_cells, kc, st);
}

extern "C" cudaError_t poa_launch_align(int gap_mode, int bits, int align_mode, const PoaJobDesc *jobs,
                                        const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, cudaStream_t st) {
    if (n_jobs <= 0) return cudaSuccess;
    if (bits == 16) {
        if (gap_mode == LG) return launch_mode<LG, int16_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
        if (gap_mode == AG) return launch_mode<AG, int16_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
        return launch_mode<CG, int16_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
    }
    if (gap_mode == LG) return launch_mode<LG, int32_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
    if (gap_mode == AG) return launch_mode<AG, int32_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
    return launch_mode<CG, int32_t>(align_mode, jobs, prm, n_jobs, ring_rows, ring_cells, st);
}


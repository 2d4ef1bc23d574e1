/* poa_chain.cu -- the device-resident progressive POA ("chain engine") behind abpoa_gpu_msa_batch.
 *
 * Reads of a group are strictly sequential (read i+1 is aligned to the graph that already contains read i; reference
 * src/abpoa_align.c:312-352).  The launch engine of poa_batch.cu pays a host round trip per read.  Here the graph of
 * every group lives in HBM and the host does nothing until its wave of groups is finished: reads go up once, results
 * come back once.  Two schedules run the same device code (the alignment in poa_kernels.cu; chain_fuse in poa_chain.cuh
 * fuses the graph-CIGAR, re-orders and flattens graph + next read into the next job):
 *
 *     free-running (default)   two persistent kernels per wave: poa_chain_dp_worker_kernel, one resident warp per group
 *                              running its alignments back to back, and poa_chain_fuse_worker_kernel, fuse CTAs fed
 *                              through the task queue of PoaChainSync.  Each group advances at its own pace in a
 *                              private plane slab.
 *     rounds                   per round and cohort of groups two kernels, poa_chain_align_kernel_p16 and
 *                              poa_chain_fuse_kernel, planes from the cohort's pool.  Taken with ABPOA_GPU_CHAIN_ROUNDS=1
 *                              and under tools that serialise kernel launches (profilers, sanitizers), where two kernels
 *                              that wait for each other cannot both run.
 *
 * The results come from the device: poa_chain_consensus_kernel (heaviest bundling or most frequent base), poa_chain_msa_kernel (row-column
 * MSA) and poa_chain_gfa_kernel (GFA) write records that come back in one copy and are installed into the caller's records.  With
 * ABPOA_GPU_CHAIN_EXPORT_GRAPH=1 the whole graph comes back instead (poa_chain_export_kernel, rebuilt by
 * poa_graph_import) and the host computes the consensus on it: the cross-check of the device graph against the host
 * code.  Groups the device cannot finish (capacity, int16 window, plane slab) are reported back and completed by the
 * launch engine -- same results either way.
 *
 * Host side: poa_chain_run reads the call's setup (chain_call), sizes the groups (plan_groups), splits them into waves
 * that fit the arena (split_waves) and runs each wave (Wave).  A group's device region is laid out by chain_slot_layout
 * (poa_chain.cuh) for the planner and the carve alike.
 *
 * Scope of the chain: global alignment, or extend alignment (-m 2, with or without z-drop -z; affine or convex gaps: the
 * alignment kernels' EXTEND instantiation, rows in the reference's Kahn order, chain_kahn_order), banded (wb >= 0),
 * packed-int16 admissible scores, heaviest-bundling or
 * most-frequent-base consensus (single cluster, no sub_aln), row-column MSA and GFA (one read set per node, not per
 * edge), base weights (-Q: a weight byte per read base, 0..255; a group with any other weight takes the other engine),
 * ambiguous strand (-s: the alignment warp retries a weak hit as the reverse complement, chain_align_read in
 * poa_kernels.cu), path scores (-G: the flatten writes every in-edge's score, chain_path_score; a group whose node weights
 * could exceed POA_PS_MAX_NODE_W takes the other engine).  Everything else takes the other engine.
 */
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <mutex>
#include <thread>
#include <vector>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include "abpoa_gpu.h"
#include "poa_internal.h"
#include "poa_engine.h"
#include "poa_device.cuh"
#include "poa_chain.cuh"
#include "poa_chain_host.h"

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    poa_die("libabpoa_b200/chain", "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); } while (0)

extern "C" cudaError_t poa_launch_chain_dp_worker(int gap_mode, const int *gaps, PoaChainSlot *slots, PoaChainSync *sync, int n_groups,
                                                  const PoaChainParams *cp, int strand, int ps, int ext, const PoaParamsDev *prm, int ring_rows,
                                                  int ring_cells, cudaStream_t st);
extern "C" cudaError_t poa_launch_chain_align_p16(int gap_mode, const int *gaps, const PoaChainSlot *slots, const int32_t *idx, int n_jobs, int round,
                                                  const PoaChainParams *cp, int strand, int ps, int ext, const PoaParamsDev *prm, int ring_rows,
                                                  int ring_cells, cudaStream_t st);
extern "C" void poa_pick_ring(int gap_mode, int bits, int band_cells, size_t smem_budget, int *ring_rows, int *ring_cells);

static_assert(offsetof(PoaChainSync, q_tail) == 128 && offsetof(PoaChainSync, total) == 256 && offsetof(PoaChainSync, abort) == 384,
              "every polled / bumped word of PoaChainSync sits in its own 128-byte line");
static_assert(POA_GFA_HDR_WORDS == POA_GFA_HDR, "the device's GFA record header is the one poa_gfa_from_record reads");

/* ------------------------------------------------------------------ kernels */
/* PS: -G runs (ChainCall::ps), whose jobs carry path scores (chain_flatten); LG: linear-gap runs, whose rows are stored in
 * whole reference vectors (chain_flatten's plane estimate); KO: extend runs, whose rows follow the reference's Kahn order
 * (chain_fuse) */
template <bool PS, bool LG>
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_seed_kernel(PoaChainSlot *slots, const PoaChainParams *cp, int n) {
    if ((int)blockIdx.x >= n) return;
    chain_seed<PS, LG>(&slots[blockIdx.x], cp);
}

template <bool PS, bool LG, bool KO = false>
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_fuse_kernel(PoaChainSlot *slots, const int32_t *idx, const PoaChainParams *cp, int n, int round) {
    if ((int)blockIdx.x >= n) return;
    chain_fuse<PS, LG, KO>(&slots[idx[blockIdx.x]], cp, round);
}

/* Free-running chain, fuse side: persistent CTAs draw tickets from PoaChainSync; ticket t is served when tasks[t] holds a group.
 * (The alignment side is poa_chain_dp_worker_kernel in poa_kernels.cu.) */
__device__ __forceinline__ int sync_ld(const int32_t *p) { int v; asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void sync_st(int32_t *p, int v) { asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned long long sync_now_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

template <bool PS, bool LG, bool KO = false>
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_fuse_worker_kernel(PoaChainSlot *slots, PoaChainSync *sync, const PoaChainParams *cp) {
    __shared__ int task_s;
    for (;;) {
        if (threadIdx.x < 32) {                                /* warp 0 waits, warp-uniformly (see poa_chain_dp_worker_kernel) */
            unsigned ticket = 0;
            if (threadIdx.x == 0) ticket = atomicAdd(&sync->q_head, 1u);
            ticket = __shfl_sync(0xffffffffu, ticket, 0);
            int g = -2; unsigned ns = 250, polls = 0;
            const unsigned long long t0 = sync_now_ns(), limit = sync->watchdog_ns;
            const int32_t *tasks = sync->tasks;
            for (;;) {
                /* the ticket's own task word is what is polled; the shared words (total, abort) and the clock only every 32nd time */
                if ((polls++ & 31u) == 0) {
                    const int tot = __shfl_sync(0xffffffffu, sync_ld(&sync->total), 0), ab = __shfl_sync(0xffffffffu, sync_ld(&sync->abort), 0);
                    if ((long long)ticket >= (long long)tot || ab) { g = -2; break; }
                    /* nobody appended a task for this long: the alignment kernel is not running next to this one (a tool that
                     * serialises kernels, a device shared with a long-running grid): give up, the launch engine finishes the groups */
                    const unsigned late = __shfl_sync(0xffffffffu, (unsigned)(polls > 1 && sync_now_ns() - t0 > limit), 0);
                    if (late) { if (threadIdx.x == 0) sync_st(&sync->abort, 1); g = -2; break; }
                }
                g = __shfl_sync(0xffffffffu, sync_ld(&tasks[ticket]), 0);
                if (g >= 0) break;
                __nanosleep(ns); if (ns < 4000) ns <<= 1;
            }
            if (threadIdx.x == 0) task_s = g;
        }
        __syncthreads();
        const int g = task_s;
        __syncthreads();
        if (g < 0) return;
        __threadfence();                                       /* acquire: graph arrays / CIGAR of this group may have been written from another SM */
        PoaChainSlot *s = &slots[g];
        const unsigned long long t0 = sync_now_ns();
        chain_fuse<PS, LG, KO>(s, cp, 0);
        __syncthreads();
        __threadfence();                                       /* release */
        __syncthreads();
        if (threadIdx.x == 0) { s->fuse_ns += sync_now_ns() - t0; __threadfence(); sync_st(&s->turn, 0); }
    }
}

/* Compact export of the final graphs (layout: poa_graph_import in poa_graph.c).  ex_off[g] = first int32 word of
 * group g's record in `ex`; a record is written only if it fits ex_cap[g] words (else word 0 = -1). */
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_export_kernel(PoaChainSlot *slots, const PoaChainParams *cp, int n,
                                                                       int32_t *ex, const int64_t *ex_off, const int32_t *ex_cap) {
    if ((int)blockIdx.x >= n) return;
    PoaChainSlot *s = &slots[blockIdx.x];
    int32_t *o = ex + ex_off[blockIdx.x];
    const int K = cp->K, A = cp->A, nn = s->n_nodes;
    if (s->failed) { if (threadIdx.x == 0) o[0] = -1; return; }
    int32_t *ci = s->scr[0], *ca = s->scr[1];
    POA_PAR_FOR(v, nn) { ci[v] = s->in_cnt[v]; ca[v] = s->aln_cnt[v]; }
    __syncthreads();
    const int n_in = cta_excl_scan(ci, nn);
    __syncthreads();
    const int n_aln = cta_excl_scan(ca, nn);
    __syncthreads();
    int32_t *co = s->scr[2];
    POA_PAR_FOR(v, nn) co[v] = s->out_cnt[v];
    __syncthreads();
    const int n_out = cta_excl_scan(co, nn);
    __syncthreads();
    const int64_t words = 4 + 5ll * nn + 4ll * n_in + n_aln;
    if (words > ex_cap[blockIdx.x] || n_out != n_in) { if (threadIdx.x == 0) o[0] = -1; return; }
    int32_t *base = o + 4, *n_read = base + nn, *in_cnt = n_read + nn, *out_cnt = in_cnt + nn, *aln_cnt = out_cnt + nn;
    int32_t *in_id = aln_cnt + nn, *in_w = in_id + n_in, *out_id = in_w + n_in, *out_w = out_id + n_in, *aln = out_w + n_in;
    if (threadIdx.x == 0) { o[0] = nn; o[1] = n_in; o[2] = n_aln; o[3] = s->fused; }
    POA_PAR_FOR(v, nn) {
        base[v] = s->base[v]; n_read[v] = s->n_read[v]; in_cnt[v] = s->in_cnt[v]; out_cnt[v] = s->out_cnt[v]; aln_cnt[v] = s->aln_cnt[v];
        for (int e = 0; e < s->in_cnt[v]; ++e) { in_id[ci[v] + e] = s->in_id[(size_t)v * K + e]; in_w[ci[v] + e] = s->in_w[(size_t)v * K + e]; }
        for (int e = 0; e < s->out_cnt[v]; ++e) { out_id[co[v] + e] = s->out_id[(size_t)v * K + e]; out_w[co[v] + e] = s->out_w[(size_t)v * K + e]; }
        for (int a = 0; a < s->aln_cnt[v]; ++a) aln[ca[v] + a] = s->aln_id[(size_t)v * A + a];
    }
}

/* consensus of every finished group (chain_cons_path: heaviest bundling on one thread per group, most frequent base on a
 * CTA per group: launched with 32 or POA_CHAIN_T threads); records are packed back to back into `out` through an atomic cursor:
 * rec_off[g] = first word of group g's record, -1 if none */
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_consensus_kernel(PoaChainSlot *slots, const PoaChainParams *cp, int n,
                                                                          int32_t *out, unsigned long long *cursor, unsigned long long out_words, int64_t *rec_off) {
    if ((int)blockIdx.x >= n) return;
    PoaChainSlot *s = &slots[blockIdx.x];
    int32_t *tmp = s->scr[2];                               /* [n_cap]: the consensus is never longer than the graph */
    chain_cons_path(s, cp, tmp, s->n_cap);
    if (threadIdx.x != 0) return;
    const int len = tmp[0];
    if (len < 0) { rec_off[blockIdx.x] = -1; return; }
    const unsigned long long at = atomicAdd(cursor, (unsigned long long)(len + 1));
    if (at + (unsigned long long)(len + 1) > out_words) { rec_off[blockIdx.x] = -1; return; }
    for (int k = 0; k <= len; ++k) out[at + k] = tmp[k];
    rec_off[blockIdx.x] = (int64_t)at;
}

/* RC-MSA of every finished group, one CTA per group: ranks on one thread (chain_msa_rank), rows by the whole CTA
 * (chain_msa_rows).  with_cons: add the consensus row, from the path chain_cons_path left in scr[1] -- run_cons: compute
 * that path here (the consensus kernel did not run).  A record is [msa_len, n_rows, rows as bytes], packed through the
 * same cursor as the consensus records, at word rec_base + cursor; rec_off[g] = -1 if the group has none (it is then
 * finished by the launch engine). */
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_msa_kernel(PoaChainSlot *slots, const PoaChainParams *cp, int n, int with_cons, int run_cons,
                                                                    int32_t *out, unsigned long long *cursor, unsigned long long rec_base,
                                                                    unsigned long long out_words, int64_t *rec_off) {
    if ((int)blockIdx.x >= n) return;
    __shared__ long long at_s;
    __shared__ int len_s;
    PoaChainSlot *s = &slots[blockIdx.x];
    if (run_cons && !s->failed && s->n_nodes >= 3) chain_cons_path(s, cp, s->scr[2], s->n_cap);
    if (threadIdx.x == 0) {
        const int msa_len = chain_msa_rank(s, cp);
        long long at = -1;
        if (msa_len > 0) {
            const unsigned long long words = 2 + ((unsigned long long)(s->n_reads + with_cons) * (unsigned long long)msa_len + 3) / 4;
            const unsigned long long a = rec_base + atomicAdd(cursor, words);
            if (a + words <= out_words) at = (long long)a;
        }
        at_s = at; len_s = msa_len;
        rec_off[blockIdx.x] = at;
        if (at >= 0) { out[at] = msa_len; out[at + 1] = s->n_reads + with_cons; }
    }
    __syncthreads();
    if (at_s < 0) return;
    chain_msa_rows(s, cp, len_s, with_cons, reinterpret_cast<uint8_t *>(out + at_s + 2));
}

/* GFA of every finished group, one CTA per group: order and size on one thread (chain_gfa_size), the record by the
 * whole CTA (chain_gfa_record).  with_cons: the record carries the consensus path chain_cons_path left in scr[1] --
 * run_cons: compute that path here (the consensus kernel did not run).  Records share the consensus records' cursor at
 * word rec_base + cursor, each 8-byte aligned; rec_off[g] = -1 if the group has none (it is then finished by the launch
 * engine). */
__global__ void __launch_bounds__(POA_CHAIN_T) poa_chain_gfa_kernel(PoaChainSlot *slots, const PoaChainParams *cp, int n, int with_cons, int run_cons,
                                                                    int32_t *out, unsigned long long *cursor, unsigned long long rec_base,
                                                                    unsigned long long out_words, int64_t *rec_off) {
    if ((int)blockIdx.x >= n) return;
    __shared__ long long at_s;
    __shared__ int32_t hdr_s[POA_GFA_HDR_WORDS];
    PoaChainSlot *s = &slots[blockIdx.x];
    if (run_cons && !s->failed && s->n_nodes >= 3) chain_cons_path(s, cp, s->scr[2], s->n_cap);
    if (threadIdx.x == 0) {
        const long long words = chain_gfa_size(s, cp, with_cons, hdr_s);
        long long at = -1;
        if (words > 0) {
            const unsigned long long a = (rec_base + atomicAdd(cursor, (unsigned long long)words + 1) + 1) & ~1ull;
            if (a + (unsigned long long)words <= out_words) at = (long long)a;
        }
        at_s = at;
        rec_off[blockIdx.x] = at;
    }
    __syncthreads();
    if (at_s < 0) return;
    chain_gfa_record(s, cp, hdr_s, out + at_s);
}

/* debugging aid (tests): the device's -G score function on n (edge weight, node weight) pairs */
__global__ void poa_chain_path_score_kernel(const int32_t *edge_w, const int32_t *node_w, int n, int32_t *out) {
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) out[i] = chain_path_score(edge_w[i], node_w[i]);
}

/* ------------------------------------------------------------------ host side */
static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

/* debugging aid (tests): out[i] = chain_path_score(edge_w[i], node_w[i]) computed on the current device */
extern "C" int poa_debug_path_scores(const int32_t *edge_w, const int32_t *node_w, int n, int32_t *out) {
    if (n <= 0) return 0;
    int32_t *d = NULL;
    const size_t b = (size_t)n * 4;
    CK(cudaMalloc((void **)&d, 3 * b));
    CK(cudaMemcpy(d, edge_w, b, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d + n, node_w, b, cudaMemcpyHostToDevice));
    poa_chain_path_score_kernel<<<(n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096, 256>>>(d, d + n, n, d + 2 * (size_t)n);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d + 2 * (size_t)n, b, cudaMemcpyDeviceToHost));
    CK(cudaFree(d));
    return n;
}

int poa_chain_eligible(const abpoa_para_t *abpt) {
    const char *off = getenv("ABPOA_GPU_NO_CHAIN");
    if (off && *off == '1') return 0;
    { const char *np = getenv("ABPOA_GPU_NO_P16"); if (np && *np == '1') return 0; }      /* the chain only has the packed int16 kernel */
    /* extend mode (-m 2, with or without z-drop): banded, affine or convex gaps (the linear-gap rows are global-only) */
    const int ext = abpt->align_mode == ABPOA_EXTEND_MODE;
    if ((abpt->align_mode != ABPOA_GLOBAL_MODE && !ext) || abpt->wb < 0) return 0;
    if (ext && abpt->gap_mode == ABPOA_LINEAR_GAP) return 0;
    /* RC-MSA and GFA run on the chain (per-node read sets, poa_chain_msa_kernel / poa_chain_gfa_kernel), and so does the
     * single-cluster most-frequent-base consensus (it needs n_read per node only; under sub_aln it needs n_span_read,
     * which the device does not keep); use_read_ids is what abpoa_post_set_para sets for them */
    const int mf = abpt->cons_algrm == ABPOA_MF && abpt->use_read_ids && !abpt->sub_aln;
    if (abpt->cons_algrm != ABPOA_HB && !mf) return 0;
    if ((abpt->use_read_ids && !abpt->out_msa && !abpt->out_gfa && !mf) || abpt->max_n_cons > 1) return 0;
    if ((abpt->zdrop > 0 && !ext) || abpt->rev_cigar || !abpt->ret_cigar) return 0;
    if (abpt->put_gap_on_right || abpt->put_gap_at_end) return 0;         /* handled by the kernels, but keep the chain on the common configuration */
    if (abpt->m > POA_MAX_M) return 0;
    if (!(abpt->disable_seeding && abpt->progressive_poa == 0)) return 0;
    return 1;
}

namespace {

/* the round schedule keeps every group listed this many rounds beyond its last read: a group that has to re-run an
 * alignment (band wider than its plane slab) falls one round behind (slots with nothing to do return at once) */
const int ROUNDS_EXTRA = 2;
/* ... and with -s one more round per read: the forward pass of a read that arrives reverse-complemented wanders off the
 * band estimate often, and every read may be re-run once */
int rounds_extra(bool strand, int n_reads) { return ROUNDS_EXTRA + (strand ? n_reads - 1 : 0); }
const double STRAND_SLAB_X = 5.0;       /* -s: plane estimate factor (plan_groups) */

struct GroupPlan {
    int g;                  /* index into the caller's groups */
    int n_reads, qmax; int64_t bases;
    int n_cap;
    size_t reads_bytes;     /* the group's part of the wave's reads region (chain_slot_reads) */
    size_t static_bytes;    /* reads_bytes + the group's own region (chain_slot_layout) */
    double pool_units_est;
    double rec_bytes;       /* RC-MSA / GFA runs: bound on the group's result records (0 otherwise) */
};

struct Cohort {
    std::vector<int> members;               /* indices into the wave's plan list */
    cudaStream_t st = NULL;
    cudaEvent_t ev_end = NULL;
    std::vector<cudaEvent_t> marks;         /* per round: before DP, between DP and fuse, after fuse */
};

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

/* Pinned staging buffers are kept for the life of the process (grow-only, one per purpose): cudaHostAlloc / cudaFreeHost of
 * half a gigabyte per batch call cost ~0.2 s, more than the copies they serve. */
struct PinnedSlot { void *p = NULL; size_t cap = 0; bool busy = false; };
std::mutex g_pin_mu; PinnedSlot g_pin[4];
void *pinned_get(int which, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    PinnedSlot &ps = g_pin[which];
    if (ps.busy) { void *q = NULL; CK(cudaHostAlloc(&q, bytes ? bytes : 1, cudaHostAllocPortable)); return q; }      /* concurrent caller: private buffer */
    if (bytes > ps.cap) {
        if (ps.p) CK(cudaFreeHost(ps.p));
        ps.cap = bytes + bytes / 4 + 4096;
        CK(cudaHostAlloc(&ps.p, ps.cap, cudaHostAllocPortable));
    }
    ps.busy = true;
    return ps.p;
}
void pinned_put(int which, void *q) {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    if (q == g_pin[which].p) g_pin[which].busy = false; else CK(cudaFreeHost(q));
}

/* two kernels that wait for each other need to run CONCURRENTLY: under a tool that injects into the CUDA driver and
 * serialises kernel launches (ncu, compute-sanitizer), or with blocking launches, use the round schedule.  Looked up once. */
bool launches_serialised() {
    static const bool serialised = [] {
        { const char *lb = getenv("CUDA_LAUNCH_BLOCKING"); if (lb && *lb == '1') return true; }      /* the second kernel would never be launched */
        for (char **v = environ; v && *v; ++v)
            if (!strncmp(*v, "CUDA_INJECTION64_PATH=", 22) || !strncmp(*v, "NV_NSIGHT_INJECTION", 19) || !strncmp(*v, "NV_COMPUTE_PROFILER", 19) ||
                !strncmp(*v, "NV_SANITIZER_INJECTION", 22) || !strncmp(*v, "NV_TPS_LAUNCH_", 14)) return true;
        /* ... or whose injection library is already mapped into this process */
        if (FILE *mp = fopen("/proc/self/maps", "r")) {
            char line[512]; bool hit = false;
            while (!hit && fgets(line, sizeof line, mp))
                hit = strstr(line, "InjectionTarget") || strstr(line, "cuda-injection") || strstr(line, "libsanitizer-collection") || strstr(line, "TreeLauncherTarget");
            fclose(mp);
            if (hit) return true;
        }
        return false;
    }();
    return serialised;
}

/* What every stage of one poa_chain_run call reads: the caller's arguments, and the parameters and knobs of the call.
 * ABPOA_GPU_CHAIN_ROUNDS, _COHORTS, _K and _EXPORT_GRAPH are read per call (the tests switch them inside one process);
 * the other knobs once per process, where they are used. */
struct ChainCall {
    int dev; poa_arena *arena; abpoa_para_t *abpt; int n_workers;
    const abpoa_gpu_group_t *groups; abpoa_gpu_group_result_t *results; PoaChainStats *stats; struct PoaEmit *emit;
    bool record, verbose;
    int m, K, A;
    int P;                  /* plane units (16 B) per 8-cell group of a DP row: the chain's kernels store H (+E1 (+E2)) and no
                               F planes (RowLayout in poa_kernels.cu) */
    bool free_run;          /* free-running schedule (default); else lock-step rounds, two kernels per round and cohort */
    int cohorts;            /* round schedule: ABPOA_GPU_CHAIN_COHORTS, or 0: as many as keep each alignment grid to one CTA per SM */
    bool want_msa; int with_cons;
    bool mf;                /* most-frequent-base consensus (-a 1); heaviest bundling otherwise */
    bool want_gfa;          /* GFA records: out_gfa with a writer attached (without one, the reference prints and computes nothing) */
    int W;                  /* RC-MSA / GFA: words per read set (W of the largest group), 0 otherwise */
    bool export_graph;      /* the whole graph comes back (compact export) and the host computes the consensus on it */
    bool strand;            /* -s: the alignment warp retries weak hits as the reverse complement; read_rc comes back */
    bool qv;                /* -Q and at least one read with weights: every group gets its weight bytes (chain_slot_reads) */
    bool ps;                /* -G: every job blob carries path scores; the kernels' path-score instantiation runs */
    bool lg;                /* linear gaps: DP rows are stored in whole reference vectors (the seed / fuse kernels' LG instantiation) */
    bool ext;               /* extend mode: the alignment kernels' EXTEND and the fuse kernels' Kahn-order (KO) instantiations */
    int sm_count;
};

ChainCall chain_call(int dev, poa_arena *arena, abpoa_para_t *abpt, int n_workers, const abpoa_gpu_group_t *groups,
                     abpoa_gpu_group_result_t *results, const std::vector<int> &todo, int flags, PoaChainStats *stats, struct PoaEmit *emit) {
    ChainCall c;
    c.dev = dev; c.arena = arena; c.abpt = abpt; c.n_workers = n_workers; c.groups = groups; c.results = results; c.stats = stats; c.emit = emit;
    c.record = (flags & ABPOA_GPU_RECORD_READS) != 0;
    c.verbose = getenv("ABPOA_GPU_PROFILE") != NULL;
    c.m = abpt->m;
    { const char *e = getenv("ABPOA_GPU_CHAIN_K"); c.K = e && *e ? atoi(e) : (c.m > 5 ? 24 : 12); }
    c.A = c.m - 1 > 1 ? c.m - 1 : 1;
    c.P = abpt->gap_mode == ABPOA_LINEAR_GAP ? 1 : (abpt->gap_mode == ABPOA_AFFINE_GAP ? 2 : 3);
    { const char *e = getenv("ABPOA_GPU_CHAIN_COHORTS"); c.cohorts = !e ? 0 : std::max(1, std::min(16, *e ? atoi(e) : 4)); }
    const bool serialised = launches_serialised();
    { const char *e = getenv("ABPOA_GPU_CHAIN_ROUNDS"); c.free_run = e && *e ? *e != '1' : !serialised; }
    { const char *e = getenv("ABPOA_GPU_CHAIN_EXPORT_GRAPH"); c.export_graph = e && *e == '1'; }
    c.want_msa = abpt->out_msa && !abpt->out_gfa;           /* with out_gfa, abpoa_output prints only the GFA */
    c.want_gfa = abpt->out_gfa && emit != NULL;
    c.with_cons = abpt->out_cons ? 1 : 0;
    c.mf = abpt->cons_algrm == ABPOA_MF;
    c.strand = abpt->amb_strand != 0;
    c.ps = abpt->inc_path_score != 0;
    c.lg = abpt->gap_mode == ABPOA_LINEAR_GAP;
    c.ext = abpt->align_mode == ABPOA_EXTEND_MODE;
    c.qv = false;
    if (abpt->use_qv)
        for (int g : todo)
            for (int i = 0; groups[g].qual_weights && i < groups[g].n_seq && !c.qv; ++i) c.qv = groups[g].qual_weights[i] != NULL;
    c.W = 0;
    if (c.want_msa || c.want_gfa) for (int g : todo) c.W = std::max(c.W, (groups[g].n_seq + 63) / 64);
    c.sm_count = 132;
    if (cudaDeviceGetAttribute(&c.sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || c.sm_count < 1) c.sm_count = 132;
    return c;
}

/* per-group sizes of the groups the chain can take; the others go to `fallback` */
std::vector<GroupPlan> plan_groups(const ChainCall &c, const std::vector<int> &todo, std::vector<int> &fallback) {
    std::vector<GroupPlan> plans;
    for (int g : todo) {
        const abpoa_gpu_group_t &in = c.groups[g];
        GroupPlan p; p.g = g; p.n_reads = in.n_seq; p.qmax = 0; p.bases = 0;
        bool ok = in.n_seq >= 2;
        for (int i = 0; i < in.n_seq; ++i) {
            const int l = in.seq_lens[i];
            if (l < 1) ok = false;
            if (l > p.qmax) p.qmax = l;
            p.bases += l;
            if (ok && !poa_p16_ok(c.abpt, l, 3 * l)) ok = false;
            /* the device keeps one byte per weight: a group with any other weight is finished by the launch engine */
            const int *qw = c.qv && in.qual_weights ? in.qual_weights[i] : NULL;
            for (int j = 0; ok && qw && j < l; ++j) ok = qw[j] >= 0 && qw[j] <= 255;
        }
        /* -G: a node weighs at most n_reads x the largest weight; past POA_PS_MAX_NODE_W the device's log is not known to round
         * as the host's does */
        if (c.ps && (int64_t)in.n_seq * (c.qv ? 255 : 1) > POA_PS_MAX_NODE_W) ok = false;
        /* extend: chain_kahn_order keeps an in-degree (<= K) in a byte */
        if (c.ext && c.K > 254) ok = false;
        if (!ok || p.qmax > (1 << 24)) { fallback.push_back(g); continue; }
        /* node capacity: 10 % growth per read, and for large groups at most 4 % plus a fixed slack (5 % error, 50 x 10 kbp:
         * 3.0 % measured, 33.8k nodes reserved for 25k used) -- a group that outgrows it goes to the launch engine */
        int64_t grow = std::min<int64_t>((int64_t)((double)p.qmax * (1.0 + 0.10 * (p.n_reads - 1))) + 256,
                                         (int64_t)((double)p.qmax * (1.0 + 0.04 * (p.n_reads - 1))) + 4096);
        /* extend runs: a read whose best cell lies before its end (z-drop, high error) threads the rest of it as new nodes:
         * room for every base up to 16k nodes (25 % error groups of a few hundred bases outgrew 10 % per read) */
        if (c.ext) grow = std::max<int64_t>(grow, 16384);
        p.n_cap = (int)std::min<int64_t>(2 + p.bases, grow);
        /* what the wave carve will take for the group, at its 256-byte granularity */
        PoaChainSlot probe;
        size_t own = 0; p.reads_bytes = 0;
        chain_slot_layout(&probe, p.n_cap, p.qmax, p.n_reads, c.K, c.A, c.m, c.W, c.record, [&](size_t b) { own += al256(b); return (uint8_t *)NULL; }, c.strand, c.ps);
        chain_slot_reads(&probe, p.n_reads, p.bases, [&](size_t b) { p.reads_bytes += al256(b); return (uint8_t *)NULL; }, c.qv);
        p.static_bytes = own + p.reads_bytes;
        const size_t nc = (size_t)p.n_cap;
        /* result records in the (then idle) plane pool: consensus + MSA rows, msa_len <= nodes */
        p.rec_bytes = c.want_msa ? (double)(nc + 1) * 4 + 8 + (double)(p.n_reads + c.with_cons) * (double)nc + 1024 : 0.0;
        /* GFA: consensus + [header, ids, bases, link counts, links (a read adds at most len + 1 edges), consensus ids, read
         * sets of the group's own words] */
        if (c.want_gfa)
            p.rec_bytes = (double)(nc + 1) * 4 + 4.0 * (POA_GFA_HDR_WORDS + 4 + 4.0 * (double)nc + (double)(p.bases + p.n_reads))
                        + 8.0 * (double)nc * (double)((p.n_reads + 63) / 64) + 1024;
        /* plane units of the group's largest (last) alignment.  Free-running, a group's slab is private and its rows take
         * what their bands really need: rows 3.2 % growth per read, 2w+1 cells plus the 8-cell grid per row (5 % error,
         * 50 x 10 kbp: 25.0k rows, 29-30.4 groups per row measured; estimate 25.8k x 30).  The round schedule bump-allocates
         * every job's band ESTIMATE (chain_flatten: +64 cells, + length drift) from a shared pool: keep the roomier figures. */
        const int wmax = poa_band_halfwidth(c.abpt, p.qmax);
        const double growth = c.free_run ? 0.032 : 0.045;
        const int band_slack = c.free_run ? 0 : 32;
        const double rows_final = std::min<double>(2.0 + (double)p.bases, (double)p.qmax * (1.0 + growth * (p.n_reads - 1)) + 64);
        const int lg_cells = c.lg ? POA_LG_ROW_CELLS(16) : 0;           /* linear gaps: rows in whole vectors (pn <= 16) */
        p.pool_units_est = rows_final * (double)((2 * wmax + 1 + band_slack + lg_cells + 7) / 8 + 2) * c.P;
        /* -s: a read that arrives reverse-complemented is first aligned on the wrong strand, and that alignment's band
         * wanders far off the estimate (50 x 10 kbp convex, every third read flipped: slabs of 1.5x the estimate handed
         * 706 of 1000 groups back, slabs of about 6x none).  Fewer groups per wave, each with a larger slab. */
        if (c.strand) p.pool_units_est *= STRAND_SLAB_X;
        plans.push_back(p);
    }
    return plans;
}

/* Waves [begin, end) of `plans`: as many groups as the arena holds (static regions + plane pool).  When several waves are
 * needed they get equal shares (a small tail wave would leave the device nearly empty for as long as a full one takes: a
 * wave lasts as long as one group's chain).  A single group that fits no wave goes to `fallback`. */
std::vector<std::pair<size_t, size_t>> split_waves(const std::vector<GroupPlan> &plans, size_t arena_cap, std::vector<int> &fallback) {
    const double pool_margin = 1.15;
    auto fit_from = [&](size_t from, size_t limit, size_t *need_static_out, double *need_pool_out) {
        size_t end = from, need_static = 0; double need_pool = 0;
        while (end < plans.size() && end - from < limit) {
            const size_t s2 = need_static + plans[end].static_bytes + sizeof(PoaChainSlot) + 4096;
            const double p2 = need_pool + std::max(plans[end].pool_units_est * 16.0 * pool_margin, plans[end].rec_bytes);
            if (end > from && (double)s2 + p2 + (64 << 20) > (double)arena_cap) break;
            need_static = s2; need_pool = p2; ++end;
        }
        if (need_static_out) *need_static_out = need_static;
        if (need_pool_out) *need_pool_out = need_pool;
        return end;
    };
    size_t n_waves = 0;
    for (size_t q = 0; q < plans.size(); ++n_waves) q = fit_from(q, plans.size(), NULL, NULL);
    const size_t per_wave = (plans.size() + n_waves - 1) / std::max<size_t>(n_waves, 1);
    std::vector<std::pair<size_t, size_t>> waves;
    for (size_t pos = 0; pos < plans.size();) {
        size_t need_static = 0; double need_pool = 0;
        const size_t end = fit_from(pos, per_wave, &need_static, &need_pool);
        if ((double)need_static + need_pool * 0.5 + (64 << 20) > (double)arena_cap) {       /* a single group that does not fit */
            fallback.push_back(plans[pos].g); ++pos; continue;
        }
        waves.push_back({pos, end});
        pos = end;
    }
    return waves;
}

/* One wave of groups on the device.  It owns the arena borrow, the pinned buffers, the streams and the events, and its
 * destructor releases them on every way out.  run(): carve + stage, the schedule (which uploads and seeds), collect the
 * results, install them into the caller's records, account. */
struct Wave {
    const ChainCall &c;
    const GroupPlan *plans;                 /* the wave's groups */
    const int nw;
    std::vector<int> &fallback;

    /* the arena borrow and its carve */
    uint8_t *d_base = NULL; size_t total = 0, doff = 0;
    PoaChainSlot *d_slots = NULL; PoaChainParams *d_cp = NULL; PoaParamsDev *d_prm = NULL;
    unsigned long long *d_cursors = NULL;   /* 2 per cohort, <= 16 cohorts */
    PoaChainSync *d_sync = NULL; int32_t *d_tasks = NULL; int64_t n_tasks = 0;
    uint8_t *d_reads = NULL; size_t reads_bytes = 0;
    int32_t *d_idx = NULL; size_t idx_n = 0;                /* round index lists */
    int64_t *d_exoff = NULL, *d_msaoff = NULL, *d_gfaoff = NULL; int32_t *d_excap = NULL;
    uint8_t *d_pool = NULL; size_t pool_bytes = 0; int32_t *d_ex = NULL;
    /* host side of the wave */
    std::vector<PoaChainSlot> hs, fin;      /* the slots as uploaded / as they came back */
    uint8_t *h_reads = NULL; int32_t *h_cons = NULL, *h_ex = NULL;
    std::vector<int64_t> h_exoff; std::vector<int32_t> h_excap; int64_t ex_words = 0;
    int band_cells = 64;
    /* streams and events */
    std::vector<Cohort> coh;
    cudaStream_t s0 = NULL, st_dp = NULL;
    cudaEvent_t ev_up = NULL, ev_t0 = NULL, ev_t1 = NULL;
    int ring_rows = 2, ring_cells = 64; int gaps[4];
    /* results */
    bool cons_kernel = false; unsigned long long rec_base = 0, cons_words = 0;
    std::vector<int64_t> recoff, msaoff, gfaoff, words, hoff2; int64_t tot_words = 0;
    std::vector<std::vector<int32_t>> rs, rn; std::vector<std::vector<uint64_t>> rh;
    std::vector<std::vector<uint8_t>> rc;  /* -s: read_rc of every group */
    int n_failed = 0;
    /* accounting */
    int64_t launches = 0; uint64_t h2d = 0, d2h = 0; float dev_ms = 0.f;
    double t_wave0 = 0, t_staged = 0, t_uploaded = 0, t_enqueued = 0, t_dev_done = 0, t_copied = 0;

    Wave(const ChainCall &c_, const GroupPlan *plans_, int nw_, std::vector<int> &fallback_) : c(c_), plans(plans_), nw(nw_), fallback(fallback_) {}
    Wave(const Wave &) = delete;
    Wave &operator=(const Wave &) = delete;
    ~Wave() {
        if (d_base) poa_arena_return(c.arena, d_base, total);
        if (h_reads) pinned_put(0, h_reads);
        if (h_cons) pinned_put(2, h_cons);
        if (h_ex) pinned_put(3, h_ex);
        for (Cohort &k : coh) {
            for (cudaEvent_t ev : k.marks) cudaEventDestroy(ev);
            if (k.ev_end) cudaEventDestroy(k.ev_end);
            if (k.st) cudaStreamDestroy(k.st);
        }
        if (st_dp) cudaStreamDestroy(st_dp);
        for (cudaEvent_t ev : { ev_up, ev_t0, ev_t1 }) if (ev) cudaEventDestroy(ev);
    }

    uint8_t *dtake(size_t b) { uint8_t *q = d_base + doff; doff += al256(b); return q; }

    void run() {
        if (!carve_and_stage()) {
            for (int t = 0; t < nw; ++t) fallback.push_back(plans[t].g);
            return;
        }
        if (c.free_run) run_free_running(); else run_rounds();
        collect();
        install();
        account();
    }

    /* Everything of the wave in one arena borrow: fixed blocks, the reads region, each group's region (chain_slot_layout),
     * the round index lists, the export offsets; the rest is the plane pool, which the export buffer reuses.  The reads
     * are staged in a pinned buffer with the same layout as their device region.  false: the export buffer does not fit. */
    bool carve_and_stage() {
        t_wave0 = now_ms();
        total = poa_arena_capacity(c.arena);
        d_base = poa_arena_borrow(c.arena, total);
        d_slots = (PoaChainSlot *)dtake((size_t)nw * sizeof(PoaChainSlot));
        d_cp = (PoaChainParams *)dtake(sizeof(PoaChainParams));
        d_prm = (PoaParamsDev *)dtake(sizeof(PoaParamsDev));
        d_cursors = (unsigned long long *)dtake((size_t)32 * sizeof(unsigned long long));
        d_sync = (PoaChainSync *)dtake(sizeof(PoaChainSync));
        for (int t = 0; t < nw; ++t) n_tasks += plans[t].n_reads - 1;
        d_tasks = (int32_t *)dtake((size_t)std::max<int64_t>(n_tasks, 1) * 4);
        for (int t = 0; t < nw; ++t) reads_bytes += plans[t].reads_bytes;
        h_reads = (uint8_t *)pinned_get(0, reads_bytes + 256);
        d_reads = dtake(reads_bytes);
        size_t roff = 0;
        auto rtake = [&](size_t b) { uint8_t *q = d_reads + roff; roff += al256(b); return q; };
        auto gtake = [&](size_t b) { return dtake(b); };
        hs.resize((size_t)nw);
        for (int t = 0; t < nw; ++t) {
            const GroupPlan &p = plans[t];
            const abpoa_gpu_group_t &in = c.groups[p.g];
            PoaChainSlot &s = hs[t]; memset(&s, 0, sizeof s);
            chain_slot_layout(&s, p.n_cap, p.qmax, p.n_reads, c.K, c.A, c.m, c.W, c.record, gtake, c.strand, c.ps);
            chain_slot_reads(&s, p.n_reads, p.bases, rtake, c.qv);
            int32_t *hoff = (int32_t *)(h_reads + ((const uint8_t *)s.read_off - d_reads)), *hw = (int32_t *)(h_reads + ((const uint8_t *)s.read_w - d_reads));
            int acc = 0;
            for (int i = 0; i < p.n_reads; ++i) {
                hoff[i] = acc; acc += in.seq_lens[i];
                hw[i] = poa_band_halfwidth(c.abpt, in.seq_lens[i]);
                const int bc = (2 * hw[i] + 1 + 104 + (c.lg ? POA_LG_ROW_CELLS(16) : 0) + 7) / 8 * 8;
                if (bc > band_cells) band_cells = bc;
            }
            hoff[p.n_reads] = acc;
        }
        /* the read bytes themselves: half a gigabyte at BASELINE size, copied into the pinned buffer by all workers; -Q: the
         * weights too (plan_groups checked that they fit a byte), 1 for a read without them */
        {
            std::atomic<int> nx(0);
            auto copy_reads = [&]() {
                for (int t; (t = nx.fetch_add(1)) < nw;) {
                    const abpoa_gpu_group_t &in = c.groups[plans[t].g];
                    uint8_t *q = h_reads + (hs[t].reads - d_reads);
                    for (int i = 0; i < in.n_seq; ++i) { memcpy(q, in.seqs[i], (size_t)in.seq_lens[i]); q += in.seq_lens[i]; }
                    if (!c.qv) continue;
                    uint8_t *w = h_reads + (hs[t].read_qw - d_reads);
                    for (int i = 0; i < in.n_seq; ++i) {
                        const int *qw = in.qual_weights ? in.qual_weights[i] : NULL;
                        if (qw) for (int j = 0; j < in.seq_lens[i]; ++j) w[j] = (uint8_t)qw[j];
                        else memset(w, 1, (size_t)in.seq_lens[i]);
                        w += in.seq_lens[i];
                    }
                }
            };
            const int nth = reads_bytes < (8u << 20) ? 1 : std::max(1, std::min(c.n_workers, 16));
            std::vector<std::thread> th;
            for (int w = 1; w < nth; ++w) th.emplace_back(copy_reads);
            copy_reads();
            for (auto &x : th) x.join();
        }
        t_staged = now_ms();
        /* round index lists (run_rounds): every group is listed from round 1 to rounds_extra() rounds past its last read.
         * Reserved on both schedules: the wave's layout up to the plane pool does not depend on the schedule. */
        idx_n = (size_t)n_tasks;
        for (int t = 0; t < nw; ++t) idx_n += (size_t)rounds_extra(c.strand, plans[t].n_reads);
        d_idx = (int32_t *)dtake(std::max<size_t>(idx_n, 1) * 4);
        /* export buffers */
        h_exoff.resize((size_t)nw); h_excap.resize((size_t)nw);
        for (int t = 0; t < nw; ++t) {
            const GroupPlan &p = plans[t];
            const int64_t cap = 4 + 5ll * p.n_cap + 4ll * 3 * p.n_cap + (int64_t)p.n_cap * 2;
            h_exoff[t] = ex_words; h_excap[t] = (int32_t)std::min<int64_t>(cap, INT32_MAX); ex_words += (cap + 63) & ~63ll;
        }
        d_exoff = (int64_t *)dtake((size_t)nw * 8); d_excap = (int32_t *)dtake((size_t)nw * 4);
        d_msaoff = c.want_msa ? (int64_t *)dtake((size_t)nw * 8) : NULL;          /* MSA record offsets */
        d_gfaoff = c.want_gfa ? (int64_t *)dtake((size_t)nw * 8) : NULL;          /* GFA record offsets */
        /* the export buffer and the plane pool share what is left: planes are dead when the export runs */
        doff = al256(doff);
        if (doff > total) poa_die("libabpoa_b200/chain", "wave layout (%zu bytes) exceeds the arena (%zu bytes)", doff, total);
        if (doff + (size_t)ex_words * 4 + (32 << 20) > total) return false;       /* cannot happen with the wave sizing; be safe */
        d_pool = d_base + doff; pool_bytes = total - doff;
        d_ex = (int32_t *)d_pool;
        return true;
    }

    /* The inputs go up on stream 0 of the wave, the seed kernel puts every group's first read into its graph, and the
     * cohort streams fork from there.  `idx`: the round index lists (round schedule only). */
    void upload_and_seed(const std::vector<int32_t> &idx) {
        for (Cohort &k : coh) { CK(cudaStreamCreateWithFlags(&k.st, cudaStreamNonBlocking)); CK(cudaEventCreate(&k.ev_end)); }
        s0 = coh[0].st;
        CK(cudaEventCreateWithFlags(&ev_up, cudaEventDisableTiming)); CK(cudaEventCreate(&ev_t0)); CK(cudaEventCreate(&ev_t1));
        const abpoa_para_t *abpt = c.abpt;
        PoaChainParams hcp; memset(&hcp, 0, sizeof hcp);
        hcp.K = c.K; hcp.A = c.A; hcp.m = c.m; hcp.max_mat = abpt->max_mat; hcp.min_mis = abpt->min_mis; hcp.o1 = abpt->gap_open1; hcp.e1 = abpt->gap_ext1;
        hcp.oe1 = abpt->gap_open1 + abpt->gap_ext1; hcp.oe2 = abpt->gap_open2 + abpt->gap_ext2; hcp.record = c.record ? 1 : 0; hcp.P = c.P; hcp.W = c.W;
        hcp.cons_algrm = c.mf ? 1 : 0; hcp.amb_strand = c.strand ? 1 : 0;
        PoaParamsDev hprm; poa_fill_params(&hprm, c.abpt, 15);
        CK(cudaMemcpyAsync(d_reads, h_reads, reads_bytes, cudaMemcpyHostToDevice, s0));
        CK(cudaMemcpyAsync(d_slots, hs.data(), (size_t)nw * sizeof(PoaChainSlot), cudaMemcpyHostToDevice, s0));
        CK(cudaMemcpyAsync(d_cp, &hcp, sizeof hcp, cudaMemcpyHostToDevice, s0));
        CK(cudaMemcpyAsync(d_prm, &hprm, sizeof hprm, cudaMemcpyHostToDevice, s0));
        if (!idx.empty()) CK(cudaMemcpyAsync(d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, s0));
        CK(cudaMemcpyAsync(d_exoff, h_exoff.data(), (size_t)nw * 8, cudaMemcpyHostToDevice, s0));
        CK(cudaMemcpyAsync(d_excap, h_excap.data(), (size_t)nw * 4, cudaMemcpyHostToDevice, s0));
        CK(cudaMemsetAsync(d_cursors, 0, (size_t)32 * sizeof(unsigned long long), s0));
        h2d = reads_bytes + (uint64_t)nw * sizeof(PoaChainSlot) + sizeof hcp + sizeof hprm + idx.size() * 4 + (uint64_t)nw * 12;
        /* timed region of the device work: inputs are resident when ev_t0 fires */
        CK(cudaEventRecord(ev_t0, s0));
        if (c.lg) { if (c.ps) poa_chain_seed_kernel<true, true><<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw);
                    else poa_chain_seed_kernel<false, true><<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw); }
        else if (c.ps) poa_chain_seed_kernel<true, false><<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw);
        else poa_chain_seed_kernel<false, false><<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw);
        CK(cudaGetLastError());
        CK(cudaEventRecord(ev_up, s0));
        static const size_t smem_budget = [] { const char *e = getenv("ABPOA_GPU_SMEM_KB"); return (size_t)(e && *e ? atoi(e) : 28) * 1024; }();
        poa_pick_ring(abpt->gap_mode, 16, band_cells, smem_budget, &ring_rows, &ring_cells);
        launches = 1;
        gaps[0] = abpt->gap_ext1; gaps[1] = abpt->gap_open1 + abpt->gap_ext1; gaps[2] = abpt->gap_ext2; gaps[3] = abpt->gap_open2 + abpt->gap_ext2;
        t_uploaded = now_ms();
        for (size_t k = 1; k < coh.size(); ++k) CK(cudaStreamWaitEvent(coh[k].st, ev_up, 0));
    }

    /* Free-running schedule: every group has a private plane slab and advances at its own pace; two persistent kernels
     * hand the groups back and forth through the task queue of PoaChainSync. */
    void run_free_running() {
        coh.resize(1);
        /* slabs: shares of the pool proportional to the estimates */
        double est_tot = 0;
        for (int t = 0; t < nw; ++t) est_tot += plans[t].pool_units_est;
        static const double slab_x = [] { const char *e = getenv("ABPOA_GPU_CHAIN_SLAB_X"); return e && *e ? atof(e) : 0.0; }();      /* experiment: compact slabs */
        size_t o = 0;
        for (int t = 0; t < nw; ++t) {
            size_t share = (size_t)((double)pool_bytes * plans[t].pool_units_est / est_tot) & ~(size_t)255;
            if (slab_x > 0) share = std::min(share, (size_t)(plans[t].pool_units_est * 16.0 * slab_x) & ~(size_t)255);
            hs[t].pool_base = d_pool + o; hs[t].pool_units = share / 16; hs[t].pool_cursor = NULL;
            o += share;
        }
        upload_and_seed({});
        /* two persistent kernels: the fuse workers first (one CTA per SM; they must be resident while alignment warps
         * wait for them -- 10 alignment CTAs, the most one SM takes, leave registers and shared memory for one), then one
         * alignment warp per group */
        static const double watchdog_s = [] { const char *e = getenv("ABPOA_GPU_CHAIN_WATCHDOG_S"); return e && *e ? atof(e) : 30.0; }();
        static const int fuse_per_sm = [] { const char *e = getenv("ABPOA_GPU_CHAIN_FUSE_PER_SM"); return e && *e ? std::max(1, atoi(e)) : 1; }();
        PoaChainSync hsync; memset(&hsync, 0, sizeof hsync);
        hsync.total = (int32_t)n_tasks; hsync.watchdog_ns = (unsigned long long)(watchdog_s * 1e9); hsync.tasks = d_tasks;
        CK(cudaMemcpyAsync(d_sync, &hsync, sizeof hsync, cudaMemcpyHostToDevice, s0));
        CK(cudaMemsetAsync(d_tasks, 0xff, (size_t)std::max<int64_t>(n_tasks, 1) * 4, s0));
        CK(cudaStreamCreateWithFlags(&st_dp, cudaStreamNonBlocking));
        cudaEvent_t ev_sync; CK(cudaEventCreateWithFlags(&ev_sync, cudaEventDisableTiming));
        CK(cudaEventRecord(ev_sync, s0));
        static const int fuse_cap = [] { const char *e = getenv("ABPOA_GPU_CHAIN_FUSE_WORKERS"); return e && *e ? std::max(1, atoi(e)) : (1 << 30); }();
        const int n_fuse = std::max(1, std::min(std::min(nw, c.sm_count * fuse_per_sm), fuse_cap));
        /* Both persistent kernels must ask for the SAME shared-memory configuration of the SM: a resident CTA pins the
         * SM's L1/shared split, and the other kernel's CTAs are only dispatched to SMs whose split matches its launch --
         * with one fuse CTA on every SM (default split of a 5 KB kernel: 64 KB) the alignment grid (split: maximum) never
         * started, and neither kernel ever ends by itself (measured: the fuse workers' watchdog fired, then the alignment
         * grid ran). */
        void (*const fuse_worker)(PoaChainSlot *, PoaChainSync *, const PoaChainParams *) =
            c.ext ? (c.ps ? poa_chain_fuse_worker_kernel<true, false, true> : poa_chain_fuse_worker_kernel<false, false, true>)
            : c.lg ? (c.ps ? poa_chain_fuse_worker_kernel<true, true> : poa_chain_fuse_worker_kernel<false, true>)
                   : (c.ps ? poa_chain_fuse_worker_kernel<true, false> : poa_chain_fuse_worker_kernel<false, false>);
        CK(cudaFuncSetAttribute(fuse_worker, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        static const bool dp_first = [] { const char *e = getenv("ABPOA_GPU_CHAIN_DP_FIRST"); return e && *e == '1'; }();     /* experiment */
        CK(cudaStreamWaitEvent(st_dp, ev_sync, 0));
        if (dp_first) CK(poa_launch_chain_dp_worker(c.abpt->gap_mode, gaps, d_slots, d_sync, nw, d_cp, c.strand, c.ps, c.ext, d_prm, ring_rows, ring_cells, st_dp));
        fuse_worker<<<n_fuse, POA_CHAIN_T, 0, s0>>>(d_slots, d_sync, d_cp);
        CK(cudaGetLastError());
        if (!dp_first) CK(poa_launch_chain_dp_worker(c.abpt->gap_mode, gaps, d_slots, d_sync, nw, d_cp, c.strand, c.ps, c.ext, d_prm, ring_rows, ring_cells, st_dp));
        cudaEvent_t ev_dp; CK(cudaEventCreateWithFlags(&ev_dp, cudaEventDisableTiming));
        CK(cudaEventRecord(ev_dp, st_dp));
        CK(cudaStreamWaitEvent(s0, ev_dp, 0));
        CK(cudaEventDestroy(ev_sync)); CK(cudaEventDestroy(ev_dp));
        launches += 2;
    }

    /* Round schedule: per round and cohort two kernels on the cohort's stream; the jobs of a cohort bump-allocate their
     * planes from the cohort's share of the pool.  Cohorts: each cohort's alignment kernel is one CTA (warp) per group; with
     * at most one CTA per SM per cohort the concurrently running kernels of all cohorts load every SM alike (a 250-CTA grid
     * next to three more would put twice as many warps on the first 118 SMs of an H100 as on the rest, and a round ends
     * when its slowest warp does). */
    void run_rounds() {
        const int n_coh = c.cohorts ? c.cohorts : std::max(1, std::min(16, (nw + c.sm_count - 1) / c.sm_count));
        coh.resize((size_t)std::min(n_coh, nw));
        for (int t = 0; t < nw; ++t) coh[(size_t)t % coh.size()].members.push_back(t);
        /* pool shares per cohort, proportional to the estimates */
        std::vector<double> est(coh.size(), 0.0); double est_tot = 0;
        for (size_t k = 0; k < coh.size(); ++k) { for (int t : coh[k].members) est[k] += plans[t].pool_units_est; est_tot += est[k]; }
        size_t o = 0;
        for (size_t k = 0; k < coh.size(); ++k) {
            const size_t share = k + 1 == coh.size() ? pool_bytes - o : (size_t)((double)pool_bytes * est[k] / est_tot) & ~(size_t)255;
            for (int t : coh[k].members) { hs[t].pool_base = d_pool + o; hs[t].pool_units = share / 16; hs[t].pool_cursor = d_cursors + 2 * k; }
            o += share;
        }
        /* round index lists per cohort: wave-local slot indices of the groups that still have a read r */
        std::vector<int32_t> h_idx; std::vector<std::vector<std::pair<size_t, int>>> round_of(coh.size());   /* (offset into h_idx, count) per round */
        int n_rounds = 0;
        for (int t = 0; t < nw; ++t) n_rounds = std::max(n_rounds, plans[t].n_reads - 1 + rounds_extra(c.strand, plans[t].n_reads));
        for (size_t k = 0; k < coh.size(); ++k)
            for (int r = 1; r <= n_rounds; ++r) {
                const size_t at = h_idx.size(); int cnt = 0;
                for (int t : coh[k].members) if (plans[t].n_reads + rounds_extra(c.strand, plans[t].n_reads) > r) { h_idx.push_back(t); ++cnt; }
                round_of[k].push_back({at, cnt});
            }
        if (h_idx.size() != idx_n) poa_die("libabpoa_b200/chain", "round index lists (%zu entries) do not fill their region (%zu)", h_idx.size(), idx_n);
        upload_and_seed(h_idx);
        /* round-major enqueue: every cohort's stream gets its first kernels at once */
        for (int r = 1; r <= n_rounds; ++r)
            for (size_t k = 0; k < coh.size(); ++k) {
                cudaStream_t st = coh[k].st;
                const std::pair<size_t, int> &ro = round_of[k][(size_t)r - 1];
                if (ro.second == 0) continue;
                cudaEvent_t e0, e1, e2; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
                coh[k].marks.push_back(e0); coh[k].marks.push_back(e1); coh[k].marks.push_back(e2);
                CK(cudaEventRecord(e0, st));
                CK(poa_launch_chain_align_p16(c.abpt->gap_mode, gaps, d_slots, d_idx + ro.first, ro.second, r, d_cp, c.strand, c.ps, c.ext, d_prm, ring_rows, ring_cells, st));
                CK(cudaEventRecord(e1, st));
                void (*const fuse)(PoaChainSlot *, const int32_t *, const PoaChainParams *, int, int) =
                    c.ext ? (c.ps ? poa_chain_fuse_kernel<true, false, true> : poa_chain_fuse_kernel<false, false, true>)
                    : c.lg ? (c.ps ? poa_chain_fuse_kernel<true, true> : poa_chain_fuse_kernel<false, true>)
                           : (c.ps ? poa_chain_fuse_kernel<true, false> : poa_chain_fuse_kernel<false, false>);
                fuse<<<ro.second, POA_CHAIN_T, 0, st>>>(d_slots, d_idx + ro.first, d_cp, ro.second, r);
                CK(cudaGetLastError());
                CK(cudaEventRecord(e2, st));
                launches += 2;
            }
    }

    /* Join the cohort streams, run the result kernels and copy back what the host needs; the arena borrow ends here.
     * Default: the consensus on the device (chain_cons_path), only consensus bytes come back.  export_graph: the whole graph
     * comes back (compact export) and the host layer computes the consensus on it -- the cross-check of the device graph
     * against the host code.  RC-MSA: the rows are always the device's (poa_chain_msa_kernel); -r1 needs no consensus.
     * GFA: the record is always the device's (poa_chain_gfa_kernel); -r3 needs no consensus, and without a writer neither
     * kernel runs. */
    void collect() {
        for (size_t k = 0; k < coh.size(); ++k) CK(cudaEventRecord(coh[k].ev_end, coh[k].st));
        t_enqueued = now_ms();
        for (size_t k = 1; k < coh.size(); ++k) CK(cudaStreamWaitEvent(s0, coh[k].ev_end, 0));
        CK(cudaEventRecord(ev_t1, s0));
        const bool export_graph = c.export_graph, want_msa = c.want_msa, want_gfa = c.want_gfa;
        unsigned long long *d_ccur = d_cursors;               /* the pool cursors are idle now: reuse the first as the record cursor */
        int64_t *d_recoff = d_exoff;                          /* and the export offsets as record offsets */
        /* the MSA / GFA records share the consensus records' cursor, behind the export records when the graph comes back too */
        if (c.abpt->out_gfa) cons_kernel = !export_graph && want_gfa && c.with_cons;
        else cons_kernel = !export_graph && (!want_msa || c.with_cons);
        const bool any_rec = cons_kernel || want_msa || want_gfa;
        rec_base = export_graph ? (unsigned long long)ex_words : 0;
        if (export_graph) poa_chain_export_kernel<<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw, d_ex, d_exoff, d_excap);
        if (any_rec) CK(cudaMemsetAsync(d_ccur, 0, sizeof(unsigned long long), s0));
        if (cons_kernel) poa_chain_consensus_kernel<<<nw, c.mf ? POA_CHAIN_T : 32, 0, s0>>>(d_slots, d_cp, nw, d_ex, d_ccur, (unsigned long long)(pool_bytes / 4), d_recoff);
        CK(cudaGetLastError());
        launches += (export_graph || cons_kernel) ? 1 : 0;
        if (want_msa) {
            poa_chain_msa_kernel<<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw, c.with_cons, export_graph && c.with_cons, d_ex, d_ccur, rec_base,
                                                            (unsigned long long)(pool_bytes / 4), d_msaoff);
            CK(cudaGetLastError());
            ++launches;
        }
        if (want_gfa) {
            poa_chain_gfa_kernel<<<nw, POA_CHAIN_T, 0, s0>>>(d_slots, d_cp, nw, c.with_cons, export_graph && c.with_cons, d_ex, d_ccur, rec_base,
                                                            (unsigned long long)(pool_bytes / 4), d_gfaoff);
            CK(cudaGetLastError());
            ++launches;
        }
        fin.resize((size_t)nw);
        PoaChainSlot *h_fin = (PoaChainSlot *)pinned_get(1, (size_t)nw * sizeof(PoaChainSlot));
        CK(cudaMemcpyAsync(h_fin, d_slots, (size_t)nw * sizeof(PoaChainSlot), cudaMemcpyDeviceToHost, s0));
        CK(cudaStreamSynchronize(s0));
        CK(cudaEventElapsedTime(&dev_ms, ev_t0, ev_t1));
        memcpy(fin.data(), h_fin, (size_t)nw * sizeof(PoaChainSlot));
        pinned_put(1, h_fin);
        if (c.free_run) {
            PoaChainSync hs2; CK(cudaMemcpy(&hs2, d_sync, sizeof hs2, cudaMemcpyDeviceToHost));
            if (hs2.abort) fprintf(stderr, "[libabpoa_b200/chain] watchdog: the alignment and the fuse kernel did not make progress together within ABPOA_GPU_CHAIN_WATCHDOG_S; "
                                           "unfinished groups go to the launch engine (ABPOA_GPU_CHAIN_ROUNDS=1 selects the round schedule)\n");
        }
        t_dev_done = now_ms();
        /* device results: record offsets, then one copy of all records */
        recoff.assign((size_t)nw, -1); msaoff.assign((size_t)nw, -1); gfaoff.assign((size_t)nw, -1);
        if (any_rec) {                             /* records: [rec_base, rec_base + cursor) words of d_ex */
            int64_t *h_ro = NULL; CK(cudaHostAlloc((void **)&h_ro, (size_t)nw * 24 + 8, cudaHostAllocDefault));
            if (cons_kernel) CK(cudaMemcpyAsync(h_ro, d_recoff, (size_t)nw * 8, cudaMemcpyDeviceToHost, s0));
            if (want_msa) CK(cudaMemcpyAsync(h_ro + nw, d_msaoff, (size_t)nw * 8, cudaMemcpyDeviceToHost, s0));
            if (want_gfa) CK(cudaMemcpyAsync(h_ro + 2 * nw, d_gfaoff, (size_t)nw * 8, cudaMemcpyDeviceToHost, s0));
            CK(cudaMemcpyAsync(h_ro + 3 * nw, d_ccur, 8, cudaMemcpyDeviceToHost, s0));
            CK(cudaStreamSynchronize(s0));
            if (cons_kernel) memcpy(recoff.data(), h_ro, (size_t)nw * 8);
            if (want_msa) memcpy(msaoff.data(), h_ro + nw, (size_t)nw * 8);
            if (want_gfa) memcpy(gfaoff.data(), h_ro + 2 * nw, (size_t)nw * 8);
            cons_words = (unsigned long long)h_ro[3 * nw];
            CK(cudaFreeHost(h_ro));
            if (rec_base + cons_words > pool_bytes / 4) cons_words = pool_bytes / 4 - rec_base;
            h_cons = (int32_t *)pinned_get(2, (size_t)std::max<unsigned long long>(cons_words, 1) * 4);
            if (cons_words) CK(cudaMemcpyAsync(h_cons, d_ex + rec_base, (size_t)cons_words * 4, cudaMemcpyDeviceToHost, s0));
        }
        /* exported graphs: word counts from header words 0..3 of every record */
        std::vector<int32_t> hdr4((size_t)nw * 4);
        if (export_graph) {
            int32_t *h_hdr = NULL; CK(cudaHostAlloc((void **)&h_hdr, (size_t)nw * 16, cudaHostAllocDefault));
            for (int t = 0; t < nw; ++t) CK(cudaMemcpyAsync(h_hdr + 4 * t, d_ex + h_exoff[t], 16, cudaMemcpyDeviceToHost, s0));
            CK(cudaStreamSynchronize(s0));
            memcpy(hdr4.data(), h_hdr, (size_t)nw * 16);
            CK(cudaFreeHost(h_hdr));
        }
        words.assign((size_t)nw, 0); hoff2.assign((size_t)nw, 0);
        for (int t = 0; t < nw; ++t) {
            const bool rec_ok = (!cons_kernel || recoff[t] >= 0) && (!want_msa || msaoff[t] >= 0) && (!want_gfa || gfaoff[t] >= 0);
            if (!export_graph) { words[t] = (!fin[t].failed && rec_ok) ? 1 : 0; continue; }
            if (fin[t].failed || hdr4[4 * t] < 2 || !rec_ok) continue;
            words[t] = 4 + 5ll * hdr4[4 * t] + 4ll * hdr4[4 * t + 1] + hdr4[4 * t + 2];
            hoff2[t] = tot_words; tot_words += words[t];
        }
        h_ex = (int32_t *)pinned_get(3, (size_t)std::max<int64_t>(tot_words, 1) * 4);
        if (export_graph) for (int t = 0; t < nw; ++t) if (words[t]) CK(cudaMemcpyAsync(h_ex + hoff2[t], d_ex + h_exoff[t], (size_t)words[t] * 4, cudaMemcpyDeviceToHost, s0));
        /* per-read records */
        rs.resize((size_t)nw); rn.resize((size_t)nw); rh.resize((size_t)nw);
        if (c.record) for (int t = 0; t < nw; ++t) {
            const int nr = plans[t].n_reads;
            rs[t].resize(nr); rn[t].resize(nr); rh[t].resize(nr);
            CK(cudaMemcpyAsync(rs[t].data(), fin[t].rec_score, (size_t)nr * 4, cudaMemcpyDeviceToHost, s0));
            CK(cudaMemcpyAsync(rn[t].data(), fin[t].rec_nops, (size_t)nr * 4, cudaMemcpyDeviceToHost, s0));
            CK(cudaMemcpyAsync(rh[t].data(), fin[t].rec_hash, (size_t)nr * 8, cudaMemcpyDeviceToHost, s0));
        }
        /* -s: which reads were fused as their reverse complement */
        rc.resize((size_t)nw);
        uint64_t rc_bytes = 0;
        if (c.strand) for (int t = 0; t < nw; ++t) {
            rc[t].resize((size_t)plans[t].n_reads);
            CK(cudaMemcpyAsync(rc[t].data(), fin[t].read_rc, (size_t)plans[t].n_reads, cudaMemcpyDeviceToHost, s0));
            rc_bytes += (uint64_t)plans[t].n_reads;
        }
        CK(cudaStreamSynchronize(s0));
        d2h = (uint64_t)tot_words * 4 + (uint64_t)cons_words * 4 + (uint64_t)nw * (sizeof(PoaChainSlot) + 16) + rc_bytes;
        poa_arena_return(c.arena, d_base, total); d_base = NULL;
        t_copied = now_ms();
    }

    /* host: each finished group's result record (rebuilt graph or the device's consensus, the device's MSA rows, per-read
     * records) on the worker threads; the groups that left the chain go to the launch engine */
    void install() {
        std::atomic<int> next(0), failed(0);
        std::vector<int> failed_groups; std::mutex fmu;
        const int nth = std::max(1, std::min(c.n_workers, nw));
        std::vector<std::thread> th;
        for (int w = 0; w < nth; ++w)
            th.emplace_back([&]() {
                abpoa_para_t *abpt = c.abpt;
                abpoa_t *ab = abpoa_init();
                for (;;) {
                    const int t = next.fetch_add(1);
                    if (t >= nw) break;
                    const GroupPlan &p = plans[t];
                    if (fin[t].failed || !words[t] || fin[t].fused != p.n_reads) {
                        if (c.verbose) fprintf(stderr, "[chain] group %d left the device chain after %d reads (flags 0x%x)\n", p.g, fin[t].fused, fin[t].failed);
                        std::lock_guard<std::mutex> lk(fmu); failed_groups.push_back(p.g); failed += 1; continue;
                    }
                    abpoa_gpu_group_result_t *o = &c.results[p.g];
                    memset(o, 0, sizeof *o);
                    abpoa_reset(ab, abpt, p.qmax);
                    abpoa_seq_t *abs = ab->abs;
                    abs->n_seq = p.n_reads; poa_seq_reserve(abs);
                    int n_rc_dp = 0;                           /* -s: second alignments (the reverse complement of a weak hit) */
                    for (int i = 0; i < p.n_reads; ++i) {
                        abs->is_rc[i] = c.strand ? rc[t][i] & 1 : 0; abs->name[i].l = 0;
                        if (c.strand) n_rc_dp += rc[t][i] >> 1 & 1;
                    }
                    if (c.export_graph) poa_graph_import(ab, abpt, h_ex + hoff2[t]);
                    else if (cons_kernel) {                    /* the device's consensus: base | coverage << 8 per position */
                        const int32_t *rec = h_cons + recoff[t];
                        const int len = rec[0];
                        std::vector<uint8_t> cb((size_t)(len > 0 ? len : 1)); std::vector<int> cc((size_t)(len > 0 ? len : 1));
                        for (int j = 0; j < len; ++j) { cb[j] = (uint8_t)(rec[1 + j] & 0xff); cc[j] = rec[1 + j] >> 8; }
                        poa_cons_install(ab, p.n_reads, len, cb.data(), cc.data());
                    }
                    if (c.want_msa) {                          /* the device's rows: [msa_len, n_rows, bytes] */
                        const int32_t *rec = h_cons + (msaoff[t] - (int64_t)rec_base);
                        poa_msa_install(ab, p.n_reads, rec[1], rec[0], reinterpret_cast<const uint8_t *>(rec + 2));
                    }
                    if (c.want_gfa) poa_gfa_install(ab, h_cons + (gfaoff[t] - (int64_t)rec_base));     /* printed by abpoa_generate_gfa */
                    poa_finish_group_result(ab, abpt, o, c.emit, p.g);
                    if (c.want_gfa) poa_gfa_install(ab, NULL);
                    o->dp_cells = fin[t].cells; o->n_aligned = p.n_reads - 1 + n_rc_dp;     /* the launch engine counts every DP */
                    if (c.record) {
                        const int nr = p.n_reads;
                        o->read_best_score = (int32_t *)poa_xcalloc((size_t)nr, sizeof(int32_t));
                        o->read_n_cigar = (int32_t *)poa_xcalloc((size_t)nr, sizeof(int32_t));
                        o->read_cigar_hash = (uint64_t *)poa_xcalloc((size_t)nr, sizeof(uint64_t));
                        o->read_cigar_hash[0] = 1469598103934665603ull;               /* FNV-1a of an empty CIGAR, as the other engine records it */
                        for (int i = 1; i < nr; ++i) { o->read_best_score[i] = rs[t][i]; o->read_n_cigar[i] = rn[t][i]; o->read_cigar_hash[i] = rh[t][i]; }
                    }
                }
                abpoa_free(ab);
            });
        for (auto &x : th) x.join();
        for (int g : failed_groups) fallback.push_back(g);
        n_failed = failed.load();
    }

    /* PoaChainStats and the ABPOA_GPU_PROFILE lines */
    void account() {
        int64_t cells = 0, alns = 0, fwd_clk = 0, bt_clk = 0;
        for (int t = 0; t < nw; ++t) if (!fin[t].failed && words[t] && fin[t].fused == plans[t].n_reads) { cells += fin[t].cells; alns += plans[t].n_reads - 1; fwd_clk += fin[t].fwd_clk; bt_clk += fin[t].bt_clk; }
        double dp_ms = 0, fuse_ms = 0, wait_ms = 0; int64_t n_marks = 0;
        if (c.free_run) {                 /* no per-launch marks: time inside the alignments (SM cycles) and inside chain_fuse, summed over groups */
            int khz = 0; if (cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, c.dev) != cudaSuccess || khz <= 0) khz = 1965000;
            for (int t = 0; t < nw; ++t) {
                dp_ms += (double)(fin[t].fwd_clk + fin[t].bt_clk) / (double)khz; fuse_ms += (double)fin[t].fuse_ns * 1e-6; wait_ms += (double)fin[t].wait_ns * 1e-6;
                n_marks += fin[t].fused > 0 ? fin[t].fused - 1 : 0;
            }
        } else {
            for (Cohort &k : coh)
                for (size_t j = 0; j + 2 < k.marks.size(); j += 3) {
                    float a = 0.f, b = 0.f;
                    CK(cudaEventElapsedTime(&a, k.marks[j], k.marks[j + 1])); CK(cudaEventElapsedTime(&b, k.marks[j + 1], k.marks[j + 2]));
                    dp_ms += a; fuse_ms += b; ++n_marks;
                }
        }
        if (PoaChainStats *stats = c.stats) {
            stats->device_ms += dev_ms; stats->cells += cells; stats->alignments += alns; stats->launches += launches;
            stats->h2d_bytes += h2d; stats->d2h_bytes += d2h; stats->groups_done += nw - n_failed; stats->groups_failed += n_failed;
            stats->fwd_clk += fwd_clk; stats->bt_clk += bt_clk;
            stats->dp_ms += dp_ms; stats->fuse_ms += fuse_ms; stats->dp_launches += n_marks; stats->fuse_launches += n_marks;
            stats->wait_ms += wait_ms; stats->free_running = c.free_run ? 1 : 0;
        }
        if (!c.verbose) return;
#ifdef POA_KPROF
        {
            double pf[6] = {0, 0, 0, 0, 0, 0}; double na = 0;
            for (int t = 0; t < nw; ++t) { for (int z = 0; z < 6; ++z) pf[z] += (double)fin[t].prof[z]; na += fin[t].fused > 0 ? fin[t].fused - 1 : 0; }
            double bd[5] = {0, 0, 0, 0, 0};
            for (int t = 0; t < nw; ++t) for (int z = 0; z < 5; ++z) bd[z] += (double)fin[t].btdiag[z];
            if (na > 0) fprintf(stderr, "[chain, backtrace per alignment] %.0f steps in %.0f speculative rounds, %.0f general steps costing %.0f k-cycles, "
                                        "%.1f rows with their F planes recomputed\n", bd[0] / na, bd[1] / na, bd[2] / na, bd[3] / na, bd[4] / na);
            if (na > 0) fprintf(stderr, "[chain, k-cycles/alignment] -DPOA_KPROF phases: setup %.0f pred %.0f compute %.0f store %.0f rowmax %.0f tail+prefetch %.0f\n",
                                pf[0] / na / 1e3, pf[1] / na / 1e3, pf[2] / na / 1e3, pf[3] / na / 1e3, pf[4] / na / 1e3, pf[5] / na / 1e3);
        }
#endif
        if (c.free_run)
            fprintf(stderr, "[chain] free-running: per group on average %.1f ms inside alignments + %.1f ms inside fuse (waited %.1f ms for fuse workers incl. the fuse itself), %lld alignments\n",
                    dp_ms / nw, fuse_ms / nw, wait_ms / nw, (long long)n_marks);
        else
            fprintf(stderr, "[chain] DP kernels %.1f ms + fuse kernels %.1f ms summed over %zu concurrent cohort streams (%lld rounds)\n", dp_ms, fuse_ms, coh.size(), (long long)n_marks);
        fprintf(stderr, "[chain] wave of %d groups (%zu cohorts, K=%d): stage %.0f + upload-enqueue %.0f + launch-enqueue %.0f ms, stage+launch+device %.0f ms (device %.1f ms), export copy %.0f ms, import+consensus %.0f ms; "
                        "static %.2f GB, pool %.2f GB, export %.1f MB; %d groups handed to the launch engine\n",
                nw, coh.size(), c.K, t_staged - t_wave0, t_uploaded - t_staged, t_enqueued - t_uploaded, t_dev_done - t_wave0, dev_ms, t_copied - t_dev_done, now_ms() - t_copied,
                (double)doff / 1e9, (double)pool_bytes / 1e9, (double)tot_words * 4 / 1e6, n_failed);
    }
};

}  // namespace

/* Run the groups listed in `todo` (eligible ones) through the device chain.  Groups that could not be
 * finished are appended to `fallback`.  Returns 0. */
int poa_chain_run(int dev, poa_arena *arena, abpoa_para_t *abpt, int n_workers, const abpoa_gpu_group_t *groups,
                  abpoa_gpu_group_result_t *results, const std::vector<int> &todo, int flags, std::vector<int> &fallback, PoaChainStats *stats,
                  struct PoaEmit *emit) {
    CK(cudaSetDevice(dev));
    const ChainCall c = chain_call(dev, arena, abpt, n_workers, groups, results, todo, flags, stats, emit);
    const std::vector<GroupPlan> plans = plan_groups(c, todo, fallback);
    if (plans.empty()) return 0;
    for (const std::pair<size_t, size_t> &w : split_waves(plans, poa_arena_capacity(arena), fallback))
        Wave(c, plans.data() + w.first, (int)(w.second - w.first), fallback).run();
    return 0;
}

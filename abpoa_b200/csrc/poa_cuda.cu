/* poa_cuda.cu -- host side of the CUDA backend: per-stream device context, job staging,
 * kernel launch, result collection.
 *
 * This is the seam the reference fills with its cpuid dispatcher
 * (src/abpoa_dispatch_simd.c:58-81 -> simd_abpoa_align_sequence_to_subgraph,
 * prototype src/abpoa_align_simd.h:12).  Here the only implementation is the sm_90a
 * kernel family in poa_kernels.cu; a missing GPU is a fatal error, never a CPU fallback.
 *
 * A "stream context" owns one CUDA stream plus grow-only pinned/HBM buffers and runs a
 * BATCH of independent alignment jobs per launch (one warp each).  The abpoa.h entry
 * point uses a batch of one; abpoa_gpu.h drives many contexts from worker threads.
 */
#include <cuda_runtime.h>
#include <atomic>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <mutex>
#include <condition_variable>
#include <algorithm>
#include <chrono>
#include <time.h>
#include "poa_internal.h"
#include "poa_device.cuh"
#include "poa_engine.h"

extern "C" cudaError_t poa_launch_align(int gap_mode, int bits, int align_mode, const PoaJobDesc *jobs,
                                        const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, cudaStream_t st);
extern "C" cudaError_t poa_launch_align_p16(int gap_mode, int align_mode, int lean, const int *gaps, const PoaJobDesc *jobs,
                                            const PoaParamsDev *prm, int n_jobs, int ring_rows, int ring_cells, cudaStream_t st);
extern "C" void poa_pick_ring(int gap_mode, int bits, int band_cells, size_t smem_budget, int *ring_rows, int *ring_cells);
extern "C" int poa_tma_enabled(void);
extern "C" int poa_lean_disabled(void);

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    poa_die("libabpoa_b200/cuda", "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); } while (0)

static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

/* ------------------------------------------------------------------ shared plane arena */
struct poa_arena {
    int dev; uint8_t *base; size_t cap;
    std::mutex mu; std::condition_variable cv;
    std::vector<std::pair<size_t, size_t>> free_list;      /* (offset, length), sorted by offset */
};

poa_arena *poa_arena_new(int dev, size_t bytes) {
    poa_arena *a = new poa_arena();
    a->dev = dev; a->cap = bytes & ~(size_t)255; a->base = NULL;
    CK(cudaSetDevice(dev));
    cudaError_t e = cudaMalloc((void **)&a->base, a->cap);
    if (e != cudaSuccess) poa_die("libabpoa_b200/cuda", "cannot reserve %zu bytes of HBM for DP planes: %s", a->cap, cudaGetErrorString(e));
    a->free_list.push_back({0, a->cap});
    return a;
}
void poa_arena_destroy(poa_arena *a) { if (!a) return; cudaSetDevice(a->dev); cudaFree(a->base); delete a; }
size_t poa_arena_capacity(const poa_arena *a) { return a->cap; }

static uint8_t *arena_take(poa_arena *a, size_t bytes) {
    bytes = al256(bytes);
    if (bytes > a->cap) poa_die("libabpoa_b200/cuda", "one launch needs %zu bytes of DP planes, arena holds %zu", bytes, a->cap);
    std::unique_lock<std::mutex> lk(a->mu);
    int waited_s = 0;
    for (;;) {
        for (size_t i = 0; i < a->free_list.size(); ++i)
            if (a->free_list[i].second >= bytes) {
                size_t off = a->free_list[i].first;
                a->free_list[i].first += bytes; a->free_list[i].second -= bytes;
                if (a->free_list[i].second == 0) a->free_list.erase(a->free_list.begin() + i);
                return a->base + off;
            }
        /* Backstop (the callers never wait here while holding planes, see poa_engine_submit): a wait
         * that lasts minutes means the arena is held by launches that cannot finish. */
        if (a->cv.wait_for(lk, std::chrono::seconds(60)) == std::cv_status::timeout) {
            waited_s += 60;
            size_t free_b = 0, largest = 0;
            for (auto &f : a->free_list) { free_b += f.second; if (f.second > largest) largest = f.second; }
            fprintf(stderr, "[libabpoa_b200/cuda] waiting %d s for %zu bytes of DP planes (arena %zu, free %zu, largest free range %zu)\n",
                    waited_s, bytes, a->cap, free_b, largest);
            if (waited_s >= 600) poa_die("libabpoa_b200/cuda", "no plane memory became available within 600 s (arena %zu bytes, request %zu)", a->cap, bytes);
        }
    }
}
static void arena_give(poa_arena *a, uint8_t *p, size_t bytes) {
    bytes = al256(bytes);
    const size_t off = (size_t)(p - a->base);
    {
        std::lock_guard<std::mutex> lk(a->mu);
        auto it = std::lower_bound(a->free_list.begin(), a->free_list.end(), std::make_pair(off, (size_t)0));
        it = a->free_list.insert(it, {off, bytes});
        if (it + 1 != a->free_list.end() && it->first + it->second == (it + 1)->first) { it->second += (it + 1)->second; a->free_list.erase(it + 1); }
        if (it != a->free_list.begin() && (it - 1)->first + (it - 1)->second == it->first) { (it - 1)->second += it->second; a->free_list.erase(it); }
    }
    a->cv.notify_all();
}

uint8_t *poa_arena_borrow(poa_arena *a, size_t bytes) { return arena_take(a, bytes); }
/* non-blocking: NULL when no free range is large enough right now */
uint8_t *poa_arena_try_borrow(poa_arena *a, size_t bytes) {
    bytes = al256(bytes);
    std::lock_guard<std::mutex> lk(a->mu);
    for (size_t i = 0; i < a->free_list.size(); ++i)
        if (a->free_list[i].second >= bytes) {
            const size_t off = a->free_list[i].first;
            a->free_list[i].first += bytes; a->free_list[i].second -= bytes;
            if (a->free_list[i].second == 0) a->free_list.erase(a->free_list.begin() + i);
            return a->base + off;
        }
    return NULL;
}
void poa_arena_return(poa_arena *a, uint8_t *p, size_t bytes) { arena_give(a, p, bytes); }

struct LaunchState {
    bool active = false;
    const abpoa_para_t *abpt = NULL; poa_job *jobs = NULL; std::vector<int> idx; int n = 0, bits = 0;
    std::vector<size_t> blob_off, work_off, cig_off;
    uint8_t *planes_base = NULL; size_t plane_bytes = 0, in_bytes = 0;
    double t_begin = 0, t_filled = 0;
};

struct poa_dev_ctx {
    LaunchState ls;
    int dev;
    poa_arena *arena;
    cudaStream_t st;
    cudaEvent_t ev_k0, ev_k1, ev_done;       /* ev_done: blocking-sync event, the host thread sleeps while the GPU works */
    uint8_t *h_in, *h_out, *d_in, *d_work, *d_planes;
    uint8_t *h_res; size_t h_res_cap;     /* mapped pinned: completion counter + PoaResultDev[] written by the kernel */
    size_t h_in_cap, h_out_cap, d_in_cap, d_work_cap, d_planes_cap;
    size_t planes_limit;              /* hard cap for the plane slab (bytes); 0 = ask the device */
    poa_engine_stats stats;
    poa_capture_fn capture; void *capture_user;
    poa_pressure_fn pressure; void *pressure_user;   /* called before this context WAITS for plane memory */
    PoaJobDesc last_desc; int last_bits, last_gap, last_rows;   /* debug: job 0 of the most recent launch */
    int last_lean, last_tma, last_ring_rows, last_ring_cells; uint64_t last_units;   /* ... how it ran, and its plane units used */
    int last_ps;                        /* ... a whole-graph global -G run of the packed kernel (LEAN but for its path scores) */
};

static void require_gpu(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        poa_die("libabpoa_b200", "no CUDA device available (%s). This library has no CPU path: the DP runs only on the GPU.",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
}

poa_dev_ctx *poa_dev_ctx_new_on(int dev) {
    require_gpu();
    poa_dev_ctx *c = new poa_dev_ctx();
    c->arena = NULL; c->st = NULL; c->h_in = c->h_out = c->d_in = c->d_work = c->d_planes = c->h_res = NULL;
    c->h_in_cap = c->h_out_cap = c->d_in_cap = c->d_work_cap = c->d_planes_cap = c->h_res_cap = c->planes_limit = 0;
    memset(&c->stats, 0, sizeof c->stats); c->capture = NULL; c->capture_user = NULL; c->pressure = NULL; c->pressure_user = NULL; memset(&c->last_desc, 0, sizeof c->last_desc);
    c->last_bits = c->last_gap = c->last_rows = 0;
    c->last_lean = c->last_tma = c->last_ring_rows = c->last_ring_cells = 0; c->last_units = 0; c->last_ps = 0;
    if (dev >= 0) { c->dev = dev; CK(cudaSetDevice(c->dev)); }
    else CK(cudaGetDevice(&c->dev));
    CK(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    CK(cudaEventCreate(&c->ev_k0)); CK(cudaEventCreate(&c->ev_k1));
    CK(cudaEventCreateWithFlags(&c->ev_done, cudaEventBlockingSync | cudaEventDisableTiming));
    return c;
}

poa_dev_ctx *poa_dev_ctx_new(void) {
    const char *env = getenv("ABPOA_GPU_DEVICE");
    return poa_dev_ctx_new_on(env && *env ? atoi(env) : -1);
}
void poa_dev_ctx_use_arena(poa_dev_ctx *c, poa_arena *a) { c->arena = a; }
void poa_dev_ctx_set_capture(poa_dev_ctx *c, poa_capture_fn fn, void *user) { c->capture = fn; c->capture_user = user; }
void poa_dev_ctx_set_pressure_cb(poa_dev_ctx *c, poa_pressure_fn fn, void *user) { c->pressure = fn; c->pressure_user = user; }

void poa_dev_ctx_free(poa_dev_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->dev);
    cudaStreamSynchronize(c->st);
    if (c->h_in) cudaFreeHost(c->h_in);
    if (c->h_out) cudaFreeHost(c->h_out);
    if (c->h_res) cudaFreeHost(c->h_res);
    if (c->d_in) cudaFree(c->d_in);
    if (c->d_work) cudaFree(c->d_work);
    if (c->d_planes) cudaFree(c->d_planes);
    cudaEventDestroy(c->ev_k0); cudaEventDestroy(c->ev_k1); cudaEventDestroy(c->ev_done);
    cudaStreamDestroy(c->st);
    delete c;
}

void poa_dev_ctx_set_planes_limit(poa_dev_ctx *c, size_t bytes) { c->planes_limit = bytes; }
const poa_engine_stats *poa_dev_ctx_stats(const poa_dev_ctx *c) { return &c->stats; }
void poa_dev_ctx_reset_stats(poa_dev_ctx *c) { memset(&c->stats, 0, sizeof c->stats); }
int poa_dev_ctx_device(const poa_dev_ctx *c) { return c->dev; }

/* wait for everything queued on the context's stream without spinning on a core */
static void stream_wait(poa_dev_ctx *c) {
    CK(cudaEventRecord(c->ev_done, c->st));
    CK(cudaEventSynchronize(c->ev_done));
}

static void release_dev(void *p) { CK(cudaFree(p)); }
static void release_host(void *p) { CK(cudaFreeHost(p)); }

static void grow_host(uint8_t **p, size_t *cap, size_t need) {
    if (need <= *cap) return;
    size_t n = al256(need * 2);
    if (*p) release_host(*p);
    CK(cudaHostAlloc((void **)p, n, cudaHostAllocDefault));
    *cap = n;
}
static void grow_dev(uint8_t **p, size_t *cap, size_t need, int slack) {
    if (need <= *cap) return;
    size_t n = al256(slack ? need * 2 : need);
    if (*p) release_dev(*p);
    cudaError_t e = cudaMalloc((void **)p, n);
    if (e != cudaSuccess && slack) { cudaGetLastError(); n = al256(need); e = cudaMalloc((void **)p, n); }
    if (e != cudaSuccess) poa_die("libabpoa_b200/cuda", "cudaMalloc of %zu bytes failed: %s", n, cudaGetErrorString(e));
    *cap = n;
}

/* Size the staging buffers once for a known workload (rows / query length per job, jobs per
 * launch) so that steady-state launches never call cudaMalloc / cudaFree (both serialise
 * the device across all streams). */
void poa_dev_ctx_reserve(poa_dev_ctx *c, int jobs, int rows_hint, int qlen_hint) {
    CK(cudaSetDevice(c->dev));
    const size_t r = (size_t)rows_hint, q = (size_t)qlen_hint, j = (size_t)jobs;
    const size_t in_b = 4096 + j * (r * 28 + q + 1024), work_b = 4096 + j * (r * (24 + 64) + (q + r + 8) * 8 + 1024 + (q + 32) * 2 * 32), out_b = 4096 + j * ((q + r + 8) * 8 + 512);
    if (in_b > c->h_in_cap) grow_host(&c->h_in, &c->h_in_cap, in_b / 2 + 1);
    if (in_b > c->d_in_cap) grow_dev(&c->d_in, &c->d_in_cap, in_b / 2 + 1, 1);
    if (work_b > c->d_work_cap) grow_dev(&c->d_work, &c->d_work_cap, work_b / 2 + 1, 1);
    if (out_b > c->h_out_cap) grow_host(&c->h_out, &c->h_out_cap, out_b / 2 + 1);
    const size_t res_b = 256 + j * sizeof(PoaResultDev);
    if (res_b > c->h_res_cap) grow_host(&c->h_res, &c->h_res_cap, res_b);
}

void poa_fill_params(PoaParamsDev *p, const abpoa_para_t *abpt, int bits) {
    memset(p, 0, sizeof *p);
    if (abpt->m > POA_MAX_M) poa_die("libabpoa_b200", "alphabet size m=%d exceeds the supported maximum %d", abpt->m, POA_MAX_M);
    p->m = abpt->m; p->align_mode = abpt->align_mode; p->gap_mode = abpt->gap_mode;
    p->e1 = abpt->gap_ext1; p->o1 = abpt->gap_open1; p->oe1 = abpt->gap_open1 + abpt->gap_ext1;
    p->e2 = abpt->gap_ext2; p->o2 = abpt->gap_open2; p->oe2 = abpt->gap_open2 + abpt->gap_ext2;
    p->zdrop = abpt->zdrop;
    p->put_gap_on_right = abpt->put_gap_on_right; p->put_gap_at_end = abpt->put_gap_at_end;
    p->ret_cigar = abpt->ret_cigar;
    (void)bits;
    memcpy(p->mat, abpt->mat, (size_t)abpt->m * abpt->m * sizeof(int));
}

/* Environment switches, read on every call (a launch costs far more than a getenv) so that tests can
 * flip them per case:
 *   ABPOA_GPU_NO_P16=1      never use the packed int16x2 kernel
 *   ABPOA_GPU_FORCE_P16=1   admit every int16/int32 job to it (the run-time range guard must then catch overflow)
 *   ABPOA_GPU_SLAB_PCT=n    give each job only n % of the estimated plane slab (forces the PLANE_OVF redo) */
static inline int env_flag(const char *name) { const char *e = getenv(name); return e && *e == '1'; }
static inline int use_p16_for(const abpoa_para_t *abpt, int qlen, int n_rows) {
    /* banded linear gaps outside local mode follow the reference's vector procedure lane for lane (band edges depend on its
     * vector width); only the generic kernel implements that ("lgx" in poa_kernels.cu) */
    if (abpt->gap_mode == ABPOA_LINEAR_GAP && abpt->align_mode != ABPOA_LOCAL_MODE && abpt->wb >= 0) return 0;
    if (env_flag("ABPOA_GPU_NO_P16")) return 0;
    if (env_flag("ABPOA_GPU_FORCE_P16")) return abpt->max_mat <= 1000 && abpt->min_mis <= 1000;
    return poa_p16_ok(abpt, qlen, n_rows);
}

static inline int planes_of(int gap_mode) { return gap_mode == ABPOA_LINEAR_GAP ? 1 : (gap_mode == ABPOA_AFFINE_GAP ? 3 : 5); }

/* plane slab (in 8-cell units) a job is given: `generous` = the full rectangle */
static uint64_t plane_units_for(const poa_job *j, int gap_mode, int generous) {
    const int P = planes_of(gap_mode);
    const uint64_t full = (uint64_t)((j->plan.qlen + 1 + 7) / 8 + 1);
    uint64_t per_row = full;
    if (!generous && j->plan.w >= 0) {
        const uint64_t est = (uint64_t)((2 * j->plan.w + 1 + 32 + 7) / 8 + 2);
        if (est < per_row) per_row = est;
        const char *pct = getenv("ABPOA_GPU_SLAB_PCT");
        if (pct && *pct) { per_row = per_row * (uint64_t)atoi(pct) / 100; if (per_row < 2) per_row = 2; }
    }
    return per_row * (uint64_t)P * (uint64_t)j->plan.n_rows;
}

/* Run `n` jobs that share parameters and score width.  Results land in pinned host memory
 * owned by the context (valid until the next run on this context). */
static inline double now_ms(void) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

/* One launch = begin (stage + H2D + kernel, returns at once) and finish (sleep until the jobs
 * report, copy CIGARs back, publish results).  A context has at most one launch outstanding;
 * a worker that owns two contexts overlaps the fusion of one half-chunk with the kernel of the other. */
/* try_only: take the planes without blocking; returns false (nothing staged, nothing held) when the arena
 * has no room right now. */
static bool run_begin(poa_dev_ctx *c, const abpoa_para_t *abpt, poa_job *jobs, const int *idx_in, int n, int bits, int generous, bool try_only = false) {
    CK(cudaSetDevice(c->dev));
    LaunchState &L = c->ls;
    L.abpt = abpt; L.jobs = jobs; L.idx.assign(idx_in, idx_in + n); L.n = n; L.bits = bits;
    const int *idx = L.idx.data();
    const double t_begin = now_ms();
    const int S = bits == 32 ? 4 : 2;          /* bits: 15 = packed int16x2 kernel, 16 / 32 = generic kernel */
    /* ---- layout of the input arena: params | descs | blobs ---- */
    size_t in_bytes = al256(sizeof(PoaParamsDev)) + al256((size_t)n * sizeof(PoaJobDesc));
    const size_t off_desc = al256(sizeof(PoaParamsDev));
    std::vector<size_t> &blob_off = L.blob_off, &work_off = L.work_off, &cig_off = L.cig_off; std::vector<size_t> qp_off(n), bt_off(n);
    blob_off.assign(n, 0); work_off.assign(n, 0); cig_off.assign(n, 0);
    std::vector<uint64_t> units(n), plane_off(n);
    for (int t = 0; t < n; ++t) { blob_off[t] = in_bytes; in_bytes += al256(jobs[idx[t]].plan.bytes); }
    /* ---- work arena: results | per job (rowinfo, rowoff, cigar) ---- */
    size_t work_bytes = al256((size_t)n * sizeof(PoaResultDev));
    for (int t = 0; t < n; ++t) {
        const poa_job &j = jobs[idx[t]];
        work_off[t] = work_bytes;
        work_bytes += al256((size_t)j.plan.n_rows * sizeof(PoaRowInfo)) + al256((size_t)j.plan.n_rows * sizeof(PoaRowOff));
        cig_off[t] = work_bytes;
        work_bytes += al256((size_t)(j.plan.qlen + j.plan.n_rows + 8) * 8);
        qp_off[t] = work_bytes;
        if (bits == 15) work_bytes += al256((size_t)abpt->m * ((((size_t)j.plan.qlen + 1 + 7) & ~(size_t)7) + 8) * 2);
        bt_off[t] = work_bytes;
        if (bits == 15) work_bytes += al256((size_t)j.plan.n_rows * sizeof(PoaBtRec));
    }
    uint64_t tot_units = 0;
    for (int t = 0; t < n; ++t) {
        units[t] = plane_units_for(&jobs[idx[t]], abpt->gap_mode, generous);
        plane_off[t] = tot_units; tot_units += units[t];
    }
    const size_t plane_bytes = (size_t)tot_units * POA_GROUP * S;
    L.plane_bytes = plane_bytes; L.in_bytes = 0;
    grow_host(&c->h_in, &c->h_in_cap, in_bytes);
    grow_host(&c->h_res, &c->h_res_cap, 256 + (size_t)n * sizeof(PoaResultDev));
    grow_dev(&c->d_in, &c->d_in_cap, in_bytes, 1);
    grow_dev(&c->d_work, &c->d_work_cap, work_bytes, 1);
    uint8_t *planes_base;
    if (c->arena) {
        planes_base = try_only ? poa_arena_try_borrow(c->arena, plane_bytes) : arena_take(c->arena, plane_bytes);
        if (!planes_base) return false;
    } else { grow_dev(&c->d_planes, &c->d_planes_cap, plane_bytes, generous ? 0 : 1); planes_base = c->d_planes; }
    L.planes_base = planes_base; L.in_bytes = in_bytes; L.active = true;

    poa_fill_params((PoaParamsDev *)c->h_in, abpt, bits);
    PoaJobDesc *desc = (PoaJobDesc *)(c->h_in + off_desc);
    for (int t = 0; t < n; ++t) {
        poa_job &j = jobs[idx[t]];
        poa_blob_fill(c->h_in + blob_off[t], &j.plan, j.abg, abpt, j.beg_node_id, j.end_node_id, j.query);
        desc[t].blob = c->d_in + blob_off[t];
        desc[t].planes = planes_base + (size_t)plane_off[t] * POA_GROUP * S;
        desc[t].plane_cap_units = units[t];
        desc[t].rowinfo = (PoaRowInfo *)(c->d_work + work_off[t]);
        desc[t].rowoff = (PoaRowOff *)(c->d_work + work_off[t] + al256((size_t)j.plan.n_rows * sizeof(PoaRowInfo)));
        desc[t].cigar = (uint64_t *)(c->d_work + cig_off[t]);
        desc[t].cigar_cap = j.plan.qlen + j.plan.n_rows + 8;
        desc[t].pad = 0;
        desc[t].result = (PoaResultDev *)(c->h_res + 256) + t;      /* mapped pinned host memory */
        desc[t].done = NULL;
        desc[t].qprof = (int16_t *)(c->d_work + qp_off[t]);
        desc[t].btrec = bits == 15 ? (PoaBtRec *)(c->d_work + bt_off[t]) : NULL;
        ((volatile PoaResultDev *)(c->h_res + 256))[t].t_end_ns = 0;
    }
    __sync_synchronize();
    c->last_desc = desc[0]; c->last_bits = bits; c->last_gap = abpt->gap_mode; c->last_rows = jobs[idx[0]].plan.n_rows;
    const double t_filled = now_ms();
    CK(cudaMemcpyAsync(c->d_in, c->h_in, in_bytes, cudaMemcpyHostToDevice, c->st));
    /* shared-memory ring: wide enough for the widest expected band of this launch */
    int band_cells = 0;
    for (int t = 0; t < n; ++t) {
        const poa_blob_plan &pl = jobs[idx[t]].plan;
        const int bc = pl.w >= 0 ? (2 * pl.w + 1 + 104 + 7) / 8 * 8 : (pl.qlen + 1 + 7) / 8 * 8 + 8;
        if (bc > band_cells) band_cells = bc;
    }
    static const size_t smem_budget = [] { const char *e = getenv("ABPOA_GPU_SMEM_KB"); return (size_t)(e && *e ? atoi(e) : 28) * 1024; }();
    int ring_rows = 2, ring_cells = 64;
    poa_pick_ring(abpt->gap_mode, bits == 32 ? 32 : 16, band_cells, smem_budget, &ring_rows, &ring_cells);
    int whole = abpt->align_mode == ABPOA_GLOBAL_MODE;
    for (int t = 0; t < n && whole; ++t) if (!jobs[idx[t]].plan.whole_graph) whole = 0;
    int lean = whole && !abpt->inc_path_score;
    c->last_ps = bits == 15 && whole && abpt->inc_path_score && !poa_lean_disabled();
    const int gaps[4] = { abpt->gap_ext1, abpt->gap_open1 + abpt->gap_ext1, abpt->gap_ext2, abpt->gap_open2 + abpt->gap_ext2 };
    /* what poa_launch_align_p16 will instantiate (the TMA variant exists only with LEAN) */
    c->last_lean = bits == 15 && lean && !poa_lean_disabled(); c->last_tma = c->last_lean && poa_tma_enabled();
    c->last_ring_rows = ring_rows; c->last_ring_cells = ring_cells;
    if (bits == 15) CK(poa_launch_align_p16(abpt->gap_mode, abpt->align_mode, lean, gaps, (const PoaJobDesc *)(c->d_in + off_desc),
                                            (const PoaParamsDev *)c->d_in, n, ring_rows, ring_cells, c->st));
    else CK(poa_launch_align(abpt->gap_mode, bits, abpt->align_mode, (const PoaJobDesc *)(c->d_in + off_desc),
                             (const PoaParamsDev *)c->d_in, n, ring_rows, ring_cells, c->st));
    L.t_begin = t_begin; L.t_filled = t_filled;
    return true;
}

static void run_finish(poa_dev_ctx *c) {
    LaunchState &L = c->ls;
    if (!L.active) return;
    L.active = false;
    CK(cudaSetDevice(c->dev));
    poa_job *jobs = L.jobs; const int *idx = L.idx.data(); const int n = L.n, bits = L.bits;
    std::vector<size_t> &blob_off = L.blob_off, &work_off = L.work_off, &cig_off = L.cig_off;
    uint8_t *planes_base = L.planes_base; const size_t plane_bytes = L.plane_bytes, in_bytes = L.in_bytes;
    const double t_begin = L.t_begin, t_filled = L.t_filled;
    /* ---- wait for the launch: every job bumps the counter in mapped host memory when its results
     *      (also written there) are complete.  No event / copy is queued behind the kernel, so
     *      streams that share a hardware channel never serialise on it. ---- */
    {
        volatile PoaResultDev *rr = (volatile PoaResultDev *)(c->h_res + 256);
        struct timespec nap = { 0, 100 * 1000 };
        const double t_wait0 = now_ms();
        int spins = 0, next = 0;
        while (next < n) {
            if (rr[next].t_end_ns != 0) { ++next; continue; }
            if (++spins > 20) nanosleep(&nap, NULL);
            if ((spins & 1023) == 0) {
                cudaError_t e = cudaStreamQuery(c->st);
                if (e != cudaSuccess && e != cudaErrorNotReady) CK(e);
                if (e == cudaSuccess && rr[next].t_end_ns == 0) { __sync_synchronize(); if (rr[next].t_end_ns == 0) poa_die("libabpoa_b200/cuda", "kernel finished without reporting job %d", next); }
                if (now_ms() - t_wait0 > 600e3) poa_die("libabpoa_b200/cuda", "alignment launch did not finish within 600 s");
            }
        }
        __sync_synchronize();
    }
    const double t_waited = now_ms();
    if (c->arena) arena_give(c->arena, planes_base, plane_bytes);      /* the backtrace is done: planes are dead */
    size_t out_bytes = 0;
    {
        const PoaResultDev *rr = (const PoaResultDev *)(c->h_res + 256);
        uint64_t t0 = UINT64_MAX, t1 = 0;
        for (int t = 0; t < n; ++t) { if (rr[t].t_start_ns < t0) t0 = rr[t].t_start_ns; if (rr[t].t_end_ns > t1) t1 = rr[t].t_end_ns; }
        if (t1 > t0) c->stats.kernel_ms += (double)(t1 - t0) * 1e-6;     /* first warp in .. last warp out, %globaltimer */
    }
    c->stats.launches += 1; c->stats.h2d_bytes += in_bytes;

    std::vector<PoaResultDev> resv(n);
    memcpy(resv.data(), c->h_res + 256, (size_t)n * sizeof(PoaResultDev));
    c->last_units = resv[0].plane_units_used;
    std::vector<size_t> out_cig(n), out_band(n);
    for (int t = 0; t < n; ++t) {
        const poa_job &j = jobs[idx[t]];
        out_cig[t] = out_bytes; out_bytes += al256((size_t)(resv[t].status == POA_ST_OK ? resv[t].n_ops : 0) * 8);
        out_band[t] = out_bytes; if (j.want_bands) out_bytes += al256((size_t)j.plan.n_rows * sizeof(PoaRowInfo));
    }
    grow_host(&c->h_out, &c->h_out_cap, out_bytes);
    for (int t = 0; t < n; ++t) {
        const poa_job &j = jobs[idx[t]];
        if (resv[t].status == POA_ST_OK && resv[t].n_ops > 0)
            CK(cudaMemcpyAsync(c->h_out + out_cig[t], c->d_work + cig_off[t], (size_t)resv[t].n_ops * 8, cudaMemcpyDeviceToHost, c->st));
        if (j.want_bands)
            CK(cudaMemcpyAsync(c->h_out + out_band[t], c->d_work + work_off[t], (size_t)j.plan.n_rows * sizeof(PoaRowInfo), cudaMemcpyDeviceToHost, c->st));
    }
    stream_wait(c);
    c->stats.d2h_bytes += out_bytes;
    c->stats.fill_ms += t_filled - t_begin; c->stats.wait_ms += t_waited - t_filled; c->stats.copy_ms += now_ms() - t_waited;
    for (int t = 0; t < n; ++t) {
        poa_job &j = jobs[idx[t]];
        j.status = resv[t].status;
        j.best_score = resv[t].best_score; j.best_i = resv[t].best_i; j.best_j = resv[t].best_j;
        j.start_i = resv[t].start_i; j.start_j = resv[t].start_j;
        j.n_aln_bases = resv[t].n_aln_bases; j.n_matched_bases = resv[t].n_matched_bases;
        j.cells = resv[t].cells; j.max_band = resv[t].max_band; j.bits = bits;
        j.n_ops = resv[t].status == POA_ST_OK ? resv[t].n_ops : 0;
        j.ops = (const uint64_t *)(c->h_out + out_cig[t]);
        j.bands = j.want_bands ? (const int32_t *)(c->h_out + out_band[t]) : NULL;
        if (c->capture && resv[t].status == POA_ST_OK) {
            poa_captured_job cj;
            cj.blob = c->h_in + blob_off[t]; cj.bytes = j.plan.bytes; cj.n_rows = j.plan.n_rows; cj.qlen = j.plan.qlen; cj.w = j.plan.w;
            cj.n_pred = ((const int32_t *)(cj.blob + ((const PoaJobHeader *)cj.blob)->off_rowmeta))[2 * j.plan.n_rows];
            cj.bits = bits; cj.best_score = resv[t].best_score; cj.n_ops = resv[t].n_ops; cj.cells = resv[t].cells; cj.plane_units = resv[t].plane_units_used;
            c->capture(c->capture_user, &cj);
        }
        if (resv[t].status == POA_ST_OK) { c->stats.cells += resv[t].cells; c->stats.alignments += 1; c->stats.fwd_clk += resv[t].fwd_clk; c->stats.bt_clk += resv[t].bt_clk; for (int z = 0; z < 6; ++z) c->stats.prof[z] += resv[t].prof[z]; for (int z = 0; z < 4; ++z) c->stats.diag[z] += resv[t].diag[z]; }
    }
}

/* Blocking launch.  A thread must not WAIT for plane memory while it holds planes of other launches
 * (every worker doing so can exhaust the arena with nobody able to finish): when the arena is short the
 * owner's pressure callback first drains whatever else the thread has in flight. */
static void run_same_width(poa_dev_ctx *c, const abpoa_para_t *abpt, poa_job *jobs, const int *idx, int n, int bits, int generous) {
    if (!run_begin(c, abpt, jobs, idx, n, bits, generous, true)) {
        if (c->pressure) c->pressure(c->pressure_user);
        run_begin(c, abpt, jobs, idx, n, bits, generous, false);
    }
    run_finish(c);
}

/* Asynchronous variant for pipelined callers: submit() stages and launches the jobs when they can
 * all go into ONE launch of one kernel variant (the normal case) and returns 1; otherwise it does
 * nothing and returns 0 (the caller uses poa_engine_run).  collect() finishes the outstanding launch,
 * redoes the rare overflow / range jobs synchronously and delivers every job to the sink. */
int poa_engine_submit(poa_dev_ctx *c, const abpoa_para_t *abpt, poa_job *jobs, int n) {
    if (n <= 0 || c->ls.active) return 0;
    int kind = -1; size_t bytes = 0;
    const size_t limit = c->arena ? poa_arena_capacity(c->arena) / 4 : c->planes_limit;
    for (int t = 0; t < n; ++t) {
        const int rb = poa_score_bits(abpt, jobs[t].plan.qlen, jobs[t].plan.n_rows);
        jobs[t].ref_bits = rb;
        const int k = use_p16_for(abpt, jobs[t].plan.qlen, jobs[t].plan.n_rows) ? 15 : rb;
        if (kind < 0) kind = k; else if (k != kind) return 0;
        bytes += (size_t)plane_units_for(&jobs[t], abpt->gap_mode, 0) * POA_GROUP * (k == 32 ? 4 : 2);
    }
    if (limit && bytes > limit) return 0;
    std::vector<int> idx(n);
    for (int t = 0; t < n; ++t) idx[t] = t;
    /* Never WAIT for planes here: the caller may hold the planes of its other sub-chunks, and if every
     * worker did that the arena could be exhausted with nobody able to finish.  -1 tells the caller
     * to drain what it has in flight first and then take the blocking path (poa_engine_run). */
    if (!run_begin(c, abpt, jobs, idx.data(), n, kind, 0, true)) return -1;
    return 1;
}

void poa_engine_collect(poa_dev_ctx *c, poa_job_sink sink, void *user) {
    if (!c->ls.active) return;
    const abpoa_para_t *abpt = c->ls.abpt; poa_job *jobs = c->ls.jobs; const int n = c->ls.n, bits = c->ls.bits;
    run_finish(c);
    /* results live in the context's pinned buffers: deliver the good ones before any re-run reuses them */
    std::vector<int> redo;
    for (int t = 0; t < n; ++t) {
        if (jobs[t].status == POA_ST_PLANE_OVF || jobs[t].status == POA_ST_RANGE) redo.push_back(t);
        else sink(user, &jobs[t]);
    }
    for (int t : redo) {
        c->stats.retries += 1;
        int b2 = bits;
        if (jobs[t].status == POA_ST_PLANE_OVF) run_same_width(c, abpt, jobs, &t, 1, b2, 1);
        if (jobs[t].status == POA_ST_RANGE) {
            b2 = jobs[t].ref_bits == 16 ? 16 : 32;
            run_same_width(c, abpt, jobs, &t, 1, b2, 0);
            if (jobs[t].status == POA_ST_PLANE_OVF) run_same_width(c, abpt, jobs, &t, 1, b2, 1);
        }
        sink(user, &jobs[t]);
    }
}

/* Public engine entry: plans must be made (poa_blob_plan_make) by the caller.  Jobs whose
 * band outgrew the estimated slab are re-run alone with the full rectangle.  Because the
 * pinned output buffer is reused between launches, results are delivered through the
 * `sink` callback right after the launch that produced them. */
void poa_engine_run(poa_dev_ctx *c, const abpoa_para_t *abpt, poa_job *jobs, int n, poa_job_sink sink, void *user) {
    if (n <= 0) return;
    std::vector<int> kinds[3];                      /* 0: packed int16x2, 1: generic int16, 2: generic int32 */
    for (int t = 0; t < n; ++t) {
        const int rb = poa_score_bits(abpt, jobs[t].plan.qlen, jobs[t].plan.n_rows);
        jobs[t].ref_bits = rb;
        if (use_p16_for(abpt, jobs[t].plan.qlen, jobs[t].plan.n_rows)) kinds[0].push_back(t);
        else kinds[rb == 16 ? 1 : 2].push_back(t);
    }
    /* a launch may borrow at most this much of the plane memory (leave room for other streams) */
    size_t limit = c->planes_limit;
    if (c->arena) limit = poa_arena_capacity(c->arena) / 4;
    static const int kind_bits[3] = { 15, 16, 32 };
    for (int pass = 0; pass < 3; ++pass) {
        std::vector<int> &v = kinds[pass];
        const int bits = kind_bits[pass];
        size_t pos = 0;
        while (pos < v.size()) {
            size_t bytes = 0, end = pos;
            while (end < v.size()) {
                const size_t b = (size_t)plane_units_for(&jobs[v[end]], abpt->gap_mode, 0) * POA_GROUP * (bits == 32 ? 4 : 2);
                if (end > pos && limit && bytes + b > limit) break;
                bytes += b; ++end;
            }
            run_same_width(c, abpt, jobs, v.data() + pos, (int)(end - pos), bits, 0);
            std::vector<int> redo;
            for (size_t t = pos; t < end; ++t) {
                const int st = jobs[v[t]].status;
                if (st == POA_ST_PLANE_OVF) redo.push_back(v[t]);
                else if (st == POA_ST_RANGE) { c->stats.retries += 1; kinds[jobs[v[t]].ref_bits == 16 ? 1 : 2].push_back(v[t]); }   /* later pass redoes it */
                else sink(user, &jobs[v[t]]);
            }
            for (int t : redo) {
                c->stats.retries += 1;
                run_same_width(c, abpt, jobs, &t, 1, bits, 1);
                if (jobs[t].status == POA_ST_RANGE) kinds[jobs[t].ref_bits == 16 ? 1 : 2].push_back(t);
                else sink(user, &jobs[t]);
            }
            pos = end;
        }
    }
}

/* ------------------------------------------------------------------ abpoa.h single-alignment path */
struct single_sink_arg { abpoa_t *ab; abpoa_para_t *abpt; abpoa_res_t *res; };

static void fail_job(const poa_job *j) {
    if (j->status == POA_ST_BT_ERROR) poa_die("poa_backtrack", "Error in %s_backtrack.", "dp");
    if (j->status == POA_ST_PLANE_OVF) poa_die("libabpoa_b200/cuda", "DP band planes exceed the device slab even at full width");
    if (j->status != POA_ST_OK) poa_die("libabpoa_b200/cuda", "alignment kernel reported status %d", j->status);
}

/* translate one finished job into the caller's abpoa_res_t (reference: tail of the
 * backtrack macros, src/abpoa_align_simd.c:187-192 and friends) */
void poa_job_to_res(const poa_job *j, const abpoa_para_t *abpt, abpoa_res_t *res) {
    fail_job(j);
    res->best_score = j->best_score;
    if (!abpt->ret_cigar) return;
    const int n = j->n_ops;
    abpoa_cigar_t *cg = NULL;
    const abpoa_graph_t *g = j->abg;
    const int *id_of_row = g->index_to_node_id + j->plan.beg_index;
    if (n > 0) {
        /* the device names graph positions by DP row; MATCH / DEL words carry node ids (abpoa.h:46-51) */
        cg = (abpoa_cigar_t *)poa_xmalloc((size_t)n * sizeof(abpoa_cigar_t));
        const int rev = abpt->rev_cigar;
        for (int t = 0; t < n; ++t) {
            abpoa_cigar_t w = j->ops[rev ? t : n - 1 - t];
            if ((w & 0xf) != ABPOA_CINS) w = ((abpoa_cigar_t)id_of_row[w >> 34] << 34) | (w & 0x3ffffffffull);
            cg[t] = w;
        }
    }
    res->graph_cigar = cg; res->n_cigar = n; res->m_cigar = n;
    res->node_e = id_of_row[j->best_i]; res->query_e = j->best_j - 1;
    res->node_s = id_of_row[j->start_i]; res->query_s = j->start_j - 1;
    res->n_aln_bases += j->n_aln_bases; res->n_matched_bases += j->n_matched_bases;
}

static void single_sink(void *user, poa_job *j) {
    single_sink_arg *a = (single_sink_arg *)user;
    poa_job_to_res(j, a->abpt, a->res);
    /* leave the band of every row where the reference leaves it (abpoa.h:139) */
    abpoa_simd_matrix_t *abm = a->ab->abm;
    const int nr = j->plan.n_rows;
    if (nr > abm->rang_m) {
        int m = poa_roundup32(nr);
        abm->dp_beg = (int *)poa_xrealloc(abm->dp_beg, (size_t)m * sizeof(int));
        abm->dp_end = (int *)poa_xrealloc(abm->dp_end, (size_t)m * sizeof(int));
        abm->dp_beg_sn = (int *)poa_xrealloc(abm->dp_beg_sn, (size_t)m * sizeof(int));
        abm->dp_end_sn = (int *)poa_xrealloc(abm->dp_end_sn, (size_t)m * sizeof(int));
        abm->rang_m = m;
    }
    const int pn = j->ref_bits == 16 ? 16 : 8;
    for (int r = 0; r < nr - 1; ++r) {
        abm->dp_beg[r] = j->bands[4 * r]; abm->dp_end[r] = j->bands[4 * r + 1];
        abm->dp_beg_sn[r] = abm->dp_beg[r] / pn; abm->dp_end_sn[r] = abm->dp_end[r] / pn;
    }
}

int poa_cuda_align_sequence_to_subgraph(abpoa_t *ab, abpoa_para_t *abpt, int beg_node_id, int end_node_id,
                                        uint8_t *query, int qlen, abpoa_res_t *res) {
    if (!ab->abm->s_mem) ab->abm->s_mem = poa_dev_ctx_new();
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    poa_job j; memset(&j, 0, sizeof j);
    j.abg = ab->abg; j.beg_node_id = beg_node_id; j.end_node_id = end_node_id; j.query = query; j.want_bands = 1;
    poa_blob_plan_make(&j.plan, ab->abg, abpt, beg_node_id, end_node_id, qlen);
    single_sink_arg a = { ab, abpt, res };
    poa_engine_run(c, abpt, &j, 1, single_sink, &a);
    return 0;
}

/* ------------------------------------------------------------------ debugging aid
 * Copy one DP row of the most recent single alignment of `ab` back from HBM: planes as
 * int32 [n_planes][cap], and the row's (beg, end, left, right).  Returns the number of
 * planes, or -1.  Used by tests/debug_planes.py to compare against the oracle cell by cell. */
extern "C" int poa_debug_fetch_row(abpoa_t *ab, int row, int32_t *out, int cap, int32_t *info4) {
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    if (!c || c->arena || row < 0 || row >= c->last_rows) return -1;
    CK(cudaSetDevice(c->dev));
    PoaRowInfo ri; PoaRowOff ro; uint32_t off;
    CK(cudaMemcpy(&ri, c->last_desc.rowinfo + row, sizeof ri, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&ro, c->last_desc.rowoff + row, sizeof ro, cudaMemcpyDeviceToHost));
    off = ro.off;
    info4[0] = ri.beg; info4[1] = ri.end; info4[2] = ri.left; info4[3] = ri.right;
    const int P = planes_of(c->last_gap), S = c->last_bits == 32 ? 4 : 2;
    const int g0 = ri.beg >> 3, ng = (ri.end >> 3) - g0 + 1, wd = ri.end - ri.beg + 1;
    if (wd <= 0 || wd > cap) return -1;
    std::vector<uint8_t> buf((size_t)ng * 8 * P * S);
    CK(cudaMemcpy(buf.data(), (uint8_t *)c->last_desc.planes + (size_t)off * POA_GROUP * S, buf.size(), cudaMemcpyDeviceToHost));
    for (int p = 0; p < P; ++p)
        for (int j = ri.beg; j <= ri.end; ++j) {
            const size_t k = (size_t)p * ng * 8 + (size_t)(j - g0 * 8);
            out[(size_t)p * cap + (j - ri.beg)] = S == 2 ? (int32_t)((int16_t *)buf.data())[k] : ((int32_t *)buf.data())[k];
        }
    return P;
}

/* debugging aid: the whole DP state of the most recent single alignment of `ab` in one copy each -- per row
 * (beg, end, left, right) into rowinfo[4 * n_rows], the row's plane offset (8-cell units) into rowoff[n_rows], and the
 * plane slab as the kernel stored it (int16 or int32 cells; a row's planes lie one after the other, each
 * ((end >> 3) - (beg >> 3) + 1) * 8 cells wide -- except the generic kernel's banded linear-gap rows outside local mode
 * ("lgx"), which are stored in whole reference vectors of pn = 16 / 8 cells, beg / pn * pn .. (end / pn + 1) * pn - 1)
 * into `planes`.  Returns the slab's size in bytes (with planes == NULL or
 * a `cap` that is too small: nothing is copied), or -1.  Rows the alignment never computed hold stale values. */
extern "C" int64_t poa_debug_fetch_planes(abpoa_t *ab, int32_t *rowinfo, uint32_t *rowoff, void *planes, int64_t cap) {
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    if (!c || c->arena || c->last_rows <= 0) return -1;
    const int64_t bytes = (int64_t)c->last_units * POA_GROUP * (c->last_bits == 32 ? 4 : 2);
    if (!planes || cap < bytes) return bytes;
    CK(cudaSetDevice(c->dev));
    std::vector<PoaRowOff> ro(c->last_rows);
    CK(cudaMemcpy(rowinfo, c->last_desc.rowinfo, (size_t)c->last_rows * sizeof(PoaRowInfo), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ro.data(), c->last_desc.rowoff, (size_t)c->last_rows * sizeof(PoaRowOff), cudaMemcpyDeviceToHost));
    for (int r = 0; r < c->last_rows; ++r) rowoff[r] = ro[r].off;
    if (bytes > 0) CK(cudaMemcpy(planes, c->last_desc.planes, (size_t)bytes, cudaMemcpyDeviceToHost));
    return bytes;
}

/* debugging aid: how the most recent single alignment of `ab` ran, as it was finally accepted (after any redo):
 * out[0] kernel (15 packed int16x2, 16 generic with int16 planes, 32 generic with int32 planes), out[1] LEAN predecessor
 * path, out[2] TMA row staging, out[3] ring rows, out[4] ring cells, out[5] DP rows, out[6] planes per row,
 * out[7] redo launches of the context so far.  Returns 0, or -1 before the first alignment. */
extern "C" int poa_debug_last_run(abpoa_t *ab, int32_t *out8) {
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    if (!c || c->last_rows <= 0) return -1;
    out8[0] = c->last_bits; out8[1] = c->last_lean; out8[2] = c->last_tma; out8[3] = c->last_ring_rows; out8[4] = c->last_ring_cells;
    out8[5] = c->last_rows; out8[6] = planes_of(c->last_gap); out8[7] = (int32_t)c->stats.retries;
    return 0;
}

/* debugging aid: replay the most recent single alignment of `ab` on the chain engine's job function (the compact row layout,
 * p16_run_job<GAP, GLOBAL, LEAN, no TMA, FB> on one warp, as poa_chain_dp_worker_kernel runs it) and rebuild every row's F
 * planes with the backtrace's recompute (poa_launch_fb_dump).  The job's blob, parameters and query profile are the ones
 * the alignment left on the device; the replay gets its own row records, a slab of the full rectangle, CIGAR, backtrace
 * records and result, so the five-plane run stays readable with poa_debug_fetch_planes.
 *   ring_rows, ring_cells  ring geometry of the replay; 0, 0: what the chain picks for this job's band (28 KB budget)
 *   buf_cells              decision-byte buffer of the recompute: > 0 as given, 0: the chain's (its ring), < 0: a whole row
 * Outputs, one copy each: rowinfo[4 * n_rows] (beg, end, left, right), rowoff[n_rows] (8-cell units), the compact slab,
 * the F slab (int16, a row's F1 (, F2) at its slab offset, ngrp * 8 cells each), the decision bytes (one per cell at the
 * row's slab offset: cap / 2 bytes), the graph-CIGAR (node ids, in abpoa_res_t order) and out[16] = status, best score,
 * node_e, query_e, node_s, query_s, n_ops, cells, max_band, plane_units_used, ring_rows, ring_cells, buf_cells,
 * windows recomputed (all rows), windows of the row with the most.
 * A -G alignment (its blob has path scores: off_predscore >= 0) that would have run LEAN but for its path scores replays on
 * the job function's path-score instantiation, as the chain runs -G jobs.
 * A banded global linear-gap alignment (the launch engine runs it on the generic kernel's lgx rows) replays on the job
 * function's linear-gap (LGX) instantiation, as the chain runs linear-gap jobs; its rows are stored in whole reference
 * vectors, there are no F planes to rebuild (fslab / fbits stay zero) and the replay brings its own query-profile scratch.
 * A banded whole-graph extend alignment (-m 2; the launch engine runs it on the packed kernel's general rows) replays on the
 * job function's EXTEND instantiation, as the chain runs extend jobs; the F-plane dump rebuilds its rows as global ones
 * (the recompute differs by mode only in local mode).
 * Returns -1 unless the last accepted run was the packed LEAN global kernel (or such a -G run, or such an extend run) with
 * affine or convex gaps, or a banded global linear-gap alignment, -2 for a ring that
 * does not fit one CTA or a buffer that does not fit shared memory; else the slab capacity the outputs need (bytes) when
 * `slab` is NULL or `cap` is smaller, else the bytes of the compact slab the replay used.  Nothing of the chain's or the
 * launch engine's own path runs here. */
extern "C" cudaError_t poa_launch_chain_replay(int gap_mode, const int *gaps, const PoaJobDesc *jd, const PoaParamsDev *prm, int ring_rows, int ring_cells,
                                               int ps, int ext, cudaStream_t st);
extern "C" cudaError_t poa_launch_fb_dump(int gap_mode, const int *gaps, const PoaJobDesc *jd, const PoaParamsDev *prm, int n_rows, int buf_cells,
                                          int16_t *fslab, uint8_t *fbits, int32_t *windows, int ps, cudaStream_t st);
extern "C" int poa_chain_fb_buf_cells(int gap_mode, int ring_rows, int ring_cells);
extern "C" int64_t poa_debug_chain_replay(abpoa_t *ab, int ring_rows, int ring_cells, int buf_cells, int32_t *rowinfo, uint32_t *rowoff,
                                          void *slab, void *fslab, uint8_t *fbits, int64_t cap, uint64_t *cigar, int64_t cigar_cap, int64_t *out16) {
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    if (!c || c->arena || c->last_rows <= 0) return -1;
    const bool lin = c->last_gap == ABPOA_LINEAR_GAP;
    CK(cudaSetDevice(c->dev));
    PoaJobHeader hd; CK(cudaMemcpy(&hd, c->last_desc.blob, sizeof hd, cudaMemcpyDeviceToHost));
    PoaParamsDev prm; CK(cudaMemcpy(&prm, c->d_in, sizeof prm, cudaMemcpyDeviceToHost));     /* what the alignment ran with */
    /* a banded whole-graph extend alignment of the packed kernel replays on the chain's EXTEND instantiation */
    const bool ext = !lin && c->last_bits == 15 && prm.align_mode == ABPOA_EXTEND_MODE && hd.w >= 0 && hd.off_live < 0;
    if (!lin && (c->last_bits != 15 || !(c->last_lean || c->last_ps || ext))) return -1;
    if (!lin && c->last_gap != ABPOA_AFFINE_GAP && c->last_gap != ABPOA_CONVEX_GAP) return -1;
    if (lin && (hd.w < 0 || prm.align_mode != ABPOA_GLOBAL_MODE)) return -1;
    const int n_rows = hd.n_rows, qlen = hd.qlen, gap = c->last_gap, ps = hd.off_predscore >= 0;
    const int n16 = lin ? 1 : (gap == ABPOA_AFFINE_GAP ? 2 : 3);
    const uint64_t units = (uint64_t)((qlen + 1 + 7) / 8 + 1) * n16 * n_rows;      /* full rectangle: no PLANE_OVF */
    const int64_t need = (int64_t)units * POA_GROUP * 2;
    if (!slab || cap < need) return need;
    if (ring_rows <= 0 || ring_cells <= 0) {
        const int band_cells = hd.w >= 0 ? (2 * hd.w + 1 + 104 + (lin ? 2 * (16 - 1) : 0) + 7) / 8 * 8 : (qlen + 1 + 7) / 8 * 8 + 8;   /* as the chain */
        poa_pick_ring(gap, 16, band_cells, (size_t)28 * 1024, &ring_rows, &ring_cells);
    }
    const int gaps[4] = { prm.e1, prm.oe1, prm.e2, prm.oe2 };
    /* fresh outputs: result | rowinfo | rowoff | cigar | btrec | slab | F slab | bytes | windows */
    const size_t o_ri = al256(sizeof(PoaResultDev)), o_ro = o_ri + al256((size_t)n_rows * sizeof(PoaRowInfo));
    const size_t o_cg = o_ro + al256((size_t)n_rows * sizeof(PoaRowOff)), cg_cap = (size_t)qlen + n_rows + 8;
    const size_t o_bt = o_cg + al256(cg_cap * 8), o_sl = o_bt + al256((size_t)n_rows * sizeof(PoaBtRec));
    const size_t o_fs = o_sl + al256((size_t)need), o_fb = o_fs + al256((size_t)need), o_wn = o_fb + al256((size_t)need / 2);
    const size_t o_qp = o_wn + al256((size_t)n_rows * 4);
    const size_t total = o_qp + al256((size_t)prm.m * ((((size_t)qlen + 1 + 7) & ~(size_t)7) + 8) * 2);
    uint8_t *d = NULL;
    CK(cudaMalloc((void **)&d, total));
    CK(cudaMemset(d, 0, total));
    PoaJobDesc jd = c->last_desc;
    jd.result = (PoaResultDev *)d; jd.rowinfo = (PoaRowInfo *)(d + o_ri); jd.rowoff = (PoaRowOff *)(d + o_ro);
    jd.cigar = (uint64_t *)(d + o_cg); jd.cigar_cap = (int32_t)cg_cap; jd.btrec = (PoaBtRec *)(d + o_bt);
    jd.planes = d + o_sl; jd.plane_cap_units = units;
    if (lin) jd.qprof = (int16_t *)(d + o_qp);         /* the generic kernel's launch has no query-profile scratch */
    const cudaError_t le = poa_launch_chain_replay(gap, gaps, &jd, (const PoaParamsDev *)c->d_in, ring_rows, ring_cells, ps, ext, c->st);
    if (le == cudaErrorInvalidValue) { cudaGetLastError(); CK(cudaFree(d)); return -2; }
    CK(le);
    PoaResultDev r; CK(cudaMemcpyAsync(&r, d, sizeof r, cudaMemcpyDeviceToHost, c->st));
    std::vector<PoaRowInfo> ri(n_rows); std::vector<PoaRowOff> ro(n_rows);
    CK(cudaMemcpyAsync(ri.data(), d + o_ri, (size_t)n_rows * sizeof(PoaRowInfo), cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(ro.data(), d + o_ro, (size_t)n_rows * sizeof(PoaRowOff), cudaMemcpyDeviceToHost, c->st));
    stream_wait(c);
    int max_ngrp = 1;
    for (int i = 0; i < n_rows - 1; ++i) if (ri[i].end >= ri[i].beg) max_ngrp = std::max(max_ngrp, (ri[i].end >> 3) - (ri[i].beg >> 3) + 1);
    if (buf_cells == 0) buf_cells = poa_chain_fb_buf_cells(gap, ring_rows, ring_cells);
    else if (buf_cells < 0) buf_cells = (max_ngrp + 31) / 32 * 256;
    std::vector<int32_t> win(n_rows, 0);
    if (r.status == POA_ST_OK && !lin) {                /* every row record is written: the dump reads inside the slab only */
        const cudaError_t de = poa_launch_fb_dump(gap, gaps, &jd, (const PoaParamsDev *)c->d_in, n_rows, buf_cells, (int16_t *)(d + o_fs), d + o_fb,
                                                  (int32_t *)(d + o_wn), ps, c->st);
        if (de == cudaErrorInvalidValue) { cudaGetLastError(); CK(cudaFree(d)); return -2; }
        CK(de);
        CK(cudaMemcpyAsync(fslab, d + o_fs, (size_t)need, cudaMemcpyDeviceToHost, c->st));
        CK(cudaMemcpyAsync(fbits, d + o_fb, (size_t)need / 2, cudaMemcpyDeviceToHost, c->st));
        CK(cudaMemcpyAsync(win.data(), d + o_wn, (size_t)n_rows * 4, cudaMemcpyDeviceToHost, c->st));
    } else if (lin) { memset(fslab, 0, (size_t)need); memset(fbits, 0, (size_t)need / 2); }
    const int n_ops = r.status == POA_ST_OK ? r.n_ops : 0;
    std::vector<uint64_t> ops((size_t)std::max(n_ops, 1));
    if (n_ops > 0) CK(cudaMemcpyAsync(ops.data(), d + o_cg, (size_t)n_ops * 8, cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(slab, d + o_sl, (size_t)need, cudaMemcpyDeviceToHost, c->st));
    stream_wait(c);
    CK(cudaFree(d));
    for (int i = 0; i < n_rows; ++i) {
        rowinfo[4 * i] = ri[i].beg; rowinfo[4 * i + 1] = ri[i].end; rowinfo[4 * i + 2] = ri[i].left; rowinfo[4 * i + 3] = ri[i].right;
        rowoff[i] = ro[i].off;
    }
    /* the device names graph positions by DP row (whole-graph job: row = node index); as poa_job_to_res */
    const int *id_of_row = ab->abg->index_to_node_id;
    for (int t = 0; t < n_ops && t < cigar_cap; ++t) {
        uint64_t w = ops[n_ops - 1 - t];
        if ((w & 0xf) != ABPOA_CINS) w = ((uint64_t)id_of_row[w >> 34] << 34) | (w & 0x3ffffffffull);
        cigar[t] = w;
    }
    int64_t wsum = 0, wmax = 0;
    for (int i = 0; i < n_rows; ++i) { wsum += win[i]; wmax = std::max<int64_t>(wmax, win[i]); }
    const int64_t o[16] = { r.status, r.best_score, id_of_row[r.best_i], r.best_j - 1, id_of_row[r.start_i], r.start_j - 1, n_ops, r.cells, r.max_band,
                            (int64_t)r.plane_units_used, ring_rows, ring_cells, buf_cells, wsum, wmax, 0 };
    memcpy(out16, o, sizeof o);
    return (int64_t)r.plane_units_used * POA_GROUP * 2;
}

/* debugging aid: redo launches (PLANE_OVF / RANGE) of the handle's single-alignment context so far */
extern "C" int64_t poa_debug_retries(abpoa_t *ab) {
    poa_dev_ctx *c = (poa_dev_ctx *)ab->abm->s_mem;
    return c ? c->stats.retries : -1;
}

/* ------------------------------------------------------------------ replay of HBM-resident jobs
 * One launch over `n` jobs whose blobs already live in device memory.  Only descriptors are
 * uploaded (outside the timed region); returns the CUDA-event time of the kernel in ms. */
double poa_dev_ctx_replay_launch(poa_dev_ctx *c, const abpoa_para_t *abpt, const poa_replay_job *rj, int n, int bits,
                                 int32_t *out_score, int32_t *out_nops, int64_t *out_cells) {
    CK(cudaSetDevice(c->dev));
    const int S = bits == 32 ? 4 : 2;
    const size_t off_desc = al256(sizeof(PoaParamsDev));
    const size_t in_bytes = off_desc + al256((size_t)n * sizeof(PoaJobDesc));
    size_t work_bytes = al256((size_t)n * sizeof(PoaResultDev));
    std::vector<size_t> work_off(n), cig_off(n), qp_off(n), bt_off(n); std::vector<uint64_t> units(n), plane_off(n);
    uint64_t tot_units = 0; int band_cells = 0;
    for (int t = 0; t < n; ++t) {
        work_off[t] = work_bytes;
        work_bytes += al256((size_t)rj[t].n_rows * sizeof(PoaRowInfo)) + al256((size_t)rj[t].n_rows * sizeof(PoaRowOff));
        cig_off[t] = work_bytes;
        work_bytes += al256((size_t)(rj[t].qlen + rj[t].n_rows + 8) * 8);
        qp_off[t] = work_bytes;
        if (bits == 15) work_bytes += al256((size_t)abpt->m * ((((size_t)rj[t].qlen + 1 + 7) & ~(size_t)7) + 8) * 2);
        bt_off[t] = work_bytes;
        if (bits == 15) work_bytes += al256((size_t)rj[t].n_rows * sizeof(PoaBtRec));
        poa_job tmp; memset(&tmp, 0, sizeof tmp); tmp.plan.n_rows = rj[t].n_rows; tmp.plan.qlen = rj[t].qlen; tmp.plan.w = rj[t].w;
        units[t] = plane_units_for(&tmp, abpt->gap_mode, 0);
        if (rj[t].plane_units > units[t]) units[t] = rj[t].plane_units;          /* a job that needed the generous slab */
        plane_off[t] = tot_units; tot_units += units[t];
        const int bc = rj[t].w >= 0 ? (2 * rj[t].w + 1 + 104 + 7) / 8 * 8 : (rj[t].qlen + 1 + 7) / 8 * 8 + 8;
        if (bc > band_cells) band_cells = bc;
    }
    const size_t plane_bytes = (size_t)tot_units * POA_GROUP * S;
    grow_host(&c->h_in, &c->h_in_cap, in_bytes);
    grow_dev(&c->d_in, &c->d_in_cap, in_bytes, 1);
    grow_dev(&c->d_work, &c->d_work_cap, work_bytes, 1);
    uint8_t *planes_base;
    if (c->arena) planes_base = arena_take(c->arena, plane_bytes);
    else { grow_dev(&c->d_planes, &c->d_planes_cap, plane_bytes, 1); planes_base = c->d_planes; }
    poa_fill_params((PoaParamsDev *)c->h_in, abpt, bits);
    PoaJobDesc *desc = (PoaJobDesc *)(c->h_in + off_desc);
    for (int t = 0; t < n; ++t) {
        desc[t].blob = rj[t].d_blob;
        desc[t].planes = planes_base + (size_t)plane_off[t] * POA_GROUP * S;
        desc[t].plane_cap_units = units[t];
        desc[t].rowinfo = (PoaRowInfo *)(c->d_work + work_off[t]);
        desc[t].rowoff = (PoaRowOff *)(c->d_work + work_off[t] + al256((size_t)rj[t].n_rows * sizeof(PoaRowInfo)));
        desc[t].cigar = (uint64_t *)(c->d_work + cig_off[t]);
        desc[t].cigar_cap = rj[t].qlen + rj[t].n_rows + 8;
        desc[t].pad = 0;
        desc[t].result = (PoaResultDev *)c->d_work + t;
        desc[t].done = NULL;
        desc[t].qprof = (int16_t *)(c->d_work + qp_off[t]);
        desc[t].btrec = bits == 15 ? (PoaBtRec *)(c->d_work + bt_off[t]) : NULL;
    }
    static const size_t smem_budget = [] { const char *e = getenv("ABPOA_GPU_SMEM_KB"); return (size_t)(e && *e ? atoi(e) : 28) * 1024; }();
    int ring_rows = 2, ring_cells = 64;
    poa_pick_ring(abpt->gap_mode, bits == 32 ? 32 : 16, band_cells, smem_budget, &ring_rows, &ring_cells);
    CK(cudaMemcpyAsync(c->d_in, c->h_in, in_bytes, cudaMemcpyHostToDevice, c->st));
    CK(cudaStreamSynchronize(c->st));
    CK(cudaEventRecord(c->ev_k0, c->st));
    /* captured jobs are whole-graph alignments (the batch engine's) */
    const int gaps[4] = { abpt->gap_ext1, abpt->gap_open1 + abpt->gap_ext1, abpt->gap_ext2, abpt->gap_open2 + abpt->gap_ext2 };
    if (bits == 15) CK(poa_launch_align_p16(abpt->gap_mode, abpt->align_mode, !abpt->inc_path_score && abpt->align_mode == ABPOA_GLOBAL_MODE, gaps,
                                            (const PoaJobDesc *)(c->d_in + off_desc), (const PoaParamsDev *)c->d_in, n, ring_rows, ring_cells, c->st));
    else CK(poa_launch_align(abpt->gap_mode, bits, abpt->align_mode, (const PoaJobDesc *)(c->d_in + off_desc),
                             (const PoaParamsDev *)c->d_in, n, ring_rows, ring_cells, c->st));
    CK(cudaEventRecord(c->ev_k1, c->st));
    grow_host(&c->h_out, &c->h_out_cap, (size_t)n * sizeof(PoaResultDev));
    CK(cudaMemcpyAsync(c->h_out, c->d_work, (size_t)n * sizeof(PoaResultDev), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    if (c->arena) arena_give(c->arena, planes_base, plane_bytes);
    float ms = 0.f; CK(cudaEventElapsedTime(&ms, c->ev_k0, c->ev_k1));
    const PoaResultDev *r = (const PoaResultDev *)c->h_out;
    for (int t = 0; t < n; ++t) {
        out_score[t] = r[t].status == POA_ST_OK ? r[t].best_score : INT32_MIN;
        out_nops[t] = r[t].n_ops; out_cells[t] = r[t].cells;
    }
    return (double)ms;
}

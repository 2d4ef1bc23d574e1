/* poa_batch.cu -- the batched engine behind abpoa_gpu.h (host-only C++; compiled by nvcc
 * only so that it shares the CUDA runtime of the library).
 *
 * Reads inside a group are sequential; groups are independent.  The engine keeps the GPU
 * full by advancing many groups at once:
 *
 *   - W worker threads, each owning a stream context (CUDA stream + pinned staging + HBM
 *     work buffers) and pulling chunks of G groups from a shared counter;
 *   - a chunk advances in rounds: round r flattens the graphs of its groups, launches ONE
 *     kernel grid (one warp per alignment of read r), receives the graph-CIGARs, and fuses
 *     them into the host graphs (abpoa_add_graph_alignment);
 *   - while one worker fuses on its core, the kernels of the other workers' chunks occupy
 *     the SMs: up to W x G alignments in flight;
 *   - the score planes (the bulk of HBM use) come from ONE arena shared by all streams and
 *     are held only from launch to result copy, so the arena bounds concurrency, not W x G.
 *
 * The per-read loop reproduces abpoa_poa (reference src/abpoa_align.c:312-352) including
 * the optional reverse-complement retry (-s); the final output step is abpoa_output
 * (reference :354-370) with out_fp = NULL.
 */
#include <cuda_runtime.h>
#include <atomic>
#include <chrono>
#include <thread>
#include <vector>
#include <mutex>
#include <algorithm>
#include <string.h>
#include <sched.h>
#include <pthread.h>
#include "abpoa_gpu.h"
#include "poa_internal.h"
#include "poa_engine.h"
#include "poa_device.cuh"
#include "poa_chain_host.h"

struct CapturedJob { uint8_t *blob; size_t bytes; int n_rows, qlen, w, n_pred, bits, best_score, n_ops; int64_t cells; uint64_t plane_units; };

struct abpoa_gpu_batch {
    std::mutex cap_mu; std::vector<CapturedJob> captured;
    int dev, n_workers, groups_per_launch;
    int pipe_depth;                 /* sub-chunks (stream contexts) each worker keeps in flight */
    int fast_order;                 /* spliced topological order in global mode (ABPOA_GPU_EXACT_ORDER=1 turns it off) */
    poa_arena *arena;
    std::vector<poa_dev_ctx *> ctx;
    double wall_ms;
    PoaChainStats chain;            /* device-resident chain engine (poa_chain.cu) */
    struct PoaEmit *emit;           /* abpoa_gpu_msa_batch_write in progress: per-group output text */
};

/* per-group text of abpoa_output(), collected while a batch runs and written in group order afterwards */
struct PoaEmit {
    const char *const *const *names;          /* [n_groups][n_seq] or NULL */
    std::vector<char *> buf; std::vector<size_t> len;
    const int *map;                           /* engine-local group index -> caller's group index (fallback sub-batches) */
};

extern "C" int abpoa_gpu_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" abpoa_gpu_batch_t *abpoa_gpu_batch_init(int device, int n_workers, int groups_per_launch) {
    if (abpoa_gpu_device_count() <= 0)
        poa_die("libabpoa_b200", "no CUDA device available. This library has no CPU path: the DP runs only on the GPU.");
    abpoa_gpu_batch *e = new abpoa_gpu_batch();
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    e->dev = device;
    { const char *eo = getenv("ABPOA_GPU_EXACT_ORDER"); e->fast_order = !(eo && *eo == '1'); }
    if (cudaSetDevice(device) != cudaSuccess) poa_die("libabpoa_b200", "cannot select CUDA device %d", device);
    unsigned hc = std::thread::hardware_concurrency();
    if (n_workers <= 0) {
        const char *env = getenv("ABPOA_GPU_WORKERS");
        n_workers = env && *env ? atoi(env) : (int)(hc ? (hc + 1) / 2 : 8);      /* ~ one per physical core */
        if (n_workers > 32 && !(env && *env)) n_workers = 32;                    /* 2 streams each: stay within the 32 hardware work queues x 2 */
        if (n_workers > 64) n_workers = 64;
        if (n_workers < 2) n_workers = 2;
    }
    if (groups_per_launch <= 0) {
        const char *env = getenv("ABPOA_GPU_GROUPS_PER_LAUNCH");
        groups_per_launch = env && *env ? atoi(env) : 0;      /* 0: chosen per batch call from the number of groups */
    }
    e->n_workers = n_workers; e->groups_per_launch = groups_per_launch;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) poa_die("libabpoa_b200", "cudaMemGetInfo failed");
    /* planes arena: most of the free HBM, leaving room for the per-stream staging buffers */
    size_t want = (size_t)((double)free_b * 0.80);
    const char *env = getenv("ABPOA_GPU_ARENA_MB");
    if (env && *env) want = (size_t)atoll(env) << 20;
    e->arena = poa_arena_new(device, want);
    {
        const char *pd = getenv("ABPOA_GPU_PIPE_DEPTH");
        e->pipe_depth = pd && *pd ? atoi(pd) : 2;
        if (e->pipe_depth < 1) e->pipe_depth = 1;
        if (e->pipe_depth > 8) e->pipe_depth = 8;
    }
    for (int w = 0; w < e->pipe_depth * n_workers; ++w) {   /* pipe_depth per worker: sub-chunks in flight */
        poa_dev_ctx *c = poa_dev_ctx_new_on(device);
        poa_dev_ctx_use_arena(c, e->arena);
        e->ctx.push_back(c);
    }
    e->wall_ms = 0; memset(&e->chain, 0, sizeof e->chain); e->emit = NULL;
    return e;
}

extern "C" void abpoa_gpu_capture_clear(abpoa_gpu_batch_t *e) {
    for (CapturedJob &c : e->captured) free(c.blob);
    e->captured.clear();
}

static void capture_cb(void *user, const poa_captured_job *cj) {
    abpoa_gpu_batch *e = (abpoa_gpu_batch *)user;
    CapturedJob c; c.bytes = cj->bytes; c.blob = (uint8_t *)poa_xmalloc(cj->bytes); memcpy(c.blob, cj->blob, cj->bytes);
    c.n_rows = cj->n_rows; c.qlen = cj->qlen; c.w = cj->w; c.n_pred = cj->n_pred; c.bits = cj->bits;
    c.best_score = cj->best_score; c.n_ops = cj->n_ops; c.cells = cj->cells; c.plane_units = cj->plane_units;
    std::lock_guard<std::mutex> lk(e->cap_mu);
    e->captured.push_back(c);
}

extern "C" int abpoa_gpu_replay(abpoa_gpu_batch_t *e, abpoa_para_t *abpt, int warmup, int repeats, abpoa_gpu_replay_t *out) {
    memset(out, 0, sizeof *out);
    if (e->captured.empty()) return -1;
    if (cudaSetDevice(e->dev) != cudaSuccess) return -1;
    /* similar-sized jobs next to each other: a launch finishes when its longest job does */
    std::vector<CapturedJob> jobs = e->captured;
    std::stable_sort(jobs.begin(), jobs.end(), [](const CapturedJob &a, const CapturedJob &b) {
        if (a.bits != b.bits) return a.bits < b.bits;
        return a.cells > b.cells; });
    size_t total = 0; std::vector<size_t> off(jobs.size());
    for (size_t t = 0; t < jobs.size(); ++t) { off[t] = total; total += (jobs[t].bytes + 255) & ~(size_t)255; }
    uint8_t *d_blobs = NULL;
    if (cudaMalloc((void **)&d_blobs, total) != cudaSuccess) poa_die(__func__, "cannot place %zu bytes of captured jobs in HBM", total);
    for (size_t t = 0; t < jobs.size(); ++t)
        if (cudaMemcpy(d_blobs + off[t], jobs[t].blob, jobs[t].bytes, cudaMemcpyHostToDevice) != cudaSuccess) poa_die(__func__, "upload failed");
    out->input_bytes = total; out->n_jobs = (int64_t)jobs.size();
    for (const CapturedJob &c : jobs) {
        out->cells += c.cells; out->rows += c.n_rows - 1; out->preds += c.n_pred;
        if (c.bits != 32) { out->jobs16 += 1; out->cells16 += c.cells; }
    }
    /* waves: as many jobs per launch as a quarter of the plane arena holds (same width only) */
    const size_t wave_bytes = poa_arena_capacity(e->arena) / 2;
    const int P = abpt->gap_mode == ABPOA_LINEAR_GAP ? 1 : (abpt->gap_mode == ABPOA_AFFINE_GAP ? 3 : 5);
    std::vector<std::pair<size_t, size_t>> waves;
    for (size_t pos = 0; pos < jobs.size();) {
        size_t end = pos, bytes = 0;
        while (end < jobs.size() && jobs[end].bits == jobs[pos].bits && end - pos < 4096) {
            const size_t per_row = jobs[end].w >= 0 ? (size_t)((2 * jobs[end].w + 1 + 32 + 7) / 8 + 2) : (size_t)((jobs[end].qlen + 8) / 8 + 1);
            size_t b = per_row * P * (size_t)jobs[end].n_rows * 8 * (jobs[end].bits == 32 ? 4 : 2);
            if (jobs[end].plane_units * 8 * (jobs[end].bits == 32 ? 4 : 2) > b) b = jobs[end].plane_units * 8 * (jobs[end].bits == 32 ? 4 : 2);
            if (end > pos && bytes + b > wave_bytes) break;
            bytes += b; ++end;
        }
        waves.push_back({pos, end}); pos = end;
    }
    poa_dev_ctx *c = e->ctx[0];
    std::vector<poa_replay_job> rj; std::vector<int32_t> sc, no; std::vector<int64_t> ce;
    double sum_ms = 0, min_ms = 1e30;
    for (int rep = 0; rep < warmup + repeats; ++rep) {
        double ms = 0; int64_t mism = 0;
        for (auto &wv : waves) {
            const size_t n = wv.second - wv.first;
            rj.resize(n); sc.resize(n); no.resize(n); ce.resize(n);
            for (size_t t = 0; t < n; ++t) { const CapturedJob &cj = jobs[wv.first + t]; rj[t].d_blob = d_blobs + off[wv.first + t]; rj[t].n_rows = cj.n_rows; rj[t].qlen = cj.qlen; rj[t].w = cj.w; rj[t].plane_units = cj.plane_units; }
            ms += poa_dev_ctx_replay_launch(c, abpt, rj.data(), (int)n, jobs[wv.first].bits, sc.data(), no.data(), ce.data());
            for (size_t t = 0; t < n; ++t) { const CapturedJob &cj = jobs[wv.first + t]; if (sc[t] != cj.best_score || no[t] != cj.n_ops || ce[t] != cj.cells) ++mism; }
        }
        if (rep >= warmup) { sum_ms += ms; if (ms < min_ms) min_ms = ms; out->mismatches += mism; }
    }
    out->kernel_ms = sum_ms / (repeats > 0 ? repeats : 1); out->kernel_ms_min = min_ms; out->launches = (int64_t)waves.size();
    cudaFree(d_blobs);
    return 0;
}

extern "C" void abpoa_gpu_batch_free(abpoa_gpu_batch_t *e) {
    if (!e) return;
    abpoa_gpu_capture_clear(e);
    for (poa_dev_ctx *c : e->ctx) poa_dev_ctx_free(c);
    poa_arena_destroy(e->arena);
    delete e;
}

extern "C" void abpoa_gpu_batch_get_stats(abpoa_gpu_batch_t *e, abpoa_gpu_stats_t *out) {
    memset(out, 0, sizeof *out);
    for (poa_dev_ctx *c : e->ctx) {
        const poa_engine_stats *s = poa_dev_ctx_stats(c);
        out->kernel_ms += s->kernel_ms; out->cells += s->cells; out->alignments += s->alignments;
        out->launches += s->launches; out->retries += s->retries; out->h2d_bytes += s->h2d_bytes; out->d2h_bytes += s->d2h_bytes;
        out->fwd_clk += s->fwd_clk; out->bt_clk += s->bt_clk;
    }
    out->wall_ms = e->wall_ms; out->n_workers = e->n_workers; out->device = e->dev;
    /* groups that ran on the device chain */
    out->cells += e->chain.cells; out->alignments += e->chain.alignments; out->launches += e->chain.launches;
    out->h2d_bytes += e->chain.h2d_bytes; out->d2h_bytes += e->chain.d2h_bytes; out->kernel_ms += e->chain.device_ms;
    out->fwd_clk += e->chain.fwd_clk; out->bt_clk += e->chain.bt_clk;
    out->chain_device_ms = e->chain.device_ms; out->chain_cells = e->chain.cells; out->chain_groups = e->chain.groups_done; out->chain_fallback_groups = e->chain.groups_failed;
    out->chain_dp_ms = e->chain.dp_ms; out->chain_fuse_ms = e->chain.fuse_ms; out->chain_dp_launches = e->chain.dp_launches;
    out->chain_wait_ms = e->chain.wait_ms; out->chain_free_running = e->chain.free_running;
}

extern "C" void abpoa_gpu_batch_reset_stats(abpoa_gpu_batch_t *e) {
    for (poa_dev_ctx *c : e->ctx) poa_dev_ctx_reset_stats(c);
    memset(&e->chain, 0, sizeof e->chain);
    e->wall_ms = 0;
}

extern "C" void abpoa_gpu_group_result_free(abpoa_gpu_group_result_t *r) {
    if (!r) return;
    for (int i = 0; i < r->n_cons; ++i) { free(r->cons_base[i]); free(r->cons_cov[i]); }
    free(r->cons_len); free(r->cons_base); free(r->cons_cov);
    for (int i = 0; i < r->n_msa_rows; ++i) free(r->msa_base[i]);
    free(r->msa_base);
    free(r->read_best_score); free(r->read_n_cigar); free(r->read_cigar_hash);
    memset(r, 0, sizeof *r);
}

extern "C" { extern __thread double poa_prof_ms[8]; }

/* Consensus / MSA of a finished group (reference abpoa_output, src/abpoa_align.c:354-370, with out_fp = NULL)
 * copied into the caller's result record.  Consensus, MSA and the public index arrays use the reference's
 * Kahn order, whatever order the alignments ran in. */
void poa_finish_group_result(abpoa_t *ab, abpoa_para_t *abpt, abpoa_gpu_group_result_t *o, struct PoaEmit *emit, int gidx) {
    poa_graph_set_fast_order(ab->abg, 0);
    /* (a consensus installed by poa_cons_install needs no graph) */
    if (ab->abg->node_n > 2 && !ab->abg->is_called_cons) { ab->abg->is_topological_sorted = 0; abpoa_topological_sort(ab->abg, abpt); }
    if (emit) {
        const int g = emit->map ? emit->map[gidx] : gidx;
        abpoa_seq_t *abs = ab->abs;
        if (emit->names && emit->names[g]) for (int i = 0; i < abs->n_seq; ++i) { const char *nm = emit->names[g][i]; poa_str_assign(&abs->name[i], nm ? nm : "", nm ? (int)strlen(nm) : 0); }
        abpoa_para_t local = *abpt;               /* the header of a list-mode consensus carries the group number (reference src/abpoa.c:154-159) */
        local.batch_index = g + 1;
        char *text = NULL; size_t tl = 0;
        FILE *mf = open_memstream(&text, &tl);
        if (!mf) poa_die(__func__, "open_memstream failed");
        abpoa_output(ab, &local, mf);
        fclose(mf);
        emit->buf[g] = text; emit->len[g] = tl;
    } else abpoa_output(ab, abpt, NULL);
    const abpoa_cons_t *abc = ab->abc;
    if (abpt->out_cons && abc->n_cons > 0) {
        o->n_cons = abc->n_cons;
        o->cons_len = (int *)poa_xmalloc(sizeof(int) * abc->n_cons);
        o->cons_base = (uint8_t **)poa_xmalloc(sizeof(uint8_t *) * abc->n_cons);
        o->cons_cov = (int **)poa_xmalloc(sizeof(int *) * abc->n_cons);
        for (int c = 0; c < abc->n_cons; ++c) {
            const int l = abc->cons_len[c];
            o->cons_len[c] = l;
            o->cons_base[c] = (uint8_t *)poa_xmalloc((size_t)(l > 0 ? l : 1));
            o->cons_cov[c] = (int *)poa_xmalloc(sizeof(int) * (size_t)(l > 0 ? l : 1));
            memcpy(o->cons_base[c], abc->cons_base[c], (size_t)l);
            memcpy(o->cons_cov[c], abc->cons_cov[c], sizeof(int) * (size_t)l);
        }
    }
    if (abpt->out_msa && abc->msa_len > 0) {
        o->msa_len = abc->msa_len; o->n_msa_rows = abc->n_seq + abc->n_cons;
        o->msa_base = (uint8_t **)poa_xmalloc(sizeof(uint8_t *) * (size_t)o->n_msa_rows);
        for (int r = 0; r < o->n_msa_rows; ++r) {
            o->msa_base[r] = (uint8_t *)poa_xmalloc((size_t)abc->msa_len);
            memcpy(o->msa_base[r], abc->msa_base[r], (size_t)abc->msa_len);
        }
    }
}

namespace {

struct GroupState {
    const abpoa_gpu_group_t *in;
    abpoa_gpu_group_result_t *out;
    abpoa_t *ab;
    int **weights;                      /* per read, as abpoa_msa builds them */
    int next_read;
};

struct Pending {                        /* one alignment in flight */
    GroupState *gs;
    abpoa_res_t res;
    bool have;
};

uint64_t fnv1a(const abpoa_cigar_t *a, int n) {
    uint64_t h = 1469598103934665603ull;
    const uint8_t *p = (const uint8_t *)a;
    for (size_t i = 0; i < (size_t)n * 8; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

/* One worker per physical core: pin worker `w` to the (base + w)-th CPU the process may use.
 * Linux numbers the first hardware thread of every core first, so consecutive workers land on
 * distinct cores; ranks of a multi-GPU job pass disjoint bases (ABPOA_GPU_CPU_BASE). */
/* CPUs the process may use, ordered so that consecutive workers land on DISTINCT physical cores
 * (one hardware thread per core first, sockets interleaved, SMT siblings only after every core has
 * a worker).  Linux numbers CPUs differently from box to box, so the order is read from sysfs. */
static std::vector<int> worker_cpu_order() {
    std::vector<int> cpus;
    cpu_set_t allowed; CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return cpus;
    struct Cpu { int cpu, pkg, core, smt; };
    std::vector<Cpu> v;
    for (int c = 0; c < CPU_SETSIZE; ++c) {
        if (!CPU_ISSET(c, &allowed)) continue;
        Cpu x = { c, 0, c, 0 };
        char path[128]; FILE *f;
        snprintf(path, sizeof path, "/sys/devices/system/cpu/cpu%d/topology/physical_package_id", c);
        if ((f = fopen(path, "r"))) { if (fscanf(f, "%d", &x.pkg) != 1) x.pkg = 0; fclose(f); }
        snprintf(path, sizeof path, "/sys/devices/system/cpu/cpu%d/topology/core_id", c);
        if ((f = fopen(path, "r"))) { if (fscanf(f, "%d", &x.core) != 1) x.core = c; fclose(f); }
        v.push_back(x);
    }
    /* smt rank = position among the allowed CPUs sharing (pkg, core) */
    for (size_t i = 0; i < v.size(); ++i) { int r = 0; for (size_t k = 0; k < i; ++k) if (v[k].pkg == v[i].pkg && v[k].core == v[i].core) ++r; v[i].smt = r; }
    /* rank of the core inside its package, to interleave the packages */
    std::vector<int> core_rank(v.size(), 0);
    for (size_t i = 0; i < v.size(); ++i) { int r = 0; for (size_t k = 0; k < v.size(); ++k) if (v[k].pkg == v[i].pkg && v[k].smt == v[i].smt && (v[k].core < v[i].core)) ++r; core_rank[i] = r; }
    std::vector<size_t> idx(v.size()); for (size_t i = 0; i < idx.size(); ++i) idx[i] = i;
    std::stable_sort(idx.begin(), idx.end(), [&](size_t a, size_t b) {
        if (v[a].smt != v[b].smt) return v[a].smt < v[b].smt;
        if (core_rank[a] != core_rank[b]) return core_rank[a] < core_rank[b];
        return v[a].pkg < v[b].pkg; });
    for (size_t i : idx) cpus.push_back(v[i].cpu);
    return cpus;
}

void pin_worker(int w) {
    const char *pin = getenv("ABPOA_GPU_PIN");
    if (pin && *pin == '0') return;
    static const std::vector<int> order = worker_cpu_order();
    if (order.empty()) return;
    const char *b = getenv("ABPOA_GPU_CPU_BASE");
    const int c = order[(size_t)((b && *b ? atoi(b) : 0) + w) % order.size()];
    cpu_set_t one; CPU_ZERO(&one); CPU_SET(c, &one);
    pthread_setaffinity_np(pthread_self(), sizeof one, &one);
}

struct Worker {
    int index;
    abpoa_gpu_batch *eng; poa_dev_ctx *ctx; poa_dev_ctx **ctxs; int n_ctx; abpoa_para_t *abpt; int flags;
    std::atomic<int> *next_chunk; int G; int slot0, slot1; int n_groups; const abpoa_gpu_group_t *groups; abpoa_gpu_group_result_t *results;
};

struct SinkCtx { abpoa_para_t *abpt; };

void sink_to_res(void *user, poa_job *j) {
    SinkCtx *sc = (SinkCtx *)user;
    Pending *pd = (Pending *)j->tag;
    memset(&pd->res, 0, sizeof pd->res);
    poa_job_to_res(j, sc->abpt, &pd->res);       /* copies the CIGAR out of the pinned buffer */
    pd->gs->out->dp_cells += j->cells;
    pd->gs->out->n_aligned += 1;
    pd->have = true;
}

void finish_group(GroupState &gs, abpoa_para_t *abpt, abpoa_gpu_batch *eng, int gidx) { poa_finish_group_result(gs.ab, abpt, gs.out, eng->emit, gidx); }

struct PhaseClock {
    double plan = 0, run = 0, fuse = 0, finish = 0, setup = 0;
    std::chrono::steady_clock::time_point t;
    void tic() { t = std::chrono::steady_clock::now(); }
    double toc() { auto n = std::chrono::steady_clock::now(); double d = std::chrono::duration<double, std::milli>(n - t).count(); t = n; return d; }
};

void worker_main(Worker wk) {
    PhaseClock pc; const bool prof = getenv("ABPOA_GPU_PROFILE") != NULL;
    pin_worker(wk.index);
    if (cudaSetDevice(wk.eng->dev) != cudaSuccess) poa_die("libabpoa_b200", "worker cannot select device %d", wk.eng->dev);
    abpoa_para_t *abpt = wk.abpt;
    const int G = wk.G;
    std::vector<abpoa_t *> handles;                     /* reused across chunks */
    SinkCtx sc = { abpt };
    for (;;) {
        const int chunk = wk.next_chunk->fetch_add(1);
        const int g0 = chunk * G;
        if (g0 >= wk.n_groups) break;
        const int g1 = g0 + G < wk.n_groups ? g0 + G : wk.n_groups;
        const int ng = g1 - g0;
        while ((int)handles.size() < ng) handles.push_back(abpoa_init());
        std::vector<GroupState> gs(ng);
        int max_reads = 0;
        pc.tic();
        for (int t = 0; t < ng; ++t) {
            GroupState &s = gs[t];
            s.in = &wk.groups[g0 + t]; s.out = &wk.results[g0 + t]; s.ab = handles[t]; s.next_read = 0;
            memset(s.out, 0, sizeof *s.out);
            const int n = s.in->n_seq;
            if (n > max_reads) max_reads = n;
            int max_len = 1024;
            for (int i = 0; i < n; ++i) if (s.in->seq_lens[i] > max_len) max_len = s.in->seq_lens[i];
            abpoa_reset(s.ab, abpt, max_len);
            poa_graph_set_fast_order(s.ab->abg, wk.eng->fast_order);
            abpoa_seq_t *abs = s.ab->abs;
            abs->n_seq = n; poa_seq_reserve(abs);
            for (int i = 0; i < n; ++i) { abs->is_rc[i] = 0; abs->name[i].l = 0; }
            s.weights = (int **)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int *));
            for (int i = 0; i < n; ++i) {
                const int l = s.in->seq_lens[i];
                const int *qw = (abpt->use_qv && s.in->qual_weights && s.in->qual_weights[i]) ? s.in->qual_weights[i] : NULL;
                if (qw) { s.weights[i] = (int *)poa_xmalloc(sizeof(int) * (size_t)(l > 0 ? l : 1)); memcpy(s.weights[i], qw, sizeof(int) * (size_t)l); }
            }
            if (wk.flags & ABPOA_GPU_RECORD_READS) {
                s.out->read_best_score = (int32_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int32_t));
                s.out->read_n_cigar = (int32_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int32_t));
                s.out->read_cigar_hash = (uint64_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(uint64_t));
            }
        }
        std::vector<poa_job> jobs; std::vector<Pending> pend(ng); std::vector<int> owner;
        {   /* graphs of ~5 % error reads end near 2.5x the read length; leave headroom */
            int qmax = 0;
            for (int t = 0; t < ng; ++t) for (int i = 0; i < gs[t].in->n_seq; ++i) if (gs[t].in->seq_lens[i] > qmax) qmax = gs[t].in->seq_lens[i];
            poa_dev_ctx_reserve(wk.ctx, ng, 3 * qmax + 64, qmax);
        }
        pc.setup += pc.toc();
        for (int r = 0; r < max_reads; ++r) {
            jobs.clear(); owner.clear();
            pc.tic();
            for (int t = 0; t < ng; ++t) {
                GroupState &s = gs[t];
                pend[t].gs = &s; pend[t].have = false; memset(&pend[t].res, 0, sizeof(abpoa_res_t));
                if (r >= s.in->n_seq) continue;
                abpoa_graph_t *abg = s.ab->abg;
                if (abg->node_n <= 2) continue;                  /* empty graph: no DP (reference :195) */
                if (!abg->is_topological_sorted) abpoa_topological_sort(abg, abpt);
                poa_job j; memset(&j, 0, sizeof j);
                j.abg = abg; j.beg_node_id = ABPOA_SRC_NODE_ID; j.end_node_id = ABPOA_SINK_NODE_ID;
                j.query = s.in->seqs[r]; j.tag = &pend[t];
                poa_blob_plan_make(&j.plan, abg, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, s.in->seq_lens[r]);
                jobs.push_back(j); owner.push_back(t);
            }
            pc.plan += pc.toc();
            if (!jobs.empty()) poa_engine_run(wk.ctx, abpt, jobs.data(), (int)jobs.size(), sink_to_res, &sc);
            pc.run += pc.toc();

            /* optional strand retry (-s): align the reverse complement of weak hits */
            std::vector<uint8_t *> rc_seq(ng, (uint8_t *)NULL); std::vector<int *> rc_w(ng, (int *)NULL);
            if (abpt->amb_strand) {
                std::vector<poa_job> rjobs; std::vector<Pending> rpend(ng);
                for (int t = 0; t < ng; ++t) {
                    GroupState &s = gs[t];
                    if (!pend[t].have) continue;
                    const int qlen = s.in->seq_lens[r];
                    const int lim = qlen < s.ab->abg->node_n - 2 ? qlen : s.ab->abg->node_n - 2;
                    if (!(pend[t].res.best_score < lim * abpt->max_mat * .3333)) continue;
                    rc_seq[t] = (uint8_t *)poa_xmalloc((size_t)qlen); rc_w[t] = (int *)poa_xmalloc(sizeof(int) * (size_t)qlen);
                    for (int k = 0; k < qlen; ++k) {
                        const uint8_t b = s.in->seqs[r][qlen - 1 - k];
                        rc_seq[t][k] = b < 4 ? (uint8_t)(3 - b) : 4;
                        rc_w[t][k] = s.weights[r] ? s.weights[r][qlen - 1 - k] : 1;
                    }
                    poa_job j; memset(&j, 0, sizeof j);
                    j.abg = s.ab->abg; j.beg_node_id = ABPOA_SRC_NODE_ID; j.end_node_id = ABPOA_SINK_NODE_ID;
                    j.query = rc_seq[t]; rpend[t].gs = &s; rpend[t].have = false; j.tag = &rpend[t];
                    poa_blob_plan_make(&j.plan, s.ab->abg, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, qlen);
                    rjobs.push_back(j);
                }
                if (!rjobs.empty()) {
                    poa_engine_run(wk.ctx, abpt, rjobs.data(), (int)rjobs.size(), sink_to_res, &sc);
                    for (int t = 0; t < ng; ++t) {
                        if (!rc_seq[t]) continue;
                        if (rpend[t].res.best_score > pend[t].res.best_score) {
                            if (pend[t].res.n_cigar) free(pend[t].res.graph_cigar);
                            pend[t].res = rpend[t].res;
                            gs[t].ab->abs->is_rc[r] = 1;
                        } else {
                            if (rpend[t].res.n_cigar) free(rpend[t].res.graph_cigar);
                            free(rc_seq[t]); free(rc_w[t]); rc_seq[t] = NULL; rc_w[t] = NULL;
                        }
                    }
                }
            }

            /* fuse: abpoa_add_graph_alignment for every group that has a read r */
            for (int t = 0; t < ng; ++t) {
                GroupState &s = gs[t];
                if (r >= s.in->n_seq) continue;
                const int qlen = s.in->seq_lens[r];
                uint8_t *q = rc_seq[t] ? rc_seq[t] : (uint8_t *)s.in->seqs[r];
                int *w = rc_seq[t] ? rc_w[t] : s.weights[r];
                if (wk.flags & ABPOA_GPU_RECORD_READS) {
                    s.out->read_best_score[r] = pend[t].have ? pend[t].res.best_score : 0;
                    s.out->read_n_cigar[r] = pend[t].res.n_cigar;
                    s.out->read_cigar_hash[r] = fnv1a(pend[t].res.graph_cigar, pend[t].res.n_cigar);
                }
                poa_add_alignment_nosync(s.ab, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, q, w, qlen, NULL, pend[t].res, r, s.in->n_seq, 1);
                if (pend[t].res.n_cigar) free(pend[t].res.graph_cigar);
                free(rc_seq[t]); free(rc_w[t]);
            }
            pc.fuse += pc.toc();
        }
        pc.tic();
        for (int t = 0; t < ng; ++t) {
            finish_group(gs[t], abpt, wk.eng, g0 + t);
            for (int i = 0; i < gs[t].in->n_seq; ++i) free(gs[t].weights[i]);
            free(gs[t].weights);
        }
    }
    pc.finish += pc.toc();
    for (abpoa_t *ab : handles) abpoa_free(ab);
    if (prof) {
        const poa_engine_stats *st = poa_dev_ctx_stats(wk.ctx);
        fprintf(stderr, "[worker-host] bfs %.0f sort_edges %.0f remain %.0f thread_cigar %.0f span %.0f ms\n",
                poa_prof_ms[0], poa_prof_ms[1], poa_prof_ms[2], poa_prof_ms[3], poa_prof_ms[4]);
        if (st->prof[0] + st->prof[1] > 0)
            fprintf(stderr, "[kernel-phases, cycles/alignment] setup %.0fk pred %.0fk compute %.0fk store %.0fk rowmax %.0fk tail+prefetch %.0fk\n",
                    st->prof[0] / 1e3 / st->alignments, st->prof[1] / 1e3 / st->alignments, st->prof[2] / 1e3 / st->alignments,
                    st->prof[3] / 1e3 / st->alignments, st->prof[4] / 1e3 / st->alignments, st->prof[5] / 1e3 / st->alignments);
        fprintf(stderr, "[worker] setup %.0f plan %.0f run %.0f (kernel %.0f, fill %.0f, wait %.0f, copy %.0f) fuse %.0f finish %.0f ms\n",
                pc.setup, pc.plan, pc.run, st->kernel_ms, st->fill_ms, st->wait_ms, st->copy_ms, pc.fuse, pc.finish);
    }
}


/* ------------------------------------------------------------------ pipelined worker
 * Two half-chunks A and B, each with its own stream context.  While A's kernel runs on the GPU
 * the thread fuses B's graph-CIGARs and stages B's next launch, and vice versa: host graph work
 * and device DP overlap inside one thread, and each half's critical chain is
 * (kernel + its own fusion), not (kernel + fusion of everything the worker owns). */
struct HalfChunk {
    poa_dev_ctx *ctx = NULL;
    int g0 = 0, ng = 0, max_reads = 0;
    std::vector<abpoa_t *> handles;
    std::vector<GroupState> gs;
    std::vector<Pending> pend;
    std::vector<poa_job> jobs;
    bool submitted = false;
    int fused_rounds = 0;              /* reads 0 .. fused_rounds-1 are in the graphs */
};

void half_setup(HalfChunk &h, const Worker &wk, int g0, int g1) {
    abpoa_para_t *abpt = wk.abpt;
    h.g0 = g0; h.ng = g1 - g0; h.max_reads = 0; h.submitted = false; h.fused_rounds = 0;
    while ((int)h.handles.size() < h.ng) h.handles.push_back(abpoa_init());
    h.gs.assign(h.ng, GroupState()); h.pend.assign(h.ng, Pending());
    int qmax = 0;
    for (int t = 0; t < h.ng; ++t) {
        GroupState &s = h.gs[t];
        s.in = &wk.groups[g0 + t]; s.out = &wk.results[g0 + t]; s.ab = h.handles[t]; s.next_read = 0;
        memset(s.out, 0, sizeof *s.out);
        const int n = s.in->n_seq;
        if (n > h.max_reads) h.max_reads = n;
        int max_len = 1024;
        for (int i = 0; i < n; ++i) { if (s.in->seq_lens[i] > max_len) max_len = s.in->seq_lens[i]; if (s.in->seq_lens[i] > qmax) qmax = s.in->seq_lens[i]; }
        abpoa_reset(s.ab, abpt, max_len);
        poa_graph_set_fast_order(s.ab->abg, wk.eng->fast_order);
        abpoa_seq_t *abs = s.ab->abs;
        abs->n_seq = n; poa_seq_reserve(abs);
        for (int i = 0; i < n; ++i) { abs->is_rc[i] = 0; abs->name[i].l = 0; }
        s.weights = (int **)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int *));
        for (int i = 0; i < n; ++i) {
            const int l = s.in->seq_lens[i];
            const int *qw = (abpt->use_qv && s.in->qual_weights && s.in->qual_weights[i]) ? s.in->qual_weights[i] : NULL;
            if (qw) { s.weights[i] = (int *)poa_xmalloc(sizeof(int) * (size_t)(l > 0 ? l : 1)); memcpy(s.weights[i], qw, sizeof(int) * (size_t)l); }
        }
        if (wk.flags & ABPOA_GPU_RECORD_READS) {
            s.out->read_best_score = (int32_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int32_t));
            s.out->read_n_cigar = (int32_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(int32_t));
            s.out->read_cigar_hash = (uint64_t *)poa_xcalloc((size_t)(n > 0 ? n : 1), sizeof(uint64_t));
        }
    }
    if (h.ng > 0) poa_dev_ctx_reserve(h.ctx, h.ng, 3 * qmax + 64, qmax);
}

/* flatten the graphs for read r of every group of the half and launch (asynchronously when possible) */
void half_start_round(HalfChunk &h, const Worker &wk, int r, SinkCtx *sc) {
    abpoa_para_t *abpt = wk.abpt;
    h.jobs.clear(); h.submitted = false;
    for (int t = 0; t < h.ng; ++t) {
        GroupState &s = h.gs[t];
        h.pend[t].gs = &s; h.pend[t].have = false; memset(&h.pend[t].res, 0, sizeof(abpoa_res_t));
        if (r >= s.in->n_seq) continue;
        abpoa_graph_t *abg = s.ab->abg;
        if (abg->node_n <= 2) continue;
        if (!abg->is_topological_sorted) abpoa_topological_sort(abg, abpt);
        poa_job j; memset(&j, 0, sizeof j);
        j.abg = abg; j.beg_node_id = ABPOA_SRC_NODE_ID; j.end_node_id = ABPOA_SINK_NODE_ID;
        j.query = s.in->seqs[r]; j.tag = &h.pend[t];
        poa_blob_plan_make(&j.plan, abg, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, s.in->seq_lens[r]);
        h.jobs.push_back(j);
    }
    if (h.jobs.empty()) return;
    /* 1: launched asynchronously.  0: mixed kernel kinds / too big for one launch, -1: the arena is short right
     * now -- both take the blocking path, which (through the context's pressure callback) first drains this
     * worker's other sub-chunks so that the thread never waits for planes while holding some. */
    if (poa_engine_submit(h.ctx, abpt, h.jobs.data(), (int)h.jobs.size()) == 1) h.submitted = true;
    else poa_engine_run(h.ctx, abpt, h.jobs.data(), (int)h.jobs.size(), sink_to_res, sc);
}

/* wait for the half's launch, then fuse read r into every group that has one */
void half_finish_round(HalfChunk &h, const Worker &wk, int r, SinkCtx *sc) {
    abpoa_para_t *abpt = wk.abpt;
    if (h.submitted) { poa_engine_collect(h.ctx, sink_to_res, sc); h.submitted = false; }
    for (int t = 0; t < h.ng; ++t) {
        GroupState &s = h.gs[t];
        if (r >= s.in->n_seq) continue;
        Pending &pd = h.pend[t];
        if (wk.flags & ABPOA_GPU_RECORD_READS) {
            s.out->read_best_score[r] = pd.have ? pd.res.best_score : 0;
            s.out->read_n_cigar[r] = pd.res.n_cigar;
            s.out->read_cigar_hash[r] = fnv1a(pd.res.graph_cigar, pd.res.n_cigar);
        }
        poa_add_alignment_nosync(s.ab, abpt, ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID, (uint8_t *)s.in->seqs[r], s.weights[r], s.in->seq_lens[r],
                                 NULL, pd.res, r, s.in->n_seq, 1);
        if (pd.res.n_cigar) free(pd.res.graph_cigar);
        memset(&pd.res, 0, sizeof pd.res); pd.have = false;
    }
    h.fused_rounds = r + 1;
}

void worker_pipelined(Worker wk) {
    const bool prof = getenv("ABPOA_GPU_PROFILE") != NULL;
    pin_worker(wk.index);
    if (cudaSetDevice(wk.eng->dev) != cudaSuccess) poa_die("libabpoa_b200", "worker cannot select device %d", wk.eng->dev);
    abpoa_para_t *abpt = wk.abpt;
    const int G = wk.G;
    SinkCtx sc = { abpt };
    /* sub-chunks in flight per worker: all contexts when there is enough work, fewer for small batches
     * (so that a few chunks spread over the workers instead of piling onto the first one) */
    int K = wk.n_ctx;
    {
        const int n_chunks = (wk.n_groups + G - 1) / G, nw = wk.eng->n_workers < n_chunks ? wk.eng->n_workers : n_chunks;
        const int per_worker = (n_chunks + nw - 1) / nw;
        if (K > per_worker) K = per_worker < 1 ? 1 : per_worker;
    }
    std::vector<HalfChunk> half((size_t)K);
    for (int k = 0; k < K; ++k) half[k].ctx = wk.ctxs[k];
    /* pressure callback of every context of this worker: collect whatever the worker has in flight (results are
     * parked in Pending records; half_finish_round fuses them later) so that their planes return to the arena */
    struct Drain { std::vector<HalfChunk> *half; SinkCtx *sc; } drain = { &half, &sc };
    auto drain_fn = [](void *user) {
        Drain *d = (Drain *)user;
        for (HalfChunk &o : *d->half) if (o.submitted) { o.submitted = false; poa_engine_collect(o.ctx, sink_to_res, d->sc); }
    };
    for (int k = 0; k < K; ++k) poa_dev_ctx_set_pressure_cb(half[k].ctx, drain_fn, &drain);
    PhaseClock pc; double t_start = 0, t_finish = 0;
    for (;;) {
        int got = 0, rounds = 0;
        for (int k = 0; k < K; ++k) {
            const int chunk = wk.next_chunk->fetch_add(1);
            const int g0 = chunk * G;
            if (g0 >= wk.n_groups) { half[k].ng = 0; half[k].max_reads = 0; continue; }
            half_setup(half[k], wk, g0, g0 + G < wk.n_groups ? g0 + G : wk.n_groups);
            if (half[k].max_reads > rounds) rounds = half[k].max_reads;
            ++got;
        }
        if (!got) break;
        for (int r = 0; r < rounds; ++r)
            for (int k = 0; k < K; ++k) {
                HalfChunk &h = half[k];
                if (h.ng == 0) continue;
                pc.tic();
                if (r > 0 && r - 1 < h.max_reads) half_finish_round(h, wk, r - 1, &sc);
                t_finish += pc.toc();
                if (r < h.max_reads) half_start_round(h, wk, r, &sc);
                t_start += pc.toc();
            }
        for (int k = 0; k < K; ++k) {
            HalfChunk &h = half[k];
            if (h.ng == 0) continue;
            pc.tic();
            if (h.fused_rounds < h.max_reads) half_finish_round(h, wk, h.max_reads - 1, &sc);
            for (int t = 0; t < h.ng; ++t) {
                finish_group(h.gs[t], abpt, wk.eng, h.g0 + t);
                for (int i = 0; i < h.gs[t].in->n_seq; ++i) free(h.gs[t].weights[i]);
                free(h.gs[t].weights);
            }
            t_finish += pc.toc();
        }
    }

    for (int k = 0; k < K; ++k) poa_dev_ctx_set_pressure_cb(half[k].ctx, NULL, NULL);
    for (int k = 0; k < K; ++k) for (abpoa_t *ab : half[k].handles) abpoa_free(ab);
    if (prof) {
        double wait = 0, fill = 0, copy = 0, kern = 0; double ph[6] = {0, 0, 0, 0, 0, 0}; int64_t alns = 0, fwd = 0, bt = 0, dg[4] = {0, 0, 0, 0};
        for (int k = 0; k < K; ++k) {
            const poa_engine_stats *st = poa_dev_ctx_stats(wk.ctxs[k]); wait += st->wait_ms; fill += st->fill_ms; copy += st->copy_ms; kern += st->kernel_ms;
            for (int z = 0; z < 6; ++z) ph[z] += (double)st->prof[z];
            for (int z = 0; z < 4; ++z) dg[z] += st->diag[z];
            alns += st->alignments; fwd += st->fwd_clk; bt += st->bt_clk;
        }
        if (dg[0] + dg[1] + dg[2] + dg[3] > 0) fprintf(stderr, "[kernel rows] straight-line %lld | generic: predecessors>2 %lld, predecessor outside the ring %lld, predecessor band wider than its ring slot %lld\n",
                                                      (long long)dg[0], (long long)dg[1], (long long)dg[2], (long long)dg[3]);
        if (alns > 0) fprintf(stderr, "[kernel, k-cycles/alignment] forward %.0f backtrace %.0f | -DPOA_KPROF phases: setup %.0f pred %.0f compute %.0f store %.0f rowmax %.0f tail+prefetch %.0f\n",
                              fwd / 1e3 / alns, bt / 1e3 / alns, ph[0] / 1e3 / alns, ph[1] / 1e3 / alns, ph[2] / 1e3 / alns, ph[3] / 1e3 / alns, ph[4] / 1e3 / alns, ph[5] / 1e3 / alns);
        fprintf(stderr, "[worker-host] bfs %.0f sort_edges %.0f remain %.0f thread_cigar %.0f ms\n", poa_prof_ms[0], poa_prof_ms[1], poa_prof_ms[2], poa_prof_ms[3]);
        fprintf(stderr, "[worker-pipe x%d] start(plan+fill+launch) %.0f finish(wait+copy+fuse) %.0f ms; launch-to-done %.0f fill %.0f copy %.0f kernel %.0f ms\n",
                K, t_start, t_finish, wait, fill, copy, kern);
    }
}


}  // namespace

extern "C" int abpoa_gpu_msa_batch(abpoa_gpu_batch_t *e, abpoa_para_t *abpt, int n_groups, const abpoa_gpu_group_t *groups,
                                   abpoa_gpu_group_result_t *results, int flags) {
    if (n_groups <= 0) return 0;
    if (!((abpt->disable_seeding && abpt->progressive_poa == 0) || abpt->align_mode != ABPOA_GLOBAL_MODE))
        poa_die(__func__, "minimizer seeding / guide-tree partitioning (-S / -p) is outside the scope of the GPU hot-path library.");
    const auto t0 = std::chrono::steady_clock::now();
    /* ---- device-resident chain (poa_chain.cu): the whole progressive loop of a group runs on the GPU; whatever it
     *      cannot take (parameters outside its scope, groups that outgrow their slot) goes through the launch engine ---- */
    if (!(flags & (ABPOA_GPU_CAPTURE_JOBS | ABPOA_GPU_NO_CHAIN)) && poa_chain_eligible(abpt)) {
        std::vector<int> todo((size_t)n_groups), rest;
        for (int g = 0; g < n_groups; ++g) todo[g] = g;
        poa_chain_run(e->dev, e->arena, abpt, e->n_workers, groups, results, todo, flags, rest, &e->chain, e->emit);
        if (!rest.empty()) {
            std::sort(rest.begin(), rest.end());
            std::vector<abpoa_gpu_group_t> sub(rest.size()); std::vector<abpoa_gpu_group_result_t> subres(rest.size());
            for (size_t k = 0; k < rest.size(); ++k) sub[k] = groups[rest[k]];
            const int *outer_map = e->emit ? e->emit->map : NULL;
            std::vector<int> map2(rest.size());
            for (size_t k = 0; k < rest.size(); ++k) map2[k] = outer_map ? outer_map[rest[k]] : rest[k];
            if (e->emit) e->emit->map = map2.data();
            abpoa_gpu_msa_batch(e, abpt, (int)rest.size(), sub.data(), subres.data(), flags | ABPOA_GPU_NO_CHAIN);
            if (e->emit) e->emit->map = outer_map;
            for (size_t k = 0; k < rest.size(); ++k) results[rest[k]] = subres[k];
        }
        e->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        return 0;
    }
    if (flags & ABPOA_GPU_CAPTURE_JOBS) abpoa_gpu_capture_clear(e);
    for (poa_dev_ctx *c : e->ctx) poa_dev_ctx_set_capture(c, (flags & ABPOA_GPU_CAPTURE_JOBS) ? capture_cb : NULL, e);
    std::atomic<int> next_chunk(0);
    /* groups per launch: as given, else spread the batch evenly over every sub-chunk slot (workers x pipe depth) */
    int G = e->groups_per_launch;
    if (G <= 0) { const int slots = e->n_workers * e->pipe_depth; G = (n_groups + slots - 1) / slots; if (G > 32) G = 32; if (G < 1) G = 1; }
    const int n_chunks = (n_groups + G - 1) / G;
    const int nw = e->n_workers < n_chunks ? e->n_workers : n_chunks;
    static const bool no_pipe = getenv("ABPOA_GPU_NO_PIPELINE") != NULL;
    const bool pipelined = !abpt->amb_strand && !no_pipe && e->pipe_depth > 1;
    std::vector<std::thread> th;
    for (int w = 0; w < nw; ++w) {
        Worker wk = { w, e, e->ctx[(size_t)e->pipe_depth * w], &e->ctx[(size_t)e->pipe_depth * w], e->pipe_depth, abpt, flags, &next_chunk, G, 0, 0, n_groups, groups, results };
        th.emplace_back(pipelined ? worker_pipelined : worker_main, wk);
    }
    for (auto &t : th) t.join();
    e->wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

/* abpoa_gpu_msa_batch + the text the reference CLI prints per group in list mode (src/abpoa.c:148-168: one
 * abpoa_msa1 per file with abpt->batch_index = file number), written to out_fp in group order. */
extern "C" int abpoa_gpu_msa_batch_write(abpoa_gpu_batch_t *e, abpoa_para_t *abpt, int n_groups, const abpoa_gpu_group_t *groups,
                                         const char *const *const *names, FILE *out_fp, abpoa_gpu_group_result_t *results, int flags) {
    if (n_groups <= 0) return 0;
    PoaEmit em; em.names = names; em.buf.assign((size_t)n_groups, (char *)NULL); em.len.assign((size_t)n_groups, 0); em.map = NULL;
    std::vector<abpoa_gpu_group_result_t> tmp;
    if (!results) { tmp.resize((size_t)n_groups); results = tmp.data(); }
    e->emit = &em;
    abpoa_gpu_msa_batch(e, abpt, n_groups, groups, results, flags);
    e->emit = NULL;
    for (int g = 0; g < n_groups; ++g) {
        if (em.buf[g]) { if (out_fp) fwrite(em.buf[g], 1, em.len[g], out_fp); free(em.buf[g]); }
        if (!tmp.empty()) abpoa_gpu_group_result_free(&results[g]);
    }
    return 0;
}

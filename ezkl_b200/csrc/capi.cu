// capi.cu — the extern "C" boundary declared in include/ezkl_b200.h: process-wide configuration, the devices of the process,
// per-(thread, device) contexts, the base-table registry with its replicas, host<->device staging, the device workers behind the
// multi-device host-pointer paths and the host-side tail (point normalisation).  No CPU fallback lives here: every compute
// entry point needs an initialised CUDA device and fails with an error code otherwise.
#include <atomic>
#include <cerrno>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/ezkl_b200.h"
#include "msm.cuh"
#include "ntt.cuh"
#include "poly.cuh"
#include "quotient.cuh"

namespace b200 {

// ---- configuration: the environment is read once, in b200_init --------------------------------------------------------------
static Config g_cfg;
const Config& config() { return g_cfg; }
int sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    int v = cache[dev].load(std::memory_order_relaxed);
    if (v == 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        cache[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}
static int env_int(const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; }
static int read_config() {
    Config c;
    if (const char* e = getenv("B200_MSM_TABLE_MB")) {
        char* end = nullptr;
        errno = 0;
        const unsigned long long mb = strtoull(e, &end, 10);
        B200_CHECK(*e >= '0' && *e <= '9' && *end == '\0' && errno == 0 && mb >= 1 && mb < ((unsigned long long)1 << 40), -1,
                   "b200_init: B200_MSM_TABLE_MB = '%s' is not a positive whole number of MiB", e);
        c.msm_table_budget = (size_t)mb << 20;
    }
    if (const char* e = getenv("B200_WS_BUDGET_MB")) c.ws_budget_call = (size_t)atol(e) << 20;
    if (const char* e = getenv("B200_WS_TOTAL_MB")) c.ws_budget_total = (size_t)atol(e) << 20;
    c.msm_reduce_m = env_int("B200_MSM_REDUCE_M", 0);
    c.msm_reduce_threads = env_int("B200_MSM_REDUCE_THREADS", 0);
    c.shard_min_logn = env_int("B200_SHARD_MIN_LOGN", 22);
    g_cfg = c;
    return 0;
}

// ---- process state ----------------------------------------------------------------------------------------------------------------
static constexpr int MAX_DEV = 8;
struct DeviceState { int id = -1; NttContext ntt; };
static DeviceState g_devs[MAX_DEV];
static std::atomic<int> g_ndev{0};
static std::atomic<bool> g_inited{false};
static std::atomic<int> g_active{0};            // entry points in flight (b200_shutdown waits for them)
static std::atomic<uint64_t> g_epoch{1};        // bumped by b200_shutdown: contexts of an older epoch are gone
static std::mutex g_mu;                         // tables, plans, context registry

// One registered base vector: a window-precomputed table replica per device of the process.
struct BaseSet {
    size_t n = 0; int c = 0, W = 0, s = 1, L = 0;
    MsmTable* t[MAX_DEV] = {};
};
static std::unordered_map<uint64_t, BaseSet*> g_tables;
static uint64_t g_next_handle = 1;

// Per (calling thread, device) context: stream, scratch, staging.  The registry owns the objects so that b200_shutdown can
// release the device memory of threads that are still alive (or already gone).
struct Ctx {
    int slot = 0, dev = 0;
    cudaStream_t stream = nullptr;
    MsmWorkspace msm_ws;
    PolyWorkspace poly_ws;
    StagingRing ring;                            // parameter blobs of every kernel launched from this context
    DevBuf stage_a, stage_b, stage_c, small;
    // pinned bounce buffers for large pageable <-> device copies (two slots, pipelined against the DMA engine)
    uint8_t* bounce[2] = {nullptr, nullptr};
    cudaEvent_t bounce_ev[2] = {nullptr, nullptr};
    // the scratch above is per thread, not per stream: a call on another stream first waits for the previous call's work
    cudaEvent_t last_ev = nullptr;
    cudaStream_t last_stream = nullptr;
    bool has_last = false;
    void release() {
        cudaSetDevice(dev);
        DevBuf* bufs[] = {&msm_ws.counts, &msm_ws.offs, &msm_ws.ents, &msm_ws.subs, &msm_ws.sums, &msm_ws.misc, &msm_ws.tile_counts, &poly_ws.scratch,
                          &stage_a, &stage_b, &stage_c, &small};
        for (DevBuf* b : bufs) b->release();
        ring.release();
        for (int i = 0; i < 2; ++i) { if (bounce[i]) cudaFreeHost(bounce[i]); if (bounce_ev[i]) cudaEventDestroy(bounce_ev[i]); bounce[i] = nullptr; bounce_ev[i] = nullptr; }
        if (last_ev) cudaEventDestroy(last_ev);
        if (stream) cudaStreamDestroy(stream);
        last_ev = nullptr; stream = nullptr;
    }
};
static std::vector<Ctx*> g_ctxs;
static std::atomic<int> g_nctx{0};

struct TlCtx {
    Ctx* c[MAX_DEV] = {};
    uint64_t epoch = 0;
    ~TlCtx() {                                   // a calling thread ends: give its device memory back
        if (epoch != g_epoch.load() || !g_inited.load()) return;
        std::lock_guard<std::mutex> lk(g_mu);
        if (epoch != g_epoch.load()) return;
        int cur = 0; cudaGetDevice(&cur);
        for (int s = 0; s < MAX_DEV; ++s) if (c[s]) {
            for (size_t i = 0; i < g_ctxs.size(); ++i) if (g_ctxs[i] == c[s]) { g_ctxs.erase(g_ctxs.begin() + i); break; }
            c[s]->release(); delete c[s]; g_nctx--;
        }
        cudaSetDevice(cur);
    }
};
static thread_local TlCtx tl;

struct CallGuard {
    bool ok;
    CallGuard() { g_active++; ok = g_inited.load(); if (!ok) set_error("b200: not initialised (call b200_init first)"); }
    ~CallGuard() { g_active--; }
};

static int get_ctx(Ctx** out, int slot = 0) {
    if (!g_inited.load()) { set_error("b200: not initialised (call b200_init first)"); return -3; }
    const uint64_t ep = g_epoch.load();
    if (tl.epoch != ep) { for (int s = 0; s < MAX_DEV; ++s) tl.c[s] = nullptr; tl.epoch = ep; }
    B200_CHECK(slot >= 0 && slot < g_ndev.load(), -1, "b200: device slot %d out of range", slot);
    if (!tl.c[slot]) {
        Ctx* c = new Ctx();
        c->slot = slot; c->dev = g_devs[slot].id;
        int cur = 0; cudaGetDevice(&cur);
        cudaError_t e = cudaSetDevice(c->dev);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->last_ev, cudaEventDisableTiming);
        if (g_ndev.load() > 1) cudaSetDevice(cur);
        if (e != cudaSuccess) { set_error("b200: context creation on device %d failed: %s", c->dev, cudaGetErrorString(e)); delete c; return -2; }
        std::lock_guard<std::mutex> lk(g_mu);
        g_ctxs.push_back(c); g_nctx++;
        tl.c[slot] = c;
    }
    *out = tl.c[slot];
    return 0;
}
// which device of the process a device pointer lives on (single-device processes skip the query)
static int slot_of(const void* dptr) {
    const int nd = g_ndev.load();
    if (nd <= 1 || !dptr) return 0;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, dptr) != cudaSuccess) { cudaGetLastError(); return 0; }
    for (int s = 0; s < nd; ++s) if (g_devs[s].id == at.device) return s;
    return 0;
}
// makes the context's device current for the duration of an entry point (multi-device processes only; a single-device process
// keeps the caller's current device, which is the one b200_init selected)
struct DevGuard {
    int prev = -1;
    explicit DevGuard(const Ctx* c) { if (g_ndev.load() > 1) { cudaGetDevice(&prev); if (prev != c->dev) cudaSetDevice(c->dev); else prev = -1; } }
    ~DevGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
// stream of a call + ordering of the per-thread scratch across streams
struct StreamScope {
    Ctx* c; cudaStream_t st;
    StreamScope(Ctx* c_, void* user) : c(c_), st(user ? (cudaStream_t)user : c_->stream) {
        if (c->has_last && c->last_stream != st) cudaStreamWaitEvent(st, c->last_ev, 0);
    }
    ~StreamScope() { if (cudaEventRecord(c->last_ev, st) == cudaSuccess) { c->last_stream = st; c->has_last = true; } else cudaGetLastError(); }
};
#define B200_ENTER(c, dptr)                                                \
    CallGuard _cg; if (!_cg.ok) return -3;                                 \
    Ctx* c; if (int _rc = get_ctx(&c, slot_of(dptr))) return _rc;          \
    DevGuard _dg(c)

// device scratch a single call may take, for batch splitting
static size_t call_budget() {
    if (g_cfg.ws_budget_call) return g_cfg.ws_budget_call;
    const int nd = g_ndev.load() > 0 ? g_ndev.load() : 1;
    const int per_dev = (g_nctx.load() + nd - 1) / nd;          // calling threads holding scratch on one device
    const size_t per = g_cfg.ws_budget_total / (size_t)(per_dev > 0 ? per_dev : 1);
    const size_t lo = (size_t)256 << 20, hi = (size_t)12 << 30;
    return per < lo ? lo : (per > hi ? hi : per);
}
// how many columns of item_bytes each one call may stage: at least one, then at most max_items
static size_t group_size(size_t item_bytes, size_t max_items) {
    size_t g = call_budget() / item_bytes;
    if (g < 1) g = 1;
    return g < max_items ? g : max_items;
}
// host Fr values arrive with 8-byte alignment (Rust / C callers); Fr is alignas(16), so always copy bytewise
static inline Fr as_fr(const b200_fr* p) { Fr r; memcpy(&r, p, sizeof r); return r; }

// ---- large host <-> device copies of PAGEABLE caller memory (what a Rust Vec<Fr> is) ------------------------------------------------
// cudaMemcpyAsync from pageable memory is limited by one driver thread copying into its own staging buffer.  Here the
// copy is cut into 16 MiB chunks that four host threads move into a pinned bounce buffer while the DMA engine drains the other one, so
// the PCIe link (Gen5 x16) is fed at memcpy-pool speed.  Copies below DIRECT_MAX_BYTES keep the plain path.  Measured with a host-pointer
// poly_op on fresh numpy buffers (two uploads and one download of S MiB) on an H100 80GB HBM3 at a 700 W power limit, median ms of
// two runs, plain vs bounce: S = 8: 1.7 / 1.6 vs 2.9 / 3.7;  16: 3.4 / 4.0 vs 4.6 / 4.6;  20: 5.5 / 5.2 vs 5.6 / 5.3;
// 24: 9.0 / 6.0 vs 5.8 / 6.1;  28: 10.1 / 8.1 vs 6.3 / 6.2;  32: 21.3 / 20.8 vs 13.0 / 11.9.  The crossover is at about 24 MiB.
static constexpr size_t BOUNCE_BYTES = (size_t)16 << 20;
static constexpr size_t DIRECT_MAX_BYTES = (size_t)24 << 20;
// One caller buffer (a column); a list of them maps onto ONE contiguous device range.  stride != 0 (uploads only): the segment is the
// field elements p[0], p[stride], p[2 stride], ... (bytes / 32 of them, stride in bytes), gathered on the host into the pinned slot.
struct HostSeg { uint8_t* p; size_t bytes; size_t stride = 0; };
// copies bytes [lo, hi) of the virtual concatenation of `segs` between the caller's buffers and `flat` (the pinned slot, offset 0 = byte lo0)
static void seg_copy_range(const HostSeg* segs, size_t nsegs, size_t lo0, size_t lo, size_t hi, uint8_t* flat, bool to_flat) {
    size_t pos = 0;
    for (size_t i = 0; i < nsegs && pos < hi; ++i) {
        const size_t s0 = pos, s1 = pos + segs[i].bytes;
        pos = s1;
        if (s1 <= lo) continue;
        const size_t a = lo > s0 ? lo : s0, b = hi < s1 ? hi : s1;
        if (segs[i].stride) {           // chunk and segment edges are multiples of 32 B, so [a, b) holds whole elements
            for (size_t e = (a - s0) / sizeof(Fr); e < (b - s0) / sizeof(Fr); ++e)
                memcpy(flat + (s0 + e * sizeof(Fr) - lo0), segs[i].p + e * segs[i].stride, sizeof(Fr));
        } else if (to_flat) memcpy(flat + (a - lo0), segs[i].p + (a - s0), b - a);
        else memcpy(segs[i].p + (a - s0), flat + (a - lo0), b - a);
    }
}
static void seg_copy_parallel(const HostSeg* segs, size_t nsegs, size_t lo, size_t hi, uint8_t* flat, bool to_flat) {
    const int T = 4;
    const size_t bytes = hi - lo;
    if (bytes < ((size_t)2 << 20)) { seg_copy_range(segs, nsegs, lo, lo, hi, flat, to_flat); return; }
    const size_t part = ((bytes / T) + 4095) & ~(size_t)4095;
    std::thread th[T - 1];
    for (int i = 1; i < T; ++i) {
        const size_t a = lo + part * i, b = a + part < hi ? a + part : hi;
        if (a < b) th[i - 1] = std::thread([=] { seg_copy_range(segs, nsegs, lo, a, b, flat, to_flat); });
    }
    seg_copy_range(segs, nsegs, lo, lo, lo + part < hi ? lo + part : hi, flat, to_flat);
    for (int i = 1; i < T; ++i) if (th[i - 1].joinable()) th[i - 1].join();
}
static int bounce_ready(Ctx* c) {
    if (c->bounce[0]) return 0;
    for (int i = 0; i < 2; ++i) {
        B200_CUDA(cudaMallocHost((void**)&c->bounce[i], BOUNCE_BYTES));
        B200_CUDA(cudaEventCreateWithFlags(&c->bounce_ev[i], cudaEventDisableTiming));
    }
    return 0;
}
// caller buffers -> contiguous device range.  When the call returns every SOURCE has been read; the device copies are ordered on `st`.
static int h2d_segments(Ctx* c, void* d_dst, const HostSeg* segs, size_t nsegs, cudaStream_t st) {
    size_t total = 0;
    bool strided = false;
    for (size_t i = 0; i < nsegs; ++i) { total += segs[i].bytes; strided |= segs[i].stride != 0; }
    if (total < DIRECT_MAX_BYTES && !strided) {
        size_t off = 0;
        for (size_t i = 0; i < nsegs; ++i) { B200_CUDA(cudaMemcpyAsync((uint8_t*)d_dst + off, segs[i].p, segs[i].bytes, cudaMemcpyHostToDevice, st)); off += segs[i].bytes; }
        return 0;
    }
    if (int rc = bounce_ready(c)) return rc;
    int slot = 0;
    for (size_t off = 0; off < total; off += BOUNCE_BYTES, slot ^= 1) {
        const size_t nb = total - off < BOUNCE_BYTES ? total - off : BOUNCE_BYTES;
        B200_CUDA(cudaEventSynchronize(c->bounce_ev[slot]));                       // the DMA that last read this slot is done
        seg_copy_parallel(segs, nsegs, off, off + nb, c->bounce[slot], true);
        B200_CUDA(cudaMemcpyAsync((uint8_t*)d_dst + off, c->bounce[slot], nb, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaEventRecord(c->bounce_ev[slot], st));
    }
    return 0;
}
// contiguous device range -> caller buffers.  Synchronous for the host: when the call returns the destinations hold the data.
static int d2h_segments(Ctx* c, const void* d_src, const HostSeg* segs, size_t nsegs, cudaStream_t st) {
    size_t total = 0;
    for (size_t i = 0; i < nsegs; ++i) total += segs[i].bytes;
    if (total < DIRECT_MAX_BYTES) {
        size_t off = 0;
        for (size_t i = 0; i < nsegs; ++i) { B200_CUDA(cudaMemcpyAsync(segs[i].p, (const uint8_t*)d_src + off, segs[i].bytes, cudaMemcpyDeviceToHost, st)); off += segs[i].bytes; }
        B200_CUDA(cudaStreamSynchronize(st));
        return 0;
    }
    if (int rc = bounce_ready(c)) return rc;
    const size_t nchunks = (total + BOUNCE_BYTES - 1) / BOUNCE_BYTES;
    for (size_t i = 0; i <= nchunks; ++i) {                                        // chunk i's DMA overlaps chunk i-1's host copy
        if (i < nchunks) {
            const size_t off = i * BOUNCE_BYTES, nb = total - off < BOUNCE_BYTES ? total - off : BOUNCE_BYTES;
            B200_CUDA(cudaMemcpyAsync(c->bounce[i & 1], (const uint8_t*)d_src + off, nb, cudaMemcpyDeviceToHost, st));
            B200_CUDA(cudaEventRecord(c->bounce_ev[i & 1], st));
        }
        if (i > 0) {
            const size_t off = (i - 1) * BOUNCE_BYTES, nb = total - off < BOUNCE_BYTES ? total - off : BOUNCE_BYTES;
            B200_CUDA(cudaEventSynchronize(c->bounce_ev[(i - 1) & 1]));
            seg_copy_parallel(segs, nsegs, off, off + nb, c->bounce[(i - 1) & 1], false);
        }
    }
    return 0;
}
// small host parameter tables -> a device buffer of the context, through the staging ring in slot-sized pieces (pinned, asynchronous, ordered
// on `st`); unlike a ring slot, the destination stays valid for as many later launches as the call makes
static int ring_upload(Ctx* c, void* d_dst, const void* h_src, size_t bytes, cudaStream_t st) {
    for (size_t off = 0; off < bytes; off += StagingRing::SLOT) {
        const size_t nb = bytes - off < StagingRing::SLOT ? bytes - off : StagingRing::SLOT;
        const void* d;
        if (int rc = c->ring.push((const uint8_t*)h_src + off, nb, st, &d)) return rc;
        B200_CUDA(cudaMemcpyAsync((uint8_t*)d_dst + off, d, nb, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}
static int h2d_one(Ctx* c, void* d_dst, const void* h_src, size_t bytes, cudaStream_t st) { HostSeg s{(uint8_t*)const_cast<void*>(h_src), bytes}; return h2d_segments(c, d_dst, &s, 1, st); }
static int d2h_one(Ctx* c, void* h_dst, const void* d_src, size_t bytes, cudaStream_t st) { HostSeg s{(uint8_t*)h_dst, bytes}; return d2h_segments(c, d_src, &s, 1, st); }
// a few bytes of device results (a counter, a check word) -> host memory, after the work queued before them on `st`
static int read_back(void* h_dst, const void* d_src, size_t bytes, cudaStream_t st) {
    B200_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// XYZZ (host) -> normalised Jacobian, one shared inversion (Montgomery's trick over zz*zzz)
static void normalize_host(const G1Xyzz* pts, size_t n, b200_g1_jac* out) {
    std::vector<Fq> prod(n), pref(n);
    Fq acc = fp_one<FqTag>();
    for (size_t i = 0; i < n; ++i) {
        pref[i] = acc;
        if (!g1_is_identity(pts[i])) { prod[i] = pts[i].zz * pts[i].zzz; acc = acc * prod[i]; }
    }
    Fq inv = fp_inv(acc);
    for (size_t i = n; i-- > 0;) {
        G1Jac j;
        if (g1_is_identity(pts[i])) {
            j.x = fp_zero<FqTag>(); j.y = fp_one<FqTag>(); j.z = fp_zero<FqTag>();
        } else {
            Fq t = inv * pref[i];            // 1 / (zz * zzz)
            inv = inv * prod[i];
            Fq zz_inv = t * pts[i].zzz, zzz_inv = t * pts[i].zz;
            j.x = pts[i].x * zz_inv; j.y = pts[i].y * zzz_inv; j.z = fp_one<FqTag>();
        }
        memcpy(&out[i], &j, sizeof j);
    }
}

// ---- profiling (CUDA events on the launching stream) ------------------------------------------------------------
static std::atomic<bool> g_prof{false};
struct ProfRec { int cls; cudaEvent_t e0, e1; };
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof_recs;
static thread_local std::vector<ProfRec> tl_prof_open;
bool prof_enabled() { return g_prof.load(std::memory_order_relaxed); }
void prof_mark(int cls, cudaStream_t st, bool begin) {
    if (begin) {
        ProfRec r; r.cls = cls;
        cudaEventCreate(&r.e0); cudaEventCreate(&r.e1);
        cudaEventRecord(r.e0, st);
        tl_prof_open.push_back(r);
    } else {
        for (size_t i = tl_prof_open.size(); i-- > 0;) {
            if (tl_prof_open[i].cls == cls) {
                ProfRec r = tl_prof_open[i];
                tl_prof_open.erase(tl_prof_open.begin() + i);
                cudaEventRecord(r.e1, st);
                std::lock_guard<std::mutex> lk(g_prof_mu);
                g_prof_recs.push_back(r);
                break;
            }
        }
    }
}

static BaseSet* find_bases(uint64_t h) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_tables.find(h);
    return it == g_tables.end() ? nullptr : it->second;
}

static NttPlan* warm_plan(int slot, uint32_t log_n, const Fr& omega, cudaStream_t st) {
    std::lock_guard<std::mutex> lk(g_mu);
    NttContext& nc = g_devs[slot].ntt;
    size_t before = nc.plans.size();
    NttPlan* p = nc.get(log_n, omega, st);
    if (p && nc.plans.size() != before) cudaStreamSynchronize(st);   // tables complete before other threads use them
    return p;
}

// the two-level power table that k_poly_coset_fold and k_perm_sigmas read: tab = [w^e, e < 2^lo_bits | w^(e << lo_bits), e < 2^(log_n - lo_bits)],
// so that w^e = tab[e mod 2^lo_bits] * tab[2^lo_bits + (e >> lo_bits)] for every e < 2^log_n
static void omega_power_table(Fr* tab, uint32_t lo_bits, uint32_t log_n, const Fr& w) {
    const size_t n_lo = (size_t)1 << lo_bits, n_hi = (size_t)1 << (log_n - lo_bits);
    Fr* lo = tab;
    Fr* hi = tab + n_lo;
    lo[0] = fp_one<FrTag>();
    for (size_t e = 1; e < n_lo; ++e) lo[e] = lo[e - 1] * w;
    const Fr step = lo[n_lo - 1] * w;
    hi[0] = fp_one<FrTag>();
    for (size_t e = 1; e < n_hi; ++e) hi[e] = hi[e - 1] * step;
}

// ---- internal call layer: <op>_on(c, st, ...) validates the device-side arguments, converts host constants and runs the
//      kernel file's *_run on `st`.  A _dev entry point is B200_ENTER + StreamScope + <op>_on; a host-pointer entry point stages
//      the caller's buffers in and out around the same <op>_on, inside one StreamScope on the thread's library stream.
static int ntt_call(Ctx* c, cudaStream_t st, const Fr* src, size_t src_stride, size_t n_in, Fr* tmp, Fr* dst, size_t dst_stride, uint32_t log_n,
                    const Fr& omega, const NttScale& pre, const NttScale& post, int batch) {
    if (log_n < 1 || log_n > 28) { set_error("ntt: log_n = %u out of range [1, 28]", log_n); return -1; }
    NttPlan* plan = warm_plan(c->slot, log_n, omega, st);         // looked up / built under g_mu; the vector of plans is never touched unlocked
    if (!plan) return -2;
    return ntt_run(plan, src, src_stride, n_in, tmp, (size_t)1 << log_n, dst, dst_stride, log_n, omega, pre, post, batch, st);
}
// the (mode, constants) pairs of the C ABI -> NttScale
static int ntt_scales(int pre_mode, const b200_fr* pre, int post_mode, const b200_fr* post, NttScale* a, NttScale* b) {
    B200_CHECK((pre_mode == 0 || pre_mode == 1 || pre_mode == 3) && (post_mode == 0 || post_mode == 1 || post_mode == 3), -1, "ntt: scale mode must be 0, 1 or 3");
    B200_CHECK((pre_mode == 0 || pre) && (post_mode == 0 || post), -1, "ntt: scale constants missing");
    a->mode = pre_mode; b->mode = post_mode;
    for (int i = 0; i < pre_mode; ++i) a->c[i] = as_fr(pre + i);
    for (int i = 0; i < post_mode; ++i) b->c[i] = as_fr(post + i);
    return 0;
}
// the zeta coset of coeff_to_extended: coefficient i is pre-scaled by zeta^(i mod 3)
static NttScale coset_pre(const Fr& zeta) { NttScale s; s.mode = 3; s.c[0] = fp_one<FrTag>(); s.c[1] = zeta; s.c[2] = zeta * zeta; return s; }
// its undoing in extended_to_coeff, with the inverse transform's divisor d: element i is post-scaled by d zeta^-(i mod 3), zeta^-1 = zeta^2
static NttScale coset_post(const Fr& d, const Fr& zeta) { NttScale s; s.mode = 3; s.c[0] = d; s.c[1] = d * (zeta * zeta); s.c[2] = d * zeta; return s; }

// ---- device workers: one host thread per extra device, so that the host-pointer entry points of a multi-device process drive
//      every PCIe link and every GPU at once (a single thread staging pageable memory serialises on its own copies) ------------
struct Job { std::function<int()> fn; int rc = 0; std::string err; bool done = false; };
struct Worker {
    std::thread th; std::mutex mu; std::condition_variable cv; std::deque<Job*> q; bool stop = false;
};
static Worker* g_workers[MAX_DEV] = {};
static std::mutex g_multi_mu;                    // multi-device host-pointer operations take every device: one at a time
static std::mutex g_done_mu;
static std::condition_variable g_done_cv;
static void worker_main(Worker* w, int dev) {
    cudaSetDevice(dev);
    for (;;) {
        Job* j;
        {
            std::unique_lock<std::mutex> lk(w->mu);
            w->cv.wait(lk, [&] { return w->stop || !w->q.empty(); });
            if (w->q.empty()) return;
            j = w->q.front(); w->q.pop_front();
        }
        j->rc = j->fn();
        if (j->rc) j->err = get_error();
        { std::lock_guard<std::mutex> lk(g_done_mu); j->done = true; }
        g_done_cv.notify_all();
    }
}
// fn(slot) for every slot < nslots: slot 0 on the calling thread, the others on their device workers; first failure wins
static int run_on_slots(int nslots, const std::function<int(int)>& fn) {
    std::vector<Job> jobs(nslots);
    for (int s = 1; s < nslots; ++s) {
        jobs[s].fn = [&fn, s] { return fn(s); };
        std::lock_guard<std::mutex> lk(g_workers[s]->mu);
        g_workers[s]->q.push_back(&jobs[s]);
        g_workers[s]->cv.notify_one();
    }
    int rc = fn(0);
    std::string err = rc ? get_error() : "";
    {
        std::unique_lock<std::mutex> lk(g_done_mu);
        g_done_cv.wait(lk, [&] { for (int s = 1; s < nslots; ++s) if (!jobs[s].done) return false; return true; });
    }
    for (int s = 1; s < nslots && !rc; ++s) if (jobs[s].rc) { rc = jobs[s].rc; err = jobs[s].err; }
    if (rc) set_error("%s", err.c_str());
    return rc;
}

// ---- MSM building blocks ------------------------------------------------------------------------------------------------------
// device-resident columns on the context's device -> XYZZ partial sums on that device (sub-batches bounded by the scratch budget)
static int msm_dev_on(Ctx* c, cudaStream_t st, const BaseSet* bs, const Fr* sc, size_t n, size_t stride, size_t batch, size_t base_off, G1Xyzz* out) {
    const MsmTable* t = bs->t[c->slot];
    B200_CHECK(t, -1, "msm: the bases have no replica on device slot %d", c->slot);
    const size_t per_col = msm_workspace_per_column(*t, n);
    const size_t max_grid = (size_t)(65535 / t->s);                 // a reduced table reduces batch * s bucket sets in one grid
    const size_t sub = group_size(per_col ? per_col : 1, max_grid < 4096 ? max_grid : 4096);
    for (size_t b0 = 0; b0 < batch; b0 += sub) {
        const size_t nb = batch - b0 < sub ? batch - b0 : sub;
        if (int rc = msm_run(*t, sc + b0 * stride, n, stride, (int)nb, out + b0, c->msm_ws, st, base_off)) return rc;
    }
    return 0;
}
// host columns cols[j][base_off .. base_off + n) for j < count -> XYZZ partial sums on the host, staged in sub-batches
static int msm_host_on(Ctx* c, const BaseSet* bs, const b200_fr* const* cols, size_t count, size_t n, size_t base_off, G1Xyzz* h_out) {
    if (count == 0) return 0;
    if (n == 0) { memset(h_out, 0, sizeof(G1Xyzz) * count); return 0; }
    DevGuard dg(c);
    const size_t sub = group_size(sizeof(Fr) * n * 2, count);
    if (c->stage_a.ensure(sizeof(Fr) * n * sub) || c->small.ensure(sizeof(G1Xyzz) * count)) return -2;
    StreamScope ss(c, nullptr);
    for (size_t b0 = 0; b0 < count; b0 += sub) {
        const size_t nb = count - b0 < sub ? count - b0 : sub;
        std::vector<HostSeg> segs(nb);
        for (size_t b = 0; b < nb; ++b) {
            B200_CHECK(cols[b0 + b], -1, "msm: scalars[%zu] is null", b0 + b);
            segs[b] = HostSeg{(uint8_t*)const_cast<b200_fr*>(cols[b0 + b] + base_off), sizeof(Fr) * n};
        }
        if (int rc = h2d_segments(c, c->stage_a.p, segs.data(), nb, ss.st)) return rc;
        if (int rc = msm_dev_on(c, ss.st, bs, c->stage_a.as<Fr>(), n, n, nb, base_off, c->small.as<G1Xyzz>() + b0)) return rc;
        if (b0 + nb < count) B200_CUDA(cudaStreamSynchronize(ss.st));      // the staging buffer is reused by the next sub-batch
    }
    B200_CUDA(cudaMemcpyAsync(h_out, c->small.p, sizeof(G1Xyzz) * count, cudaMemcpyDeviceToHost, ss.st));
    B200_CUDA(cudaStreamSynchronize(ss.st));
    return 0;
}
static void slice_bounds(size_t n, int g, int world, size_t* lo, size_t* hi) {
    const size_t base = n / world, rem = n % world;
    *lo = (size_t)g * base + ((size_t)g < rem ? (size_t)g : rem);
    *hi = *lo + base + ((size_t)g < rem ? 1 : 0);
}

}  // namespace b200

using namespace b200;

#pragma GCC visibility push(default)
extern "C" {

int b200_version(void) { return 200; }
const char* b200_last_error(void) { return get_error(); }
uint64_t b200_launch_count(void) { return g_launches.load(); }
int b200_device_count(void) { return g_inited.load() ? g_ndev.load() : 0; }

static int init_devices(const int* ids, int n) {
    if (g_inited.load()) {               // idempotent for the same device set; a different set needs b200_shutdown first
        bool same = n == g_ndev.load();
        for (int s = 0; same && s < n; ++s) same = ids[s] < 0 || ids[s] == g_devs[s].id;
        B200_CHECK(same, -1, "b200_init: already initialised with another device set (call b200_shutdown first)");
        return 0;
    }
    if (int rc = read_config()) return rc;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) { set_error("b200_init: no CUDA device (%s)", cudaGetErrorString(e)); return -2; }
    int first = 0;
    for (int s = 0; s < n; ++s) {
        int device = ids[s];
        if (device < 0) { B200_CUDA(cudaGetDevice(&device)); }
        B200_CHECK(device < count, -1, "b200_init: device %d >= device count %d", device, count);
        cudaDeviceProp prop;
        B200_CUDA(cudaGetDeviceProperties(&prop, device));
        B200_CHECK(prop.major == 9 && prop.minor == 0, -2, "b200_init: device %d is sm_%d%d; this library carries sm_90a code only", device, prop.major, prop.minor);
        B200_CUDA(cudaSetDevice(device));
        B200_CUDA(cudaFree(0));
        g_devs[s].id = device;
        if (s == 0) first = device;
    }
    for (int s = 0; s < n && n > 1; ++s) {          // NVLink peer mappings: every device may load from / store to every other
        B200_CUDA(cudaSetDevice(g_devs[s].id));
        for (int q = 0; q < n; ++q) if (q != s) {
            cudaError_t pe = cudaDeviceEnablePeerAccess(g_devs[q].id, 0);
            if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) { set_error("b200_init: no peer access %d -> %d (%s)", g_devs[s].id, g_devs[q].id, cudaGetErrorString(pe)); return -2; }
            cudaGetLastError();
        }
    }
    B200_CUDA(cudaSetDevice(first));
    g_ndev.store(n);
    for (int s = 1; s < n; ++s) {
        g_workers[s] = new Worker();
        g_workers[s]->th = std::thread(worker_main, g_workers[s], g_devs[s].id);
    }
    g_inited.store(true);
    return 0;
}
int b200_init(int device) { return init_devices(&device, 1); }
int b200_init_multi(int n_devices) {
    B200_CHECK(n_devices == 1 || n_devices == 2 || n_devices == 4 || n_devices == 8, -1, "b200_init_multi: n_devices = %d, want 1, 2, 4 or 8", n_devices);
    int ids[MAX_DEV];
    for (int i = 0; i < n_devices; ++i) ids[i] = i;
    return init_devices(ids, n_devices);
}

void b200_shutdown(void) {
    if (!g_inited.exchange(false)) return;                    // new entry points now fail with -3
    while (g_active.load() > 0) std::this_thread::yield();    // calls in flight on other threads finish first
    for (int s = 1; s < MAX_DEV; ++s) if (g_workers[s]) {
        { std::lock_guard<std::mutex> lk(g_workers[s]->mu); g_workers[s]->stop = true; }
        g_workers[s]->cv.notify_all();
        g_workers[s]->th.join();
        delete g_workers[s]; g_workers[s] = nullptr;
    }
    std::lock_guard<std::mutex> lk(g_mu);
    int cur = 0; cudaGetDevice(&cur);
    for (auto& kv : g_tables) {
        for (int s = 0; s < MAX_DEV; ++s) if (kv.second->t[s]) { cudaSetDevice(kv.second->t[s]->device); msm_table_free(kv.second->t[s]); delete kv.second->t[s]; }
        delete kv.second;
    }
    g_tables.clear();
    for (Ctx* c : g_ctxs) { c->release(); delete c; }          // streams and scratch of every calling thread, alive or not
    g_ctxs.clear(); g_nctx.store(0);
    g_epoch++;
    for (int s = 0; s < g_ndev.load(); ++s) { cudaSetDevice(g_devs[s].id); g_devs[s].ntt.release(); g_devs[s].id = -1; }
    cudaSetDevice(cur);
    g_ndev.store(0);
}

// ---- profiling -------------------------------------------------------------------------------------------------
int b200_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto& r : g_prof_recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    g_prof_recs.clear();
    g_prof.store(on != 0);
    return 0;
}
int b200_profile_read(int cls, double* total_ms, uint64_t* count) {
    B200_CHECK(cls >= 0 && cls < PROF_NCLASS && total_ms && count, -1, "profile_read: bad argument");
    int cur = 0; cudaGetDevice(&cur);
    for (int s = 0; s < g_ndev.load(); ++s) { B200_CUDA(cudaSetDevice(g_devs[s].id)); B200_CUDA(cudaDeviceSynchronize()); }
    cudaSetDevice(cur);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    double ms = 0; uint64_t n = 0;
    for (auto& r : g_prof_recs) if (r.cls == cls) { float t = 0; if (cudaEventElapsedTime(&t, r.e0, r.e1) == cudaSuccess) { ms += t; ++n; } else cudaGetLastError(); }
    *total_ms = ms; *count = n;
    return 0;
}

// ---- memory helpers ---------------------------------------------------------------------------------------
int b200_dev_alloc(void** d_ptr, size_t bytes) { B200_ENTER(c, nullptr); B200_CUDA(cudaMalloc(d_ptr, bytes)); return 0; }
int b200_dev_alloc_on(int slot, void** d_ptr, size_t bytes) {
    CallGuard cg; if (!cg.ok) return -3;
    Ctx* c; if (int rc = get_ctx(&c, slot)) return rc;
    DevGuard dg(c);
    B200_CUDA(cudaMalloc(d_ptr, bytes));
    return 0;
}
int b200_dev_free(void* d_ptr) { B200_CUDA(cudaFree(d_ptr)); return 0; }
int b200_dev_upload(void* d_dst, const void* h_src, size_t bytes) {
    B200_ENTER(c, d_dst);
    if (bytes == 0) return 0;
    B200_CHECK(d_dst && h_src, -1, "dev_upload: null pointer");
    if (int rc = h2d_one(c, d_dst, h_src, bytes, c->stream)) return rc;
    B200_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int b200_dev_upload_async(void* d_dst, const void* h_src, size_t bytes, void* stream) {
    B200_ENTER(c, d_dst);
    B200_CHECK(d_dst && h_src, -1, "dev_upload_async: null pointer");
    B200_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, stream ? (cudaStream_t)stream : c->stream));     // truly asynchronous only from pinned memory
    return 0;
}
int b200_dev_download(void* h_dst, const void* d_src, size_t bytes) {
    B200_ENTER(c, d_src);
    if (bytes == 0) return 0;
    B200_CHECK(h_dst && d_src, -1, "dev_download: null pointer");
    return d2h_one(c, h_dst, d_src, bytes, c->stream);
}
int b200_host_alloc(void** h_ptr, size_t bytes) { B200_CUDA(cudaMallocHost(h_ptr, bytes)); return 0; }
int b200_host_free(void* h_ptr) { B200_CUDA(cudaFreeHost(h_ptr)); return 0; }
int b200_sync(void) { B200_ENTER(c, nullptr); B200_CUDA(cudaStreamSynchronize(c->stream)); return 0; }
// the calling thread's library stream on every device of the process
int b200_sync_all(void) {
    CallGuard cg; if (!cg.ok) return -3;
    for (int s = 0; s < g_ndev.load(); ++s) { Ctx* c; if (int rc = get_ctx(&c, s)) return rc; B200_CUDA(cudaStreamSynchronize(c->stream)); }
    return 0;
}

// ---- bases ---------------------------------------------------------------------------------------------------
// Registration in the steps that b200_bases_register* and b200_srs_register share: bases_alloc makes a BaseSet whose table on the
// context's device is allocated with level 0 left for the caller to fill, bases_build fills the other levels and enqueues the replica
// copies, bases_drop is the failure cleanup (it frees every table of the set) and bases_publish hands out the handle once the stream
// has finished.  `who` names the entry point in the error messages.
static int bases_drop(BaseSet* bs, int rc) {
    int cur = 0; cudaGetDevice(&cur);
    for (int s = 0; s < MAX_DEV; ++s) if (bs->t[s]) { cudaSetDevice(bs->t[s]->device); msm_table_free(bs->t[s]); delete bs->t[s]; }
    cudaSetDevice(cur);
    delete bs; return rc;
}
static int bases_alloc(Ctx* c, size_t n, int window_bits, size_t max_table_bytes, BaseSet** out) {
    BaseSet* bs = new BaseSet();
    MsmTable* t = new MsmTable();
    bs->t[c->slot] = t;
    if (int rc = msm_table_alloc(t, n, window_bits, max_table_bytes ? max_table_bytes : config().msm_table_budget)) return bases_drop(bs, rc);
    *out = bs;
    return 0;
}
static int bases_build(Ctx* c, cudaStream_t st, BaseSet* bs, const void* d_bases, const char* who) {
    MsmTable* t = bs->t[c->slot];
    if (int rc = msm_table_build(t, reinterpret_cast<const G1Affine*>(d_bases), st)) return rc;
    bs->n = t->n; bs->c = t->c; bs->W = t->W; bs->s = t->s; bs->L = t->L;
    // replicas: the finished table crosses NVLink once per extra device (cheaper than rebuilding: one inversion per point and level)
    for (int s = 0; s < g_ndev.load(); ++s) if (s != c->slot) {
        MsmTable* r = new MsmTable();
        *r = *t; r->d_table = nullptr; r->device = g_devs[s].id;
        bs->t[s] = r;
        cudaSetDevice(r->device);
        cudaError_t e = cudaMalloc(&r->d_table, t->bytes());
        cudaSetDevice(c->dev);
        if (e != cudaSuccess) { set_error("%s: replica on device %d: %s", who, r->device, cudaGetErrorString(e)); return -2; }
        e = cudaMemcpyPeerAsync(r->d_table, r->device, t->d_table, t->device, t->bytes(), st);
        if (e != cudaSuccess) { set_error("%s: peer copy: %s", who, cudaGetErrorString(e)); return -2; }
    }
    return 0;
}
static uint64_t bases_publish(BaseSet* bs) {
    std::lock_guard<std::mutex> lk(g_mu);
    const uint64_t h = g_next_handle++;
    g_tables[h] = bs;
    return h;
}
// The bases come from the device (d_bases, copied into level 0) or from the host (h_bases, uploaded straight into level 0 of the
// new table, so no staging buffer of the calling thread grows to the size of an SRS vector).  max_table_bytes = 0: the configured budget.
static int bases_register_on(Ctx* c, cudaStream_t st, const void* d_bases, const b200_g1_affine* h_bases, size_t n, int window_bits, size_t max_table_bytes,
                             uint64_t* handle) {
    B200_CHECK((d_bases || h_bases) && handle && n > 0, -1, "bases_register: null argument or n == 0");
    B200_CHECK(window_bits == 0 || (window_bits >= 4 && window_bits <= 24), -1, "bases_register: window_bits %d not in {0, 4..24}", window_bits);
    BaseSet* bs = nullptr;
    if (int rc = bases_alloc(c, n, window_bits, max_table_bytes, &bs)) return rc;
    if (h_bases) {
        if (int rc = h2d_one(c, bs->t[c->slot]->d_table, h_bases, sizeof(G1Affine) * n, st)) return bases_drop(bs, rc);
    }
    if (int rc = bases_build(c, st, bs, d_bases, "bases_register")) return bases_drop(bs, rc);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("bases_register: %s", cudaGetErrorString(e)); return bases_drop(bs, -2); }
    *handle = bases_publish(bs);
    return 0;
}
int b200_bases_register_ex_dev(const void* d_bases, size_t n, int window_bits, size_t max_table_bytes, uint64_t* handle) {
    B200_ENTER(c, d_bases); StreamScope ss(c, nullptr);
    return bases_register_on(c, ss.st, d_bases, nullptr, n, window_bits, max_table_bytes, handle);
}
int b200_bases_register_ex(const b200_g1_affine* bases, size_t n, int window_bits, size_t max_table_bytes, uint64_t* handle) {
    B200_ENTER(c, nullptr);
    B200_CHECK(bases && handle && n > 0, -1, "bases_register: null argument or n == 0");
    StreamScope ss(c, nullptr);
    return bases_register_on(c, ss.st, nullptr, bases, n, window_bits, max_table_bytes, handle);
}
int b200_bases_register_dev(const void* d_bases, size_t n, int window_bits, uint64_t* handle) {
    return b200_bases_register_ex_dev(d_bases, n, window_bits, 0, handle);
}
int b200_bases_register(const b200_g1_affine* bases, size_t n, int window_bits, uint64_t* handle) {
    return b200_bases_register_ex(bases, n, window_bits, 0, handle);
}
int b200_bases_release(uint64_t handle) {
    CallGuard cg; if (!cg.ok) return -3;
    BaseSet* bs = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_tables.find(handle);
        B200_CHECK(it != g_tables.end(), -1, "bases_release: unknown handle %llu", (unsigned long long)handle);
        bs = it->second;
        g_tables.erase(it);
    }
    int cur = 0; cudaGetDevice(&cur);
    for (int s = 0; s < MAX_DEV; ++s) if (bs->t[s]) { cudaSetDevice(bs->t[s]->device); cudaDeviceSynchronize(); msm_table_free(bs->t[s]); delete bs->t[s]; }
    cudaSetDevice(cur);
    delete bs;
    return 0;
}
int b200_bases_info(uint64_t handle, size_t* n, int* window_bits, int* windows) {
    BaseSet* t = find_bases(handle);
    B200_CHECK(t, -1, "bases_info: unknown handle %llu", (unsigned long long)handle);
    if (n) *n = t->n;
    if (window_bits) *window_bits = t->c;
    if (windows) *windows = t->W;
    return 0;
}
int b200_bases_table(uint64_t handle, int* levels, int* windows_per_level, size_t* table_bytes) {
    BaseSet* t = find_bases(handle);
    B200_CHECK(t, -1, "bases_table: unknown handle %llu", (unsigned long long)handle);
    if (levels) *levels = t->L;
    if (windows_per_level) *windows_per_level = t->s;
    if (table_bytes) *table_bytes = sizeof(G1Affine) * t->n * (size_t)t->L;
    return 0;
}

// ---- MSM -----------------------------------------------------------------------------------------------------
int b200_msm_batch_dev(uint64_t bases, const void* d_scalars, size_t n, size_t stride, size_t batch, void* d_out_xyzz, void* stream) {
    B200_ENTER(c, d_scalars);
    BaseSet* t = find_bases(bases);
    B200_CHECK(t, -1, "msm: unknown bases handle %llu", (unsigned long long)bases);
    B200_CHECK(d_scalars && d_out_xyzz, -1, "msm: null pointer");
    B200_CHECK(n <= t->n, -1, "msm: %zu scalars per column, %zu bases registered", n, t->n);
    B200_CHECK(batch <= 1 || stride >= n, -1, "msm: column stride %zu < column length %zu", stride, n);
    if (batch == 0) return 0;
    StreamScope ss(c, stream);
    return msm_dev_on(c, ss.st, t, reinterpret_cast<const Fr*>(d_scalars), n, stride, batch, 0, reinterpret_cast<G1Xyzz*>(d_out_xyzz));
}
int b200_msm_batch(uint64_t bases, const b200_fr* const* scalars, size_t n, size_t batch, b200_g1_jac* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(scalars && out, -1, "msm: null pointer");
    if (batch == 0) return 0;
    BaseSet* t = find_bases(bases);
    B200_CHECK(t, -1, "msm: unknown bases handle %llu", (unsigned long long)bases);
    B200_CHECK(n <= t->n, -1, "msm: %zu scalars but only %zu bases registered", n, t->n);
    for (size_t b = 0; b < batch; ++b) B200_CHECK(scalars[b] || n == 0, -1, "msm: scalars[%zu] is null", b);
    std::vector<G1Xyzz> h(batch);
    const int nd = g_ndev.load();
    if (nd == 1 || n * batch < ((size_t)1 << 16)) {
        if (int rc = msm_host_on(c, t, scalars, batch, n, 0, h.data())) return rc;
    } else if (batch >= (size_t)nd) {
        // columns dealt round-robin over the devices: no exchange at all, every device stages and commits its own columns
        std::lock_guard<std::mutex> lk(g_multi_mu);
        std::vector<std::vector<const b200_fr*>> mine(nd);
        for (size_t b = 0; b < batch; ++b) mine[b % nd].push_back(scalars[b]);
        std::vector<std::vector<G1Xyzz>> part(nd);
        int rc = run_on_slots(nd, [&](int s) -> int {
            Ctx* cs; if (int r = get_ctx(&cs, s)) return r;
            part[s].resize(mine[s].size());
            return msm_host_on(cs, t, mine[s].data(), mine[s].size(), n, 0, part[s].data());
        });
        if (rc) return rc;
        for (size_t b = 0; b < batch; ++b) h[b] = part[b % nd][b / nd];
    } else {
        // fewer columns than devices: split the (scalar, base) pairs of every column into one contiguous range per device
        // (each against its table replica), then add the per-device partial sums in device order
        std::lock_guard<std::mutex> lk(g_multi_mu);
        std::vector<std::vector<G1Xyzz>> part(nd, std::vector<G1Xyzz>(batch));
        int rc = run_on_slots(nd, [&](int s) -> int {
            Ctx* cs; if (int r = get_ctx(&cs, s)) return r;
            size_t lo, hi; slice_bounds(n, s, nd, &lo, &hi);
            return msm_host_on(cs, t, scalars, batch, hi - lo, lo, part[s].data());
        });
        if (rc) return rc;
        for (size_t b = 0; b < batch; ++b) { G1Xyzz acc = part[0][b]; for (int s = 1; s < nd; ++s) acc = g1_add(acc, part[s][b]); h[b] = acc; }
    }
    normalize_host(h.data(), batch, out);
    return 0;
}
int b200_msm(uint64_t bases, const b200_fr* scalars, size_t n, b200_g1_jac* out) {
    const b200_fr* cols[1] = {scalars};
    return b200_msm_batch(bases, cols, n, 1, out);
}
// base-split MSM on device-resident slices (north star: bases split across the GPUs, partial sums reduced over NVLink)
int b200_msm_sharded_dev(uint64_t bases, const void* const* d_scalar_slices, size_t n, size_t batch, b200_g1_jac* out) {
    CallGuard cg; if (!cg.ok) return -3;
    const int nd = g_ndev.load();
    B200_CHECK(d_scalar_slices && out, -1, "msm_sharded: null pointer");
    BaseSet* t = find_bases(bases);
    B200_CHECK(t, -1, "msm: unknown bases handle %llu", (unsigned long long)bases);
    B200_CHECK(n <= t->n && batch >= 1 && batch <= 4096, -1, "msm_sharded: bad sizes");
    Ctx* cs[MAX_DEV];
    for (int s = 0; s < nd; ++s) if (int rc = get_ctx(&cs[s], s)) return rc;
    int cur = 0; cudaGetDevice(&cur);
    // gather buffer on device 0: [column][device] XYZZ partials
    if (cs[0]->small.ensure(sizeof(G1Xyzz) * batch * (nd + 2))) return -2;
    G1Xyzz* gather = cs[0]->small.as<G1Xyzz>();
    for (int s = 0; s < nd; ++s) {
        B200_CHECK(d_scalar_slices[s], -1, "msm_sharded: slice %d is null", s);
        size_t lo, hi; slice_bounds(n, s, nd, &lo, &hi);
        B200_CUDA(cudaSetDevice(cs[s]->dev));
        StreamScope ss(cs[s], nullptr);
        G1Xyzz* part = gather + batch * nd;           // device 0: a staging row behind the gather matrix
        if (s != 0) { if (cs[s]->small.ensure(sizeof(G1Xyzz) * batch)) { cudaSetDevice(cur); return -2; } part = cs[s]->small.as<G1Xyzz>(); }
        if (int rc = msm_dev_on(cs[s], ss.st, t, reinterpret_cast<const Fr*>(d_scalar_slices[s]), hi - lo, hi - lo, batch, lo, part)) { cudaSetDevice(cur); return rc; }
        // partial sums travel to device 0 over NVLink: column b of device s lands at gather[b * nd + s]
        B200_CUDA(cudaMemcpy2DAsync(gather + s, sizeof(G1Xyzz) * nd, part, sizeof(G1Xyzz), sizeof(G1Xyzz), batch, cudaMemcpyDefault, ss.st));
    }
    for (int s = 1; s < nd; ++s) { B200_CUDA(cudaSetDevice(cs[s]->dev)); B200_CUDA(cudaStreamSynchronize(cs[s]->stream)); }
    B200_CUDA(cudaSetDevice(cs[0]->dev));
    std::vector<G1Xyzz> h(batch);
    {
        StreamScope ss(cs[0], nullptr);
        G1Xyzz* sums = gather + batch * (nd + 1);
        if (int rc = g1_sum_run(gather, batch, nd, sums, ss.st)) { cudaSetDevice(cur); return rc; }
        B200_CUDA(cudaMemcpyAsync(h.data(), sums, sizeof(G1Xyzz) * batch, cudaMemcpyDeviceToHost, ss.st));
        B200_CUDA(cudaStreamSynchronize(ss.st));
    }
    cudaSetDevice(cur);
    normalize_host(h.data(), batch, out);
    return 0;
}
int b200_g1_sum_dev(const void* d_points_xyzz, size_t groups, size_t count, void* d_out_xyzz, void* stream) {
    B200_ENTER(c, d_points_xyzz);
    B200_CHECK(d_points_xyzz && d_out_xyzz, -1, "g1_sum: null pointer");
    StreamScope ss(c, stream);
    return g1_sum_run(reinterpret_cast<const G1Xyzz*>(d_points_xyzz), groups, count, reinterpret_cast<G1Xyzz*>(d_out_xyzz), ss.st);
}
static int g1_fft_on(Ctx* c, cudaStream_t st, const void* d_in_affine, uint32_t log_n, const b200_fr* omega, const b200_fr* scale, void* d_out_affine) {
    B200_CHECK(d_in_affine && omega && d_out_affine, -1, "g1_fft: null pointer");
    const Fr w = as_fr(omega);
    Fr sc = fp_one<FrTag>();
    if (scale) sc = as_fr(scale);
    return g1_fft_run(reinterpret_cast<const G1Affine*>(d_in_affine), log_n, w, scale ? &sc : nullptr, reinterpret_cast<G1Affine*>(d_out_affine), c->msm_ws.misc, st);
}
int b200_g1_fft_dev(const void* d_in_affine, uint32_t log_n, const b200_fr* omega, const b200_fr* scale, void* d_out_affine, void* stream) {
    B200_ENTER(c, d_in_affine); StreamScope ss(c, stream);
    return g1_fft_on(c, ss.st, d_in_affine, log_n, omega, scale, d_out_affine);
}
int b200_g1_fft(const b200_g1_affine* in, uint32_t log_n, const b200_fr* omega, const b200_fr* scale, b200_g1_affine* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(in && omega && out && log_n <= 26, -1, "g1_fft: bad argument");
    const size_t n = (size_t)1 << log_n;
    if (c->stage_a.ensure(sizeof(G1Affine) * n) || c->stage_b.ensure(sizeof(G1Affine) * n)) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, in, sizeof(G1Affine) * n, ss.st)) return rc;
    if (int rc = g1_fft_on(c, ss.st, c->stage_a.p, log_n, omega, scale, c->stage_b.p)) return rc;
    return d2h_one(c, out, c->stage_b.p, sizeof(G1Affine) * n, ss.st);
}
int b200_g1_fixed_base_mul_dev(const void* d_scalars, size_t n, const b200_g1_affine* base, void* d_out_affine, void* stream) {
    B200_ENTER(c, d_scalars);
    B200_CHECK(d_scalars && base && d_out_affine, -1, "g1_fixed_base_mul: null pointer");
    G1Affine b; memcpy(&b, base, sizeof b);
    StreamScope ss(c, stream);
    return g1_fixed_base_mul_run(reinterpret_cast<const Fr*>(d_scalars), n, b, reinterpret_cast<G1Affine*>(d_out_affine), ss.st);
}
int b200_g1_generate_dev(uint64_t seed, size_t n, void* d_out_affine, void* stream) {
    B200_ENTER(c, d_out_affine);
    B200_CHECK(d_out_affine, -1, "g1_generate: null pointer");
    StreamScope ss(c, stream);
    return g1_generate_run(seed, n, reinterpret_cast<G1Affine*>(d_out_affine), ss.st);
}
int b200_g1_normalize(const b200_g1_xyzz* points, size_t n, b200_g1_jac* out) {
    B200_CHECK(points && out, -1, "g1_normalize: null pointer");
    if (n == 0) return 0;
    std::vector<G1Xyzz> tmp(n);
    memcpy(tmp.data(), points, sizeof(G1Xyzz) * n);
    normalize_host(tmp.data(), n, out);
    return 0;
}

// ---- NTT -----------------------------------------------------------------------------------------------------
int b200_ntt_dev(const void* d_src, size_t src_stride, size_t n_in, void* d_tmp, void* d_dst, size_t dst_stride, uint32_t log_n,
                 const b200_fr* omega, int pre_mode, const b200_fr* pre, int post_mode, const b200_fr* post, size_t batch, void* stream) {
    B200_ENTER(c, d_src);
    B200_CHECK(d_src && d_tmp && d_dst && omega, -1, "ntt: null pointer");
    NttScale a, b;
    if (int rc = ntt_scales(pre_mode, pre, post_mode, post, &a, &b)) return rc;
    B200_CHECK(batch <= 65535, -1, "ntt: batch %zu out of range [0, 65535]", batch);     // before it narrows to the grid's int
    if (batch == 0) return 0;
    StreamScope ss(c, stream);
    return ntt_call(c, ss.st, reinterpret_cast<const Fr*>(d_src), src_stride, n_in, reinterpret_cast<Fr*>(d_tmp), reinterpret_cast<Fr*>(d_dst), dst_stride,
                    log_n, as_fr(omega), a, b, (int)batch);
}

// one transform of 2^log_n elements split across the devices of the process in contiguous natural-order slices (slice g of
// 2^log_n / n_devices elements on device g).  Enqueued on the calling thread's library stream of every device; b200_sync_all
// (or any later call on those streams) orders after it.  The exchanges of the six-step scheme are peer loads / stores inside
// the butterfly kernels (ntt.cu: ntt_run_sharded).
static int ntt_sharded_on(Ctx* const* cs, int nd, const Fr* const* src, Fr* const* tmp, Fr* const* dst, uint32_t log_n, uint64_t n_in, const Fr& omega,
                          const NttScale& pre, const NttScale& post) {
    NttPlan* plans[MAX_DEV]; int ids[MAX_DEV]; cudaStream_t st[MAX_DEV]; cudaEvent_t ev[MAX_DEV];
    int cur = 0; cudaGetDevice(&cur);
    for (int s = 0; s < nd; ++s) {
        cudaSetDevice(cs[s]->dev);
        plans[s] = warm_plan(s, log_n, omega, cs[s]->stream);
        if (!plans[s]) { cudaSetDevice(cur); return -2; }
        ids[s] = cs[s]->dev; st[s] = cs[s]->stream; ev[s] = cs[s]->last_ev;
        if (cs[s]->has_last && cs[s]->last_stream != st[s]) cudaStreamWaitEvent(st[s], cs[s]->last_ev, 0);
    }
    cudaSetDevice(cur);
    int rc = ntt_run_sharded(plans, nd, ids, src, tmp, dst, log_n, omega, pre, post, n_in, st, ev);
    for (int s = 0; s < nd && !rc; ++s) { cs[s]->last_stream = st[s]; cs[s]->has_last = true; }       // ev[s] was recorded after the last pass
    return rc;
}
int b200_ntt_sharded_dev(const void* const* d_src_slices, void* const* d_tmp_slices, void* const* d_dst_slices, uint32_t log_n, size_t n_in, const b200_fr* omega,
                         int pre_mode, const b200_fr* pre, int post_mode, const b200_fr* post) {
    CallGuard cg; if (!cg.ok) return -3;
    const int nd = g_ndev.load();
    B200_CHECK(nd >= 2, -1, "ntt_sharded: needs a multi-device process (b200_init_multi)");
    B200_CHECK(d_src_slices && d_tmp_slices && d_dst_slices && omega, -1, "ntt_sharded: null pointer");
    NttScale a, b;
    if (int rc = ntt_scales(pre_mode, pre, post_mode, post, &a, &b)) return rc;
    Ctx* cs[MAX_DEV];
    for (int s = 0; s < nd; ++s) {
        if (int rc = get_ctx(&cs[s], s)) return rc;
        B200_CHECK(d_src_slices[s] && d_tmp_slices[s] && d_dst_slices[s], -1, "ntt_sharded: slice %d is null", s);
    }
    return ntt_sharded_on(cs, nd, reinterpret_cast<const Fr* const*>(d_src_slices), reinterpret_cast<Fr* const*>(d_tmp_slices), reinterpret_cast<Fr* const*>(d_dst_slices),
                          log_n, n_in, as_fr(omega), a, b);
}

// host path on ONE device: polynomials src[p] (n_in each) -> dst[p] (2^log_n each), staged in sub-batches
static int ntt_host_on(Ctx* c, const b200_fr* const* src, b200_fr* const* dst, size_t batch, size_t n_in, uint32_t log_n, const Fr& omega,
                       const NttScale& pre, const NttScale& post) {
    if (batch == 0) return 0;
    DevGuard dg(c);
    const size_t N = (size_t)1 << log_n;
    const size_t sub = group_size(sizeof(Fr) * N * 3, batch);
    if (c->stage_a.ensure(sizeof(Fr) * n_in * sub) || c->stage_b.ensure(sizeof(Fr) * N * sub) || c->stage_c.ensure(sizeof(Fr) * N * sub)) return -2;
    StreamScope ss(c, nullptr);
    for (size_t b0 = 0; b0 < batch; b0 += sub) {
        const size_t nb = batch - b0 < sub ? batch - b0 : sub;
        std::vector<HostSeg> up(nb), down(nb);
        for (size_t p = 0; p < nb; ++p) {
            B200_CHECK(src[b0 + p] && dst[b0 + p], -1, "ntt: polynomial %zu is null", b0 + p);
            up[p] = HostSeg{(uint8_t*)const_cast<b200_fr*>(src[b0 + p]), sizeof(Fr) * n_in};
            down[p] = HostSeg{(uint8_t*)dst[b0 + p], sizeof(Fr) * N};
        }
        if (int rc = h2d_segments(c, c->stage_a.p, up.data(), nb, ss.st)) return rc;
        if (int rc = ntt_call(c, ss.st, c->stage_a.as<Fr>(), n_in, n_in, c->stage_b.as<Fr>(), c->stage_c.as<Fr>(), N, log_n, omega, pre, post, (int)nb)) return rc;
        if (int rc = d2h_segments(c, c->stage_c.p, down.data(), nb, ss.st)) return rc;
    }
    return 0;
}
// shared host path: on a multi-device process a batch is dealt over the devices; a single large transform is sharded
static int ntt_host(const b200_fr* const* src, b200_fr* const* dst, size_t batch, size_t n_in, uint32_t log_n, const Fr& omega,
                    const NttScale& pre, const NttScale& post) {
    B200_ENTER(c, nullptr);
    B200_CHECK(log_n >= 1 && log_n <= 28, -1, "ntt: log_n = %u out of range [1, 28]", log_n);
    const size_t N = (size_t)1 << log_n;
    B200_CHECK(n_in <= N, -1, "ntt: %zu input elements > 2^%u", n_in, log_n);
    if (batch == 0) return 0;
    const int nd = g_ndev.load();
    if (nd > 1 && batch >= 2 && N * batch >= ((size_t)1 << 18)) {
        std::lock_guard<std::mutex> lk(g_multi_mu);
        std::vector<std::vector<const b200_fr*>> s_in(nd);
        std::vector<std::vector<b200_fr*>> s_out(nd);
        for (size_t p = 0; p < batch; ++p) { s_in[p % nd].push_back(src[p]); s_out[p % nd].push_back(dst[p]); }
        return run_on_slots(nd, [&](int s) -> int {
            Ctx* cs; if (int r = get_ctx(&cs, s)) return r;
            return ntt_host_on(cs, s_in[s].data(), s_out[s].data(), s_in[s].size(), n_in, log_n, omega, pre, post);
        });
    }
    if (nd > 1 && batch == 1 && (int)log_n >= g_cfg.shard_min_logn) {
        // one large transform: every device uploads its contiguous slice over its own PCIe link, the passes exchange over NVLink
        std::lock_guard<std::mutex> lk(g_multi_mu);
        B200_CHECK(src[0] && dst[0], -1, "ntt: polynomial 0 is null");
        const size_t slice = N / nd;
        Fr* sl_src[MAX_DEV]; Fr* sl_tmp[MAX_DEV]; Fr* sl_dst[MAX_DEV]; Ctx* wcs[MAX_DEV];
        int rc = run_on_slots(nd, [&](int s) -> int {
            Ctx* cs; if (int r = get_ctx(&cs, s)) return r;
            DevGuard dg(cs);
            if (cs->stage_a.ensure(sizeof(Fr) * slice) || cs->stage_b.ensure(sizeof(Fr) * slice)) return -2;
            wcs[s] = cs; sl_src[s] = cs->stage_a.as<Fr>(); sl_tmp[s] = cs->stage_b.as<Fr>(); sl_dst[s] = cs->stage_a.as<Fr>();
            const size_t lo = slice * s, hi = lo + slice < n_in ? lo + slice : n_in;
            if (hi > lo) { if (int r = h2d_one(cs, sl_src[s], src[0] + lo, sizeof(Fr) * (hi - lo), cs->stream)) return r; }
            B200_CUDA(cudaStreamSynchronize(cs->stream));
            return 0;
        });
        if (rc) return rc;
        // the passes are enqueued on the worker contexts' streams from this thread (the workers are idle under g_multi_mu)
        if ((rc = ntt_sharded_on(wcs, nd, sl_src, sl_tmp, sl_dst, log_n, n_in, omega, pre, post))) return rc;
        return run_on_slots(nd, [&](int s) -> int {
            Ctx* cs = wcs[s];
            DevGuard dg(cs);
            return d2h_one(cs, dst[0] + slice * s, sl_dst[s], sizeof(Fr) * slice, cs->stream);
        });
    }
    return ntt_host_on(c, src, dst, batch, n_in, log_n, omega, pre, post);
}
int b200_fft_batch(b200_fr* const* a, size_t batch, uint32_t log_n, const b200_fr* omega) {
    B200_CHECK(a && omega, -1, "fft: null pointer");
    NttScale none;
    return ntt_host(a, a, batch, (size_t)1 << (log_n <= 28 ? log_n : 0), log_n, as_fr(omega), none, none);
}
int b200_fft(b200_fr* a, uint32_t log_n, const b200_fr* omega) { b200_fr* p[1] = {a}; return b200_fft_batch(p, 1, log_n, omega); }
int b200_ifft_batch(b200_fr* const* a, size_t batch, uint32_t log_n, const b200_fr* omega_inv, const b200_fr* divisor) {
    B200_CHECK(a && omega_inv && divisor, -1, "ifft: null pointer");
    NttScale none, post;
    post.mode = 1; post.c[0] = as_fr(divisor);
    return ntt_host(a, a, batch, (size_t)1 << (log_n <= 28 ? log_n : 0), log_n, as_fr(omega_inv), none, post);
}
int b200_ifft(b200_fr* a, uint32_t log_n, const b200_fr* omega_inv, const b200_fr* divisor) {
    b200_fr* p[1] = {a};
    return b200_ifft_batch(p, 1, log_n, omega_inv, divisor);
}
int b200_coeff_to_extended_batch(const b200_fr* const* coeffs, size_t batch, size_t n_coeffs, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta, b200_fr* const* out) {
    B200_CHECK(coeffs && out && ext_omega && zeta, -1, "coeff_to_extended: null pointer");
    NttScale none;
    return ntt_host(coeffs, out, batch, n_coeffs, ext_k, as_fr(ext_omega), coset_pre(as_fr(zeta)), none);
}
int b200_coeff_to_extended(const b200_fr* coeffs, size_t n_coeffs, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta, b200_fr* out) {
    const b200_fr* s[1] = {coeffs}; b200_fr* d[1] = {out};
    return b200_coeff_to_extended_batch(s, 1, n_coeffs, ext_k, ext_omega, zeta, d);
}
int b200_extended_to_coeff(b200_fr* a, uint32_t ext_k, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor, const b200_fr* zeta) {
    B200_CHECK(a && ext_omega_inv && ext_ifft_divisor && zeta, -1, "extended_to_coeff: null pointer");
    NttScale none;
    b200_fr* p[1] = {a};
    return ntt_host(p, p, 1, (size_t)1 << (ext_k <= 28 ? ext_k : 0), ext_k, as_fr(ext_omega_inv), none, coset_post(as_fr(ext_ifft_divisor), as_fr(zeta)));
}

// ---- polynomial ops --------------------------------------------------------------------------------------------
static int poly_op_on(Ctx*, cudaStream_t st, int op, const void* d_a, const void* d_b, const b200_fr* s, void* d_out, size_t n) {
    B200_CHECK(op >= 0 && op <= 4, -1, "poly_op: unknown op %d", op);
    B200_CHECK(d_a && d_out && (op == POLY_SCALE || d_b) && (op < POLY_SCALE || s), -1, "poly_op: missing operand for op %d", op);
    Fr sv = fp_zero<FrTag>();
    if (s) sv = as_fr(s);
    return poly_binary(op, reinterpret_cast<const Fr*>(d_a), reinterpret_cast<const Fr*>(d_b), s ? &sv : nullptr, reinterpret_cast<Fr*>(d_out), n, st);
}
int b200_poly_op_dev(int op, const void* d_a, const void* d_b, const b200_fr* s, void* d_out, size_t n, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return poly_op_on(c, ss.st, op, d_a, d_b, s, d_out, n);
}
int b200_poly_op(int op, const b200_fr* a, const b200_fr* b, const b200_fr* s, b200_fr* out, size_t n) {
    B200_ENTER(c, nullptr);
    B200_CHECK(a && out, -1, "poly_op: null pointer");
    if (n == 0) return 0;
    const bool need_b = op != POLY_SCALE;
    B200_CHECK(!need_b || b, -1, "poly_op: missing operand b");
    if (c->stage_a.ensure(sizeof(Fr) * n) || (need_b && c->stage_b.ensure(sizeof(Fr) * n))) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, a, sizeof(Fr) * n, ss.st)) return rc;
    if (need_b) { if (int rc = h2d_one(c, c->stage_b.p, b, sizeof(Fr) * n, ss.st)) return rc; }
    if (int rc = poly_op_on(c, ss.st, op, c->stage_a.p, need_b ? c->stage_b.p : nullptr, s, c->stage_a.p, n)) return rc;
    return d2h_one(c, out, c->stage_a.p, sizeof(Fr) * n, ss.st);
}
static int lincomb_on(Ctx* c, cudaStream_t st, const void* const* d_polys, const b200_fr* scalars, size_t count, size_t n, void* d_out) {
    B200_CHECK(d_out && (count == 0 || (d_polys && scalars)), -1, "poly_lincomb: null pointer");
    std::vector<Fr> sv(count);
    if (count) memcpy(sv.data(), scalars, sizeof(Fr) * count);
    return poly_lincomb(reinterpret_cast<const Fr* const*>(d_polys), sv.data(), count, reinterpret_cast<Fr*>(d_out), n, c->ring, st);
}
int b200_poly_lincomb_dev(const void* const* d_polys, const b200_fr* scalars, size_t count, size_t n, void* d_out, void* stream) {
    B200_ENTER(c, d_out); StreamScope ss(c, stream);
    return lincomb_on(c, ss.st, d_polys, scalars, count, n, d_out);
}
int b200_poly_lincomb(const b200_fr* const* polys, const b200_fr* scalars, size_t count, size_t n, b200_fr* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(out && (count == 0 || (polys && scalars)), -1, "poly_lincomb: null pointer");
    if (n == 0) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * n * (count ? count : 1)) || c->stage_b.ensure(sizeof(Fr) * n)) return -2;
    std::vector<const void*> ptrs(count);
    std::vector<HostSeg> up(count);
    for (size_t j = 0; j < count; ++j) {
        B200_CHECK(polys[j], -1, "poly_lincomb: polys[%zu] is null", j);
        ptrs[j] = c->stage_a.as<Fr>() + j * n;
        up[j] = HostSeg{(uint8_t*)const_cast<b200_fr*>(polys[j]), sizeof(Fr) * n};
    }
    StreamScope ss(c, nullptr);
    if (int rc = h2d_segments(c, c->stage_a.p, up.data(), count, ss.st)) return rc;
    if (int rc = lincomb_on(c, ss.st, ptrs.data(), scalars, count, n, c->stage_b.p)) return rc;
    return d2h_one(c, out, c->stage_b.p, sizeof(Fr) * n, ss.st);
}
static int scale_cycle_on(Ctx* c, cudaStream_t st, void* d_a, size_t n, const b200_fr* consts, uint32_t period) {
    B200_CHECK(d_a && consts && period > 0 && period <= 1024, -1, "poly_scale_cycle: bad argument");
    return poly_scale_cycle(reinterpret_cast<const Fr*>(d_a), reinterpret_cast<const Fr*>(consts), period, reinterpret_cast<Fr*>(d_a), n, c->ring, st);
}
int b200_poly_scale_cycle_dev(void* d_a, size_t n, const b200_fr* consts, uint32_t period, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return scale_cycle_on(c, ss.st, d_a, n, consts, period);
}
int b200_poly_scale_cycle(b200_fr* a, size_t n, const b200_fr* consts, uint32_t period) {
    B200_ENTER(c, nullptr);
    B200_CHECK(a && consts, -1, "poly_scale_cycle: null pointer");
    if (n == 0) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * n)) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, a, sizeof(Fr) * n, ss.st)) return rc;
    if (int rc = scale_cycle_on(c, ss.st, c->stage_a.p, n, consts, period)) return rc;
    return d2h_one(c, a, c->stage_a.p, sizeof(Fr) * n, ss.st);
}
static int eval_batch_on(Ctx* c, cudaStream_t st, const void* d_polys, size_t stride, size_t n, const b200_fr* x, size_t batch, void* d_out) {
    B200_CHECK(d_polys && x && d_out, -1, "poly_eval: null pointer");
    if (batch == 0) return 0;
    std::vector<Fr> xv(batch);
    memcpy(xv.data(), x, sizeof(Fr) * batch);
    return poly_eval(reinterpret_cast<const Fr*>(d_polys), stride, n, xv.data(), reinterpret_cast<Fr*>(d_out), (int)batch, c->poly_ws, c->ring, st);
}
int b200_poly_eval_batch_dev(const void* d_polys, size_t stride, size_t n, const b200_fr* x, size_t batch, void* d_out, void* stream) {
    B200_ENTER(c, d_polys); StreamScope ss(c, stream);
    return eval_batch_on(c, ss.st, d_polys, stride, n, x, batch, d_out);
}
int b200_poly_eval_batch(const b200_fr* const* polys, size_t n, const b200_fr* x, size_t batch, b200_fr* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(polys && x && out, -1, "poly_eval: null pointer");
    if (batch == 0) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * (n ? n : 1) * batch) || c->small.ensure(sizeof(Fr) * batch)) return -2;
    std::vector<HostSeg> up(batch);
    for (size_t p = 0; p < batch; ++p) {
        B200_CHECK(n == 0 || polys[p], -1, "poly_eval: polys[%zu] is null", p);
        up[p] = HostSeg{(uint8_t*)const_cast<b200_fr*>(polys[p]), sizeof(Fr) * n};
    }
    StreamScope ss(c, nullptr);
    if (n) { if (int rc = h2d_segments(c, c->stage_a.p, up.data(), batch, ss.st)) return rc; }
    if (int rc = eval_batch_on(c, ss.st, c->stage_a.p, n, n, x, batch, c->small.p)) return rc;
    return d2h_one(c, out, c->small.p, sizeof(Fr) * batch, ss.st);
}
int b200_poly_eval(const b200_fr* coeffs, size_t n, const b200_fr* x, b200_fr* out) {
    const b200_fr* p[1] = {coeffs};
    return b200_poly_eval_batch(p, n, x, 1, out);
}
static int batch_invert_on(Ctx* c, cudaStream_t st, void* d_a, size_t n) {
    B200_CHECK(d_a, -1, "batch_invert: null pointer");
    return poly_batch_invert(reinterpret_cast<Fr*>(d_a), n, c->poly_ws, st);
}
int b200_batch_invert_dev(void* d_a, size_t n, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return batch_invert_on(c, ss.st, d_a, n);
}
int b200_batch_invert(b200_fr* a, size_t n) {
    B200_ENTER(c, nullptr);
    B200_CHECK(a, -1, "batch_invert: null pointer");
    if (n == 0) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * n)) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, a, sizeof(Fr) * n, ss.st)) return rc;
    if (int rc = batch_invert_on(c, ss.st, c->stage_a.p, n)) return rc;
    return d2h_one(c, a, c->stage_a.p, sizeof(Fr) * n, ss.st);
}
static int prefix_scan_on(Ctx* c, cudaStream_t st, int product, const void* d_a, size_t a_stride, size_t n, size_t batch, const b200_fr* inits, void* d_out, size_t out_stride) {
    B200_CHECK(d_a && inits && d_out, -1, "prefix_scan: null pointer");
    B200_CHECK(batch <= 1 || (a_stride >= n && out_stride >= n), -1, "prefix_scan: column stride smaller than the column");
    if (batch == 0) return 0;
    std::vector<Fr> iv(batch);
    memcpy(iv.data(), inits, sizeof(Fr) * batch);
    return poly_prefix_scan(product != 0, reinterpret_cast<const Fr*>(d_a), a_stride, n, iv.data(), reinterpret_cast<Fr*>(d_out), out_stride, (int)batch, c->poly_ws, c->ring, st);
}
int b200_prefix_scan_dev(int product, const void* d_a, size_t n, const b200_fr* init, void* d_out, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return prefix_scan_on(c, ss.st, product, d_a, n, n, 1, init, d_out, n);
}
int b200_prefix_scan_batch_dev(int product, const void* d_a, size_t a_stride, size_t n, size_t batch, const b200_fr* inits, void* d_out, size_t out_stride, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return prefix_scan_on(c, ss.st, product, d_a, a_stride, n, batch, inits, d_out, out_stride);
}
int b200_prefix_scan(int product, const b200_fr* a, size_t n, const b200_fr* init, b200_fr* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(a && init && out, -1, "prefix_scan: null pointer");
    if (n == 0) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * n) || c->stage_b.ensure(sizeof(Fr) * n)) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, a, sizeof(Fr) * n, ss.st)) return rc;
    if (int rc = prefix_scan_on(c, ss.st, product, c->stage_a.p, n, n, 1, init, c->stage_b.p, n)) return rc;
    return d2h_one(c, out, c->stage_b.p, sizeof(Fr) * n, ss.st);
}
static int kate_division_on(Ctx* c, cudaStream_t st, const void* d_a, size_t n, const b200_fr* b, void* d_q) {
    B200_CHECK(d_a && b && d_q, -1, "kate_division: null pointer");
    // q[e] is computed from a[e + 1 ..]: a thread's stores would overwrite the coefficient its neighbour still has to read
    B200_CHECK(d_q != d_a, -1, "kate_division: q must not alias a (the quotient cannot be computed in place)");
    const Fr bv = as_fr(b);
    return poly_kate_division(reinterpret_cast<const Fr*>(d_a), n, &bv, reinterpret_cast<Fr*>(d_q), c->poly_ws, c->ring, st);
}
int b200_kate_division_dev(const void* d_a, size_t n, const b200_fr* b, void* d_q, void* stream) {
    B200_ENTER(c, d_a); StreamScope ss(c, stream);
    return kate_division_on(c, ss.st, d_a, n, b, d_q);
}
int b200_kate_division(const b200_fr* a, size_t n, const b200_fr* b, b200_fr* q) {
    B200_ENTER(c, nullptr);
    B200_CHECK(a && b && q, -1, "kate_division: null pointer");
    B200_CHECK(n >= 1, -1, "kate_division: empty polynomial");
    if (n == 1) return 0;
    if (c->stage_a.ensure(sizeof(Fr) * n) || c->stage_b.ensure(sizeof(Fr) * n)) return -2;
    StreamScope ss(c, nullptr);
    if (int rc = h2d_one(c, c->stage_a.p, a, sizeof(Fr) * n, ss.st)) return rc;
    if (int rc = kate_division_on(c, ss.st, c->stage_a.p, n, b, c->stage_b.p)) return rc;
    return d2h_one(c, q, c->stage_b.p, sizeof(Fr) * (n - 1), ss.st);
}

// ---- mv-lookup multiplicities --------------------------------------------------------------------------------------------------
static int lookup_multiplicities_on(Ctx* c, cudaStream_t st, const void* d_table, size_t n_table, const void* const* d_inputs, size_t n_inputs, size_t n_rows, void* d_m,
                                    uint64_t* missing) {
    B200_CHECK(d_table && d_m && d_inputs && n_inputs >= 1, -1, "lookup_multiplicities: null pointer");
    unsigned long long* d_missing = nullptr;
    if (int rc = lookup_multiplicities_run(reinterpret_cast<const Fr*>(d_table), n_table, reinterpret_cast<const Fr* const*>(d_inputs), n_inputs, n_rows,
                                           reinterpret_cast<Fr*>(d_m), c->msm_ws.misc, c->ring, &d_missing, st)) return rc;
    if (missing) {
        unsigned long long h = 0;
        if (int rc = read_back(&h, d_missing, sizeof h, st)) return rc;
        *missing = h;
    }
    return 0;
}
int b200_lookup_multiplicities_dev(const void* d_table, size_t n_table, const void* const* d_inputs, size_t n_inputs, size_t n_rows, void* d_m, uint64_t* missing, void* stream) {
    B200_ENTER(c, d_table); StreamScope ss(c, stream);
    return lookup_multiplicities_on(c, ss.st, d_table, n_table, d_inputs, n_inputs, n_rows, d_m, missing);
}
int b200_lookup_multiplicities(const b200_fr* table, size_t n_table, const b200_fr* const* inputs, size_t n_inputs, size_t n_rows, b200_fr* m, uint64_t* missing) {
    B200_ENTER(c, nullptr);
    B200_CHECK(table && inputs && m && n_inputs >= 1, -1, "lookup_multiplicities: null pointer");
    if (c->stage_a.ensure(sizeof(Fr) * (n_table + n_inputs * (n_rows ? n_rows : 1))) || c->stage_b.ensure(sizeof(Fr) * n_table)) return -2;
    // the table and then every input column, back to back in stage_a
    std::vector<const void*> ptrs(n_inputs);
    std::vector<HostSeg> up(1 + (n_rows ? n_inputs : 0));
    up[0] = HostSeg{(uint8_t*)const_cast<b200_fr*>(table), sizeof(Fr) * n_table};
    for (size_t j = 0; j < n_inputs; ++j) {
        B200_CHECK(inputs[j] || n_rows == 0, -1, "lookup_multiplicities: inputs[%zu] is null", j);
        ptrs[j] = c->stage_a.as<Fr>() + n_table + j * n_rows;
        if (n_rows) up[1 + j] = HostSeg{(uint8_t*)const_cast<b200_fr*>(inputs[j]), sizeof(Fr) * n_rows};
    }
    StreamScope ss(c, nullptr);
    if (int rc = h2d_segments(c, c->stage_a.p, up.data(), up.size(), ss.st)) return rc;
    uint64_t miss = 0;
    if (int rc = lookup_multiplicities_on(c, ss.st, c->stage_a.p, n_table, ptrs.data(), n_inputs, n_rows, c->stage_b.p, &miss)) return rc;
    if (int rc = d2h_one(c, m, c->stage_b.p, sizeof(Fr) * n_table, ss.st)) return rc;
    if (missing) *missing = miss;
    return 0;
}

// ---- permutation keygen ------------------------------------------------------------------------------------------------------------
// n_map_columns mapping columns at d_map -> sigma columns at d_out (stride out_stride); a cell is valid when its column is < n_columns and its
// row < 2^k.  The host-pointer entry point calls this once per column group, with n_columns = every column of the key.
static int perm_sigmas_on(Ctx* c, cudaStream_t st, const void* d_map, size_t n_map_columns, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta,
                          void* d_out, size_t out_stride, unsigned long long* d_invalid) {
    B200_CHECK(d_map && d_out && omega && delta, -1, "permutation_sigmas: null pointer");
    B200_CHECK(n_columns < (1ull << 32), -1, "permutation_sigmas: %zu columns, at most 2^32 - 1", n_columns);
    const uint32_t lo_bits = (k + 1) / 2;
    std::vector<Fr> tab(n_columns + ((size_t)1 << lo_bits) + ((size_t)1 << (k - lo_bits)));
    const Fr d = as_fr(delta);
    tab[0] = fp_one<FrTag>();
    for (size_t j = 1; j < n_columns; ++j) tab[j] = tab[j - 1] * d;
    omega_power_table(tab.data() + n_columns, lo_bits, k, as_fr(omega));
    return perm_sigmas_run(reinterpret_cast<const uint32_t*>(d_map), n_map_columns, k, tab.data(), n_columns, lo_bits, reinterpret_cast<Fr*>(d_out), out_stride, d_invalid,
                           c->ring, st);
}
int b200_permutation_sigmas_dev(const void* d_mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, void* d_out, size_t out_stride,
                                uint64_t* invalid, void* stream) {
    B200_ENTER(c, d_out);
    B200_CHECK(k <= 28, -1, "permutation_sigmas_dev: k = %u out of range [0, 28]", k);
    B200_CHECK(out_stride >= ((size_t)1 << k), -1, "permutation_sigmas_dev: out_stride %zu < 2^%u", out_stride, k);
    if (n_columns == 0) return 0;
    B200_CHECK(d_mapping && d_out && omega && delta, -1, "permutation_sigmas_dev: null pointer");
    StreamScope ss(c, stream);
    unsigned long long* d_inv = nullptr;
    if (invalid) {
        if (c->small.ensure(sizeof(unsigned long long))) return -2;
        d_inv = c->small.as<unsigned long long>();
        B200_CUDA(cudaMemsetAsync(d_inv, 0, sizeof *d_inv, ss.st));
    }
    if (int rc = perm_sigmas_on(c, ss.st, d_mapping, n_columns, n_columns, k, omega, delta, d_out, out_stride, d_inv)) return rc;
    if (invalid) {
        unsigned long long h = 0;
        if (int rc = read_back(&h, d_inv, sizeof h, ss.st)) return rc;
        *invalid = h;
    }
    return 0;
}
// index of the first cell (column >= n_columns or row >= n) of the host mapping, or `cells` when every cell is valid; large mappings are
// scanned by several host threads
static size_t first_invalid_cell(const uint32_t* map, size_t cells, size_t n_columns, size_t n) {
    auto scan = [=](size_t lo, size_t hi) { for (size_t e = lo; e < hi; ++e) if (map[2 * e] >= n_columns || map[2 * e + 1] >= n) return e; return cells; };
    const size_t T = cells >= ((size_t)1 << 22) ? 8 : 1, part = (cells + T - 1) / T;
    std::vector<size_t> first(T, cells);
    std::vector<std::thread> th;
    for (size_t t = 1; t < T; ++t) th.emplace_back([&, t] { first[t] = scan(t * part < cells ? t * part : cells, (t + 1) * part < cells ? (t + 1) * part : cells); });
    first[0] = scan(0, part < cells ? part : cells);
    for (auto& x : th) x.join();
    for (size_t t = 0; t < T; ++t) if (first[t] < cells) return first[t];
    return cells;
}
// host path on ONE device: the columns cols[0 .. count) of the mapping -> out[cols[.]], staged in column groups bounded by the call budget
static int perm_sigmas_host_on(Ctx* c, const uint32_t* mapping, const size_t* cols, size_t count, size_t n_columns, uint32_t k, const b200_fr* omega,
                               const b200_fr* delta, b200_fr* const* out) {
    if (count == 0) return 0;
    DevGuard dg(c);
    const size_t n = (size_t)1 << k, map_bytes = 2 * sizeof(uint32_t) * n, col_bytes = sizeof(Fr) * n;
    const size_t sub = group_size(map_bytes + col_bytes, count);
    if (c->stage_a.ensure(map_bytes * sub) || c->stage_b.ensure(col_bytes * sub)) return -2;
    StreamScope ss(c, nullptr);
    for (size_t b0 = 0; b0 < count; b0 += sub) {
        const size_t nb = count - b0 < sub ? count - b0 : sub;
        std::vector<HostSeg> up, down;            // adjacent columns (in the mapping, and in the caller's output) merge into one segment
        for (size_t b = b0; b < b0 + nb; ++b) {
            uint8_t* m = (uint8_t*)const_cast<uint32_t*>(mapping + 2 * n * cols[b]);
            uint8_t* o = (uint8_t*)out[cols[b]];
            if (!up.empty() && up.back().p + up.back().bytes == m) up.back().bytes += map_bytes; else up.push_back(HostSeg{m, map_bytes});
            if (!down.empty() && down.back().p + down.back().bytes == o) down.back().bytes += col_bytes; else down.push_back(HostSeg{o, col_bytes});
        }
        if (int rc = h2d_segments(c, c->stage_a.p, up.data(), up.size(), ss.st)) return rc;
        if (int rc = perm_sigmas_on(c, ss.st, c->stage_a.p, nb, n_columns, k, omega, delta, c->stage_b.p, n, nullptr)) return rc;
        if (int rc = d2h_segments(c, c->stage_b.p, down.data(), down.size(), ss.st)) return rc;
    }
    return 0;
}
int b200_permutation_sigmas(const uint32_t* mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, b200_fr* const* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(k <= 28, -1, "permutation_sigmas: k = %u out of range [0, 28]", k);
    if (n_columns == 0) return 0;
    B200_CHECK(mapping && omega && delta && out, -1, "permutation_sigmas: null pointer");
    B200_CHECK(n_columns < (1ull << 32), -1, "permutation_sigmas: %zu columns, at most 2^32 - 1", n_columns);
    for (size_t j = 0; j < n_columns; ++j) B200_CHECK(out[j], -1, "permutation_sigmas: out[%zu] is null", j);
    const size_t n = (size_t)1 << k, cells = n_columns * n;
    const size_t bad = first_invalid_cell(mapping, cells, n_columns, n);
    B200_CHECK(bad == cells, -1, "permutation_sigmas: cell (column %zu, row %zu) maps to (%u, %u), outside %zu columns of 2^%u rows", bad / n, bad % n,
               mapping[2 * bad], mapping[2 * bad + 1], n_columns, k);
    const int nd = g_ndev.load();
    if (nd > 1 && n_columns >= 2 && cells >= ((size_t)1 << 18)) {
        // column groups dealt round-robin over the devices, as the batched transforms deal polynomials
        std::lock_guard<std::mutex> lk(g_multi_mu);
        std::vector<std::vector<size_t>> mine(nd);
        for (size_t j = 0; j < n_columns; ++j) mine[j % nd].push_back(j);
        return run_on_slots(nd, [&](int s) -> int {
            Ctx* cs; if (int r = get_ctx(&cs, s)) return r;
            return perm_sigmas_host_on(cs, mapping, mine[s].data(), mine[s].size(), n_columns, k, omega, delta, out);
        });
    }
    std::vector<size_t> all(n_columns);
    for (size_t j = 0; j < n_columns; ++j) all[j] = j;
    return perm_sigmas_host_on(c, mapping, all.data(), n_columns, n_columns, k, omega, delta, out);
}

// ---- quotient numerator (evaluate_h) ------------------------------------------------------------------------------
static_assert(sizeof(b200_instr) == sizeof(QInstr) && sizeof(b200_col_ref) == sizeof(QLoad), "ABI structs must match the kernel's");
static int quotient_eval_on(Ctx* c, cudaStream_t st, const void* const* d_columns, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_col_ref* loads, size_t n_loads,
                            const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr, void* d_out, uint32_t out_shift = 0, uint32_t out_off = 0,
                            const uint32_t* col_shifts = nullptr) {
    B200_CHECK(d_out && (n_columns == 0 || d_columns) && (n_loads == 0 || loads) && (n_constants == 0 || constants) && (n_instr == 0 || program), -1, "quotient_eval: null pointer");
    B200_CHECK(ext_k >= k && ext_k <= 28, -1, "quotient_eval: need k <= ext_k <= 28");
    const uint64_t N = 1ull << ext_k, scale = 1ull << (ext_k - k);
    std::vector<QLoad> ql(n_loads);
    for (size_t i = 0; i < n_loads; ++i) {
        ql[i].column = loads[i].column;
        const int64_t off = (int64_t)loads[i].rotation * (int64_t)scale;           // Rotation(r) on the extended domain = r * 2^(ext_k - k)
        ql[i].offset = (uint32_t)(((off % (int64_t)N) + (int64_t)N) % (int64_t)N);
    }
    return quotient_eval_run(reinterpret_cast<const Fr* const*>(d_columns), col_shifts, n_columns, ext_k, ql.data(), n_loads, reinterpret_cast<const Fr*>(constants), n_constants,
                             reinterpret_cast<const QInstr*>(program), n_instr, reinterpret_cast<Fr*>(d_out), out_shift, out_off, c->ring, st);
}
int b200_quotient_eval_dev(const void* const* d_columns, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_col_ref* loads, size_t n_loads,
                           const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr, void* d_out, void* stream) {
    B200_ENTER(c, d_out); StreamScope ss(c, stream);
    return quotient_eval_on(c, ss.st, d_columns, n_columns, k, ext_k, loads, n_loads, constants, n_constants, program, n_instr, d_out);
}
int b200_quotient_eval(const b200_fr* const* columns, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_col_ref* loads, size_t n_loads,
                       const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr, b200_fr* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(out && (n_columns == 0 || columns), -1, "quotient_eval: null pointer");
    B200_CHECK(ext_k >= 1 && ext_k <= 28, -1, "quotient_eval: ext_k out of range");
    const size_t N = (size_t)1 << ext_k;
    if (c->stage_a.ensure(sizeof(Fr) * N * (n_columns ? n_columns : 1)) || c->stage_b.ensure(sizeof(Fr) * N)) return -2;
    std::vector<const void*> ptrs(n_columns);
    std::vector<HostSeg> up(n_columns);
    for (size_t i = 0; i < n_columns; ++i) {
        B200_CHECK(columns[i], -1, "quotient_eval: column %zu is null", i);
        ptrs[i] = c->stage_a.as<Fr>() + i * N;
        up[i] = HostSeg{(uint8_t*)const_cast<b200_fr*>(columns[i]), sizeof(Fr) * N};
    }
    StreamScope ss(c, nullptr);
    if (int rc = h2d_segments(c, c->stage_a.p, up.data(), n_columns, ss.st)) return rc;
    if (int rc = quotient_eval_on(c, ss.st, ptrs.data(), n_columns, k, ext_k, loads, n_loads, constants, n_constants, program, n_instr, c->stage_b.p)) return rc;
    return d2h_one(c, out, c->stage_b.p, sizeof(Fr) * N, ss.st);
}

// evaluate_h by parts: for any p <= ext_k - k the extended domain of N = 2^ext_k points is the disjoint union of P = 2^p cosets of
// m = N / P points; part c holds the extended indices c + P i (the points g_c w_m^i, g_c = zeta w_N^c, w_m = w_N^P).  A rotation by r
// rows moves an index by r 2^(ext_k - k), a multiple of P, so it stays inside part c: the numerator on part c reads only part c of every
// column, m elements per column.  p = 0 is one part, the whole extended coset; p = ext_k - k is 2^(ext_k - k) parts of n points.  Per part:
//   coefficient columns: p = 0: the size-N coset NTT of each column from its coefficients (pre-scaled by [1, zeta, zeta^2], n_in = its
//                        length, so the transform skips the zero padding), one column per transform (tmp holds one coset);
//                        p > 0: part c of column q is the size-m NTT (w_m) of b_s = sum_j q_{s+jm} g_c^{s+jm}, folded and pre-scaled
//                        by ONE poly_coset_fold launch for every coefficient column (a device table of (address, length) per column) from
//                        two small power tables of w_N, then transformed in batches of at most P columns (tmp holds P parts);
//   extended columns:    read in place by the interpreter, elements c, c + P, c + 2P, ... of cols[i] (a load of stride P from cols[i] + c);
//                        or, when stage_ext is given, staged by stage_ext(c) as m contiguous elements at cols[i] and read densely;
//   numerator:           the interpreter on m rows (rotations scale by 2^(ext_k - p - k), wrap mod m), storing row i at index c + P i of h.
// cols[i] = device address of column i, lengths[i] < N: coefficient form, == N: extended.  Device memory: parts = n_coeff * m elements (the
// coefficient columns' parts, in column order), tmp = N elements, and for p > 0 the power and fold tables in c->small.  Both evaluate_h
// entry points run this loop: the host one on columns it uploads, the _dev one on the caller's.
static int evaluate_h_parts_on(Ctx* c, cudaStream_t st, const Fr* const* cols, const size_t* lengths, size_t n_columns, uint32_t k, uint32_t ext_k, uint32_t p,
                               const Fr& ext_omega, const Fr& zeta, const b200_col_ref* loads, size_t n_loads, const b200_fr* constants, size_t n_constants,
                               const b200_instr* program, size_t n_instr, Fr* parts, Fr* tmp, Fr* h, const std::function<int(size_t)>& stage_ext) {
    const size_t N = (size_t)1 << ext_k, P = (size_t)1 << p, m = N >> p;
    std::vector<FoldCol> fold;
    for (size_t i = 0; i < n_columns; ++i) if (lengths[i] < N) fold.push_back(FoldCol{cols[i], lengths[i]});
    const uint32_t lo_bits = (ext_k + 1) / 2;
    const Fr* d_tab = nullptr;
    const FoldCol* d_fold = nullptr;
    NttScale zeta_cycle = coset_pre(zeta), none;
    if (p > 0 && !fold.empty()) {
        const size_t n_lo = (size_t)1 << lo_bits, n_hi = N >> lo_bits, n_tab = 3 + n_lo + n_hi;
        // [1, zeta, zeta^2 | w_N^e, e < n_lo | w_N^(e n_lo), e < n_hi | the fold table], staged once for every part
        const size_t tab_bytes = sizeof(Fr) * n_tab, fold_bytes = sizeof(FoldCol) * fold.size();
        if (c->small.ensure(tab_bytes + fold_bytes)) return -2;
        std::vector<uint8_t> blob(tab_bytes + fold_bytes);
        Fr* tab = reinterpret_cast<Fr*>(blob.data());
        for (int i = 0; i < 3; ++i) tab[i] = zeta_cycle.c[i];
        omega_power_table(tab + 3, lo_bits, ext_k, ext_omega);
        memcpy(blob.data() + tab_bytes, fold.data(), fold_bytes);
        if (int rc = ring_upload(c, c->small.p, blob.data(), blob.size(), st)) return rc;
        d_tab = c->small.as<Fr>();
        d_fold = reinterpret_cast<const FoldCol*>(c->small.as<uint8_t>() + tab_bytes);
    }
    Fr omega_m = ext_omega;
    for (uint32_t i = 0; i < p; ++i) omega_m = omega_m * omega_m;
    std::vector<const void*> ptrs(n_columns);
    std::vector<uint32_t> shifts(n_columns, 0);
    for (size_t i = 0, j = 0; i < n_columns; ++i) if (lengths[i] < N) ptrs[i] = parts + m * j++;
    for (size_t part = 0; part < P; ++part) {
        if (p == 0) {
            for (size_t j = 0; j < fold.size(); ++j) {
                const size_t len = fold[j].len;
                if (int rc = ntt_call(c, st, fold[j].a, len, len, tmp, parts + j * m, m, ext_k, ext_omega, zeta_cycle, none, 1)) return rc;
            }
        } else if (!fold.empty()) {
            if (int rc = poly_coset_fold(d_fold, fold.size(), d_tab, lo_bits, ext_k, part, parts, m, m, st)) return rc;
            for (size_t j0 = 0; j0 < fold.size(); j0 += P) {
                const int nb = (int)(fold.size() - j0 < P ? fold.size() - j0 : P);
                if (int rc = ntt_call(c, st, parts + j0 * m, m, m, tmp, parts + j0 * m, m, ext_k - p, omega_m, none, none, nb)) return rc;
            }
        }
        if (stage_ext) { if (int rc = stage_ext(part)) return rc; }
        for (size_t i = 0; i < n_columns; ++i) if (lengths[i] == N) {
            ptrs[i] = stage_ext ? cols[i] : cols[i] + part;
            shifts[i] = stage_ext ? 0 : p;
        }
        if (int rc = quotient_eval_on(c, st, ptrs.data(), n_columns, k, ext_k - p, loads, n_loads, constants, n_constants, program, n_instr, h, p, (uint32_t)part,
                                      shifts.data())) return rc;
    }
    return 0;
}
// the finishing step of both evaluate_h entry points, in place in h: h * t_evaluations[i mod t_period], then extended_to_coeff (scratch: N elements)
static int evaluate_h_finish(Ctx* c, cudaStream_t st, Fr* h, Fr* scratch, uint32_t ext_k, const b200_fr* zeta, const b200_fr* t_evaluations, uint32_t t_period,
                             const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor) {
    const size_t N = (size_t)1 << ext_k;
    if (int rc = scale_cycle_on(c, st, h, N, t_evaluations, t_period)) return rc;
    NttScale none;
    return ntt_call(c, st, h, N, N, scratch, h, N, ext_k, as_fr(ext_omega_inv), none, coset_post(as_fr(ext_ifft_divisor), as_fr(zeta)), 1);
}

// evaluate_h at its natural boundary: the CPU evaluator receives coefficient-form polynomials and builds their cosets itself
// (UPSTREAM plonk/evaluation.rs: `advice_polys.iter().map(|a| domain.coeff_to_extended(a))`), and vanishing/prover.rs then divides by
// the vanishing polynomial and converts back.  One call does the same on the device, so a coefficient column crosses PCIe once
// (n elements) instead of its coset twice (2^ext_k down, 2^ext_k up).  When every column's extended coset fits the call budget the
// loop runs one part, the whole coset of every column (p = 0); otherwise the numerator is evaluated one n-point coset part at a time
// (p = ext_k - k).  Device memory: stage_a = the coefficient columns (uploaded once), stage_c = the current m = 2^(ext_k - p) element part
// of every column (the coefficient columns' in column order, then the extended columns', gathered on the host into the pinned bounce
// slots per part), stage_b = h (N elements) followed by the N-element NTT scratch of the loop and of the finishing step.
int b200_evaluate_h(const b200_fr* const* polys, const size_t* lengths, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta,
                    const b200_col_ref* loads, size_t n_loads, const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr,
                    const b200_fr* t_evaluations, uint32_t t_period, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor, b200_fr* out) {
    B200_ENTER(c, nullptr);
    B200_CHECK(out && ext_omega && zeta && (n_columns == 0 || (polys && lengths)), -1, "evaluate_h: null pointer");
    B200_CHECK(ext_k >= k && ext_k >= 1 && ext_k <= 28, -1, "evaluate_h: need k <= ext_k <= 28");
    B200_CHECK(!t_evaluations || (t_period >= 1 && t_period <= 1024 && ext_omega_inv && ext_ifft_divisor), -1, "evaluate_h: finishing needs t_evaluations, its period and the inverse-transform constants");
    const size_t N = (size_t)1 << ext_k;
    for (size_t i = 0; i < n_columns; ++i)
        B200_CHECK(polys[i] && lengths[i] >= 1 && lengths[i] <= N, -1, "evaluate_h: column %zu is null or longer than 2^ext_k", i);
    StreamScope ss(c, nullptr);
    const uint32_t p = k >= 1 && sizeof(Fr) * N * n_columns > call_budget() ? ext_k - k : 0;
    const size_t m = N >> p, P = (size_t)1 << p;
    std::vector<size_t> coeff, exts;
    size_t coeff_elems = 0;
    for (size_t i = 0; i < n_columns; ++i) {
        if (lengths[i] < N) { coeff.push_back(i); coeff_elems += lengths[i]; }
        else exts.push_back(i);
    }
    if (c->stage_c.ensure(sizeof(Fr) * m * n_columns) || c->stage_a.ensure(sizeof(Fr) * (coeff_elems ? coeff_elems : 1)) || c->stage_b.ensure(sizeof(Fr) * 2 * N)) return -2;
    Fr* parts = c->stage_c.as<Fr>();
    Fr* h = c->stage_b.as<Fr>();
    std::vector<HostSeg> up(coeff.size()), ext_up(exts.size());
    std::vector<const Fr*> cols(n_columns);
    size_t off = 0;
    for (size_t j = 0; j < coeff.size(); ++j) {
        up[j] = HostSeg{(uint8_t*)const_cast<b200_fr*>(polys[coeff[j]]), sizeof(Fr) * lengths[coeff[j]]};
        cols[coeff[j]] = c->stage_a.as<Fr>() + off;
        off += lengths[coeff[j]];
    }
    for (size_t j = 0; j < exts.size(); ++j) cols[exts[j]] = parts + (coeff.size() + j) * m;
    if (!coeff.empty()) { if (int rc = h2d_segments(c, c->stage_a.p, up.data(), up.size(), ss.st)) return rc; }
    auto stage_ext = [&](size_t part) -> int {
        if (exts.empty()) return 0;
        for (size_t j = 0; j < exts.size(); ++j) ext_up[j] = HostSeg{(uint8_t*)const_cast<b200_fr*>(polys[exts[j]] + part), sizeof(Fr) * m, P > 1 ? sizeof(Fr) * P : 0};
        return h2d_segments(c, parts + coeff.size() * m, ext_up.data(), ext_up.size(), ss.st);
    };
    if (int rc = evaluate_h_parts_on(c, ss.st, cols.data(), lengths, n_columns, k, ext_k, p, as_fr(ext_omega), as_fr(zeta), loads, n_loads, constants, n_constants,
                                     program, n_instr, parts, h + N, h, stage_ext)) return rc;
    if (t_evaluations) {
        if (int rc = evaluate_h_finish(c, ss.st, h, h + N, ext_k, zeta, t_evaluations, t_period, ext_omega_inv, ext_ifft_divisor)) return rc;
    }
    return d2h_one(c, out, h, sizeof(Fr) * N, ss.st);
}

// evaluate_h on device-resident columns: always by parts, on the caller's columns where they are
int b200_evaluate_h_dev(const void* const* d_polys, const size_t* lengths, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta,
                        const b200_col_ref* loads, size_t n_loads, const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr,
                        const b200_fr* t_evaluations, uint32_t t_period, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor, void* d_out, void* stream) {
    B200_ENTER(c, d_out);
    B200_CHECK(d_out && ext_omega && zeta && (n_columns == 0 || (d_polys && lengths)), -1, "evaluate_h_dev: null pointer");
    B200_CHECK(k >= 1 && ext_k >= k && ext_k <= 28, -1, "evaluate_h_dev: need 1 <= k <= ext_k <= 28 (k = %u, ext_k = %u)", k, ext_k);
    B200_CHECK(!t_evaluations || (t_period >= 1 && t_period <= 1024 && ext_omega_inv && ext_ifft_divisor), -1,
               "evaluate_h_dev: finishing needs t_evaluations, a period in 1 ... 1024 and the inverse-transform constants");
    const size_t N = (size_t)1 << ext_k, n = (size_t)1 << k;
    const uintptr_t out_lo = (uintptr_t)d_out, out_hi = out_lo + sizeof(Fr) * N;
    size_t n_coeff = 0;
    for (size_t i = 0; i < n_columns; ++i) {
        B200_CHECK(d_polys[i] && lengths[i] >= 1 && lengths[i] <= N, -1, "evaluate_h_dev: column %zu is null, empty or longer than 2^ext_k", i);
        const uintptr_t lo = (uintptr_t)d_polys[i], hi = lo + sizeof(Fr) * lengths[i];
        B200_CHECK(hi <= out_lo || lo >= out_hi, -1, "evaluate_h_dev: d_out overlaps column %zu", i);
        if (lengths[i] < N) ++n_coeff;
    }
    StreamScope ss(c, stream);
    if (c->stage_c.ensure(sizeof(Fr) * n * (n_coeff ? n_coeff : 1)) || c->stage_b.ensure(sizeof(Fr) * N)) return -2;
    Fr* h = reinterpret_cast<Fr*>(d_out);
    if (int rc = evaluate_h_parts_on(c, ss.st, reinterpret_cast<const Fr* const*>(d_polys), lengths, n_columns, k, ext_k, ext_k - k, as_fr(ext_omega), as_fr(zeta),
                                     loads, n_loads, constants, n_constants, program, n_instr, c->stage_c.as<Fr>(), c->stage_b.as<Fr>(), h, nullptr)) return rc;
    if (!t_evaluations) return 0;
    return evaluate_h_finish(c, ss.st, h, c->stage_b.as<Fr>(), ext_k, zeta, t_evaluations, t_period, ext_omega_inv, ext_ifft_divisor);
}

// ---- SRS --------------------------------------------------------------------------------------------------------------------------
// Fr's 2^28-th root of unity (halo2curves Fr::ROOT_OF_UNITY = 7^((r - 1) / 2^28)) in Montgomery form
static Fr fr_root_of_unity() {
    Fr w;
    const uint32_t v[8] = {0x60c37c9cu, 0xd34f1ed9u, 0xd39329c8u, 0x3215cf6du, 0x3dd31f74u, 0x98865ea9u, 0x166d18b7u, 0x03ddb9f5u};
    memcpy(w.l, v, sizeof v);
    return fp_to_mont(w);
}
// the 2^log_n-th root of unity of halo2's EvaluationDomain, ROOT_OF_UNITY^(2^(28 - log_n)), log_n <= 28
static Fr fr_omega(uint32_t log_n) {
    Fr w = fr_root_of_unity();
    for (uint32_t i = log_n; i < 28; ++i) w = w * w;
    return w;
}
// 1 / x for a small integer x, Montgomery form
static Fr fr_inv_u64(uint64_t x) {
    Fr f = fp_zero<FrTag>();
    f.l[0] = (uint32_t)x; f.l[1] = (uint32_t)(x >> 32);
    return fp_inv(fp_to_mont(f));
}
static const char* g1_invalid_reason(unsigned r) {
    return r == G1_X_NOT_CANONICAL ? "x is not below p" : r == G1_Y_NOT_CANONICAL ? "y is not below p" : "is not on the curve";
}
// Both vectors go straight into level 0 of their new tables and are checked there; only when every point passed is valid does the group
// FFT (for a NULL g_lagrange) run, from level 0 of g's table into level 0 of the other, so a rejected file costs no FFT scratch.
static int srs_register_on(Ctx* c, cudaStream_t st, const b200_g1_affine* g, const b200_g1_affine* gl, uint32_t k, int window_bits, size_t max_table_bytes,
                           uint64_t* g_handle, uint64_t* g_lagrange_handle) {
    const size_t n = (size_t)1 << k;
    BaseSet* bs[2] = {nullptr, nullptr};
    auto fail = [&](int rc) { for (BaseSet* b : bs) if (b) bases_drop(b, rc); return rc; };
    auto cuda_fail = [&](cudaError_t e) { set_error("srs_register: %s", cudaGetErrorString(e)); return fail(-2); };
    for (int v = 0; v < 2; ++v) if (int rc = bases_alloc(c, n, window_bits, max_table_bytes, &bs[v])) return fail(rc);
    G1Affine* lv0[2] = {bs[0]->t[c->slot]->d_table, bs[1]->t[c->slot]->d_table};
    const b200_g1_affine* src[2] = {g, gl};
    if (c->small.ensure(2 * sizeof(unsigned long long))) return fail(-2);
    unsigned long long* d_first = c->small.as<unsigned long long>();
    if (cudaError_t e = cudaMemsetAsync(d_first, 0xff, 2 * sizeof(unsigned long long), st)) return cuda_fail(e);
    for (int v = 0; v < 2; ++v) if (src[v]) {
        if (int rc = h2d_one(c, lv0[v], src[v], sizeof(G1Affine) * n, st)) return fail(rc);
        if (int rc = g1_validate_run(lv0[v], n, d_first + v, st)) return fail(rc);
    }
    unsigned long long first[2];
    if (cudaError_t e = cudaMemcpyAsync(first, d_first, sizeof first, cudaMemcpyDeviceToHost, st)) return cuda_fail(e);
    if (cudaError_t e = cudaStreamSynchronize(st)) return cuda_fail(e);
    for (int v = 0; v < 2; ++v) if (first[v] != ~0ull) {
        set_error("srs_register: %s[%llu] %s", v ? "g_lagrange" : "g", first[v] >> 2, g1_invalid_reason((unsigned)(first[v] & 3)));
        return fail(-1);
    }
    if (!gl) {                                  // ParamsKZG::downsize: g_lagrange = n^-1 * FFT_{omega^-1}(g)
        const Fr w_inv = fp_inv(fr_omega(k)), n_inv = fr_inv_u64(n);
        if (int rc = g1_fft_on(c, st, lv0[0], k, reinterpret_cast<const b200_fr*>(&w_inv), reinterpret_cast<const b200_fr*>(&n_inv), lv0[1])) return fail(rc);
    }
    for (int v = 0; v < 2; ++v) if (int rc = bases_build(c, st, bs[v], nullptr, "srs_register")) return fail(rc);
    if (cudaError_t e = cudaStreamSynchronize(st)) return cuda_fail(e);
    *g_handle = bases_publish(bs[0]);
    *g_lagrange_handle = bases_publish(bs[1]);
    return 0;
}
int b200_srs_register(const b200_g1_affine* g, const b200_g1_affine* g_lagrange, uint32_t k, int window_bits, size_t max_table_bytes,
                      uint64_t* g_handle, uint64_t* g_lagrange_handle) {
    B200_ENTER(c, nullptr);
    B200_CHECK(g && g_handle && g_lagrange_handle, -1, "srs_register: null argument (g, g_handle and g_lagrange_handle are required)");
    B200_CHECK(k <= 26, -1, "srs_register: k = %u out of range [0, 26]", k);
    B200_CHECK(window_bits == 0 || (window_bits >= 4 && window_bits <= 24), -1, "srs_register: window_bits %d not in {0, 4..24}", window_bits);
    StreamScope ss(c, nullptr);
    return srs_register_on(c, ss.st, g, g_lagrange, k, window_bits, max_table_bytes, g_handle, g_lagrange_handle);
}

// ---- proving key ------------------------------------------------------------------------------------------------------------------
// Fr::ZETA (halo2curves), the cube root of unity that coeff_to_extended distributes as [1, zeta, zeta^2], in Montgomery form
static Fr fr_zeta() {
    Fr z;
    const uint32_t v[8] = {0x36636f23u, 0xb8ca0b2du, 0xec2bc5e9u, 0xcc37a73fu, 0x3fd84104u, 0x048b6e19u, 0xe131a029u, 0x30644e72u};
    memcpy(z.l, v, sizeof v);
    return fp_to_mont(z);
}
// the device that owns a caller's buffer, or -1 when it is not device memory
static int device_of(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged ? at.device : -1;
}
// cols[j] (j < n_cols, fixed columns first) -> values, checked; only when every element passed is canonical are polys and l written.
// polys: iNTT (omega^-1, then 2^-k) of the values in column groups bounded by the call budget.  l: the Lagrange indicators of rows {0},
// {u} and [0, u) -- whose interpolants are L_0, L_u and 1 - L_u - sum_{r > u} L_r -- to coefficients, then coeff_to_extended.
static int pk_load_on(Ctx* c, cudaStream_t st, const void* const* cols, size_t n_cols, size_t n_fixed, uint32_t k, uint32_t ext_k, uint32_t blinding_factors,
                      Fr* values, Fr* polys, size_t stride, Fr* l) {
    const size_t n = (size_t)1 << k, N = (size_t)1 << ext_k;
    if (c->small.ensure(sizeof(unsigned long long))) return -2;
    unsigned long long* d_first = c->small.as<unsigned long long>();
    B200_CUDA(cudaMemsetAsync(d_first, 0xff, sizeof *d_first, st));
    for (size_t j = 0; j < n_cols; ++j) {               // column j's check runs while the host stages column j + 1
        if (int rc = h2d_one(c, values + j * stride, cols[j], sizeof(Fr) * n, st)) return rc;
        if (int rc = fr_validate_run(values + j * stride, n, j, d_first, st)) return rc;
    }
    unsigned long long first = ~0ull;
    if (int rc = read_back(&first, d_first, sizeof first, st)) return rc;
    if (first != ~0ull) {
        const size_t col = (size_t)(first >> 32), row = (size_t)(first & 0xffffffffu);
        set_error("pk_load: %s[%zu][%zu] is not below r", col < n_fixed ? "fixed_values" : "permutations", col < n_fixed ? col : col - n_fixed, row);
        return -1;
    }
    const size_t g = group_size(sizeof(Fr) * n, n_cols < 65535 ? n_cols : 65535), s = group_size(sizeof(Fr) * N, 3);
    const size_t tmp_elems = g * n > s * N ? g * n : s * N;
    if (c->stage_a.ensure(sizeof(Fr) * 3 * n) || c->stage_b.ensure(sizeof(Fr) * tmp_elems)) return -2;
    Fr* coef = c->stage_a.as<Fr>();
    Fr* tmp = c->stage_b.as<Fr>();
    const Fr w_inv = fp_inv(fr_omega(k));
    const NttScale zeta_cycle = coset_pre(fr_zeta());
    NttScale none, div_n;
    div_n.mode = 1; div_n.c[0] = fr_inv_u64(n);
    for (size_t j0 = 0; j0 < n_cols; j0 += g) {
        const int nb = (int)(n_cols - j0 < g ? n_cols - j0 : g);
        if (int rc = ntt_call(c, st, values + j0 * stride, stride, n, tmp, polys + j0 * stride, stride, k, w_inv, none, div_n, nb)) return rc;
    }
    const uint64_t u = n - blinding_factors - 1, lo[3] = {0, u, 0}, hi[3] = {1, u + 1, u};
    if (int rc = fr_indicator_run(coef, n, lo, hi, st)) return rc;
    for (size_t j0 = 0; j0 < 3; j0 += s) {
        const int nb = (int)(3 - j0 < s ? 3 - j0 : s);
        if (int rc = ntt_call(c, st, coef + j0 * n, n, n, tmp, coef + j0 * n, n, k, w_inv, none, div_n, nb)) return rc;
        if (int rc = ntt_call(c, st, coef + j0 * n, n, n, tmp, l + j0 * N, N, ext_k, fr_omega(ext_k), zeta_cycle, none, nb)) return rc;
    }
    B200_CUDA(cudaStreamSynchronize(st));
    return 0;
}
int b200_pk_load(const void* const* h_fixed_values, size_t n_fixed, const void* const* h_permutations, size_t n_perm, uint32_t k, uint32_t ext_k,
                 uint32_t blinding_factors, void* d_values, void* d_polys, size_t stride, void* d_l) {
    B200_ENTER(c, d_values ? d_values : d_l);
    B200_CHECK(k >= 1 && ext_k >= k && ext_k <= 28, -1, "pk_load: need 1 <= k <= ext_k <= 28 (k = %u, ext_k = %u)", k, ext_k);
    const size_t n = (size_t)1 << k, n_cols = n_fixed + n_perm;
    B200_CHECK(blinding_factors < n, -1, "pk_load: blinding_factors = %u, need fewer than 2^k = %zu", blinding_factors, n);
    B200_CHECK(stride >= n, -1, "pk_load: stride %zu < 2^k = %zu", stride, n);
    B200_CHECK(n_cols < ((size_t)1 << 32) && (n_cols == 0 || stride <= ((size_t)1 << 58) / n_cols), -1, "pk_load: %zu columns of stride %zu exceed the address space",
               n_cols, stride);
    B200_CHECK(d_l && (n_cols == 0 || (d_values && d_polys)) && (n_fixed == 0 || h_fixed_values) && (n_perm == 0 || h_permutations), -1,
               "pk_load: null pointer (d_l is required; d_values, d_polys and the column arrays may be NULL only when there are no columns)");
    std::vector<const void*> cols(n_cols);
    for (size_t j = 0; j < n_cols; ++j) {
        cols[j] = j < n_fixed ? h_fixed_values[j] : h_permutations[j - n_fixed];
        B200_CHECK(cols[j], -1, "pk_load: %s[%zu] is null", j < n_fixed ? "h_fixed_values" : "h_permutations", j < n_fixed ? j : j - n_fixed);
    }
    const char* names[3] = {"d_values", "d_polys", "d_l"};
    const uintptr_t lo[3] = {(uintptr_t)d_values, (uintptr_t)d_polys, (uintptr_t)d_l};
    const size_t col_bytes = n_cols ? sizeof(Fr) * ((n_cols - 1) * stride + n) : 0;
    const uintptr_t hi[3] = {lo[0] + col_bytes, lo[1] + col_bytes, lo[2] + sizeof(Fr) * 3 * ((size_t)1 << ext_k)};
    for (int a = 0; a < 3; ++a) {
        if (hi[a] == lo[a]) continue;
        B200_CHECK((lo[a] & 15) == 0, -1, "pk_load: %s is not 16-byte aligned", names[a]);
        const int dev = device_of((const void*)lo[a]);
        B200_CHECK(dev == c->dev, -1, dev < 0 ? "pk_load: %s is not device memory" : "pk_load: %s is on another device than the other outputs", names[a]);
        for (int b = 0; b < a; ++b)
            B200_CHECK(hi[b] == lo[b] || hi[a] <= lo[b] || lo[a] >= hi[b], -1, "pk_load: %s overlaps %s", names[a], names[b]);
    }
    StreamScope ss(c, nullptr);
    return pk_load_on(c, ss.st, cols.data(), n_cols, n_fixed, k, ext_k, blinding_factors, reinterpret_cast<Fr*>(d_values), reinterpret_cast<Fr*>(d_polys),
                      stride, reinterpret_cast<Fr*>(d_l));
}

}  // extern "C"
#pragma GCC visibility pop

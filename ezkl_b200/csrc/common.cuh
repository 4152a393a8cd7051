// common.cuh — error plumbing, device scratch arena and block-level helpers shared by the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <string>

namespace b200 {

// Thread-local last-error string behind b200_last_error() (include/ezkl_b200.h).
void set_error(const char* fmt, ...);
const char* get_error();

// Kernels launched by libezkl_b200.so since load (b200_launch_count): every launch site of the operation kernels calls
// count_launch() right after issuing its launch, so a launch that then fails is counted too.  The test-only debug library
// (debug.cu, libezkl_b200_dbg.so) has its own copy of this counter, which nothing reads.
inline std::atomic<uint64_t> g_launches{0};
inline void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

#define B200_CUDA(call)                                                                                  \
    do {                                                                                                 \
        cudaError_t _e = (call);                                                                         \
        if (_e != cudaSuccess) {                                                                         \
            ::b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e));     \
            return -2;                                                                                   \
        }                                                                                                \
    } while (0)

#define B200_CHECK(cond, code, ...)                                                                      \
    do {                                                                                                 \
        if (!(cond)) { ::b200::set_error(__VA_ARGS__); return (code); }                                  \
    } while (0)

// Growable device scratch buffer (one per call-site purpose per context); never shrinks.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); p = nullptr; return -2; }
        cap = want;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() { return reinterpret_cast<T*>(p); }
};

// Host->device parameter blobs (programs, pointer tables, per-call constants): one ring per (thread, device) context, pushed
// only by the kernel files, at most one blob per launch sequence.  push() stages `bytes` from `src`, sets *d_out to the device
// copy and returns 0; when it returns, the host source may be reused.
//   * A blob of at most SLOT bytes goes without a stream synchronisation: it is copied into a slot of a pinned ring and an async
//     H2D copy into the matching slot of a device ring is enqueued on the caller's stream, followed by an event.  A slot is reused
//     only after its own event has completed (a host-side wait on that one event — never a device-wide synchronisation), so
//     neither the pinned source nor the device copy can be overwritten while a kernel may still read it.
//   * A larger blob, or any blob while the pinned ring cannot be allocated, is copied into `overflow` and the stream is
//     synchronised.  An overflow blob is valid until the next push on this ring: the caller enqueues the kernels that read it
//     before it pushes again, so the next overflow copy is ordered after them.
//   * A failing CUDA call returns -2 with the error set.
// Not capturable in a CUDA graph (a replay would re-read the pinned slot).
struct StagingRing {
    static constexpr size_t SLOT = (size_t)256 << 10;
    static constexpr int NSLOT = 96;
    uint8_t* h = nullptr;
    uint8_t* d = nullptr;
    cudaEvent_t ev[NSLOT] = {};
    bool used[NSLOT] = {};
    int head = 0;
    DevBuf overflow;
    int push(const void* src, size_t bytes, cudaStream_t st, const void** d_out) {
        if (bytes <= SLOT && !h && !alloc_ring()) { cudaGetLastError(); release_ring(); }
        if (bytes > SLOT || !h) {
            if (overflow.ensure(bytes)) return -2;
            B200_CUDA(cudaMemcpyAsync(overflow.p, src, bytes, cudaMemcpyHostToDevice, st));
            B200_CUDA(cudaStreamSynchronize(st));
            *d_out = overflow.p;
            return 0;
        }
        const int s = head;
        head = (head + 1) % NSLOT;
        if (used[s]) B200_CUDA(cudaEventSynchronize(ev[s]));
        memcpy(h + s * SLOT, src, bytes);
        B200_CUDA(cudaMemcpyAsync(d + s * SLOT, h + s * SLOT, bytes, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaEventRecord(ev[s], st));
        used[s] = true;
        *d_out = d + s * SLOT;
        return 0;
    }
    void release() { release_ring(); overflow.release(); }
private:
    bool alloc_ring() {
        if (cudaMallocHost((void**)&h, SLOT * NSLOT) != cudaSuccess) { h = nullptr; return false; }
        if (cudaMalloc((void**)&d, SLOT * NSLOT) != cudaSuccess) { d = nullptr; return false; }
        for (int i = 0; i < NSLOT; ++i) if (cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) != cudaSuccess) { ev[i] = nullptr; return false; }
        return true;
    }
    void release_ring() {
        if (h) cudaFreeHost(h);
        if (d) cudaFree(d);
        for (int i = 0; i < NSLOT; ++i) { if (ev[i]) cudaEventDestroy(ev[i]); ev[i] = nullptr; used[i] = false; }
        h = d = nullptr; head = 0;
    }
};

// Process-wide tuning knobs, read from the environment ONCE in b200_init (never on a launch path).
struct Config {
    size_t ws_budget_call = 0;      // B200_WS_BUDGET_MB: fixed per-call scratch budget (tests use it to force the batch-split paths); 0 = derive
    size_t ws_budget_total = (size_t)24 << 30;   // scratch the library may hold across all calling threads of a device (of an 80 GB H100)
    int msm_reduce_m = 0;           // B200_MSM_REDUCE_M: buckets per thread of the bucket reduction (1..4096), 0 = automatic
    int msm_reduce_threads = 0;     // B200_MSM_REDUCE_THREADS: CTA size of the bucket reduction (32 / 64 / 128 / 256), 0 = automatic
    int shard_min_logn = 22;        // B200_SHARD_MIN_LOGN: a single transform of at least this size is sharded across the devices
    size_t msm_table_budget = (size_t)16 << 30;   // B200_MSM_TABLE_MB: base-table bytes per registered vector and device (msm_pick_levels)
};
const Config& config();
// Streaming multiprocessors of the current device (132 on an H100 SXM); grids are sized in multiples of it.
int sm_count();

// Optional device-side timing of kernel classes with CUDA events on the launching stream (bench.py's roofline leg).
enum ProfClass { PROF_MSM_ACCUMULATE = 0, PROF_MSM_TOTAL = 1, PROF_NTT = 2, PROF_POLY = 3, PROF_MSM_RECODE = 4, PROF_MSM_TAIL = 5, PROF_QUOTIENT = 6,
                 PROF_MSM_SCAN = 7, PROF_MSM_REDUCE = 8, PROF_MSM_FOLD = 9, PROF_NCLASS = 10 };
bool prof_enabled();
void prof_mark(int cls, cudaStream_t st, bool begin);
struct ProfScope {
    int cls; cudaStream_t st; bool on;
    ProfScope(int c, cudaStream_t s) : cls(c), st(s), on(prof_enabled()) { if (on) prof_mark(cls, st, true); }
    ~ProfScope() { if (on) prof_mark(cls, st, false); }
};

static inline unsigned div_up(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

#if defined(__CUDACC__)
// Exclusive scan of one uint32 per thread across the block (blockDim.x <= 1024, multiple of 32).
// Returns the exclusive prefix; *total gets the block sum (valid in every thread).
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t block_total;
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (unsigned)d) incl += t;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < nw ? warp_sums[lane] : 0, wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= (unsigned)d) wi += t;
        }
        if (lane < nw) warp_sums[lane] = wi - w;
        if (lane == 31) block_total = wi;
    }
    __syncthreads();
    uint32_t r = warp_sums[wid] + incl - v;
    *total = block_total;
    __syncthreads();
    return r;
}
#endif

}  // namespace b200

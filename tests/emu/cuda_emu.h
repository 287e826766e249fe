// cuda_emu.h -- TEST INFRASTRUCTURE: a host-side stand-in for the slice of CUDA that libsph_b200 uses, so that
// the UNMODIFIED kernel and host sources under sph_taichi_b200/csrc/ can be compiled by g++ and executed
// thread-for-thread on the CPU (optionally under AddressSanitizer).  Built only by tests/emu/build_emu.py;
// the product never defines SPH_EMU and never sees this file.
//
// Execution model: a launch runs its blocks one after the other; every CUDA thread of a block is a host
// thread (taken from a pool), warp collectives and __syncthreads are real barriers, atomics are real
// atomics, "device memory" is host memory.  TMA bulk copies complete synchronously in the issuing lane and
// flip an emulated mbarrier phase.  Streams are synchronous; stream capture records the launches and
// cudaGraphLaunch replays them (kernel arguments frozen at capture time, as in CUDA).
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <tuple>
#include <vector>

// ---- language surface ---------------------------------------------------------------------------------
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct uint3 { unsigned x = 0, y = 0, z = 0; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }

inline thread_local uint3 threadIdx, blockIdx;
inline thread_local dim3 blockDim, gridDim;

using std::max;
using std::min;

// ---- thread model ---------------------------------------------------------------------------------------
namespace emu {

struct Warp {
    std::barrier<> bar;
    uint32_t slot[32] = {};
    std::atomic<uint32_t> exited{0};
    explicit Warp(int lanes) : bar(lanes) {}
};
struct Block {
    std::barrier<> bar;
    std::vector<std::unique_ptr<Warp>> warps;
    explicit Block(int threads) : bar(threads) {
        for (int t = 0; t < threads; t += 32) warps.emplace_back(new Warp(std::min(32, threads - t)));
    }
};
inline thread_local Warp *tw = nullptr;
inline thread_local Block *tb = nullptr;
inline thread_local int lane = 0;

// persistent worker pool: worker t runs CUDA thread t of the current block
class Pool {
public:
    static Pool &get() { static Pool p; return p; }
    void run_block(int threads, const std::function<void(int)> &fn) {
        grow(threads);
        {
            std::lock_guard<std::mutex> lk(m_);
            fn_ = &fn; active_ = threads; pending_ = threads; ++epoch_;
        }
        cv_.notify_all();
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [&] { return pending_ == 0; });
    }
    ~Pool() {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; ++epoch_; }
        cv_.notify_all();
        for (auto &t : workers_) t.join();
    }
private:
    void grow(int n) {
        while ((int)workers_.size() < n) {
            int id = (int)workers_.size();
            uint64_t seen;
            { std::lock_guard<std::mutex> lk(m_); seen = epoch_; }
            workers_.emplace_back([this, id, seen]() mutable {
                for (;;) {
                    const std::function<void(int)> *fn = nullptr;
                    {
                        std::unique_lock<std::mutex> lk(m_);
                        cv_.wait(lk, [&] { return epoch_ != seen; });
                        seen = epoch_;
                        if (stop_) return;
                        if (id >= active_) continue;
                        fn = fn_;
                    }
                    (*fn)(id);
                    std::lock_guard<std::mutex> lk(m_);
                    if (--pending_ == 0) done_.notify_all();
                }
            });
        }
    }
    std::mutex m_;
    std::condition_variable cv_, done_;
    std::vector<std::thread> workers_;
    const std::function<void(int)> *fn_ = nullptr;
    int active_ = 0, pending_ = 0;
    uint64_t epoch_ = 0;
    bool stop_ = false;
};

inline void run_grid(dim3 grid, dim3 block, const std::function<void()> &body) {
    const int threads = (int)block.x;
    for (unsigned bb = 0; bb < grid.x * grid.y; ++bb) {
        const unsigned b = bb % grid.x, by = bb / grid.x;
        Block blk(threads);
        std::function<void(int)> fn = [&](int t) {
            threadIdx = uint3{(unsigned)t, 0, 0};
            blockIdx = uint3{b, by, 0};
            blockDim = block;
            gridDim = grid;
            tb = &blk;
            tw = blk.warps[t >> 5].get();
            lane = t & 31;
            body();
            tw->exited.fetch_or(1u << lane);
            tw->bar.arrive_and_drop();
            blk.bar.arrive_and_drop();
        };
        Pool::get().run_block(threads, fn);
    }
}

// ---- streams, events, graphs ---------------------------------------------------------------------------
struct Graph { std::vector<std::function<void()>> ops; };
struct Stream { Graph *capturing = nullptr; };
inline Stream default_stream;
inline Stream *as_stream(void *s) { return s ? static_cast<Stream *>(s) : &default_stream; }
inline void submit(void *stream, std::function<void()> op) {
    Stream *s = as_stream(stream);
    if (s->capturing) s->capturing->ops.push_back(std::move(op));
    else op();
}
struct LaunchCfg { dim3 grid, block; void *stream; };
inline LaunchCfg cfg(dim3 g, dim3 b, size_t = 0, void *stream = nullptr) { return LaunchCfg{g, b, stream}; }

// kernel<<<grid, block, smem, stream>>>(args...)  ==>  emu::launch(emu::cfg(grid, block, smem, stream), kernel, args...)
template <class K, class... A>
inline void launch(LaunchCfg c, K kernel, A... args) {
    auto call = [kernel, c, tup = std::make_tuple(args...)]() {
        run_grid(c.grid, c.block, [&] { std::apply(kernel, tup); });
    };
    submit(c.stream, call);
}

}  // namespace emu

inline void __syncthreads() { emu::tb->bar.arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::tw->bar.arrive_and_wait(); }

// ---- warp collectives (full-mask use only) -------------------------------------------------------------
namespace emu {
template <class F>
inline uint32_t collective(uint32_t mine, F &&combine) {
    tw->slot[lane] = mine;
    tw->bar.arrive_and_wait();
    uint32_t r = combine(tw->slot, ~tw->exited.load());
    tw->bar.arrive_and_wait();
    return r;
}
}  // namespace emu
inline unsigned __ballot_sync(unsigned, int pred) {
    return emu::collective(pred ? 1u : 0u, [](const uint32_t *s, uint32_t alive) {
        uint32_t r = 0;
        for (int l = 0; l < 32; ++l) if (((alive >> l) & 1u) && s[l]) r |= 1u << l;
        return r;
    });
}
inline unsigned __match_any_sync(unsigned, int v) {
    const int me = emu::lane;
    return emu::collective((uint32_t)v, [me](const uint32_t *s, uint32_t alive) {
        uint32_t r = 0;
        for (int l = 0; l < 32; ++l) if (((alive >> l) & 1u) && s[l] == s[me]) r |= 1u << l;
        return r;
    });
}
inline uint32_t emu_shfl_bits(uint32_t v, int src) {
    return emu::collective(v, [src](const uint32_t *s, uint32_t) { return s[src & 31]; });
}
template <class T>
inline T emu_shfl(T v, int src) {
    static_assert(sizeof(T) == 4 || sizeof(T) == 8, "32- and 64-bit shuffles only");
    uint32_t b[2] = {0, 0};
    std::memcpy(b, &v, sizeof(T));
    b[0] = emu_shfl_bits(b[0], src);
    if (sizeof(T) == 8) b[1] = emu_shfl_bits(b[1], src);
    T r; std::memcpy(&r, b, sizeof(T));
    return r;
}
template <class T> inline T __shfl_sync(unsigned, T v, int src) { return emu_shfl(v, src); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) { return emu_shfl(v, emu::lane ^ m); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d) { return emu_shfl(v, emu::lane >= (int)d ? emu::lane - (int)d : emu::lane); }
inline int __reduce_min_sync(unsigned, int v) {
    return (int)emu::collective((uint32_t)v, [](const uint32_t *s, uint32_t alive) {
        int r = INT32_MAX;
        for (int l = 0; l < 32; ++l) if ((alive >> l) & 1u) r = std::min(r, (int)s[l]);
        return (uint32_t)r;
    });
}
inline int __reduce_max_sync(unsigned, int v) {
    return (int)emu::collective((uint32_t)v, [](const uint32_t *s, uint32_t alive) {
        int r = INT32_MIN;
        for (int l = 0; l < 32; ++l) if ((alive >> l) & 1u) r = std::max(r, (int)s[l]);
        return (uint32_t)r;
    });
}

// ---- scalar intrinsics -----------------------------------------------------------------------------------
inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline int __float_as_int(float f) { int u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
inline float __int_as_float(int u) { float f; std::memcpy(&f, &u, 4); return f; }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }  // built with -ffp-contract=off
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fdividef(float a, float b) { return a / b; }
inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline unsigned __brev(unsigned x) {
    unsigned r = 0;
    for (int k = 0; k < 32; ++k) r |= ((x >> k) & 1u) << (31 - k);
    return r;
}
inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t s) {
    uint64_t v = ((uint64_t)hi << 32) | lo;
    return (uint32_t)((v << (s & 31)) >> 32);
}
template <class T> inline T __ldg(const T *p) { return *p; }

// ---- atomics ---------------------------------------------------------------------------------------------
inline int atomicAdd(int *p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline int atomicMax(int *p, int v) {
    int old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
inline float atomicAdd(float *p, float v) {
    uint32_t *u = reinterpret_cast<uint32_t *>(p);
    uint32_t old = __atomic_load_n(u, __ATOMIC_SEQ_CST);
    for (;;) {
        float f = __uint_as_float(old) + v;
        uint32_t nw = __float_as_uint(f);
        if (__atomic_compare_exchange_n(u, &old, nw, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) return __uint_as_float(old);
    }
}
inline double atomicAdd(double *p, double v) {
    uint64_t *u = reinterpret_cast<uint64_t *>(p);
    uint64_t old = __atomic_load_n(u, __ATOMIC_SEQ_CST);
    for (;;) {
        double d; std::memcpy(&d, &old, 8); d += v;
        uint64_t nw; std::memcpy(&nw, &d, 8);
        if (__atomic_compare_exchange_n(u, &old, nw, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) { std::memcpy(&d, &old, 8); return d; }
    }
}

// ---- stand-ins for sph_ptx.cuh ---------------------------------------------------------------------------
inline float rsqrt_ftz(float x) { return 1.0f / std::sqrt(x); }
inline float rcp_ftz(float x) { return 1.0f / x; }
inline void ldg256(const float4 *p, float4 &a, float4 &b) { a = p[0]; b = p[1]; }
inline int ldg_stream(const int32_t *p) { return *p; }
inline void pdl_wait() {}
// mbarrier (arrival count 1): low word = completed phases, bits 32..62 = transaction count (signed: complete_tx may
// run ahead of expect_tx), bit 63 = the arrive of the current phase has happened.  A phase completes when it has
// arrived and its transaction count is zero.  Only the issuing lane writes; the waiting lanes poll.
inline void emu_mbar_update(uint64_t *bar, int64_t tx_delta, bool arrive) {
    uint64_t v = __atomic_load_n(bar, __ATOMIC_SEQ_CST);
    uint32_t done = (uint32_t)v;
    int64_t tx = (int64_t)((v >> 32) & 0x7fffffffull);
    if (tx & 0x40000000) tx -= 0x80000000ll;  // sign-extend 31 bits
    bool arrived = (v >> 63) != 0 || arrive;
    tx += tx_delta;
    if (arrived && tx == 0) { ++done; arrived = false; }
    __atomic_store_n(bar, ((uint64_t)arrived << 63) | (((uint64_t)tx & 0x7fffffffull) << 32) | done, __ATOMIC_SEQ_CST);
}
inline void mbar_init(uint64_t *bar, int) { __atomic_store_n(bar, 0ull, __ATOMIC_SEQ_CST); }
inline void mbar_fence_init() {}
inline void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { emu_mbar_update(bar, (int64_t)bytes, true); }
inline void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    if ((reinterpret_cast<uintptr_t>(dst_smem) | reinterpret_cast<uintptr_t>(src_gmem) | bytes) & 15u) {
        std::fprintf(stderr, "emu: cp.async.bulk needs 16-byte aligned addresses and size (dst %p src %p bytes %u)\n",
                     dst_smem, src_gmem, bytes);
        std::abort();
    }
    std::memcpy(dst_smem, src_gmem, bytes);
    emu_mbar_update(bar, -(int64_t)bytes, false);
}
inline void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (((uint32_t)__atomic_load_n(bar, __ATOMIC_SEQ_CST) & 1u) == parity) std::this_thread::yield();
}

// packed fp32 pairs: two independent IEEE fp32 operations (lo = first element in memory)
typedef unsigned long long f32x2;
inline f32x2 pack2(float lo, float hi) { return ((f32x2)__float_as_uint(hi) << 32) | __float_as_uint(lo); }
inline float emu_lo(f32x2 v) { return __uint_as_float((uint32_t)v); }
inline float emu_hi(f32x2 v) { return __uint_as_float((uint32_t)(v >> 32)); }
inline f32x2 add2(f32x2 a, f32x2 b) { return pack2(__fadd_rn(emu_lo(a), emu_lo(b)), __fadd_rn(emu_hi(a), emu_hi(b))); }
inline f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
    return pack2(std::fmaf(emu_lo(a), emu_lo(b), emu_lo(c)), std::fmaf(emu_hi(a), emu_hi(b), emu_hi(c)));
}

// ---- runtime API -----------------------------------------------------------------------------------------
typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0;
typedef void *cudaStream_t;
typedef emu::Graph *cudaGraph_t;
typedef emu::Graph *cudaGraphExec_t;
struct EmuEvent { std::chrono::steady_clock::time_point t; };
typedef EmuEvent *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum cudaStreamCaptureMode { cudaStreamCaptureModeThreadLocal, cudaStreamCaptureModeRelaxed };
constexpr unsigned cudaStreamNonBlocking = 1;

inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char *cudaGetErrorString(cudaError_t) { return "emulated CUDA runtime"; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int) { *v = 4; return cudaSuccess; }
inline cudaError_t cudaMemset(void *p, int v, size_t n) { std::memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void *p, int v, size_t n, cudaStream_t s) {
    emu::submit(s, [=] { std::memset(p, v, n); });
    return cudaSuccess;
}
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t st) {
    emu::submit(st, [=] { std::memcpy(d, s, n); });
    return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaMalloc(void **p, size_t n) { *p = std::malloc(n); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFree(void *p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new emu::Stream(); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete static_cast<emu::Stream *>(s); return cudaSuccess; }
inline cudaError_t cudaStreamBeginCapture(cudaStream_t s, cudaStreamCaptureMode) {
    emu::as_stream(s)->capturing = new emu::Graph();
    return cudaSuccess;
}
inline cudaError_t cudaStreamEndCapture(cudaStream_t s, cudaGraph_t *g) {
    *g = emu::as_stream(s)->capturing;
    emu::as_stream(s)->capturing = nullptr;
    return cudaSuccess;
}
inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t *e, cudaGraph_t g, unsigned long long = 0) {
    *e = new emu::Graph(*g);
    return cudaSuccess;
}
inline cudaError_t cudaGraphLaunch(cudaGraphExec_t e, cudaStream_t s) {
    for (auto &op : e->ops) emu::submit(s, op);
    return cudaSuccess;
}
inline cudaError_t cudaGraphDestroy(cudaGraph_t g) { delete g; return cudaSuccess; }
inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new EmuEvent(); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
    return cudaSuccess;
}

// invariants the kernels state about their own staging windows (compiled out of the product)
#define SPH_EMU_CHECK(cond)                                                                          \
    do {                                                                                             \
        if (!(cond)) {                                                                               \
            std::fprintf(stderr, "emu: kernel invariant violated at %s:%d: %s (block %u thread %u)\n", __FILE__, \
                         __LINE__, #cond, blockIdx.x, threadIdx.x);                                  \
            std::abort();                                                                            \
        }                                                                                            \
    } while (0)

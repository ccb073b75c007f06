// Thin device abstraction for the k-mer pipeline.
//
// Product build (nvcc, sm_90a): kernels are functor bodies launched as grid-stride CUDA kernels, memory
// is cudaMalloc'd HBM, atomics are the hardware atomics.
//
// AC_EMULATE build (g++, tests/emu only): the same functor bodies run serially on the host so that the
// per-thread device logic can be exercised by the CPU test-suite in a container that has no GPU.  The
// emulation library is test infrastructure; the product library never falls back to it.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

// Kernels launched by this process (bench.py's "gpu_launches"); defined in pipeline.cu
extern unsigned long long g_ac_kernel_launches;

#ifdef AC_EMULATE
// ------------------------------------------------------------------------------------------------
#define AC_HD inline
#define AC_D inline

template <class T> inline T ac_atomic_cas(T* p, T cmp, T val) { T old = *p; if (old == cmp) *p = val; return old; }
template <class T> inline T ac_atomic_add(T* p, T v) { T old = *p; *p = (T)(old + v); return old; }
template <class T> inline T ac_atomic_or(T* p, T v) { T old = *p; *p = (T)(old | v); return old; }
template <class T> inline T ac_atomic_and(T* p, T v) { T old = *p; *p = (T)(old & v); return old; }
template <class T> inline T ac_atomic_min(T* p, T v) { T old = *p; if (v < old) *p = v; return old; }
template <class T> inline T ac_atomic_max(T* p, T v) { T old = *p; if (v > old) *p = v; return old; }
template <class T> inline T ac_ld_volatile(const T* p) { return *p; }
template <class T> inline T ac_ld_cg(const T* p) { return *p; }
inline void ac_st_stream(uint32_t* p, uint32_t v) { *p = v; }
inline void ac_ld_group(const uint64_t* p, uint64_t out[4]) { out[0] = p[0]; out[1] = p[1]; out[2] = p[2]; out[3] = p[3]; }
inline uint64_t ac_umul64hi(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
inline uint32_t ac_popc(uint32_t v) { return (uint32_t)__builtin_popcount(v); }
inline int ac_ctz(uint32_t v) { return __builtin_ctz(v); }

struct AcStream { int dummy; };

inline void* ac_dev_alloc(size_t bytes) { void* p = malloc(bytes ? bytes : 1); if (!p) throw std::runtime_error("emu alloc failed"); return p; }
inline void ac_dev_free(void* p) { free(p); }
inline void ac_memset(void* p, int v, size_t bytes, AcStream*) { memset(p, v, bytes); }
inline void ac_h2d(void* d, const void* h, size_t bytes, AcStream*) { memcpy(d, h, bytes); }
inline void ac_d2h(void* h, const void* d, size_t bytes, AcStream*) { memcpy(h, d, bytes); }
inline void ac_copy_dd(void* dst, const void* src, size_t bytes, AcStream*) { memcpy(dst, src, bytes); }
inline void ac_sync(AcStream*) {}
inline void* ac_host_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
inline void ac_host_free(void* p) { free(p); }
inline int ac_smem_optin() { return 227 * 1024; }         // what an H100 grants one CTA
struct AcTimer { explicit AcTimer(AcStream*) {} void stop() {} float ms() const { return 0.f; } };
struct DeviceContext {
    int device; AcStream stream{};
    DeviceContext(int device, void*) : device(device) {}
    void make_current() const {}
};

template <class Body> inline void ac_launch(const char*, AcStream*, const Body& body, uint64_t n);
template <int CTAS, class Body> inline void ac_launch_occ(const char* name, AcStream* st, const Body& body, uint64_t n) { ac_launch(name, st, body, n); }
template <class Body> inline void ac_launch(const char*, AcStream*, const Body& body, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) body(i);
}
// Cooperative launch: body(thread, n_threads, sync) walks its items with stride n_threads and may call sync() — a barrier over the
// whole grid — between phases.  Emulated by one thread.
struct AcGridSync { void operator()() const {} };
template <class Body> inline void ac_launch_coop(const char*, AcStream*, const Body& body, uint64_t, uint64_t = 256) { AcGridSync sync; body(0, 1, sync); }
// Events that order one stream after another (no timing): no-ops under emulation, where every copy is done when it is issued
struct AcEvent {};
inline void ac_record(AcEvent*, AcStream*) {}
inline void ac_wait(AcStream*, AcEvent*) {}

#else
// ------------------------------------------------------------------------------------------------
#include <cuda_runtime.h>

#ifdef __CUDACC__
#define AC_HD __host__ __device__ __forceinline__
#define AC_D __device__ __forceinline__
#else   // host translation units of the product build only see the host-callable part
#define AC_HD inline
#define AC_D inline
#endif

#define AC_CUDA_CHECK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) \
    throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e)); } while (0)

#ifdef __CUDACC__
AC_D uint64_t ac_atomic_cas(uint64_t* p, uint64_t cmp, uint64_t val) {
    return (uint64_t)atomicCAS((unsigned long long*)p, (unsigned long long)cmp, (unsigned long long)val);
}
AC_D uint32_t ac_atomic_cas(uint32_t* p, uint32_t cmp, uint32_t val) { return atomicCAS(p, cmp, val); }
AC_D uint32_t ac_atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
AC_D uint64_t ac_atomic_add(uint64_t* p, uint64_t v) { return (uint64_t)atomicAdd((unsigned long long*)p, (unsigned long long)v); }
AC_D unsigned long long ac_atomic_add(unsigned long long* p, unsigned long long v) { return atomicAdd(p, v); }
AC_D uint32_t ac_atomic_or(uint32_t* p, uint32_t v) { return atomicOr(p, v); }
AC_D uint32_t ac_atomic_min(uint32_t* p, uint32_t v) { return atomicMin(p, v); }
AC_D uint32_t ac_atomic_max(uint32_t* p, uint32_t v) { return atomicMax(p, v); }
AC_D uint64_t ac_atomic_min(uint64_t* p, uint64_t v) { return (uint64_t)atomicMin((unsigned long long*)p, (unsigned long long)v); }
AC_D uint64_t ac_atomic_max(uint64_t* p, uint64_t v) { return (uint64_t)atomicMax((unsigned long long*)p, (unsigned long long)v); }
template <class T> AC_D T ac_ld_volatile(const T* p) { return *(const volatile T*)p; }
AC_D uint64_t ac_ld_cg(const uint64_t* p) { return (uint64_t)__ldcg(reinterpret_cast<const unsigned long long*>(p)); }   // L2 (cache-global) load: sees other threads' atomics
// four consecutive 8-byte records (one 32-byte sector) in two 128-bit L2 loads (sm_90 has no 256-bit load); every record is read
// whole, and callers treat each one on its own (a record may lag the table, as any load may)
AC_D void ac_ld_group(const uint64_t* p, uint64_t out[4]) {
    asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(out[0]), "=l"(out[1]) : "l"(p) : "memory");
    asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(out[2]), "=l"(out[3]) : "l"(p + 2) : "memory");
}
AC_D void ac_st_stream(uint32_t* p, uint32_t v) { __stcs(p, v); }      // written once, read much later: evict first, leave the L2 to the table
AC_D uint64_t ac_umul64hi(uint64_t a, uint64_t b) { return __umul64hi(a, b); }
AC_D uint32_t ac_popc(uint32_t v) { return (uint32_t)__popc(v); }
AC_D int ac_ctz(uint32_t v) { return __ffs((int)v) - 1; }
AC_D uint64_t ac_atomic_or(uint64_t* p, uint64_t v) { return (uint64_t)atomicOr((unsigned long long*)p, (unsigned long long)v); }
AC_D uint64_t ac_atomic_and(uint64_t* p, uint64_t v) { return (uint64_t)atomicAnd((unsigned long long*)p, (unsigned long long)v); }
#endif

struct AcStream { cudaStream_t s; };

inline void* ac_dev_alloc(size_t bytes) { void* p = nullptr; AC_CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1)); return p; }
inline void ac_dev_free(void* p) { if (p) cudaFree(p); }
inline void ac_memset(void* p, int v, size_t bytes, AcStream* st) { AC_CUDA_CHECK(cudaMemsetAsync(p, v, bytes, st->s)); }
inline void ac_h2d(void* d, const void* h, size_t bytes, AcStream* st) { AC_CUDA_CHECK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st->s)); }
inline void ac_d2h(void* h, const void* d, size_t bytes, AcStream* st) { AC_CUDA_CHECK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st->s)); }
inline void ac_copy_dd(void* dst, const void* src, size_t bytes, AcStream* st) { AC_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st->s)); }
inline void ac_sync(AcStream* st) { AC_CUDA_CHECK(cudaStreamSynchronize(st->s)); }
// AC_SYNC_LAUNCHES=1 (debugging): wait for every kernel right after its launch and name the one that failed.
inline void ac_debug_sync(const char* name, AcStream* st) {
    static const bool on = getenv("AC_SYNC_LAUNCHES") != nullptr;
    if (!on) return;
    const cudaError_t e = cudaStreamSynchronize(st->s);
    if (e != cudaSuccess) throw std::runtime_error(std::string("kernel ") + name + " failed: " + cudaGetErrorString(e));
}
inline void* ac_host_alloc(size_t bytes) { void* p = nullptr; AC_CUDA_CHECK(cudaMallocHost(&p, bytes ? bytes : 1)); return p; }
inline void ac_host_free(void* p) { if (p) cudaFreeHost(p); }
// SMs of the current device (132 on an H100 SXM), read once: every device a process drives is the same model
inline uint64_t ac_sm_count() {
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    return (uint64_t)sms;
}
// Opt-in shared memory one CTA may ask for (227 KiB on an H100), read once: every device a process drives is the same model
inline int ac_smem_optin() {
    static int optin = -1;
    if (optin < 0) { int dev = 0; AC_CUDA_CHECK(cudaGetDevice(&dev)); AC_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)); }
    return optin;
}
// An event that orders one stream after another (no timing)
struct AcEvent {
    cudaEvent_t e = nullptr;
    AcEvent() { AC_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); }
    AcEvent(const AcEvent&) = delete; AcEvent& operator=(const AcEvent&) = delete;
    ~AcEvent() { cudaEventDestroy(e); }
};
inline void ac_record(AcEvent* ev, AcStream* st) { AC_CUDA_CHECK(cudaEventRecord(ev->e, st->s)); }
inline void ac_wait(AcStream* st, AcEvent* ev) { AC_CUDA_CHECK(cudaStreamWaitEvent(st->s, ev->e, 0)); }
// Device time of what a stream runs between the constructor and stop() (two CUDA events); ms() once the stream has synced
class AcTimer {
    cudaEvent_t e0 = nullptr, e1 = nullptr; AcStream* st;
public:
    explicit AcTimer(AcStream* st) : st(st) { AC_CUDA_CHECK(cudaEventCreate(&e0)); AC_CUDA_CHECK(cudaEventCreate(&e1)); AC_CUDA_CHECK(cudaEventRecord(e0, st->s)); }
    AcTimer(const AcTimer&) = delete; AcTimer& operator=(const AcTimer&) = delete;
    ~AcTimer() { cudaEventDestroy(e0); cudaEventDestroy(e1); }
    void stop() { AC_CUDA_CHECK(cudaEventRecord(e1, st->s)); }
    float ms() const { float t = 0.f; AC_CUDA_CHECK(cudaEventElapsedTime(&t, e0, e1)); return t; }
};
// The device and stream a device object runs on: the caller's stream, or (null) a non-blocking stream of its own
struct DeviceContext {
    int device; AcStream stream; bool own_stream = false;
    DeviceContext(int device, void* s) : device(device) {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n == 0)
            throw std::runtime_error(std::string("autocycler_gpu: no CUDA device available (") + cudaGetErrorString(e) + "); this library has no CPU path");
        AC_CUDA_CHECK(cudaSetDevice(device));
        if (s) stream.s = (cudaStream_t)s;
        else { AC_CUDA_CHECK(cudaStreamCreateWithFlags(&stream.s, cudaStreamNonBlocking)); own_stream = true; }
    }
    DeviceContext(const DeviceContext&) = delete; DeviceContext& operator=(const DeviceContext&) = delete;
    ~DeviceContext() { if (own_stream) { cudaSetDevice(device); cudaStreamDestroy(stream.s); } }
    void make_current() const { AC_CUDA_CHECK(cudaSetDevice(device)); }
};

#ifdef __CUDACC__
#include <cooperative_groups.h>
// Every kernel but the cooperative ones is launched here: a dynamic shared-memory size is opted into, a launch error names the kernel, the launch is counted
// and AC_SYNC_LAUNCHES waits for it.
template <class... P, class... A> inline void ac_launch_kernel(const char* name, AcStream* st, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A... args) {
    if (smem > 0) AC_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, block, smem, st->s>>>(args...);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("launch ") + name + ": " + cudaGetErrorString(e));
    ++g_ac_kernel_launches;
    ac_debug_sync(name, st);
}

// The trip count is the same for every lane of a warp and the lanes meet again after each unit: bodies with data-dependent
// latency (hash probes) otherwise let the lanes drift into different iterations and the warp issues every instruction for a
// fraction of its lanes.
template <class Body> __global__ void __launch_bounds__(256) ac_body_kernel(const Body body, uint64_t n) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint32_t lane = threadIdx.x & 31u;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
        const uint64_t i = base + lane;
        if (i < n) body(i);
        __syncwarp();
    }
}

// The same loop compiled for a given number of resident 256-thread CTAs per SM (a register budget).  For the insert, a budget
// without spills beats more resident CTAs with spills (DESIGN.md §4).
template <class Body, int CTAS> __global__ void __launch_bounds__(256, CTAS) ac_body_kernel_occ(const Body body, uint64_t n) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint32_t lane = threadIdx.x & 31u;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
        const uint64_t i = base + lane;
        if (i < n) body(i);
        __syncwarp();
    }
}
template <int CTAS, class Body> inline void ac_launch_occ(const char* name, AcStream* st, const Body& body, uint64_t n) {
    if (n == 0) return;
    const int threads = 256;
    const uint64_t want = (n + threads - 1) / threads, max_blocks = ac_sm_count() * (uint64_t)CTAS * 2;   // two waves of resident CTAs, grid-stride beyond
    ac_launch_kernel(name, st, ac_body_kernel_occ<Body, CTAS>, (unsigned)(want < max_blocks ? want : max_blocks), threads, 0, body, n);
}

// Cooperative launch (all CTAs co-resident): body(thread, n_threads, sync) walks its items with stride n_threads and may call
// sync() — a barrier over the whole grid — between phases, so that a chain of small dependent steps costs one launch instead of one
// launch (and often one host round trip) per step.  `work` / `per_block` sizes the grid — a barrier over few CTAs is cheap (a microsecond
// or two against five to ten over every SM), so steps with little work per phase ask for few — never more CTAs than fit.
struct AcGridSync { __device__ __forceinline__ void operator()() const { cooperative_groups::this_grid().sync(); } };
template <class Body> __global__ void __launch_bounds__(256) ac_coop_kernel(const Body body) {
    AcGridSync sync;
    body((uint64_t)blockIdx.x * blockDim.x + threadIdx.x, (uint64_t)gridDim.x * blockDim.x, sync);
}
template <class Body> inline void ac_launch_coop(const char* name, AcStream* st, const Body& body, uint64_t work, uint64_t per_block = 256) {
    static int resident = 0;                  // per kernel instantiation; one device per process in this library
    if (!resident) {
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ac_coop_kernel<Body>, 256, 0);
        resident = per_sm * (int)ac_sm_count();
        if (resident <= 0) throw std::runtime_error(std::string("cooperative launch ") + name + ": kernel does not fit");
    }
    uint64_t want = (work + per_block - 1) / per_block;
    if (want < 1) want = 1;
    const int sms = (int)ac_sm_count();
    const uint64_t cap = resident < sms ? (uint64_t)resident : (uint64_t)sms;     // one CTA per SM is plenty for these small steps, and keeps the barrier cheap
    const unsigned blocks = (unsigned)(want < cap ? want : cap);
    void* args[] = {(void*)&body};
    cudaError_t e = cudaLaunchCooperativeKernel((void*)ac_coop_kernel<Body>, dim3(blocks), dim3(256), args, 0, st->s);
    if (e != cudaSuccess) throw std::runtime_error(std::string("cooperative launch ") + name + ": " + cudaGetErrorString(e));
    ++g_ac_kernel_launches;
    ac_debug_sync(name, st);
}

template <class Body> inline void ac_launch(const char* name, AcStream* st, const Body& body, uint64_t n) {
    if (n == 0) return;
    const int threads = 256;
    uint64_t want = (n + threads - 1) / threads;
    const uint64_t max_blocks = ac_sm_count() * 16;   // every SM x 16 256-thread CTAs (two waves of the 8 an SM holds), grid-stride beyond that
    ac_launch_kernel(name, st, ac_body_kernel<Body>, (unsigned)(want < max_blocks ? want : max_blocks), threads, 0, body, n);
}
#endif   // __CUDACC__
#endif

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    void ensure(size_t bytes) {
        if (bytes > cap) {
            ac_dev_free(p); p = nullptr; cap = 0; p = ac_dev_alloc(bytes); cap = bytes;
#ifdef AC_EMULATE
            static const bool poison = getenv("AC_EMU_POISON") != nullptr;
            if (poison) memset(p, 0xA5, cap);
#endif
        }
    }
    template <class T> T* as() { return (T*)p; }
    ~DevBuf() { ac_dev_free(p); }
};

struct PinBuf {   // pinned host memory: D2H lands at DMA speed and the host graph works on it in place
    void* p = nullptr; size_t cap = 0;
    void ensure(size_t bytes) { if (bytes > cap) { ac_host_free(p); p = nullptr; cap = 0; p = ac_host_alloc(bytes); cap = bytes; } }
    template <class T> T* as() { return (T*)p; }
    ~PinBuf() { ac_host_free(p); }
};

// Exclusive scan from serial pieces, for small volumes: one thread sums each tile of TILE values, the tile sums are scanned the same way
// one level up, then each thread writes its tile's prefixes.  out may alias in.  Returns the total when asked (one host round trip).
template <class T, uint64_t TILE, int LEVELS> struct SerialScan {
    DevBuf level[LEVELS];                    // the tile sums of every level
    T run(AcStream* st, const T* in, T* out, uint64_t n, bool want_total, int l = 0);
};
#if defined(AC_EMULATE) || defined(__CUDACC__)
template <class T, uint64_t TILE> struct ScanSumBody {
    const T* in; uint64_t n; T* sums;
    AC_D void operator()(uint64_t t) const {
        const uint64_t lo = t * TILE, hi = lo + TILE < n ? lo + TILE : n;
        T s = 0;
        for (uint64_t x = lo; x < hi; ++x) s += in[x];
        sums[t] = s;
    }
};
template <class T, uint64_t TILE> struct ScanApplyBody {
    const T* in; T* out; uint64_t n; const T* tile_off;
    AC_D void operator()(uint64_t t) const {
        const uint64_t lo = t * TILE, hi = lo + TILE < n ? lo + TILE : n;
        T acc = tile_off ? tile_off[t] : 0;
        for (uint64_t x = lo; x < hi; ++x) { const T v = in[x]; out[x] = acc; acc += v; }
    }
};
template <class T, uint64_t TILE, int LEVELS> T SerialScan<T, TILE, LEVELS>::run(AcStream* st, const T* in, T* out, uint64_t n, bool want_total, int l) {
    if (n == 0) return 0;
    if (l >= LEVELS) throw std::runtime_error("scan too deep");
    const uint64_t nb = (n + TILE - 1) / TILE;
    if (nb == 1 && !want_total) { ac_launch("scan_apply", st, ScanApplyBody<T, TILE>{in, out, n, nullptr}, 1); return 0; }
    level[l].ensure(nb * sizeof(T));
    T* sums = level[l].template as<T>();
    T total = 0;
    ac_launch("scan_sum", st, ScanSumBody<T, TILE>{in, n, sums}, nb);
    if (nb == 1) { ac_d2h(&total, sums, sizeof(T), st); ac_sync(st); }
    else total = run(st, sums, sums, nb, want_total, l + 1);
    ac_launch("scan_apply", st, ScanApplyBody<T, TILE>{in, out, n, nb == 1 ? nullptr : sums}, nb);
    return total;
}
#endif

// Exclusive scan of n u32 values in one launch (ac_scan_chained_kernel; serial tiles of 256 under emulation), with the state it keeps
// from one scan to the next.  out may alias in.  Returns the total when asked: that costs one host round trip.
struct DeviceScan {
    uint32_t operator()(AcStream* st, const uint32_t* in, uint32_t* out, uint64_t n, bool want_total = true);
    // in place; x[n-1] must be 0, so that the scanned x[n-1] is the total, which stays on the device (copied to total_dst)
    void keep_total(AcStream* st, uint32_t* x, uint64_t n, uint32_t* total_dst) { (*this)(st, x, x, n, false); ac_copy_dd(total_dst, x + (n - 1), 4, st); }
#ifndef AC_EMULATE
    DevBuf state; unsigned long long epoch = 0, tickets = 0;
#else
    SerialScan<uint32_t, 256, 4> serial;
#endif
};

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

template <class Body> inline void ac_launch(const char*, AcStream*, const Body& body, uint64_t n);
template <int CTAS, class Body> inline void ac_launch_occ(const char* name, AcStream* st, const Body& body, uint64_t n) { ac_launch(name, st, body, n); }
template <class Body> inline void ac_launch(const char*, AcStream*, const Body& body, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) body(i);
}
// Cooperative launch: body(thread, n_threads, sync) walks its items with stride n_threads and may call sync() — a barrier over the
// whole grid — between phases.  Emulated by one thread.
struct AcGridSync { void operator()() const {} };
template <class Body> inline void ac_launch_coop(const char*, AcStream*, const Body& body, uint64_t, uint64_t = 256) { AcGridSync sync; body(0, 1, sync); }

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

#ifdef __CUDACC__
#include <cooperative_groups.h>
// Every functor-body kernel is launched through this one grid-stride template; the launch counter
// feeds bench.py's "gpu_launches".
extern unsigned long long g_ac_kernel_launches;

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
    const unsigned blocks = (unsigned)(want < max_blocks ? want : max_blocks);
    ac_body_kernel_occ<Body, CTAS><<<blocks, threads, 0, st->s>>>(body, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("launch ") + name + ": " + cudaGetErrorString(e));
    ++g_ac_kernel_launches;
    ac_debug_sync(name, st);
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
    unsigned blocks = (unsigned)(want < max_blocks ? want : max_blocks);
    ac_body_kernel<Body><<<blocks, threads, 0, st->s>>>(body, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("launch ") + name + ": " + cudaGetErrorString(e));
    ++g_ac_kernel_launches;
    ac_debug_sync(name, st);
}
#endif   // __CUDACC__
#endif

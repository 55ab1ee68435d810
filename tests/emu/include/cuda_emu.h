// cuda_emu.h — TEST INFRASTRUCTURE ONLY.  A minimal SIMT emulation that lets tests/ run the *kernel source* of
// csrc/*.cuh on the host, one OS thread per CUDA thread, so that kernel logic can be checked against the oracle
// in a container without a GPU.  It is never linked into libbigclam_b200.so and nothing in the package can
// reach it: the product has no CPU path.
//
//   * a warp = 32 threads sharing a pthread barrier and a 32-slot exchange buffer: __shfl*_sync, __ballot_sync,
//     __any_sync and __syncwarp are barrier rounds, so a collective reached by only part of a warp (a bug on
//     the GPU as well) shows up here as a hang -> run under a timeout;
//   * a block = its warps plus one more barrier (__syncthreads); blocks run one after the other (fine for
//     kernels without inter-block waits);
//   * `extern __shared__` / `__shared__` are rewritten by tests/emu/build.sh (dynamic -> emu::dyn_smem(),
//     static -> function-local static);
//   * inline PTX is replaced in the kernel headers under #ifdef BIGCLAM_EMU.
#pragma once
#include <pthread.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <thread>
#include <type_traits>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __grid_constant__
#define __align__(n) alignas(n)

struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
using emu_dim3 = dim3;
extern thread_local emu_dim3 threadIdx, blockIdx, blockDim, gridDim;

struct alignas(16) double2 { double x, y; };
inline double2 make_double2(double x, double y) { return double2{x, y}; }
struct alignas(8) float2 { float x, y; };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float __double2float_ru(double d) {
    float f = (float)d;
    if ((double)f < d) f = std::nextafterf(f, INFINITY);
    return f;
}
inline float __log2f(float v) { return std::log2(v); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __double2float_rd(double d) {
    float f = (float)d;
    if ((double)f > d) f = std::nextafterf(f, -INFINITY);
    return f;
}

namespace emu {
struct WarpCtx {
    pthread_barrier_t bar;
    uint64_t slot[2][32];          // two exchange buffers used alternately: one barrier round per collective
};
struct BlockCtx {
    pthread_barrier_t bar;
};
extern thread_local WarpCtx *warp;
extern thread_local BlockCtx *block;
extern thread_local int lane;
extern thread_local int xpar;      // which exchange buffer this lane's next collective uses (same on all lanes of a warp)
extern unsigned char *g_dyn_smem;
inline unsigned char *dyn_smem() { return g_dyn_smem; }
inline void wsync() { pthread_barrier_wait(&warp->bar); }
template <class T>
inline T exch(T v, int src) {
    static_assert(sizeof(T) <= 8, "emulated shuffles move at most 8 bytes");
    uint64_t u = 0;
    std::memcpy(&u, &v, sizeof(T));
    // the next collective writes the other buffer, and the one after that can only start once every lane has
    // passed the next barrier, i.e. has finished reading this one: no second barrier needed
    const int p = (xpar ^= 1);
    warp->slot[p][lane] = u;
    wsync();
    const uint64_t r = warp->slot[p][src & 31];
    T out;
    std::memcpy(&out, &r, sizeof(T));
    return out;
}
}  // namespace emu

template <class T> inline T __shfl_sync(unsigned, T v, int src, int = 32) { return emu::exch(v, src); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return emu::exch(v, emu::lane ^ m); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) {
    const int src = emu::lane - (int)d;
    return emu::exch(v, src < 0 ? emu::lane : src);
}
inline unsigned __ballot_sync(unsigned, int pred) {
    const int p = (emu::xpar ^= 1);
    emu::warp->slot[p][emu::lane] = pred ? 1u : 0u;
    emu::wsync();
    unsigned m = 0;
    for (int i = 0; i < 32; ++i) m |= (unsigned)emu::warp->slot[p][i] << i;
    return m;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::wsync(); }
inline void __syncthreads() { pthread_barrier_wait(&emu::block->bar); }

struct alignas(16) uint4 { unsigned x, y, z, w; };
inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline double atomicAdd(double *p, double v) {
    uint64_t *q = reinterpret_cast<uint64_t *>(p);
    uint64_t old = __atomic_load_n(q, __ATOMIC_SEQ_CST);
    for (;;) {
        double d;
        std::memcpy(&d, &old, 8);
        d += v;
        uint64_t nu;
        std::memcpy(&nu, &d, 8);
        if (__atomic_compare_exchange_n(q, &old, nu, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
            double r;
            std::memcpy(&r, &old, 8);
            return r;
        }
    }
}

template <class T> inline T __ldg(const T *p) { return *p; }
template <class T> inline T __ldcg(const T *p) { return *p; }
inline int __double2hiint(double d) { int64_t u; std::memcpy(&u, &d, 8); return (int)(u >> 32); }
inline int __double2loint(double d) { int64_t u; std::memcpy(&u, &d, 8); return (int)(u & 0xffffffff); }
inline double __hiloint2double(int hi, int lo) {
    const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo;
    double d;
    std::memcpy(&d, &u, 8);
    return d;
}
inline double __dadd_rn(double a, double b) { return a + b; }     // build with -ffp-contract=off
inline double __dmul_rn(double a, double b) { return a * b; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
inline void __nanosleep(unsigned) {}
inline void __threadfence() { __sync_synchronize(); }
inline void __threadfence_system() { __sync_synchronize(); }
using std::fma;

template <class A, class B> inline std::common_type_t<A, B> min(A a, B b) {
    using T = std::common_type_t<A, B>;
    return (T)a < (T)b ? (T)a : (T)b;
}
template <class A, class B> inline std::common_type_t<A, B> max(A a, B b) {
    using T = std::common_type_t<A, B>;
    return (T)a > (T)b ? (T)a : (T)b;
}

namespace emu {
// <<<grid, block, smem>>> : blocks one after the other, `block` OS threads each
template <class K, class... A>
inline void launch(K kernel, dim3 grid3, unsigned block, size_t smem, A... args) {
    const unsigned grid = grid3.x * grid3.y;
    for (unsigned b = 0; b < grid; ++b) {
        std::vector<unsigned char> sm(smem + 64);
        g_dyn_smem = reinterpret_cast<unsigned char *>(((uintptr_t)sm.data() + 63) & ~(uintptr_t)63);
        BlockCtx bc;
        pthread_barrier_init(&bc.bar, nullptr, block);
        const unsigned nw = (block + 31) / 32;
        std::vector<WarpCtx> wc(nw);
        for (unsigned w = 0; w < nw; ++w) pthread_barrier_init(&wc[w].bar, nullptr, std::min(32u, block - 32 * w));
        std::vector<std::thread> th;
        th.reserve(block);
        for (unsigned t = 0; t < block; ++t)
            th.emplace_back([=, &bc, &wc]() {
                threadIdx.x = t;
                blockIdx.x = b % grid3.x;
                blockIdx.y = b / grid3.x;
                blockDim.x = block;
                gridDim.x = grid3.x;
                gridDim.y = grid3.y;
                lane = (int)(t & 31);
                xpar = 0;
                warp = &wc[t / 32];
                emu::block = &bc;
                kernel(args...);
            });
        for (auto &x : th) x.join();
        for (unsigned w = 0; w < nw; ++w) pthread_barrier_destroy(&wc[w].bar);
        pthread_barrier_destroy(&bc.bar);
    }
}
}  // namespace emu

// ---------------------------------------------------------------------------------------------------------------
// BIGCLAM_EMU_HOST: a synchronous stand-in for the part of the CUDA runtime csrc/bigclam_capi.cu uses, so that the
// HOST LOGIC of the C API (speculation, buffer flips, device-side loop bookkeeping, sparse-row plumbing) can be
// driven by the existing `-m gpu` tests on a machine without a GPU (tools only; see tests/emu/build_hostemu.sh).
// "Device" memory is host memory, streams and events are no-ops / wall clocks, one SM, kernels run on launch.
#ifdef BIGCLAM_EMU_HOST
typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0;
typedef void *cudaStream_t;
struct emu_event { std::chrono::steady_clock::time_point t; };
typedef emu_event *cudaEvent_t;
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp { int major = 9, minor = 0, multiProcessorCount = 1; };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyHostToHost };
enum { cudaStreamNonBlocking = 1, cudaIpcMemLazyEnablePeerAccess = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
inline const char *cudaGetErrorString(cudaError_t) { return "emulated runtime error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 8; return cudaSuccess; }     // (bigclam_multi_*: several emulated devices)
constexpr cudaError_t cudaErrorPeerAccessAlreadyEnabled = 704;
inline cudaError_t cudaDeviceCanAccessPeer(int *can, int, int) { *can = 1; return cudaSuccess; }
inline cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { *p = cudaDeviceProp(); return cudaSuccess; }
template <class K> inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }
template <class K> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *b, K, int, size_t) { *b = 2; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
template <class T> inline cudaError_t cudaMalloc(T **p, size_t bytes) { *p = static_cast<T *>(std::malloc(bytes ? bytes : 1)); return *p ? cudaSuccess : 2; }
template <class T> inline cudaError_t cudaMallocHost(T **p, size_t bytes) { return cudaMalloc(p, bytes); }
inline cudaError_t cudaFree(void *p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaFreeHost(void *p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind k, cudaStream_t) { return cudaMemcpy(d, s, n, k); }
inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t) {
    for (size_t r = 0; r < h; ++r) std::memmove(static_cast<char *>(d) + r * dp, static_cast<const char *>(s) + r * sp, w);
    return cudaSuccess;
}
inline cudaError_t cudaMemset(void *d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { return cudaMemset(d, v, n); }
inline cudaError_t cudaMemGetInfo(size_t *f, size_t *t) { *f = *t = (size_t)8 << 30; return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new emu_event(); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
    return cudaSuccess;
}
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { std::memset(h, 0, sizeof(*h)); std::memcpy(h, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { std::memcpy(p, &h, sizeof(*p)); return cudaSuccess; }
inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
#endif  // BIGCLAM_EMU_HOST

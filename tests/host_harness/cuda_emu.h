// cuda_emu.h -- TEST-ONLY.  Just enough of the CUDA execution model to run the kernels of
// irbpp_b200/csrc/ on host threads, so that kernel-level logic (barrier structure, warp collectives,
// shared-memory hand-overs) can be checked against the oracle in a container without a GPU:
//   * one host thread per CUDA thread of ONE thread block at a time (blocks run one after another);
//   * __shared__ variables become function-local statics (one block alive at a time);
//   * __syncthreads / __syncwarp are real barriers; every warp collective is an exchange through a
//     32-entry slot array between two warp barriers (full masks only, as the kernels use them);
//   * the runtime API is mapped onto the host heap; "device" and "host" pointers are the same.
// It is slow (thousands of thread switches per launch) and is never linked into the product: the
// library built from it exports emu_irbpp_* names that irbpp_b200/_lib.py cannot bind.
#pragma once
#define IRBPP_HOST_EMULATION 1      // csrc/irbpp_tma.cuh: bulk copies become memcpy, mbarrier waits no-ops
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) alignas(n)

using std::max;
using std::min;

struct uint3_emu { unsigned x = 0, y = 0, z = 0; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a) : x(a) {} dim3(int a) : x((unsigned)a) {} };
static thread_local uint3_emu threadIdx, blockIdx;
static uint3_emu blockDim, gridDim;

struct uint4 { uint32_t x, y, z, w; };
struct float4 { float x, y, z, w; };
struct double2 { double x, y; };
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline double2 make_double2(double a, double b) { return double2{a, b}; }

namespace cuda_emu {

struct Barrier {
    std::mutex m;
    std::condition_variable cv;
    int count = 0, gen = 0;
    void wait(int n) {
        std::unique_lock<std::mutex> lk(m);
        const int g = gen;
        if (++count == n) { count = 0; ++gen; cv.notify_all(); }
        else cv.wait(lk, [&] { return gen != g; });
    }
};

constexpr int MAX_WARPS = 32;
static unsigned char* dyn_smem = nullptr;      // the launch's dynamic shared memory, exactly as many bytes as requested
static Barrier cta_bar;
static Barrier warp_bar[MAX_WARPS];
static uint64_t slots[MAX_WARPS][32];
static int cta_threads = 0;

static inline int lane() { return (int)(threadIdx.x & 31u); }
static inline int warp() { return (int)(threadIdx.x >> 5); }

// all-to-all exchange of one 64-bit value inside the calling thread's warp
static inline void exchange(uint64_t v, uint64_t (&out)[32]) {
    const int w = warp();
    slots[w][lane()] = v;
    warp_bar[w].wait(32);
    for (int i = 0; i < 32; ++i) out[i] = slots[w][i];
    warp_bar[w].wait(32);
}
template <class T> static inline uint64_t pack(T v) { uint64_t u = 0; memcpy(&u, &v, sizeof(T)); return u; }
template <class T> static inline T unpack(uint64_t u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

template <class K, class... A>
static void launch(K kernel, int grid, int block, size_t smem_bytes, A... args) {
    gridDim.x = (unsigned)grid; blockDim.x = (unsigned)block; cta_threads = block;
    // a heap block of exactly the requested size: an address sanitizer then sees any access beyond it
    void* mem = nullptr;
    if (posix_memalign(&mem, 16, smem_bytes ? smem_bytes : 16)) abort();
    dyn_smem = static_cast<unsigned char*>(mem);
    for (int b = 0; b < grid; ++b) {
        std::vector<std::thread> th;
        th.reserve(block);
        for (int t = 0; t < block; ++t)
            th.emplace_back([=] { threadIdx.x = (unsigned)t; blockIdx.x = (unsigned)b; kernel(args...); });
        for (auto& x : th) x.join();
    }
    dyn_smem = nullptr;
    free(mem);
}

}  // namespace cuda_emu

static inline void __syncthreads() { cuda_emu::cta_bar.wait(cuda_emu::cta_threads); }
static inline void __syncwarp(unsigned = 0xffffffffu) { cuda_emu::warp_bar[cuda_emu::warp()].wait(32); }

template <class T> static inline T __shfl_sync(unsigned, T v, int src) {
    uint64_t o[32]; cuda_emu::exchange(cuda_emu::pack(v), o); return cuda_emu::unpack<T>(o[src & 31]);
}
template <class T> static inline T __shfl_up_sync(unsigned, T v, int delta) {
    uint64_t o[32]; cuda_emu::exchange(cuda_emu::pack(v), o);
    const int l = cuda_emu::lane(); return l >= delta ? cuda_emu::unpack<T>(o[l - delta]) : v;
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int x) {
    uint64_t o[32]; cuda_emu::exchange(cuda_emu::pack(v), o); return cuda_emu::unpack<T>(o[(cuda_emu::lane() ^ x) & 31]);
}
static inline unsigned __ballot_sync(unsigned, int pred) {
    uint64_t o[32]; cuda_emu::exchange(pred ? 1u : 0u, o);
    unsigned r = 0; for (int i = 0; i < 32; ++i) r |= (unsigned)(o[i] & 1u) << i; return r;
}
static inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }
static inline unsigned __reduce_or_sync(unsigned, unsigned v) {
    uint64_t o[32]; cuda_emu::exchange(v, o); unsigned r = 0; for (int i = 0; i < 32; ++i) r |= (unsigned)o[i]; return r;
}
static inline unsigned __reduce_max_sync(unsigned, unsigned v) {
    uint64_t o[32]; cuda_emu::exchange(v, o); unsigned r = 0; for (int i = 0; i < 32; ++i) r = std::max(r, (unsigned)o[i]); return r;
}

static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
// position of the offset-th set bit of mask at or above bit `base` (offset > 0), 0xffffffff if there is none
static inline unsigned __fns(unsigned mask, unsigned base, int offset) {
    for (unsigned b = base; b < 32; ++b)
        if ((mask >> b) & 1u) { if (--offset == 0) return b; }
    return 0xffffffffu;
}
static inline long long clock64() { return 0; }

template <class T> static inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicOr(uint32_t* p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicMax(int* p, int v) {
    int o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return o;
}
static inline int atomicMin(int* p, int v) {
    int o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (o > v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return o;
}

// ---- runtime API on the host heap ------------------------------------------------------------------------
typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0;
constexpr cudaError_t cudaErrorInvalidDevice = 101;
typedef void* cudaStream_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
constexpr unsigned cudaHostAllocMapped = 2;
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount };
enum cudaLaunchAttributeID { cudaLaunchAttributeProgrammaticStreamSerialization };
struct cudaLaunchAttribute { cudaLaunchAttributeID id; struct { int programmaticStreamSerializationAllowed; } val; };
struct cudaLaunchConfig_t { dim3 gridDim, blockDim; size_t dynamicSmemBytes; cudaStream_t stream; cudaLaunchAttribute* attrs; unsigned numAttrs; };

static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 1; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaMalloc(void** p, size_t n) { return posix_memalign(p, 256, n ? n : 256) ? 1 : cudaSuccess; }
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMalloc(p, n); }
template <class T> static inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned f) { return cudaHostAlloc(reinterpret_cast<void**>(p), n, f); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaHostGetDevicePointer(void** d, void* h, unsigned) { *d = h; return cudaSuccess; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
template <class K, class... A>
static inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* c, K kernel, A... args) {
    cuda_emu::launch(kernel, (int)c->gridDim.x, (int)c->blockDim.x, c->dynamicSmemBytes, args...);
    return cudaSuccess;
}
#define CUDA_EMU_LAUNCH(kernel, grid, block, smem, stream, ...) cuda_emu::launch(kernel, (int)(grid), (int)(block), (size_t)(smem), __VA_ARGS__)

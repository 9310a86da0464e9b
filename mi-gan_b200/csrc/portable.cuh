// What differs between the two builds of every CUDA source here, written once.
//
// The product library is compiled by nvcc for sm_90a.  The emulation build (tests/emul/build_emul.py) compiles the same
// sources as plain C++ with -DMIGAN_EMULATE -ffp-contract=off and runs the kernels' functors and block functions as
// host loops, so their arithmetic and index math are checked on a machine without a GPU.  This header decides, per
// build, the function qualifiers, the half type, the item launch, the block layer, the rounding of arithmetic and device
// memory; the host loops that stand in for a GEMM stay next to the kernel they emulate.
//
// Rounding: an operation written with one of the *_rn functions below is rounded on its own.  On the device that is
// the matching __f*_rn / __d*_rn intrinsic, which nvcc never contracts into an FMA; in the emulation build it is the
// plain operator, which -ffp-contract=off keeps uncontracted.  fma_rn is a single fused rounding in both builds.  So an
// expression written with them gives the same bits in both builds.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

#ifdef MIGAN_EMULATE
#include <vector>
#define CK_HD inline
#define CK_D inline
typedef void* ck_stream_t;
typedef _Float16 ck_half;                       // IEEE binary16, round-to-nearest-even conversions (GCC, x86-64)
CK_HD ck_half ck_f2h(float v) { return (ck_half)v; }
CK_HD float ck_h2f(ck_half h) { return (float)h; }
#else
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#define CK_HD __host__ __device__ __forceinline__
#define CK_D __device__ __forceinline__   // device-only: the function may call device intrinsics
typedef cudaStream_t ck_stream_t;
typedef __half ck_half;
CK_HD ck_half ck_f2h(float v) { return __float2half_rn(v); }
CK_HD float ck_h2f(ck_half h) { return __half2float(h); }
#endif

// ---- arithmetic rounded operation by operation ----------------------------------------------------------------------
#ifdef __CUDA_ARCH__
CK_HD float fadd_rn(float a, float b) { return __fadd_rn(a, b); }
CK_HD float fsub_rn(float a, float b) { return __fsub_rn(a, b); }
CK_HD float fmul_rn(float a, float b) { return __fmul_rn(a, b); }
CK_HD float fdiv_rn(float a, float b) { return __fdiv_rn(a, b); }
CK_HD float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
CK_HD float fsqrt_rn(float a) { return __fsqrt_rn(a); }
CK_HD double dadd_rn(double a, double b) { return __dadd_rn(a, b); }
CK_HD double dsub_rn(double a, double b) { return __dsub_rn(a, b); }
CK_HD double dmul_rn(double a, double b) { return __dmul_rn(a, b); }
CK_HD double ddiv_rn(double a, double b) { return __ddiv_rn(a, b); }
#else
CK_HD float fadd_rn(float a, float b) { return a + b; }
CK_HD float fsub_rn(float a, float b) { return a - b; }
CK_HD float fmul_rn(float a, float b) { return a * b; }
CK_HD float fdiv_rn(float a, float b) { return a / b; }
CK_HD float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
CK_HD float fsqrt_rn(float a) { return sqrtf(a); }
CK_HD double dadd_rn(double a, double b) { return a + b; }
CK_HD double dsub_rn(double a, double b) { return a - b; }
CK_HD double dmul_rn(double a, double b) { return a * b; }
CK_HD double ddiv_rn(double a, double b) { return a / b; }
#endif

// ---- alignment --------------------------------------------------------------------------------------------------------
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int round_up(int v, int a) { return (v + a - 1) / a * a; }
CK_HD size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// ---- item launches and device memory ----------------------------------------------------------------------------------
// ck_launch runs f(i) for i in [0, items): one thread per item on the device, a host loop in the emulation build.
// dev_copy is asynchronous on the stream; to_host waits for its copy, to_device does not (a pageable source is staged
// before the call returns, so the caller may free it at once).
#ifdef MIGAN_EMULATE
namespace comod {
template <class F>
inline int ck_launch(const F& f, int64_t items, ck_stream_t) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < items; ++i) f(i);
    return 0;
}
}  // namespace comod
inline int dev_set(int) { return 0; }
inline int dev_alloc(void** p, size_t bytes) { *p = aligned_alloc(256, align_up(std::max<size_t>(bytes, 1), 256)); return *p ? 0 : 1; }
inline void dev_free(void* p) { free(p); }
inline int dev_copy(void* d, const void* s, size_t bytes, ck_stream_t) { memcpy(d, s, bytes); return 0; }
inline int dev_sync() { return 0; }
inline const char* dev_err(int) { return "emulation"; }
inline int to_host(void* dst, const void* src, size_t bytes, ck_stream_t) { memcpy(dst, src, bytes); return 0; }
inline int to_device(void* dst, const void* src, size_t bytes, ck_stream_t) { memcpy(dst, src, bytes); return 0; }
#else
namespace comod {
template <class F>
__global__ void __launch_bounds__(256) ck_items_kernel(const F f, const int64_t items) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < items) f(i);
}
template <class F>
inline cudaError_t ck_launch(const F& f, int64_t items, ck_stream_t s) {
    if (items <= 0) return cudaSuccess;
    ck_items_kernel<F><<<(unsigned)((items + 255) / 256), 256, 0, s>>>(f, items);
    return cudaGetLastError();
}
}  // namespace comod
inline int dev_set(int d) { return (int)cudaSetDevice(d); }
inline int dev_alloc(void** p, size_t bytes) { return (int)cudaMalloc(p, std::max<size_t>(bytes, 256)); }
inline void dev_free(void* p) { cudaFree(p); }
inline int dev_copy(void* d, const void* s, size_t bytes, ck_stream_t st) { return (int)cudaMemcpyAsync(d, s, bytes, cudaMemcpyDefault, st); }
inline int dev_sync() { return (int)cudaDeviceSynchronize(); }
inline const char* dev_err(int e) { return cudaGetErrorString((cudaError_t)e); }
inline int to_host(void* dst, const void* src, size_t bytes, ck_stream_t s) {
    if (cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s)) return (int)e;
    return (int)cudaStreamSynchronize(s);
}
inline int to_device(void* dst, const void* src, size_t bytes, ck_stream_t s) {
    return (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s);
}
// Opt a kernel in to more than 48 KB of dynamic shared memory.
template <class K>
int set_smem(K kernel, size_t bytes) {
    return (int)cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}
#endif

// ---- block kernels ----------------------------------------------------------------------------------------------------
// A block kernel is one body over a block blk, run by both builds: blk.each(f) runs f(t) for every thread t of the
// block (on the device, f(threadIdx.x) in all threads at once; in the emulation build, t = 0, 1, ... in turn),
// blk.sync() is the barrier between two phases, and blk.any(f) is a barrier that returns whether f(t) is nonzero in
// some thread.  A value that every thread of a block holds equal is a plain local of the body; a value that differs per
// thread is a Local<T>, indexed by the thread.  Code between two barriers must not race.  ck_blocks runs a body over a
// grid of blocks on the host, each with an arena in place of the block's shared memory.
#ifdef MIGAN_EMULATE
template <int N>
struct HostBlock {
    template <class T>
    struct Local {
        T v[N];
        T& operator[](int t) { return v[t]; }
    };
    template <class F> void each(F f) const { for (int t = 0; t < N; ++t) f(t); }
    void sync() const {}
    template <class F> bool any(F f) const {
        int r = 0;
        for (int t = 0; t < N; ++t) r |= f(t);
        return r != 0;
    }
};
// body(blk, b, smem) for every block b in [0, blocks); smem is smem_bytes, 16-byte aligned, the block's own.
template <int N, class F>
int ck_blocks(int64_t blocks, size_t smem_bytes, const F& body) {
#pragma omp parallel
    {
        std::vector<double> arena(smem_bytes / sizeof(double) + 1);
        const HostBlock<N> blk;
#pragma omp for schedule(dynamic)
        for (int64_t b = 0; b < blocks; ++b) body(blk, b, static_cast<void*>(arena.data()));
    }
    return 0;
}
#else
struct DeviceBlock {
    template <class T>
    struct Local {
        T v;
        CK_D T& operator[](int) { return v; }
    };
    template <class F> CK_D void each(F f) const { f((int)threadIdx.x); }
    CK_D void sync() const { __syncthreads(); }
    template <class F> CK_D bool any(F f) const { return __syncthreads_or(f((int)threadIdx.x)) != 0; }
};
#endif

// s[0] = s[0] + ... + s[N - 1] in a fixed tree (stride N / 2, N / 4, ..., 1), visible to every thread on return.  s
// holds one partial per thread, written before the call.
template <int N, class B>
CK_D void block_tree(const B& blk, double* s) {
    blk.sync();
    for (int stride = N / 2; stride > 0; stride >>= 1) {
        blk.each([&](int t) {
            if (t < stride) s[t] = dadd_rn(s[t], s[t + stride]);
        });
        blk.sync();
    }
}

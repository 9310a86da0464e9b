// Tensor-core convolution of the FID InceptionV3 forward (sm_90a): an implicit GEMM on wgmma with TF32 operands.
//
//   M = output pixels n*OH*OW, N = cout (packed to NP, a multiple of 64), K = kh*kw*cinp (packed to KP, a multiple of 32).
//   CTA: 256 threads = two warpgroups; tile 128 pixels x 64 channels, each warpgroup owns 64 pixel rows.
//   K loop in chunks of 32: every thread gathers four float4 of the A chunk (pixel row, 16 consecutive k) straight from
//   the NHWC input -- halo and zero padding included, no im2col buffer -- splits them into TF32 hi / lo in registers and
//   stores both into the 128-byte-swizzled K-major tile; the pre-split B chunk arrives by cp.async.  Two stages: the
//   gathers of chunk k+1 run while the wgmma of chunk k execute.
//   Precision: three passes hi*hi + hi*lo + lo*hi (m64n64k8 .tf32), the hi*hi products in one accumulator and the two
//   corrections in their own, added in the epilogue (fp32-faithful, the generator kernel's scheme of DESIGN section 3
//   with TF32 instead of fp16 halves: fp32's exponent range, so no activation clamp is needed).
//   Epilogue: + folded BatchNorm bias, ReLU, store into the channel slice [c0, c0 + cout) of a ct-channel NHWC tensor.
#include <cuda_runtime.h>
#include <stdint.h>

#include "inception_kernels.cuh"

namespace migan {
namespace {

constexpr int kBM = 128, kBN = 64, kBK = 32, kThreads = 256;
constexpr int kATile = kBM * kBK * 4;                 // 16 KB per half (hi or lo)
constexpr int kBTile = kBN * kBK * 4;                 // 8 KB per half
constexpr int kStage = 2 * kATile + 2 * kBTile;       // 48 KB
constexpr int kSmem = 2 * kStage + 1024;              // two stages + alignment slack

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major operand, 128-byte swizzle: rows of 32 fp32 (128 B), 8-row groups 1024 B apart.  +32 B steps k by 8.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr) {
    uint64_t d = 0;
    d |= (uint64_t)((addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// Byte offset of the 16-byte chunk q (k = 4q .. 4q+3) of row r in a swizzled tile.
__device__ __forceinline__ uint32_t sw_off(int r, int q) { return (uint32_t)(r * 128 + ((q ^ (r & 7)) << 4)); }

// D[64 x 64] (+)= A[64 x 8] * B[64 x 8]^T, TF32 operands K-major in shared memory, fp32 accumulators.
__device__ __forceinline__ void mma_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

struct Gather {
    float4 v[4];
};

__global__ void __launch_bounds__(kThreads, 1) incep_conv_tf32_kernel(const __grid_constant__ IncepConvArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
    const int tid = threadIdx.x, wg = tid >> 7;
    const int64_t P = (int64_t)a.n * a.OH * a.OW;
    const int64_t m0 = (int64_t)blockIdx.x * kBM;
    const int n0 = blockIdx.y * kBN;
    const int taps = a.kh * a.kw, nk = a.KP / kBK;

    // this thread's A row (pixel) and its 16 k of each chunk
    const int arow = tid >> 1, aq0 = (tid & 1) * 4;
    const int64_t p = m0 + arow;
    const bool prow = p < P;
    int ay0 = 0, ax0 = 0;
    const float* xin = a.x;
    if (prow) {
        const int ox = (int)(p % a.OW);
        const int64_t t = p / a.OW;
        const int oy = (int)(t % a.OH);
        const int64_t img = t / a.OH;
        ay0 = oy * a.stride - a.ph;
        ax0 = ox * a.stride - a.pw;
        xin = a.x + img * a.H * (int64_t)a.W * a.cinp;
    }
    // this thread's B row and chunks: 4 x 16 B of hi (tid & 1 == 0) or lo
    const int brow = tid >> 2, bq0 = (tid & 3) * 2;

    auto gather = [&](int kc, Gather& g) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = kc * kBK + (aq0 + j) * 4;
            const int tap = k / a.cinp, ci = k - tap * a.cinp;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (prow && tap < taps) {
                const int ky = tap / a.kw, kx = tap - ky * a.kw;
                const int iy = ay0 + ky, ix = ax0 + kx;
                if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W)
                    v = __ldg(reinterpret_cast<const float4*>(xin + ((int64_t)iy * a.W + ix) * a.cinp + ci));
            }
            g.v[j] = v;
        }
    };
    auto store_a = [&](int st, const Gather& g) {
        uint8_t* hi = smem + st * kStage;
        uint8_t* lo = hi + kATile;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float4 h, l;
            incep::tf32_split(g.v[j].x, h.x, l.x);
            incep::tf32_split(g.v[j].y, h.y, l.y);
            incep::tf32_split(g.v[j].z, h.z, l.z);
            incep::tf32_split(g.v[j].w, h.w, l.w);
            const uint32_t off = sw_off(arow, aq0 + j);
            *reinterpret_cast<float4*>(hi + off) = h;
            *reinterpret_cast<float4*>(lo + off) = l;
        }
    };
    auto load_b = [&](int st, int kc) {
        const uint32_t base = smem_u32(smem + st * kStage + 2 * kATile);
        const int64_t row = (int64_t)(n0 + brow) * a.KP + kc * kBK;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int q = bq0 + j;
            cp_async16(base + sw_off(brow, q), a.bhi + row + q * 4);
            cp_async16(base + kBTile + sw_off(brow, q), a.blo + row + q * 4);
        }
    };

    float acc[32], cor[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { acc[i] = 0.f; cor[i] = 0.f; }

    {
        Gather g;
        gather(0, g);
        load_b(0, 0);
        store_a(0, g);
    }
    for (int kc = 0; kc < nk; ++kc) {
        const int st = kc & 1;
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
        const uint32_t s0 = smem_u32(smem + st * kStage);
        const uint32_t ahi = s0 + wg * (kATile / 2), alo = ahi + kATile;
        const uint32_t bhi = s0 + 2 * kATile, blo = bhi + kBTile;
        fence_acc(acc);
        fence_acc(cor);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < kBK / 8; ++ks) {
            const uint32_t o = ks * 32;
            mma_tf32(acc, desc_sw128(ahi + o), desc_sw128(bhi + o), 1);
            mma_tf32(cor, desc_sw128(ahi + o), desc_sw128(blo + o), 1);
            mma_tf32(cor, desc_sw128(alo + o), desc_sw128(bhi + o), 1);
        }
        wg_commit();
        if (kc + 1 < nk) {   // the other stage was last read by chunk kc - 1, whose wgmma completed before the barrier
            Gather g;
            gather(kc + 1, g);
            load_b(st ^ 1, kc + 1);
            store_a(st ^ 1, g);
        }
        wg_wait0();
        fence_acc(acc);
        fence_acc(cor);
    }

    // epilogue: accumulator fragment of m64n64: d[4j + 2h + e] = (row 16*warp + lane/4 + 8h, col 8j + 2*(lane%4) + e)
    const int warp = (tid >> 5) & 3, lane = tid & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t pr = m0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * h;
        if (pr >= P) continue;
        float* yrow = a.y + pr * a.ct + a.c0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int co = n0 + 8 * j + 2 * (lane & 3) + e;
                if (co < a.cout) {
                    const int i = 4 * j + 2 * h + e;
                    yrow[co] = fmaxf(acc[i] + cor[i] + a.bias[co], 0.f);
                }
            }
        }
    }
}

}  // namespace

cudaError_t launch_incep_conv(const IncepConvArgs& a, cudaStream_t s) {
    // per device; cheap next to the launch
    const cudaError_t e = cudaFuncSetAttribute(incep_conv_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return e;
    const int64_t P = (int64_t)a.n * a.OH * a.OW;
    const dim3 grid((unsigned)((P + kBM - 1) / kBM), (unsigned)(a.NP / kBN));
    incep_conv_tf32_kernel<<<grid, kThreads, kSmem, s>>>(a);
    return cudaGetLastError();
}

}  // namespace migan

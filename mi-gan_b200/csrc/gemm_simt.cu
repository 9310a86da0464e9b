// fp32 CUDA-core GEMM for the 1x1 pointwise conv (SeparableConv2d.conv2,
// lib/model_zoo/migan_inference.py:161) with the fused "+noise -> lrelu_agc" epilogue
// (:165-169).  This is the bring-up / cross-check path (MIGAN_B200_PATH=simt): exact fp32
// FMA arithmetic, no tensor cores.  The production path is sepconv_tc.cu (wgmma).
//
//   out[p][n] = epi( sum_k A[p][k] * Bt[k][n] )      A [P][K] row-major (NHWC pixels x Cin)
//                                                    Bt [K][N] (conv2.weight transposed)
// Tile 128 x 64 x 16, 256 threads, 8 x 4 outputs per thread, register double buffering.
#include "common.cuh"
#include "kernels.h"

namespace migan {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4;

__global__ void __launch_bounds__(256)
pw_gemm_simt_kernel(const float* __restrict__ A, const float* __restrict__ Bt, float* __restrict__ out,
                    int64_t P, int K, int N, const float* __restrict__ noise, int HW, int W, int noise_pitch, int act) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN];
    const int tid = threadIdx.x;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int ty = tid / (BN / TN);  // 0..15 -> rows ty*8 .. +7
    const int tx = tid % (BN / TN);  // 0..15 -> cols tx*4 .. +3

    // A tile loader: 128 rows x 16 k = 512 float4, 2 per thread
    const int a_row = tid >> 2;      // 0..63 (+64)
    const int a_kq = (tid & 3) * 4;  // k offset 0,4,8,12
    // B tile loader: 16 k x 64 n = 256 float4, 1 per thread
    const int b_k = tid >> 4;        // 0..15
    const int b_n = (tid & 15) * 4;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = a_row + h * 64;
            const int64_t p = m0 + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < P) v = ldg4(A + p * K + k0 + a_kq);
            As[a_kq + 0][r] = v.x; As[a_kq + 1][r] = v.y; As[a_kq + 2][r] = v.z; As[a_kq + 3][r] = v.w;
        }
        *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = ldg4(Bt + (int64_t)(k0 + b_k) * N + n0 + b_n);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * TM]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * TM + 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * TN]);
            const float a[TM] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bb[TN] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t p = m0 + ty * TM + i;
        if (p >= P) continue;
        float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        if (noise) {
            const int q = (int)(p % HW);               // pixel of the image; the plane's rows are noise_pitch apart
            const float nz = __ldg(noise + q + (q / W) * (noise_pitch - W));
            v.x += nz; v.y += nz; v.z += nz; v.w += nz;
        }
        if (act) v = lrelu_agc4(v);
        stg4(out + p * N + n0 + tx * TN, v);
    }
}

cudaError_t launch_pw_gemm_simt(const float* A, const float* Bt, float* out, int64_t P, int K, int N,
                                const float* noise, int H, int W, int noise_pitch, int act, cudaStream_t s) {
    if (K % BK != 0 || N % BN != 0) return cudaErrorInvalidValue;
    dim3 grid((unsigned)((P + BM - 1) / BM), N / BN);
    pw_gemm_simt_kernel<<<grid, 256, 0, s>>>(A, Bt, out, P, K, N, noise, H * W, W, noise_pitch, act);
    return cudaGetLastError();
}

}  // namespace migan

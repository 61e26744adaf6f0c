// pd_gemm_simt.cu — plain fp32 CUDA-core tile GEMM with the same contract as the tensor-core kernel.
// It exists as the validation arm for tests (PD_GEMM_SIMT): every composite test can be run with
// either implementation, which separates "is the tensor-core pipeline right" from "is the model
// math right".  Not used by the product path (pd_create selects PD_GEMM_TC).
#include "pd_common.cuh"
#include <cuda_fp16.h>

namespace {
constexpr int TM = 64, TN = 64, TK = 16;

__global__ void __launch_bounds__(256)
pd_gemm_simt_kernel(int M, int N, int K, const float* __restrict__ A, long sAm, long sAk,
                    const float* __restrict__ B, long sBn, long sBk, PdEpilogue e, int kchunk) {
    __shared__ float As[TK][TM + 1];
    __shared__ float Bs[TK][TN + 1];
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int kbeg = blockIdx.z * kchunk;
    const int kend = min(K, kbeg + kchunk);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int k0 = kbeg; k0 < kend; k0 += TK) {
        for (int i = threadIdx.x; i < TM * TK; i += 256) {
            int mm, kk;
            if (sAk == 1) { kk = i % TK; mm = i / TK; } else { mm = i % TM; kk = i / TM; }
            int m = m0 + mm, k = k0 + kk;
            As[kk][mm] = (m < M && k < kend) ? A[(long)m * sAm + (long)k * sAk] : 0.f;
        }
        for (int i = threadIdx.x; i < TN * TK; i += 256) {
            int nn, kk;
            if (sBk == 1) { kk = i % TK; nn = i / TK; } else { nn = i % TN; kk = i / TN; }
            int n = n0 + nn, k = k0 + kk;
            Bs[kk][nn] = (n < N && k < kend) ? B[(long)n * sBn + (long)k * sBk] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < TK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int row = m0 + ty * 4 + i;
        if (row >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int col = n0 + tx * 4 + j;
            if (col >= N) continue;
            if (e.c_f16) {                                  // fp16 output matrix (ldc in halfs)
                reinterpret_cast<__half*>(e.C)[(long)row * e.ldc + col] = __float2half_rn(pd_epi_value(e, row, col, acc[i][j]));
                continue;
            }
            float* c = e.C + (long)row * e.ldc + col;
            if (e.accumulate) atomicAdd(c, acc[i][j]);
            else *c = pd_epi_value(e, row, col, acc[i][j]);
        }
    }
}

// y[m, n] = sum_k A[m, k] * B[n, k]  for N <= 4 (scalar heads): one warp per row, HBM-bound on A.
__global__ void __launch_bounds__(256)
gemv_rows_kernel(int M, int N, int K, const float* __restrict__ A, long lda, const float* __restrict__ B, long ldb,
                 PdEpilogue e) {
    const int lane = threadIdx.x & 31;
    const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= M) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float* a = A + row * lda;
    for (int k = lane; k < K; k += 32) {
        const float av = a[k];
#pragma unroll
        for (int n = 0; n < 4; ++n) if (n < N) acc[n] = fmaf(av, __ldg(B + (long)n * ldb + k), acc[n]);
    }
#pragma unroll
    for (int n = 0; n < 4; ++n) {
        if (n < N) {
            float v = pd_warp_sum(acc[n]);
            if (lane == 0) e.C[row * e.ldc + n] = pd_epi_value(e, (int)row, n, v);
        }
    }
}

// C[m, n] += sum_k A[k, m] * B[k, n]  for M <= 4 (weight gradient of a scalar head): blockDim (32, 8), a warp owns
// 32 consecutive n; rows k are strided over blockIdx.y, whose partials the last block of the column group adds in order.
__global__ void wcolsum_kernel(int M, int N, long K, const float* __restrict__ A, long lda, const float* __restrict__ B,
                               long ldb, float* C, long ldc, float* ws, unsigned* tickets) {
    const int n = blockIdx.x * 32 + threadIdx.x;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (n < N) {
        for (long k = (long)blockIdx.y * blockDim.y + threadIdx.y; k < K; k += (long)gridDim.y * blockDim.y) {
            const float bv = B[k * ldb + n];
#pragma unroll
            for (int m = 0; m < 4; ++m) if (m < M) acc[m] = fmaf(__ldg(A + k * lda + m), bv, acc[m]);
        }
    }
    __shared__ float sh[4][8][33];
#pragma unroll
    for (int m = 0; m < 4; ++m) sh[m][threadIdx.y][threadIdx.x] = acc[m];
    __syncthreads();
    float* part = ws + (long)blockIdx.x * gridDim.y * 128 + threadIdx.x;      // [y][m][32]
    if (threadIdx.y == 0) {
        for (int m = 0; m < M; ++m) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += sh[m][i][threadIdx.x];
            part[blockIdx.y * 128 + m * 32] = s;
        }
    }
    if (pd_last_block(tickets + blockIdx.x, gridDim.y) && threadIdx.y == 0 && n < N) {
        for (int m = 0; m < M; ++m) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.y; ++b) s += __ldcg(part + b * 128 + m * 32);
            C[(long)m * ldc + n] += s;
        }
    }
}
}  // namespace

int pd_gemm_simt_launch(pd_handle* h, int M, int N, int K, const float* A, long lda, int a_mn, const float* B,
                        long ldb, int b_mn, const PdEpilogue& epi, cudaStream_t stream) {
    if (h->gemm_impl != PD_GEMM_SIMT) {      // shape-specialised paths of the product (the validation arm stays generic)
        if (!epi.accumulate && !epi.c_f16 && N <= 4 && !a_mn && !b_mn) {
            gemv_rows_kernel<<<pd_cdiv(M, 8), 256, 0, stream>>>(M, N, K, A, lda, B, ldb, epi);
            PD_CHECK_LAUNCH(h, "gemv_rows_kernel");
            return PD_OK;
        }
        if (epi.accumulate && M <= 4 && a_mn && b_mn) {
            long gy = (K + 63) / 64;
            long cap = (long)h->num_sms * 8 / ((N + 31) / 32);
            if (cap < 1) cap = 1;
            if (gy > cap) gy = cap;
            float* ws;
            unsigned* tk;
            const int gx = (N + 31) / 32;
            int rc = pd_scratch(h, stream, (long)gx * gy * 128, gx, &ws, &tk);
            if (rc) return rc;
            wcolsum_kernel<<<dim3(gx, (unsigned)gy), dim3(32, 8), 0, stream>>>(M, N, K, A, lda, B, ldb, epi.C, epi.ldc, ws, tk);
            PD_CHECK_LAUNCH(h, "wcolsum_kernel");
            return PD_OK;
        }
    }
    long sAm = a_mn ? 1 : lda, sAk = a_mn ? lda : 1;
    long sBn = b_mn ? 1 : ldb, sBk = b_mn ? ldb : 1;
    // one block per output tile over the whole of K: an accumulating launch adds each element once (no split-K, whose
    // atomic partial sums would land in arrival order)
    int gx = pd_cdiv(N, TN), gy = pd_cdiv(M, TM);
    int kchunk = pd_cdiv(K, TK) * TK;
    dim3 grid(gx, gy, 1);
    pd_gemm_simt_kernel<<<grid, 256, 0, stream>>>(M, N, K, A, sAm, sAk, B, sBn, sBk, epi, kchunk);
    PD_CHECK_LAUNCH(h, "pd_gemm_simt_kernel");
    return PD_OK;
}

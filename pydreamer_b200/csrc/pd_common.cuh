// pydreamer_b200 — shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>

#include "../../include/pd_b200.h"

// ---------------------------------------------------------------------------
// Deterministic cross-block reductions.  A kernel that sums per-block partials into a gradient writes them to a scratch
// area and the LAST block to finish adds them up in block order (atomicAdd would sum in arrival order, so two runs of the
// same step would differ in the last bits and a training run would drift).  Kernels on one stream run one after the
// other, so each stream the handle sees gets its own scratch area (allocated with the handle; a CUDA graph keeps the
// capture streams' areas).
// ---------------------------------------------------------------------------
constexpr int PD_SCRATCH_SLOTS = 8;             // distinct streams per handle
constexpr long PD_SCRATCH_FLOATS = 4L << 20;    // partials per stream (16 MB)
constexpr int PD_SCRATCH_TICKETS = 4096;        // reduction groups per launch
struct PdScratch {
    cudaStream_t stream;
    int used;
    float* ws;
    unsigned* tickets;          // all zero between launches: the last block of a group resets its ticket
};

// ---------------------------------------------------------------------------
// Handle: host-side state plus the reduction scratch areas
// ---------------------------------------------------------------------------
struct pd_handle {
    int device;
    int num_sms;
    int gemm_impl;            // PD_GEMM_TC / PD_GEMM_SIMT
    int max_smem_optin;
    long launches;            // kernels launched through this handle
    char err[512];
    void* encode_tiled;       // cuTensorMapEncodeTiled entry point
    void* encode_im2col;      // cuTensorMapEncodeIm2col entry point (lazy)
    int gemm_smem_configured;
    int skinny_smem_configured;   // pd_gemm_skinny_kernel's shared-memory opt-in done
    int round_ops;            // round tensor-core operands to tf32 (rna) where they are produced
    int k1_configured;        // persistent RSSM kernels: shared-memory opt-in done on THIS handle's device
    int k1_ctas;              // ... and the co-resident grid they launch (one CTA per SM)
    int k1b_configured;
    int k1b_ctas;
    PdScratch scratch[PD_SCRATCH_SLOTS];
};

// The scratch area of `stream` (PD_OK), or an error when the handle has seen more streams than it has areas or the
// launch needs more than one area holds.
int pd_scratch(pd_handle* h, cudaStream_t stream, long nfloats, int ngroups, float** ws, unsigned** tickets);

// 2-D tensor map of a row-major matrix (dim0 = the contiguous dimension, rows ld_elems apart), 128-byte swizzle, zero
// fill out of bounds (pd_gemm_sm90.cu).
int make_map(pd_handle* h, CUtensorMap* tm, const void* base, uint64_t dim0, uint64_t dim1, uint64_t ld_elems,
             uint32_t box0, uint32_t box1, int elt_bytes = 4);
// K splits of a storing dense GEMM of M x N outputs and kb_total 32-k blocks (pd_gemm_sm90.cu); pd_gemm_tf32_kernel and
// pd_gemm_skinny_kernel both split at these k-blocks.
int pd_gemm_store_splits(const pd_handle* h, int M, int N, int kb_total);

// Launch wrappers run on the handle's device whatever the caller's current device is (and put it back).
struct PdDeviceGuard {
    int prev;
    bool switched;
    explicit PdDeviceGuard(const pd_handle* h) : prev(-1), switched(false) {
        if (h && cudaGetDevice(&prev) == cudaSuccess && prev != h->device) {
            cudaSetDevice(h->device);
            switched = true;
        }
    }
    ~PdDeviceGuard() {
        if (switched) cudaSetDevice(prev);
    }
};

#define PD_FAIL(h, code, ...)                                        \
    do {                                                             \
        if (h) snprintf((h)->err, sizeof((h)->err), __VA_ARGS__);    \
        return (code);                                               \
    } while (0)

#define PD_CHECK_LAUNCH(h, name)                                                  \
    do {                                                                          \
        cudaError_t e__ = cudaGetLastError();                                     \
        if (e__ != cudaSuccess)                                                   \
            PD_FAIL(h, PD_ERR_LAUNCH, "%s: %s", name, cudaGetErrorString(e__));   \
        (h)->launches++;                                                          \
    } while (0)

#define PD_REQUIRE(h, cond, ...)                                     \
    do {                                                             \
        if (!(cond)) PD_FAIL(h, PD_ERR_ARG, __VA_ARGS__);            \
    } while (0)

static inline int pd_cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------------------
// Device math helpers
// ---------------------------------------------------------------------------
// Round-to-nearest(-away) to TF32 precision (10 explicit mantissa bits).  Producers of
// tensor-core operands apply this so the hardware's operand truncation is exact
// (no systematic shrink of every product) — see DESIGN.md "precision".
__device__ __forceinline__ float pd_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float pd_round_if(float x, int on) { return on ? pd_tf32(x) : x; }

// ELU(alpha = 1).  exp(x) - 1 for x <= 0 without libm's expm1f (~45 instructions with branches — the GEMM epilogues that fuse
// the activation were bound by it, r02 ncu of the conv1 GEMM): a degree-7 Taylor polynomial where exp(x) - 1 would cancel
// (|x| < 0.25, truncation error < 4e-10) and ex2.approx elsewhere (result magnitude >= 0.22, relative error < 5e-7).
__device__ __forceinline__ float pd_selp(float a, float b, bool p) {   // p ? a : b as ONE select: the compiler otherwise turns
    float r;                                                            // the two-sided expressions below into a branch per element
    asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\tselp.f32 %0, %1, %2, q;\n\t}" : "=f"(r) : "f"(a), "f"(b), "r"((int)p));
    return r;
}
__device__ __forceinline__ float pd_expm1_nonpos(float x) {
    float p = fmaf(x, 1.f / 5040.f, 1.f / 720.f);
    p = fmaf(p, x, 1.f / 120.f);
    p = fmaf(p, x, 1.f / 24.f);
    p = fmaf(p, x, 1.f / 6.f);
    p = fmaf(p, x, 0.5f);
    p = fmaf(p, x, 1.f);
    p *= x;
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 1.4426950408889634f));
    return pd_selp(p, e - 1.f, x > -0.25f);
}
// both sides are evaluated on min(x, 0) and selected (r02 ncu of the conv1 GEMM: one BSSY / BSYNC region per element)
__device__ __forceinline__ float pd_elu(float x) { return pd_selp(x, pd_expm1_nonpos(fminf(x, 0.f)), x > 0.f); }
// d ELU / dx expressed through the ELU *output* y (alpha = 1): x>0 -> 1, else exp(x) = y + 1
__device__ __forceinline__ float pd_elu_grad_from_out(float y) { return y > 0.f ? 1.f : y + 1.f; }
__device__ __forceinline__ float pd_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float pd_softplus(float x) {
    // torch.nn.functional.softplus(beta=1, threshold=20)
    return x > 20.f ? x : log1pf(expf(x));
}

// Called by every thread of every block of a reduction group of n blocks after the block wrote its partials: true in the
// last block to arrive, which then sees all partials (read them with __ldcg) and resets the group's ticket.
__device__ __forceinline__ bool pd_last_block(unsigned* ticket, unsigned n) {
    __shared__ unsigned s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
        s_last = atomicAdd(ticket, 1u) == n - 1;
        if (s_last) atomicExch(ticket, 0u);
    }
    __syncthreads();
    if (s_last) __threadfence();
    return s_last;
}

__device__ __forceinline__ float pd_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float pd_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum for blockDim.x <= 1024 (result valid in all threads).
__device__ __forceinline__ float pd_block_sum(float v, float* sh /* >= 33 floats */) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = pd_warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[w] = v;
    __syncthreads();
    float r = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
    if (w == 0) {
        r = pd_warp_sum(r);
        if (lane == 0) sh[32] = r;
    }
    __syncthreads();
    return sh[32];
}

// ---------------------------------------------------------------------------
// GEMM epilogue shared by the tensor-core and the SIMT kernels
// ---------------------------------------------------------------------------
struct PdEpilogue {
    float* C;
    long ldc;
    const float* bias;   // [N] or nullptr
    const float* R;      // residual, row (m / r_div), or nullptr
    long ldr;
    int r_div;
    int act;             // PD_ACT_NONE / PD_ACT_ELU
    int round_out;       // round result to tf32 precision
    int accumulate;      // 0: C = v ; 1: C += v (one addition per element and launch, no bias/act)
    int c_f16;           // C is an fp16 matrix (ldc in halfs): the epilogue converts and stores rows with vector stores
    // backward through the ELU that FOLLOWED the layer whose input gradient this GEMM produces (pd_gemm_actbwd):
    // v *= elu'(dact[m, n]) (dact = that layer's saved output); the bias gradient is a column sum of C afterwards
    const float* dact;
    long lddact;
};

__device__ __forceinline__ float pd_epi_value(const PdEpilogue& e, int row, int col, float acc) {
    float v = acc;
    if (e.bias) v += __ldg(e.bias + col);
    if (e.R) v += __ldg(e.R + (long)(row / e.r_div) * e.ldr + col);
    if (e.act == PD_ACT_ELU) v = pd_elu(v);
    if (e.round_out) v = pd_tf32(v);
    return v;
}

// pd_gemm_sm90.cu — persistent, warp-specialised TF32 / fp16 GEMM for sm_90a.
//
//   C[M,N] (=|+=) sum_k A(m,k) * B(n,k) (+bias)(+residual) -> act
//
// Pipeline (one CTA per SM, 416 threads):
//   warp 8      : TMA producer  — cp.async.bulk.tensor tiles (SWIZZLE_128B) into a 5-stage shared-memory ring guarded by
//                                 full / empty mbarriers
//   warps 9..12 : transposers   — only with an MN-major operand: rewrite each landed MN-major tile in place into the
//                                 K-major layout, then arrive on the stage's ready mbarrier
//   warps 0..7  : consumers     — two warpgroups of wgmma.m64n128k8 (tf32) / m64n128k16 (fp16), a warp owns 16 rows x 128
//                                 columns of the 128 x 128 output tile, fp32 accumulators in registers, one wgmma group in
//                                 flight; then the epilogue straight from the registers: bias / residual / ELU /
//                                 ELU-backward / tf32 rounding -> four 128B-swizzled 32 x 16 smem boxes -> TMA store (or
//                                 TMA reduce-add for accumulate)
// Work units are (tile, k-split); the producer runs ahead into the next unit while the consumers drain the last.  A tile
// split over K (few output tiles, long K: weight gradients, one-timestep layers) writes each split's partial tile to a
// scratch area; the last split of the tile to finish adds the partials in split order and runs the epilogue, so the
// result does not depend on scheduling.
//
// Operand layouts: both operands may be K-major ([rows][K], K contiguous) or MN-major ([K][rows]); the second form lets the
// backward contractions dX = dY*W and dW = dY^T*X read the forward tensors in place (no transposes in HBM).  Every shared
// tile is made of 128-byte rows with the 16-byte chunk c of row r stored at c ^ (r & 7) (TMA SWIZZLE_128B):
//   K-major : row = m (or n), 32 fp32 / 64 fp16 k per row; read by wgmma through a shared-memory descriptor
//   MN-major: row = k, 32 m per row, groups of 32 m 4096 B apart; as it lands from TMA, before the transposers turn each
//             4 KB group into the K-major rows of its 32 m (wgmma reads tf32 operands only K-major)
// The implicit-GEMM convolution operands (TMA im2col mode on an NHWC tensor) land in the same two layouts.
#include "pd_common.cuh"
#include <cuda_fp16.h>
#include <stdlib.h>

namespace {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 32;                          // fp32 elements per k-block = 128 B = one swizzle row
constexpr int STAGES = 5;
constexpr int A_BYTES = BM * BK * 4;            // 16 KB
constexpr int B_BYTES = BN * BK * 4;            // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int GSTR = 4096;                      // bytes between the 32-wide MN groups of an MN-major tile
constexpr int CONS_WARPS = 8;
constexpr int TR_WARPS = BM / 32;              // transposer warps: one per 4 KB MN group of a tile
constexpr int NUM_THREADS = 32 * (CONS_WARPS + 1 + TR_WARPS);
constexpr int NJ = BN / 8;                      // n8 blocks of a consumer warp's 16 x 128 slice
constexpr int EPI_ROWS = 16;                    // rows of the epilogue's TMA store boxes: one consumer warp's slice
constexpr int EPI_STAGING = CONS_WARPS * 2 * 4096;   // per consumer warp: four 32 x 16 fp32 swizzled TMA-store boxes
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + EPI_STAGING;
static_assert(SMEM_BYTES <= 227 * 1024, "H100 allows 227 KB of shared memory per block");

struct GemmArgs {
    int M, N, K;
    int a_mn, b_mn;
    int num_m, num_n, kb_total, splits, kb_per_split;
    float* part;               // splits > 1: [tile][split][BM * BN] partial tiles
    unsigned* tickets;         // splits > 1: [tile] splits finished
    // MN-major tiled operands: one 3-D box {32 columns, 32 k-rows, 4 column groups} (16 KB) instead of four 2-D boxes of
    // 4 KB.  a3_on / b3_on: the 3-D map is valid; a3_part / b3_part: index of the one partial column group (MN % 32 != 0;
    // tiles holding it keep the 2-D boxes), or -1.
    int a3_on, b3_on, a3_part, b3_part;
    // implicit-GEMM convolution operands (TMA im2col mode on an NHWC tensor, k x k taps, stride 2, no padding):
    //   a_mode 1: A rows = output pixels, K = (tap, channel)            (conv forward / deconv input-gradient)
    //   a_mode 2: A' rows = (tap, channel padded to 32), K = output pixels  (deconv weight gradient)
    //   b_mode 2: B' rows = (tap, channel padded to 32), K = output pixels  (conv weight gradient)
    int a_mode, b_mode;
    int cv_PQ, cv_Q, cv_C, cv_k, cv_cblocks, cv_cpad;
    int f16;                   // operands are fp16 (64 elements per 128-byte k-block) instead of tf32
    int tma_store;             // C is TMA-addressable: epilogue uses cp.async.bulk.tensor store / reduce
    PdEpilogue epi;
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    uint32_t spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (done) break;
        if (++spins > (1u << 24)) __trap();   // watchdog: a broken pipeline must not hang the GPU
    }
}
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* smem, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* tmap, uint64_t* bar, void* smem, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// MN-major tile whose first column group is gi: may it be fetched as one 3-D box (no partial column group inside)?
__device__ __forceinline__ bool mn3_ok(int on, int part, int gi) { return on && !(part >= gi && part < gi + 4); }
__device__ __forceinline__ void tma_load_im2col(const void* tmap, uint64_t* bar, void* smem, int c, int w, int h, int n,
                                                int off_w, int off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(smem_u32(smem)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n),
          "h"((uint16_t)off_w), "h"((uint16_t)off_h)
        : "memory");
}
// byte offset of 16-byte chunk c of row r in a 128B-swizzled tile
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// In-place transpose of one 4 KB block of an MN-major tile (32 k-rows of 32 mn) into the K-major layout the wgmma
// descriptors read (32 mn-rows of 32 k).  Both layouts are 128B-swizzled and hold the same 32 x 32 elements in the same
// 4 KB, so one warp transposes a block on its own.  Lane (q, p) = (lane >> 3, lane & 7) moves the two 4 x 4 sub-blocks
// (mn chunk p, k chunk a = p ^ d), d = 2q and 2q + 1: four 16-byte loads of k-rows 4a .. 4a+3 at chunk p, a transpose in
// registers, four 16-byte stores of mn-rows 4p .. 4p+3 at chunk a.  The 8 lanes of a quarter-warp (one phase of a
// 16-byte access) reach 8 different chunk columns on both sides, so neither side has a bank conflict: load r lands in
// column p ^ r ^ 4 ((p ^ d) & 1), store i in column p ^ d ^ i ^ 4 (p & 1), each a permutation of p.
__device__ __forceinline__ void transpose_block(uint32_t base, int lane) {
    const int q = lane >> 3, p = lane & 7;
    uint32_t v[2][4][4];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int a = p ^ (2 * q + s);
#pragma unroll
        for (int r = 0; r < 4; ++r)
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(v[s][r][0]), "=r"(v[s][r][1]), "=r"(v[s][r][2]), "=r"(v[s][r][3])
                         : "r"(base + swz(4 * a + r, p)) : "memory");
    }
    __syncwarp();
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int a = p ^ (2 * q + s);
#pragma unroll
        for (int i = 0; i < 4; ++i)
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                         ::"r"(base + swz(4 * p + i, a)), "r"(v[s][0][i]), "r"(v[s][1][i]), "r"(v[s][2][i]), "r"(v[s][3][i])
                         : "memory");
    }
}

// wgmma shared-memory descriptor of a K-major SWIZZLE_128B tile: start >> 4, LBO (unused when swizzled) = 1, SBO = 1024 B
// between 8-row groups, layout 1 = 128-byte swizzle.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// The 64 accumulators of a warpgroup's m64n128 slice as read-write asm operands %0 .. %63.  Every asm statement from the
// first wgmma of a tile to the last wait names all of them, so the compiler never moves or reads them while the tensor
// cores own them.
#define PD_ACC4(j) "+f"(acc[j][0]), "+f"(acc[j][1]), "+f"(acc[j][2]), "+f"(acc[j][3])
#define PD_ACC64 PD_ACC4(0), PD_ACC4(1), PD_ACC4(2), PD_ACC4(3), PD_ACC4(4), PD_ACC4(5), PD_ACC4(6), PD_ACC4(7), \
                 PD_ACC4(8), PD_ACC4(9), PD_ACC4(10), PD_ACC4(11), PD_ACC4(12), PD_ACC4(13), PD_ACC4(14), PD_ACC4(15)
#define PD_D64 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28," \
               "%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54," \
               "%55,%56,%57,%58,%59,%60,%61,%62,%63}"

// Issues one 128-byte k-block of the warpgroup's 64 x 128 slice (rows 64 wgi .. of the A tile, all 128 rows of the B
// tile), both tiles K-major, as one wgmma group: four wgmma.m64n128k8 (tf32) / m64n128k16 (fp16), each 32 bytes further
// along the swizzled rows.  Thread (warp w of the group, lane) holds per n8 block j the same four elements as an mma.sync
// m16n8 C fragment of rows 16 w ..
__device__ __forceinline__ void wg_issue(const uint8_t* sa, const uint8_t* sb, int f16, int wgi, float (&acc)[16][4]) {
    const uint64_t a0 = wg_desc(smem_u32(sa) + wgi * 64 * 128), b0 = wg_desc(smem_u32(sb));
    if (f16) {
        asm volatile(
            "{\n\t"
            "wgmma.fence.sync.aligned;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PD_D64 ", %64, %68, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PD_D64 ", %65, %69, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PD_D64 ", %66, %70, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PD_D64 ", %67, %71, 1, 1, 1, 0, 0;\n\t"
            "wgmma.commit_group.sync.aligned;\n\t"
            "}"
            : PD_ACC64
            : "l"(a0), "l"(a0 + 2), "l"(a0 + 4), "l"(a0 + 6), "l"(b0), "l"(b0 + 2), "l"(b0 + 4), "l"(b0 + 6)
            : "memory");
    } else {
        asm volatile(
            "{\n\t"
            "wgmma.fence.sync.aligned;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " PD_D64 ", %64, %68, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " PD_D64 ", %65, %69, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " PD_D64 ", %66, %70, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " PD_D64 ", %67, %71, 1, 1, 1;\n\t"
            "wgmma.commit_group.sync.aligned;\n\t"
            "}"
            : PD_ACC64
            : "l"(a0), "l"(a0 + 2), "l"(a0 + 4), "l"(a0 + 6), "l"(b0), "l"(b0 + 2), "l"(b0 + 4), "l"(b0 + 6)
            : "memory");
    }
}
// Waits until at most N of the warpgroup's wgmma groups are pending.
template <int N>
__device__ __forceinline__ void wg_wait(float (&acc)[16][4]) {
    asm volatile("wgmma.wait_group.sync.aligned %64;" : PD_ACC64 : "n"(N) : "memory");
}
#undef PD_ACC4
#undef PD_ACC64
#undef PD_D64

// The epilogue of a thread's accumulators, acc[j][x] at row r0 + 8 (x >> 1), column c0 + 8 j + (x & 1): bias and residual
// unless C accumulates, then, when `finish` (the value is stored, or reduced by TMA), ELU, ELU backward and tf32 rounding.
// Elements outside C are computed but never stored.  The bias, residual and ELU-backward loads of CH n8 blocks are all
// issued before the first is used, so that their latencies overlap: one load at a time, each waited for by its use, made
// the epilogue take longer than the k-loop.  The residual's row offsets (a division) are computed once per tile.  The
// arithmetic per element is unchanged, so the results are the same bits.
template <int CH, int NJT>
__device__ __forceinline__ void epi_apply(const PdEpilogue& e, float (&acc)[NJT][4], int r0, int c0, int M, int N, bool finish) {
    const bool add = !e.accumulate;
    const bool in_r[2] = {r0 < M, r0 + 8 < M};
    const float* rrow[2];
    const float* drow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        rrow[h] = (add && e.R && in_r[h]) ? e.R + (long)((r0 + 8 * h) / e.r_div) * e.ldr : nullptr;
        drow[h] = (finish && e.dact && in_r[h]) ? e.dact + (long)(r0 + 8 * h) * e.lddact : nullptr;
    }
    const float* bias = add ? e.bias : nullptr;
#pragma unroll
    for (int j0 = 0; j0 < NJT; j0 += CH) {
        float bv[CH][2], rv[CH][4], dv[CH][4];
#pragma unroll
        for (int j = 0; j < CH; ++j)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
                const int col = c0 + 8 * (j0 + j) + x;
                bv[j][x] = (bias && col < N) ? __ldg(bias + col) : 0.f;
            }
#pragma unroll
        for (int j = 0; j < CH; ++j)
#pragma unroll
            for (int x = 0; x < 4; ++x) {
                const int col = c0 + 8 * (j0 + j) + (x & 1);
                const bool in = in_r[x >> 1] && col < N;
                rv[j][x] = (add && e.R && in) ? __ldg(rrow[x >> 1] + col) : 0.f;
                dv[j][x] = (finish && e.dact && in) ? __ldg(drow[x >> 1] + col) : 0.f;
            }
#pragma unroll
        for (int j = 0; j < CH; ++j)
#pragma unroll
            for (int x = 0; x < 4; ++x) {
                const bool in = in_r[x >> 1] && c0 + 8 * (j0 + j) + (x & 1) < N;
                float v = acc[j0 + j][x];
                if (add && in) {
                    if (e.bias) v += bv[j][x & 1];
                    if (e.R) v += rv[j][x];
                }
                if (finish) {
                    if (e.act == PD_ACT_ELU) v = pd_elu(v);
                    if (e.dact && in) v *= pd_elu_grad_from_out(dv[j][x]);
                    if (e.round_out) v = pd_tf32(v);
                }
                acc[j0 + j][x] = v;
            }
    }
}

// 8 consumer warps: two warpgroups of wgmma, a warp owns 16 rows x 128 columns of the output tile.  Warp 8: TMA producer.
// Warps 9 .. 12: with an MN-major operand, transpose each landed stage to K-major (warp 9 + j takes the 4 KB block j of
// every MN-major tile) and release it to the consumers through ready[]; otherwise they exit at once.
__global__ void __launch_bounds__(NUM_THREADS, 1)
pd_gemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmA3,
                    const __grid_constant__ CUtensorMap tmB3, const GemmArgs g) {
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full = (uint64_t*)(smem + STAGES * STAGE_BYTES + EPI_STAGING);   // [STAGES] TMA landed
    uint64_t* empty = full + STAGES;                                            // [STAGES] consumers done
    uint64_t* ready = empty + STAGES;                                           // [STAGES] transposed to K-major

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const bool tr = g.a_mn || g.b_mn;

    if (warp == CONS_WARPS && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmB) : "memory");
        if (g.a3_on) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmA3) : "memory");
        if (g.b3_on) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmB3) : "memory");
        if (g.tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmC) : "memory");
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1); mbar_init(&empty[i], CONS_WARPS); mbar_init(&ready[i], TR_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int units = g.num_m * g.num_n * g.splits;

    if (warp == CONS_WARPS) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int u = blockIdx.x; u < units; u += gridDim.x) {
                const int tile = u / g.splits, split = u % g.splits;
                const int m0 = (tile / g.num_n) * BM;
                const int n0 = (tile % g.num_n) * BN;
                const int kb1 = min(g.kb_total, (split + 1) * g.kb_per_split);
                for (int kb = split * g.kb_per_split; kb < kb1; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * STAGE_BYTES;
                    uint8_t* sb = sa + A_BYTES;
                    mbar_expect_tx(&full[stage], STAGE_BYTES);
                    int k0 = kb * (g.f16 ? 2 * BK : BK);
                    if (g.a_mode == 1) {
                        // implicit im2col rows: k-block = 32 channels of one filter tap; pixel tile starts at m0
                        const int tap = kb / g.cv_cblocks, c0 = (kb - tap * g.cv_cblocks) * 32;
                        const int kh = tap / g.cv_k, kw = tap - kh * g.cv_k;
                        const int n_ = m0 / g.cv_PQ, r_ = m0 - n_ * g.cv_PQ;
                        const int p_ = r_ / g.cv_Q, q_ = r_ - p_ * g.cv_Q;
                        tma_load_im2col(&tmA, &full[stage], sa, c0, 2 * q_, 2 * p_, n_, kw, kh);   // 128 pixels x 32 ch
                        k0 = tap * g.cv_C + c0;                       // matching rows of the (tap, channel)-major weight
                    }
                    if (g.a_mode == 2 || g.b_mode == 2) {
                        // K = output pixels: k-block = 32 consecutive pixels starting at kb*32
                        const int pix = kb * BK;
                        const int n_ = pix / g.cv_PQ, r_ = pix - n_ * g.cv_PQ;
                        const int p_ = r_ / g.cv_Q, q_ = r_ - p_ * g.cv_Q;
                        const void* tm = g.a_mode == 2 ? (const void*)&tmA : (const void*)&tmB;
                        uint8_t* dst = g.a_mode == 2 ? sa : sb;
                        const int base = g.a_mode == 2 ? m0 : n0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {                 // 4 boxes of 32 (tap, channel) rows x 32 pixels
                            const int idx = base + 32 * j;
                            int tap = idx / g.cv_cpad, c0 = idx - tap * g.cv_cpad;
                            if (tap >= g.cv_k * g.cv_k) { tap = 0; c0 = g.cv_cpad + 32; }        // past the last tap: all-OOB -> zeros
                            const int kh = tap / g.cv_k, kw = tap - kh * g.cv_k;
                            tma_load_im2col(tm, &full[stage], dst + j * GSTR, c0, 2 * q_, 2 * p_, n_, kw, kh);
                        }
                    }
                    if (g.a_mode == 0) {
                        if (!g.a_mn) {
                            tma_load_2d(&tmA, &full[stage], sa, k0, m0);              // box {32 k, 128 m}
                        } else if (mn3_ok(g.a3_on, g.a3_part, m0 >> 5)) {
                            tma_load_3d(&tmA3, &full[stage], sa, 0, k0, m0 >> 5);     // box {32 m, 32 k, 4 groups}
                        } else {
#pragma unroll
                            for (int j = 0; j < BM / 32; ++j)                        // box {32 m, 32 k} x 4
                                tma_load_2d(&tmA, &full[stage], sa + j * GSTR, m0 + j * 32, k0);
                        }
                    }
                    if (g.b_mode == 0) {
                        if (!g.b_mn) {
                            tma_load_2d(&tmB, &full[stage], sb, k0, n0);
                        } else if (mn3_ok(g.b3_on, g.b3_part, n0 >> 5)) {
                            tma_load_3d(&tmB3, &full[stage], sb, 0, k0, n0 >> 5);
                        } else {
#pragma unroll
                            for (int j = 0; j < BN / 32; ++j)
                                tma_load_2d(&tmB, &full[stage], sb + j * GSTR, n0 + j * 32, k0);
                        }
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    if (warp > CONS_WARPS) {
        // ===================== transposers: MN-major tiles -> K-major, in place =====================
        if (!tr) return;
        const int blk = (warp - CONS_WARPS - 1) * 4096;
        int stage = 0; uint32_t phase = 0;
        for (int u = blockIdx.x; u < units; u += gridDim.x) {
            const int split = u % g.splits;
            const int kb1 = min(g.kb_total, (split + 1) * g.kb_per_split);
            for (int kb = split * g.kb_per_split; kb < kb1; ++kb) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
                if (g.a_mn) transpose_block(sa + blk, lane);
                if (g.b_mn) transpose_block(sa + A_BYTES + blk, lane);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stores, before wgmma reads them
                __syncwarp();
                if (lane == 0) mbar_arrive(&ready[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===================== consumers: wgmma + epilogue =====================
    const int g8 = lane >> 2, t4 = lane & 3;
    const int wm = (warp >> 2) * 64 + (warp & 3) * 16;                // this warp's 16 rows of the 128 x 128 tile
    const PdEpilogue& e = g.epi;
    uint8_t* stg = smem + STAGES * STAGE_BYTES + warp * 2 * 4096;     // NJ / 4 fp32 boxes {32, 16} (or NJ / 8 fp16 {64, 16})
    int stage = 0; uint32_t phase = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int tile = u / g.splits, split = u % g.splits;
        const int m0 = (tile / g.num_n) * BM;
        const int n0 = (tile % g.num_n) * BN;
        const int kb1 = min(g.kb_total, (split + 1) * g.kb_per_split);
        float acc[NJ][4];
#pragma unroll
        for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
            for (int x = 0; x < 4; ++x) acc[nj][x] = 0.f;
        // One wgmma group in flight: k-block kb is issued before kb - 1 is waited for, and kb - 1's stage is freed then.
        int prev = -1;
        for (int kb = split * g.kb_per_split; kb < kb1; ++kb) {
            mbar_wait(&full[stage], phase);
            if (tr) mbar_wait(&ready[stage], phase);                 // the MN-major tiles are K-major now
            const uint8_t* sa = smem + stage * STAGE_BYTES;
            wg_issue(sa, sa + A_BYTES, g.f16, warp >> 2, acc);
            wg_wait<1>(acc);
            if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wg_wait<0>(acc);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }

        // Fragment element x of nj: row wm + g8 + 8*(x>>1), column nj*8 + 2*t4 + (x&1).
        if (g.splits > 1) {
            // ---- split-K: partial tile to scratch; the last split of the tile sums all partials in split order
            float* tp = g.part + (long)tile * g.splits * (BM * BN);
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int off = (wm + g8 + 8 * h) * BN + nj * 8 + 2 * t4;
                    *reinterpret_cast<float2*>(tp + (long)split * (BM * BN) + off) = make_float2(acc[nj][2 * h], acc[nj][2 * h + 1]);
                }
            __threadfence();
            asm volatile("bar.sync 1, %0;" ::"n"(32 * CONS_WARPS) : "memory");      // consumer warps only
            __shared__ unsigned s_last;
            if (threadIdx.x == 0) {
                s_last = atomicAdd(g.tickets + tile, 1u) == (unsigned)(g.splits - 1);
                if (s_last) atomicExch(g.tickets + tile, 0u);
            }
            asm volatile("bar.sync 1, %0;" ::"n"(32 * CONS_WARPS) : "memory");
            if (!s_last) continue;
            __threadfence();
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int off = (wm + g8 + 8 * h) * BN + nj * 8 + 2 * t4;
                    float2 sum = make_float2(0.f, 0.f);
                    for (int sp = 0; sp < g.splits; ++sp) {
                        const float2 v = __ldcg(reinterpret_cast<const float2*>(tp + (long)sp * (BM * BN) + off));
                        sum.x += v.x; sum.y += v.y;
                    }
                    acc[nj][2 * h] = sum.x; acc[nj][2 * h + 1] = sum.y;
                }
        }
        // ---- epilogue
        const int rbase = m0 + wm, cbase = n0;
        if (rbase >= g.M || cbase >= g.N) continue;                  // warp-uniform: nothing of this slice is real
        // two n8 blocks per batch of loads: four spill at this kernel's 128 registers and measured slower
        epi_apply<2>(e, acc, rbase + g8, cbase + 2 * t4, g.M, g.N, g.tma_store || !e.accumulate);
        if (!g.tma_store) {
            // generic path (C not TMA-addressable: ldc % 4 != 0, e.g. N = 1 / 18 outputs)
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    const int row = rbase + g8 + 8 * (x >> 1), col = cbase + nj * 8 + 2 * t4 + (x & 1);
                    if (row < g.M && col < g.N) {
                        float* cp = e.C + (long)row * e.ldc + col;
                        if (e.accumulate) atomicAdd(cp, acc[nj][x]);
                        else *cp = acc[nj][x];
                    }
                }
            continue;
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // staging boxes free again
        __syncwarp();
        const uint32_t sbase = smem_u32(stg);
        if (e.c_f16) {
            // NJ / 8 boxes {64 halfs, 16 rows}: 128-byte rows, 16-byte chunk = 8 columns
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = g8 + 8 * h;
                    const __half2 v2 = __floats2half2_rn(acc[nj][2 * h], acc[nj][2 * h + 1]);
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + (nj >> 3) * (EPI_ROWS * 128) + swz(r, nj & 7) + t4 * 4),
                                 "r"(*reinterpret_cast<const uint32_t*>(&v2))
                                 : "memory");
                }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                for (int b = 0; b < NJ / 8 && cbase + 64 * b < g.N; ++b)
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (EPI_ROWS * 128)), "r"(cbase + 64 * b), "r"(rbase) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            continue;
        }
        // NJ / 4 boxes {32 fp32, 16 rows}: box b holds columns 32b .. 32b+31 of the slice
#pragma unroll
        for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = g8 + 8 * h, lc = (nj & 3) * 8 + 2 * t4;
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};"
                             ::"r"(sbase + (nj >> 2) * (EPI_ROWS * 128) + swz(r, lc >> 2) + (lc & 3) * 4), "f"(acc[nj][2 * h]),
                               "f"(acc[nj][2 * h + 1])
                             : "memory");
            }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        const int nbox = min(NJ / 4, (g.N - cbase + 31) / 32);
        if (lane == 0) {
            for (int b = 0; b < nbox; ++b) {
                if (e.accumulate)
                    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (EPI_ROWS * 128)), "r"(cbase + 32 * b), "r"(rbase) : "memory");
                else
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (EPI_ROWS * 128)), "r"(cbase + 32 * b), "r"(rbase) : "memory");
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");    // all stores/reductions landed
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

int make_map(pd_handle* h, CUtensorMap* tm, const void* base, uint64_t dim0, uint64_t dim1, uint64_t ld_elems,
             uint32_t box0, uint32_t box1, int elt_bytes) {
    cuuint64_t gdim[2] = {dim0, dim1};
    cuuint64_t gstride[1] = {ld_elems * (uint64_t)elt_bytes};
    cuuint32_t box[2] = {box0, box1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = ((EncodeTiledFn)h->encode_tiled)(tm, elt_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstride,
                                                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) PD_FAIL(h, PD_ERR_ARG, "cuTensorMapEncodeTiled failed (%d): dims %llu x %llu ld %llu", (int)r,
                                   (unsigned long long)dim0, (unsigned long long)dim1, (unsigned long long)ld_elems);
    return PD_OK;
}

namespace {

// 3-D view of an MN-major fp32 operand [K rows][MN columns, ld]: (32 columns of a group, k, column group) with strides
// (ld * 4 B, 128 B), box {32, 32, 4} — in shared memory the same bytes as four 2-D {32, 32} boxes 4096 B apart.  Only the
// MN / 32 FULL column groups are addressable (a partial last group would read past the row); *on = 0 if there is none.
int make_map3(pd_handle* h, CUtensorMap* tm, const void* base, uint64_t mn, uint64_t k, uint64_t ld_elems, int* on, int* part) {
    const uint64_t groups = mn / 32;
    *part = (mn % 32) ? (int)groups : -1;
    *on = 0;
    if (groups == 0) return PD_OK;
    cuuint64_t gdim[3] = {32, k, groups};
    cuuint64_t gstride[2] = {ld_elems * 4, 128};
    cuuint32_t box[3] = {32, (cuuint32_t)BK, 4};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = ((EncodeTiledFn)h->encode_tiled)(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)base, gdim, gstride, box, estr,
                                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) PD_FAIL(h, PD_ERR_ARG, "cuTensorMapEncodeTiled(3-D MN-major) failed (%d): mn %llu k %llu ld %llu", (int)r,
                                   (unsigned long long)mn, (unsigned long long)k, (unsigned long long)ld_elems);
    *on = 1;
    return PD_OK;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// TMA im2col-mode map over an NHWC fp32 tensor (k x k taps, stride 2, no padding): lower corner 0, upper corner -(k-1).
int make_im2col_map(pd_handle* h, CUtensorMap* tm, const float* base, int NB, int H, int W, int C, int k, int pixels) {
    if (!h->encode_im2col) {
        cudaDriverEntryPointQueryResult q;
        void* p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
            PD_FAIL(h, PD_ERR_DEVICE, "cuTensorMapEncodeIm2col entry point not found");
        h->encode_im2col = p;
    }
    cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)NB};
    cuuint64_t gstr[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
    int lo[2] = {0, 0}, up[2] = {-(k - 1), -(k - 1)};
    cuuint32_t estr[4] = {1, 2, 2, 1};
    CUresult r = ((EncodeIm2colFn)h->encode_im2col)(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, gdim, gstr, lo, up, 32,
                                                   (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) PD_FAIL(h, PD_ERR_ARG, "cuTensorMapEncodeIm2col failed (%d): %dx%dx%dx%d k=%d", (int)r, NB, H, W, C, k);
    return PD_OK;
}

int configure(pd_handle* h) {
    if (h->gemm_smem_configured) return PD_OK;
    cudaError_t e = cudaFuncSetAttribute(pd_gemm_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) PD_FAIL(h, PD_ERR_DEVICE, "cudaFuncSetAttribute(smem=%d): %s", SMEM_BYTES, cudaGetErrorString(e));
    h->gemm_smem_configured = 1;
    return PD_OK;
}

// Split-K factor: the one that minimises waves x (k-blocks per unit + per-unit epilogue), waves = ceil(tiles * splits /
// slots) — 96 tiles on 132 SMs leave a quarter of the chip idle unsplit, 3 splits give 288 units = 2.2 waves of a third of
// the work each — among those whose partial tiles fit the scratch area.  1 for problems with enough tiles.
int pick_splits(int tiles, int kb_total, int slots, int min_kb) {
    int maxs = kb_total / min_kb;
    const int fit = (int)(PD_SCRATCH_FLOATS / (BM * BN)) / tiles;
    if (maxs > fit) maxs = fit;
    if (tiles > PD_SCRATCH_TICKETS || maxs < 2) return 1;
    const double epi_kb = 6.0;                 // a unit's drain (partial tile out, sums in) in k-block times
    int best = 1;
    double best_cost = 1e300;
    for (int sp = 1; sp <= maxs; ++sp) {
        const int kbs = pd_cdiv(kb_total, sp);
        if (pd_cdiv(kb_total, kbs) != sp) continue;            // no empty units
        const long waves = ((long)tiles * sp + slots - 1) / slots;
        const double cost = (double)waves * ((double)kbs + epi_kb);
        if (cost < best_cost - 1e-9) { best_cost = cost; best = sp; }
    }
    return best;
}

}  // namespace

// Splits of a storing (not accumulating) dense launch: skinny-M layers (the per-timestep RSSM GEMMs, M = B*I = 50: too few
// output tiles to pull their weights through more than a handful of SMs) split K over the idle SMs.  pd_gemm_skinny_kernel
// splits its K at the same k-blocks, so both kernels add the same partial sums in the same order.
int pd_gemm_store_splits(const pd_handle* h, int M, int N, int kb_total) {
    const int num_m = pd_cdiv(M, BM), tiles = num_m * pd_cdiv(N, BN);
    const bool skinny = num_m == 1 && tiles * 2 <= h->num_sms && kb_total >= 8;
    return skinny ? pick_splits(tiles, kb_total, h->num_sms, 4) : 1;
}

namespace {

int launch(pd_handle* h, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmA3,
           const CUtensorMap& tmB3, GemmArgs& g, int splits, cudaStream_t stream, const char* name) {
    const int tiles = g.num_m * g.num_n;
    g.kb_per_split = pd_cdiv(g.kb_total, splits);
    g.splits = pd_cdiv(g.kb_total, g.kb_per_split);
    if (g.splits > 1) {
        int rc = pd_scratch(h, stream, (long)tiles * g.splits * (BM * BN), tiles, &g.part, &g.tickets);
        if (rc) return rc;
    }
    const int units = tiles * g.splits;
    const int grid = units < h->num_sms ? units : h->num_sms;
    pd_gemm_tf32_kernel<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tmA, tmB, tmC, tmA3, tmB3, g);
    PD_CHECK_LAUNCH(h, name);
    return PD_OK;
}

}  // namespace

// Implicit-GEMM convolution launcher.  mode 1: C[pixels, N] = im2col(X) * B   (B: [N][K] or, b_mn, [K][N]; K = (tap, c))
//                                      mode 2: C[(tap,cpad), N] += im2col(X)^T * Bt   (Bt stored [pixels][N])
//                                      mode 3: C[M, (tap,cpad)] += At^T * im2col(X)   (At stored [pixels][M])
int pd_conv_gemm_launch(pd_handle* h, int mode, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo,
                        int o_mn, int ODIM, const PdEpilogue& epi, cudaStream_t stream) {
    PD_REQUIRE(h, (C % 4) == 0 && ((((uintptr_t)X) & 15) == 0), "pd_conv_gemm: C %% 4 and 16-byte alignment required");
    PD_REQUIRE(h, (ldo % 4) == 0 && ((((uintptr_t)O) & 15) == 0), "pd_conv_gemm: operand alignment");
    PD_REQUIRE(h, (epi.ldc % 4) == 0 && ((((uintptr_t)epi.C) & 15) == 0), "pd_conv_gemm: C must be TMA-addressable");
    int rc = configure(h);
    if (rc) return rc;
    const int P = (H - k) / 2 + 1, Q = (W - k) / 2 + 1;
    const long pixels = (long)NB * P * Q;
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.cv_PQ = P * Q; g.cv_Q = Q; g.cv_C = C; g.cv_k = k; g.cv_cblocks = pd_cdiv(C, 32); g.cv_cpad = g.cv_cblocks * 32;
    g.epi = epi; g.tma_store = 1;
    CUtensorMap tmA, tmB, tmC, tmA3, tmB3;
    memset(&tmA3, 0, sizeof(tmA3)); memset(&tmB3, 0, sizeof(tmB3));
    g.a3_part = g.b3_part = -1;
    int M, N;
    if (mode == 1) {
        M = (int)pixels; N = ODIM;
        g.a_mode = 1; g.a_mn = 0; g.b_mode = 0; g.b_mn = o_mn;
        g.kb_total = k * k * g.cv_cblocks;
        rc = make_im2col_map(h, &tmA, X, NB, H, W, C, k, BM); if (rc) return rc;
        const long Ktot = (long)k * k * C;
        if (!o_mn) rc = make_map(h, &tmB, O, (uint64_t)Ktot, (uint64_t)N, (uint64_t)ldo, BK, BN);
        else       rc = make_map(h, &tmB, O, (uint64_t)N, (uint64_t)Ktot, (uint64_t)ldo, 32, BK);
        if (rc) return rc;
        if (o_mn) { rc = make_map3(h, &tmB3, O, (uint64_t)N, (uint64_t)Ktot, (uint64_t)ldo, &g.b3_on, &g.b3_part); if (rc) return rc; }
    } else if (mode == 2) {
        M = k * k * g.cv_cpad; N = ODIM;
        g.a_mode = 2; g.a_mn = 1; g.b_mode = 0; g.b_mn = 1;
        g.kb_total = pd_cdiv(pixels, BK);
        rc = make_im2col_map(h, &tmA, X, NB, H, W, C, k, BK); if (rc) return rc;
        rc = make_map(h, &tmB, O, (uint64_t)N, (uint64_t)pixels, (uint64_t)ldo, 32, BK); if (rc) return rc;
        rc = make_map3(h, &tmB3, O, (uint64_t)N, (uint64_t)pixels, (uint64_t)ldo, &g.b3_on, &g.b3_part); if (rc) return rc;
    } else {
        M = ODIM; N = k * k * g.cv_cpad;
        g.a_mode = 0; g.a_mn = 1; g.b_mode = 2; g.b_mn = 1;
        g.kb_total = pd_cdiv(pixels, BK);
        rc = make_map(h, &tmA, O, (uint64_t)M, (uint64_t)pixels, (uint64_t)ldo, 32, BK); if (rc) return rc;
        rc = make_map3(h, &tmA3, O, (uint64_t)M, (uint64_t)pixels, (uint64_t)ldo, &g.a3_on, &g.a3_part); if (rc) return rc;
        rc = make_im2col_map(h, &tmB, X, NB, H, W, C, k, BK); if (rc) return rc;
    }
    rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 32, EPI_ROWS);
    if (rc) return rc;
    g.M = M; g.N = N; g.K = 0;
    g.num_m = pd_cdiv(M, BM); g.num_n = pd_cdiv(N, BN);
    const int splits = epi.accumulate ? pick_splits(g.num_m * g.num_n, g.kb_total, h->num_sms, 8) : 1;
    return launch(h, tmA, tmB, tmC, tmA3, tmB3, g, splits, stream, "pd_gemm_tf32_kernel(im2col)");
}

int pd_gemm_tc_launch(pd_handle* h, int M, int N, int K, const void* A, long lda, int a_mn, const void* B,
                      long ldb, int b_mn, const PdEpilogue& epi, cudaStream_t stream, int f16) {
    PD_REQUIRE(h, !f16 || (!a_mn && !b_mn && (lda % 8) == 0 && (ldb % 8) == 0), "pd_gemm_f16: K-major operands with ld %% 8 == 0 only");
    PD_REQUIRE(h, (lda % 4) == 0 && (ldb % 4) == 0, "pd_gemm(tensor core): lda/ldb must be multiples of 4 (got %ld, %ld)",
               lda, ldb);
    PD_REQUIRE(h, (((uintptr_t)A) & 15) == 0 && (((uintptr_t)B) & 15) == 0, "pd_gemm(tensor core): A/B must be 16B aligned");
    int rc = configure(h);
    if (rc) return rc;
    CUtensorMap tmA, tmB, tmC, tmA3, tmB3;
    memset(&tmA3, 0, sizeof(tmA3)); memset(&tmB3, 0, sizeof(tmB3));
    if (f16)        rc = make_map(h, &tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 2 * BK, BM, 2);
    else if (!a_mn) rc = make_map(h, &tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
    else            rc = make_map(h, &tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 32, BK);
    if (rc) return rc;
    if (f16)        rc = make_map(h, &tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 2 * BK, BN, 2);
    else if (!b_mn) rc = make_map(h, &tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, BN);
    else            rc = make_map(h, &tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 32, BK);
    if (rc) return rc;

    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.M = M; g.N = N; g.K = K; g.a_mn = a_mn; g.b_mn = b_mn;
    g.num_m = pd_cdiv(M, BM); g.num_n = pd_cdiv(N, BN);
    g.f16 = f16;
    g.kb_total = pd_cdiv(K, f16 ? 2 * BK : BK);
    g.epi = epi;
    g.a3_part = g.b3_part = -1;
    if (!f16 && a_mn) { rc = make_map3(h, &tmA3, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, &g.a3_on, &g.a3_part); if (rc) return rc; }
    if (!f16 && b_mn) { rc = make_map3(h, &tmB3, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, &g.b3_on, &g.b3_part); if (rc) return rc; }
    g.tma_store = ((epi.ldc % 4) == 0) && ((((uintptr_t)epi.C) & 15) == 0);
    if (epi.c_f16) {
        PD_REQUIRE(h, !epi.accumulate && !epi.R && !epi.round_out, "pd_gemm: an fp16 output takes bias / activation only");
        PD_REQUIRE(h, (epi.ldc % 8) == 0 && ((((uintptr_t)epi.C) & 15) == 0), "pd_gemm: fp16 output needs ldc %% 8 == 0 (16-byte rows)");
        g.tma_store = 1;
        rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 64, EPI_ROWS, 2);
        if (rc) return rc;
    } else if (g.tma_store) {
        rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 32, EPI_ROWS);
        if (rc) return rc;
    } else {
        tmC = tmA;
    }
    PD_REQUIRE(h, !epi.dact || (g.tma_store && !epi.c_f16 && !epi.accumulate), "pd_gemm(actbwd): needs a TMA-addressable fp32 C");
    // Weight gradients (accumulate) and skinny-M layers split K over the idle SMs.
    const int splits = epi.accumulate ? pick_splits(g.num_m * g.num_n, g.kb_total, h->num_sms, 8)
                                      : pd_gemm_store_splits(h, M, N, g.kb_total);
    return launch(h, tmA, tmB, tmC, tmA3, tmB3, g, splits, stream, "pd_gemm_tf32_kernel");
}

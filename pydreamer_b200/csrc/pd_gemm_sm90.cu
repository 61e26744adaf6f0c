// pd_gemm_sm90.cu — persistent, warp-specialised TF32 / fp16 GEMM for sm_90a.
//
//   C[M,N] (=|+=) sum_k A(m,k) * B(n,k) (+bias)(+residual) -> act
//
// Pipeline (one CTA per SM, 288 threads):
//   warp 8      : TMA producer  — cp.async.bulk.tensor tiles (SWIZZLE_128B) into a 5-stage shared-memory ring guarded by
//                                 full / empty mbarriers
//   warps 0..7  : consumers     — each owns a 32 x 64 sub-tile of the 128 x 128 output tile: mma.sync m16n8k8 (tf32) or
//                                 m16n8k16 (fp16) with fp32 accumulators in registers, then the epilogue straight from the
//                                 registers: bias / residual / ELU / ELU-backward / tf32 rounding -> two 128B-swizzled
//                                 32 x 32 smem boxes -> TMA store (or TMA reduce-add for accumulate)
// Work units are (tile, k-split); the producer runs ahead into the next unit while the consumers drain the last.  A tile
// split over K (few output tiles, long K: weight gradients, one-timestep layers) writes each split's partial tile to a
// scratch area; the last split of the tile to finish adds the partials in split order and runs the epilogue, so the
// result does not depend on scheduling.
//
// Operand layouts: both operands may be K-major ([rows][K], K contiguous) or MN-major ([K][rows]); the second form lets the
// backward contractions dX = dY*W and dW = dY^T*X read the forward tensors in place (no transposes in HBM).  Every shared
// tile is made of 128-byte rows with the 16-byte chunk c of row r stored at c ^ (r & 7) (TMA SWIZZLE_128B):
//   K-major : row = m (or n), 32 fp32 / 64 fp16 k per row; fragments by ldmatrix (conflict-free)
//   MN-major: row = k, 32 m per row, groups of 32 m 4096 B apart; fragments by scalar loads
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
constexpr int NUM_THREADS = 32 * CONS_WARPS + 32;
constexpr int EPI_STAGING = CONS_WARPS * 2 * 4096;   // per consumer warp: two 32x32 fp32 swizzled TMA-store boxes
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
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// byte offset of 16-byte chunk c of row r in a 128B-swizzled tile
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
// 32-bit element (mn, k) of an MN-major tile (k-rows of 32 mn, groups of 32 mn GSTR apart)
__device__ __forceinline__ uint32_t ld_mn(const uint8_t* t, int mn, int k) {
    return *reinterpret_cast<const uint32_t*>(t + (mn >> 5) * GSTR + swz(k, (mn & 31) >> 2) + (mn & 3) * 4);
}

// One 128-byte k-block of the warp's 32 x 64 sub-tile (rows wm .. wm+31 of the A tile, rows wn .. wn+63 of the B tile):
// four k-steps of 32 bytes, i.e. m16n8k8 tf32 or m16n8k16 fp16.  K-major fragments come from ldmatrix: viewed as b16 pairs, an
// 8 x 16-byte block of a K-major tile hands lane (g, t) its element (row g, 32-bit word t) — exactly the tf32 A / B fragment
// pattern, and for fp16 the standard one.
__device__ __forceinline__ void mma_kblock(const uint8_t* sa, const uint8_t* sb, int a_mn, int b_mn, int f16, int wm, int wn,
                                           float (&acc)[2][8][4]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, q = lane >> 3, l8 = lane & 7;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        uint32_t a[2][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
            if (!a_mn) {
                const int r = wm + mi * 16 + (q & 1) * 8 + l8;
                ldsm_x4(smem_u32(sa) + swz(r, 2 * s + (q >> 1)), a[mi]);
            } else {
                const int m = wm + mi * 16 + g, k = 8 * s + t;
                a[mi][0] = ld_mn(sa, m, k); a[mi][1] = ld_mn(sa, m + 8, k);
                a[mi][2] = ld_mn(sa, m, k + 4); a[mi][3] = ld_mn(sa, m + 8, k + 4);
            }
        }
#pragma unroll
        for (int nj = 0; nj < 8; nj += 2) {
            uint32_t b[4];                                     // b0, b1 of n8-tile nj, then of nj + 1
            if (!b_mn) {
                const int r = wn + (nj + (q >> 1)) * 8 + l8;
                ldsm_x4(smem_u32(sb) + swz(r, 2 * s + (q & 1)), b);
            } else {
                const int n = wn + nj * 8 + g, k = 8 * s + t;
                b[0] = ld_mn(sb, n, k); b[1] = ld_mn(sb, n, k + 4);
                b[2] = ld_mn(sb, n + 8, k); b[3] = ld_mn(sb, n + 8, k + 4);
            }
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                if (f16) { mma_f16(acc[mi][nj], a[mi], b[0], b[1]); mma_f16(acc[mi][nj + 1], a[mi], b[2], b[3]); }
                else     { mma_tf32(acc[mi][nj], a[mi], b[0], b[1]); mma_tf32(acc[mi][nj + 1], a[mi], b[2], b[3]); }
            }
        }
    }
}


// wgmma shared-memory descriptor of a K-major SWIZZLE_128B tile: start >> 4, LBO (unused when swizzled) = 1, SBO = 1024 B
// between 8-row groups, layout 1 = 128-byte swizzle.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// One 128-byte k-block of the warpgroup's 64 x 128 slice (rows 64 wgi .. of the A tile, all 128 rows of the B tile), both
// operands K-major: four wgmma.m64n128k8 (tf32) / m64n128k16 (fp16), each 32 bytes further along the swizzled rows.  One asm
// statement from fence to wait, so the compiler never touches the accumulators while the tensor cores own them.  Thread
// (warp w of the group, lane) holds per n8 block j the same four elements as an mma.sync m16n8 C fragment of rows 16 w ..
__device__ __forceinline__ void wg_kblock(const uint8_t* sa, const uint8_t* sb, int f16, int wgi, float (&acc)[1][16][4]) {
    const uint64_t a0 = wg_desc(smem_u32(sa) + wgi * 64 * 128), b0 = wg_desc(smem_u32(sb));
    if (f16) {
        asm volatile(
            "{\n\t"
            "wgmma.fence.sync.aligned;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %68, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %65, %69, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %66, %70, 1, 1, 1, 0, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %67, %71, 1, 1, 1, 0, 0;\n\t"
            "wgmma.commit_group.sync.aligned;\n\t"
            "wgmma.wait_group.sync.aligned 0;\n\t"
            "}"
            : "+f"(acc[0][0][0]), "+f"(acc[0][0][1]), "+f"(acc[0][0][2]), "+f"(acc[0][0][3]), "+f"(acc[0][1][0]), "+f"(acc[0][1][1]), "+f"(acc[0][1][2]), "+f"(acc[0][1][3]), "+f"(acc[0][2][0]), "+f"(acc[0][2][1]), "+f"(acc[0][2][2]), "+f"(acc[0][2][3]), "+f"(acc[0][3][0]), "+f"(acc[0][3][1]), "+f"(acc[0][3][2]), "+f"(acc[0][3][3]), "+f"(acc[0][4][0]), "+f"(acc[0][4][1]), "+f"(acc[0][4][2]), "+f"(acc[0][4][3]), "+f"(acc[0][5][0]), "+f"(acc[0][5][1]), "+f"(acc[0][5][2]), "+f"(acc[0][5][3]), "+f"(acc[0][6][0]), "+f"(acc[0][6][1]), "+f"(acc[0][6][2]), "+f"(acc[0][6][3]), "+f"(acc[0][7][0]), "+f"(acc[0][7][1]), "+f"(acc[0][7][2]), "+f"(acc[0][7][3]), "+f"(acc[0][8][0]), "+f"(acc[0][8][1]), "+f"(acc[0][8][2]), "+f"(acc[0][8][3]), "+f"(acc[0][9][0]), "+f"(acc[0][9][1]), "+f"(acc[0][9][2]), "+f"(acc[0][9][3]), "+f"(acc[0][10][0]), "+f"(acc[0][10][1]), "+f"(acc[0][10][2]), "+f"(acc[0][10][3]), "+f"(acc[0][11][0]), "+f"(acc[0][11][1]), "+f"(acc[0][11][2]), "+f"(acc[0][11][3]), "+f"(acc[0][12][0]), "+f"(acc[0][12][1]), "+f"(acc[0][12][2]), "+f"(acc[0][12][3]), "+f"(acc[0][13][0]), "+f"(acc[0][13][1]), "+f"(acc[0][13][2]), "+f"(acc[0][13][3]), "+f"(acc[0][14][0]), "+f"(acc[0][14][1]), "+f"(acc[0][14][2]), "+f"(acc[0][14][3]), "+f"(acc[0][15][0]), "+f"(acc[0][15][1]), "+f"(acc[0][15][2]), "+f"(acc[0][15][3])
            : "l"(a0), "l"(a0 + 2), "l"(a0 + 4), "l"(a0 + 6), "l"(b0), "l"(b0 + 2), "l"(b0 + 4), "l"(b0 + 6)
            : "memory");
    } else {
        asm volatile(
            "{\n\t"
            "wgmma.fence.sync.aligned;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %68, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %65, %69, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %66, %70, 1, 1, 1;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %67, %71, 1, 1, 1;\n\t"
            "wgmma.commit_group.sync.aligned;\n\t"
            "wgmma.wait_group.sync.aligned 0;\n\t"
            "}"
            : "+f"(acc[0][0][0]), "+f"(acc[0][0][1]), "+f"(acc[0][0][2]), "+f"(acc[0][0][3]), "+f"(acc[0][1][0]), "+f"(acc[0][1][1]), "+f"(acc[0][1][2]), "+f"(acc[0][1][3]), "+f"(acc[0][2][0]), "+f"(acc[0][2][1]), "+f"(acc[0][2][2]), "+f"(acc[0][2][3]), "+f"(acc[0][3][0]), "+f"(acc[0][3][1]), "+f"(acc[0][3][2]), "+f"(acc[0][3][3]), "+f"(acc[0][4][0]), "+f"(acc[0][4][1]), "+f"(acc[0][4][2]), "+f"(acc[0][4][3]), "+f"(acc[0][5][0]), "+f"(acc[0][5][1]), "+f"(acc[0][5][2]), "+f"(acc[0][5][3]), "+f"(acc[0][6][0]), "+f"(acc[0][6][1]), "+f"(acc[0][6][2]), "+f"(acc[0][6][3]), "+f"(acc[0][7][0]), "+f"(acc[0][7][1]), "+f"(acc[0][7][2]), "+f"(acc[0][7][3]), "+f"(acc[0][8][0]), "+f"(acc[0][8][1]), "+f"(acc[0][8][2]), "+f"(acc[0][8][3]), "+f"(acc[0][9][0]), "+f"(acc[0][9][1]), "+f"(acc[0][9][2]), "+f"(acc[0][9][3]), "+f"(acc[0][10][0]), "+f"(acc[0][10][1]), "+f"(acc[0][10][2]), "+f"(acc[0][10][3]), "+f"(acc[0][11][0]), "+f"(acc[0][11][1]), "+f"(acc[0][11][2]), "+f"(acc[0][11][3]), "+f"(acc[0][12][0]), "+f"(acc[0][12][1]), "+f"(acc[0][12][2]), "+f"(acc[0][12][3]), "+f"(acc[0][13][0]), "+f"(acc[0][13][1]), "+f"(acc[0][13][2]), "+f"(acc[0][13][3]), "+f"(acc[0][14][0]), "+f"(acc[0][14][1]), "+f"(acc[0][14][2]), "+f"(acc[0][14][3]), "+f"(acc[0][15][0]), "+f"(acc[0][15][1]), "+f"(acc[0][15][2]), "+f"(acc[0][15][3])
            : "l"(a0), "l"(a0 + 2), "l"(a0 + 4), "l"(a0 + 6), "l"(b0), "l"(b0 + 2), "l"(b0 + 4), "l"(b0 + 6)
            : "memory");
    }
}

// WG: both operands K-major (plain or im2col rows) — two warpgroups of wgmma, a warp owns 16 rows x 128 columns.
// Otherwise (an MN-major operand: wgmma reads tf32 only K-major) eight mma.sync warps of 32 rows x 64 columns.
template <bool WG>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pd_gemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmA3,
                    const __grid_constant__ CUtensorMap tmB3, const GemmArgs g) {
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full = (uint64_t*)(smem + STAGES * STAGE_BYTES + EPI_STAGING);   // [STAGES]
    uint64_t* empty = full + STAGES;                                            // [STAGES]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == CONS_WARPS && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmB) : "memory");
        if (g.a3_on) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmA3) : "memory");
        if (g.b3_on) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmB3) : "memory");
        if (g.tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmC) : "memory");
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONS_WARPS); }
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

    // ===================== consumers: MMA + epilogue =====================
    constexpr int MI = WG ? 1 : 2, NJ = WG ? 16 : 8;                // m16 x n8 fragments per warp
    constexpr int RB = 16 * MI;                                      // rows of the warp's slice = rows of its store boxes
    const int g8 = lane >> 2, t4 = lane & 3;
    const int wm = WG ? (warp >> 2) * 64 + (warp & 3) * 16 : (warp & 3) * 32;   // this warp's slice of the 128 x 128 tile
    const int wn = WG ? 0 : (warp >> 2) * 64;
    const PdEpilogue& e = g.epi;
    uint8_t* stg = smem + STAGES * STAGE_BYTES + warp * 2 * 4096;     // NJ / 4 fp32 boxes {32, RB} (or NJ / 8 fp16 {64, RB})
    int stage = 0; uint32_t phase = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int tile = u / g.splits, split = u % g.splits;
        const int m0 = (tile / g.num_n) * BM;
        const int n0 = (tile % g.num_n) * BN;
        const int kb1 = min(g.kb_total, (split + 1) * g.kb_per_split);
        float acc[MI][NJ][4];
#pragma unroll
        for (int mi = 0; mi < MI; ++mi)
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[mi][nj][x] = 0.f;
        for (int kb = split * g.kb_per_split; kb < kb1; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint8_t* sa = smem + stage * STAGE_BYTES;
            if constexpr (WG) wg_kblock(sa, sa + A_BYTES, g.f16, warp >> 2, acc);
            else              mma_kblock(sa, sa + A_BYTES, g.a_mn, g.b_mn, g.f16, wm, wn, acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }

        // Fragment element x of (mi, nj): row wm + mi*16 + g8 + 8*(x>>1), column wn + nj*8 + 2*t4 + (x&1).
        if (g.splits > 1) {
            // ---- split-K: partial tile to scratch; the last split of the tile sums all partials in split order
            float* tp = g.part + (long)tile * g.splits * (BM * BN);
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int off = (wm + mi * 16 + g8 + 8 * h) * BN + wn + nj * 8 + 2 * t4;
                        *reinterpret_cast<float2*>(tp + (long)split * (BM * BN) + off) = make_float2(acc[mi][nj][2 * h], acc[mi][nj][2 * h + 1]);
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
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int off = (wm + mi * 16 + g8 + 8 * h) * BN + wn + nj * 8 + 2 * t4;
                        float2 sum = make_float2(0.f, 0.f);
                        for (int sp = 0; sp < g.splits; ++sp) {
                            const float2 v = __ldcg(reinterpret_cast<const float2*>(tp + (long)sp * (BM * BN) + off));
                            sum.x += v.x; sum.y += v.y;
                        }
                        acc[mi][nj][2 * h] = sum.x; acc[mi][nj][2 * h + 1] = sum.y;
                    }
        }
        // ---- epilogue
        const int rbase = m0 + wm, cbase = n0 + wn;
        if (rbase >= g.M || cbase >= g.N) continue;                  // warp-uniform: nothing of this sub-tile is real
#pragma unroll
        for (int mi = 0; mi < MI; ++mi)
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    const int row = rbase + mi * 16 + g8 + 8 * (x >> 1), col = cbase + nj * 8 + 2 * t4 + (x & 1);
                    float v = acc[mi][nj][x];
                    const bool in = row < g.M && col < g.N;
                    if (!e.accumulate && in) {
                        if (e.bias) v += __ldg(e.bias + col);
                        if (e.R) v += __ldg(e.R + (long)(row / e.r_div) * e.ldr + col);
                    }
                    if (g.tma_store || !e.accumulate) {
                        if (e.act == PD_ACT_ELU) v = pd_elu(v);
                        if (e.dact && in) v *= pd_elu_grad_from_out(__ldg(e.dact + (long)row * e.lddact + col));
                        if (e.round_out) v = pd_tf32(v);
                    }
                    acc[mi][nj][x] = v;
                }
        if (!g.tma_store) {
            // generic path (C not TMA-addressable: ldc % 4 != 0, e.g. N = 1 / 18 outputs)
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                    for (int x = 0; x < 4; ++x) {
                        const int row = rbase + mi * 16 + g8 + 8 * (x >> 1), col = cbase + nj * 8 + 2 * t4 + (x & 1);
                        if (row < g.M && col < g.N) {
                            float* cp = e.C + (long)row * e.ldc + col;
                            if (e.accumulate) atomicAdd(cp, acc[mi][nj][x]);
                            else *cp = acc[mi][nj][x];
                        }
                    }
            continue;
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // staging boxes free again
        __syncwarp();
        const uint32_t sbase = smem_u32(stg);
        if (e.c_f16) {
            // NJ / 8 boxes {64 halfs, RB rows}: 128-byte rows, 16-byte chunk = 8 columns
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
                for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int r = mi * 16 + g8 + 8 * h;
                        const __half2 v2 = __floats2half2_rn(acc[mi][nj][2 * h], acc[mi][nj][2 * h + 1]);
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sbase + (nj >> 3) * (RB * 128) + swz(r, nj & 7) + t4 * 4),
                                     "r"(*reinterpret_cast<const uint32_t*>(&v2))
                                     : "memory");
                    }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                for (int b = 0; b < NJ / 8 && cbase + 64 * b < g.N; ++b)
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (RB * 128)), "r"(cbase + 64 * b), "r"(rbase) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            continue;
        }
        // NJ / 4 boxes {32 fp32, RB rows}: box b holds columns 32b .. 32b+31 of the slice
#pragma unroll
        for (int mi = 0; mi < MI; ++mi)
#pragma unroll
            for (int nj = 0; nj < NJ; ++nj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = mi * 16 + g8 + 8 * h, lc = (nj & 3) * 8 + 2 * t4;
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};"
                                 ::"r"(sbase + (nj >> 2) * (RB * 128) + swz(r, lc >> 2) + (lc & 3) * 4), "f"(acc[mi][nj][2 * h]),
                                   "f"(acc[mi][nj][2 * h + 1])
                                 : "memory");
                }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        const int nbox = min(NJ / 4, (g.N - cbase + 31) / 32);
        if (lane == 0) {
            for (int b = 0; b < nbox; ++b) {
                if (e.accumulate)
                    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (RB * 128)), "r"(cbase + 32 * b), "r"(rbase) : "memory");
                else
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"((uint64_t)&tmC), "r"(sbase + b * (RB * 128)), "r"(cbase + 32 * b), "r"(rbase) : "memory");
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");    // all stores/reductions landed
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D tensor map with 128-byte swizzle: dim0 = contiguous dimension.
int make_map(pd_handle* h, CUtensorMap* tm, const void* base, uint64_t dim0, uint64_t dim1, uint64_t ld_elems,
             uint32_t box0, uint32_t box1, int elt_bytes = 4) {
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

// wgmma reads tf32 operands only K-major: both operands K-major (plain, fp16 or im2col rows) take the wgmma instantiation.
bool wgmma_ok(const GemmArgs& g) { return !g.a_mn && !g.b_mn && g.a_mode != 2 && g.b_mode != 2; }
// rows of the epilogue's TMA store boxes: one warp's slice (16 rows under wgmma, 32 under mma.sync)
uint32_t store_rows(const GemmArgs& g) { return wgmma_ok(g) ? 16 : 32; }

int configure(pd_handle* h) {
    if (h->gemm_smem_configured) return PD_OK;
    cudaError_t e = cudaFuncSetAttribute(pd_gemm_tf32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(pd_gemm_tf32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
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
    if (wgmma_ok(g)) pd_gemm_tf32_kernel<true><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tmA, tmB, tmC, tmA3, tmB3, g);
    else             pd_gemm_tf32_kernel<false><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(tmA, tmB, tmC, tmA3, tmB3, g);
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
    rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 32, store_rows(g));
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
        rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 64, store_rows(g), 2);
        if (rc) return rc;
    } else if (g.tma_store) {
        rc = make_map(h, &tmC, epi.C, (uint64_t)N, (uint64_t)M, (uint64_t)epi.ldc, 32, store_rows(g));
        if (rc) return rc;
    } else {
        tmC = tmA;
    }
    PD_REQUIRE(h, !epi.dact || (g.tma_store && !epi.c_f16 && !epi.accumulate), "pd_gemm(actbwd): needs a TMA-addressable fp32 C");
    // Weight gradients (accumulate) and skinny-M layers (the per-timestep RSSM GEMMs, M = B*I = 50: too few output tiles to
    // pull their weights through more than a handful of SMs) split K over the idle SMs.
    const int tiles = g.num_m * g.num_n;
    const bool skinny = g.num_m == 1 && tiles * 2 <= h->num_sms && g.kb_total >= 8;
    const int splits = (epi.accumulate || skinny) ? pick_splits(tiles, g.kb_total, h->num_sms, epi.accumulate ? 8 : 4) : 1;
    return launch(h, tmA, tmB, tmC, tmA3, tmB3, g, splits, stream, "pd_gemm_tf32_kernel");
}

// pd_gemm_skinny.cu — weight-streaming TF32 GEMM for few rows and a weight stored as it is in the forward pass.
//
//   C[M <= 64, N] = sum_k A(m, k) * B[k][n]  (+bias)(+residual) -> act -> (tf32 rounding)
//
// The BPTT input gradients of the posterior unroll (dX[B*I, in] = dY[B*I, out] . W[out, in], one launch per weight and
// timestep) read a whole weight matrix for 50 rows of output: the time is the weight's trip from HBM, and the general kernel
// (pd_gemm_sm90.cu) spends it on 128-row tiles, in-place transposes and a partial-tile round trip through global memory.
// This kernel streams the weight in its stored [K][N] orientation instead, and computes the same bits as the general
// kernel: it splits K at the same k-blocks (pd_gemm_store_splits), accumulates each split over the same 8-k tensor-core
// steps in the same order, and adds the splits' partial sums in split order from 0, as that kernel's last CTA does.
//   * grid = (S, N / BN), BN = 32 NG columns (NG = 4 when 64-column slabs would need more CTAs than SMs, else 2), clusters
//     of S <= 8 CTAs along K.  Rank r takes `spc` (1 or 2) consecutive splits, so up to 16 splits fit one cluster.
//   * the last warp: TMA producer.  A stage is one 32-k block: the A box {32 k, 64 m} (rows past M are zero-filled, not
//     read) and NG weight boxes {32 n, 32 k}, all 128-byte swizzled, into a 6-stage ring guarded by full / empty mbarriers.
//   * warps 0 .. 2 NG - 1: mma.sync.m16n8k8 tf32, warp w owns the 32 columns of group w % NG and the rows 32 (w / NG) ..
//     + 31 (only the m16 blocks below M run), one accumulator set per split it takes.  The B fragment is read straight
//     from the [k][n] tile: the mma's n index g of n8 block j is column 16 (g >> 2) + (g & 3) + 4 j of the group, which
//     puts the 32 lanes of each fragment load (k rows t and t + 4, swizzled by t) on 32 different banks.  Operands are the
//     fp32 bits read as tf32, as in pd_gemm_sm90.cu.
//   * split-K without scratch: each CTA stores its splits' [64, BN] partial tiles in its own shared memory; after a
//     cluster barrier, rank r sums rows r, r + S, ... over splits 0 .. splits-1 in order through distributed shared memory
//     and stores them with the epilogue.  C is written outright (no pre-clear).
#include "pd_k1_pipe.cuh"

namespace {

using k1::mbar_arrive;
using k1::mbar_expect_tx;
using k1::mbar_init;
using k1::mbar_wait;
using k1::mma_tf32;
using k1::s_u32;
using k1::tma_box;

constexpr int BM = 64;                             // rows of the A box: M <= 64
constexpr int BK = 32;                             // k per stage: one 128-byte swizzle row of A (= the general kernel's k-block)
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * BK * 4;               // 8 KB
constexpr int G_BYTES = 32 * BK * 4;               // 4 KB: one {32 n, 32 k} weight box
constexpr int MAX_RANKS = 8;                       // portable cluster size
constexpr int MAX_SPC = 2;                         // splits per CTA
constexpr int MAX_SPLITS = MAX_RANKS * MAX_SPC;

template <int NG>
struct Cfg {
    static constexpr int BN = 32 * NG;
    static constexpr int STAGE_BYTES = A_BYTES + NG * G_BYTES;
    static constexpr int CONS_WARPS = 2 * NG;
    static constexpr int NUM_THREADS = 32 * (CONS_WARPS + 1);
    static constexpr int PLD = BN + 4;             // row stride (floats) of a partial tile
    static constexpr int PART = BM * PLD;          // floats per partial tile
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 2 * STAGES * 8;
    static_assert(MAX_SPC * PART * 4 <= STAGES * STAGE_BYTES, "the partial tiles reuse the stage ring");
};

struct SkinnyArgs {
    int M, N, kb_total, kb_per_split, splits, spc;
    PdEpilogue epi;
};

// byte offset of fp32 element (row r, column c) of a 128B-swizzled tile of 32-float rows
__device__ __forceinline__ uint32_t swz4(int r, int c) { return (uint32_t)(r * 128 + ((((c >> 2) ^ r) & 7) << 4) + (c & 3) * 4); }
__device__ __forceinline__ uint32_t lds(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

template <int NG>
__global__ void __launch_bounds__(Cfg<NG>::NUM_THREADS, 1)
pd_gemm_skinny_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const SkinnyArgs g) {
    using C_ = Cfg<NG>;
    constexpr int BN = C_::BN, CONS_WARPS = C_::CONS_WARPS, PLD = C_::PLD;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full = (uint64_t*)(smem + STAGES * C_::STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t rank;
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const int n0 = blockIdx.y * BN;
    const int s0 = rank * g.spc, s1 = min(g.splits, s0 + g.spc);            // this CTA's splits
    const int kb0 = s0 * g.kb_per_split, kb1 = min(g.kb_total, s1 * g.kb_per_split);

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&tmB) : "memory");
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int g8 = lane >> 2, t4 = lane & 3;
    const int cg = warp % NG, rh = warp / NG;
    float acc[MAX_SPC][2][4][4];
#pragma unroll
    for (int h = 0; h < MAX_SPC; ++h)
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[h][mb][j][x] = 0.f;

    if (warp == CONS_WARPS) {
        // ===================== TMA producer: the CTA's splits are one contiguous k range =====================
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * C_::STAGE_BYTES;
                mbar_expect_tx(&full[stage], C_::STAGE_BYTES);
                tma_box(&tmA, &full[stage], sa, kb * BK, 0);                                  // {32 k, 64 m}
#pragma unroll
                for (int j = 0; j < NG; ++j)
                    tma_box(&tmB, &full[stage], sa + A_BYTES + j * G_BYTES, n0 + 32 * j, kb * BK);   // {32 n, 32 k}
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        __syncwarp();
    } else {
        // ===================== consumers: one accumulator set per split =====================
        const bool on0 = 32 * rh < g.M, on1 = 32 * rh + 16 < g.M;     // m16 blocks of this warp holding real rows
        const int r0 = 32 * rh + g8;
        int stage = 0; uint32_t phase = 0;
#pragma unroll
        for (int h = 0; h < MAX_SPC; ++h) {
            if (s0 + h >= s1) break;
            const int ka = (s0 + h) * g.kb_per_split, kz = min(g.kb_total, ka + g.kb_per_split);
            for (int kb = ka; kb < kz; ++kb) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = s_u32(smem + stage * C_::STAGE_BYTES);
                const uint32_t sb = sa + A_BYTES + cg * G_BYTES;
                if (on0) {
#pragma unroll
                    for (int kk = 0; kk < BK / 8; ++kk) {
                        uint32_t b[4][2];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int col = 16 * (g8 >> 2) + (g8 & 3) + 4 * j;
                            b[j][0] = lds(sb + swz4(8 * kk + t4, col));
                            b[j][1] = lds(sb + swz4(8 * kk + t4 + 4, col));
                        }
#pragma unroll
                        for (int mb = 0; mb < 2; ++mb) {
                            if (mb == 1 && !on1) break;
                            const int r = r0 + 16 * mb;
                            const uint32_t a0 = lds(sa + swz4(r, 8 * kk + t4)), a1 = lds(sa + swz4(r + 8, 8 * kk + t4));
                            const uint32_t a2 = lds(sa + swz4(r, 8 * kk + t4 + 4)), a3 = lds(sa + swz4(r + 8, 8 * kk + t4 + 4));
#pragma unroll
                            for (int j = 0; j < 4; ++j) mma_tf32(acc[h][mb][j], a0, a1, a2, a3, b[j][0], b[j][1]);
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    }
    __syncthreads();                               // every stage consumed: the ring becomes the partial tiles

    float* part = (float*)smem;                    // [MAX_SPC][BM][PLD]
    if (warp < CONS_WARPS) {
        // fragment element x of n8 block j: row g8 + 8 (x >> 1), mma column 2 t4 + (x & 1) -> group column below
        const int c = 32 * cg + 16 * (t4 >> 1) + 2 * (t4 & 1);
#pragma unroll
        for (int h = 0; h < MAX_SPC; ++h) {
            if (s0 + h >= s1) break;
            float* ph = part + h * C_::PART;
#pragma unroll
            for (int mb = 0; mb < 2; ++mb) {
                const int r = 32 * rh + 16 * mb + g8;
                if (r - g8 >= g.M) break;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    *reinterpret_cast<float2*>(ph + r * PLD + c + 4 * j) = make_float2(acc[h][mb][j][0], acc[h][mb][j][1]);
                    *reinterpret_cast<float2*>(ph + (r + 8) * PLD + c + 4 * j) = make_float2(acc[h][mb][j][2], acc[h][mb][j][3]);
                }
            }
        }
    }
    cluster_sync();                                // all partial tiles of the cluster written

    // rank r: rows r, r + S, ..., 4 columns per thread; split s lives in rank s / spc, slot s % spc
    const int S = gridDim.x;                       // the cluster spans the grid's x dimension
    const int my_rows = (g.M - (int)rank + S - 1) / S;
    const uint32_t pbase = s_u32(part);
    for (int it = threadIdx.x; it < my_rows * (BN / 4); it += C_::NUM_THREADS) {
        const int row = (int)rank + S * (it / (BN / 4)), c4 = 4 * (it % (BN / 4));
        const uint32_t off = pbase + (uint32_t)(row * PLD + c4) * 4;
        float4 v[MAX_SPLITS];                      // all loads in flight before the first addition
#pragma unroll
        for (int s = 0; s < MAX_SPLITS; ++s) {
            if (s >= g.splits) break;
            uint32_t ra;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;"
                         : "=r"(ra) : "r"(off + (uint32_t)((s % g.spc) * C_::PART * 4)), "r"(s / g.spc));
            asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(v[s].x), "=f"(v[s].y), "=f"(v[s].z), "=f"(v[s].w) : "r"(ra) : "memory");
        }
        // the general kernel's order: one split as it is, several summed from 0 in split order
        float4 sum = g.splits > 1 ? make_float4(0.f, 0.f, 0.f, 0.f) : v[0];
#pragma unroll
        for (int s = 0; s < MAX_SPLITS; ++s) {
            if (s >= g.splits || g.splits == 1) break;
            sum.x += v[s].x; sum.y += v[s].y; sum.z += v[s].z; sum.w += v[s].w;
        }
        const float sv[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
        for (int x = 0; x < 4; ++x) {
            const int col = n0 + c4 + x;
            if (col < g.N) g.epi.C[(long)row * g.epi.ldc + col] = pd_epi_value(g.epi, row, col, sv[x]);
        }
    }
    cluster_sync();                                // no CTA leaves while another still reads its partial tiles
}

// K splits (normalised: none empty) of the general kernel for this shape, and the k-blocks per split.
int skinny_splits(const pd_handle* h, int M, int N, int K, int* kb_per_split) {
    const int kb_total = pd_cdiv(K, BK);
    *kb_per_split = pd_cdiv(kb_total, pd_gemm_store_splits(h, M, N, kb_total));
    return pd_cdiv(kb_total, *kb_per_split);
}

template <int NG>
int launch(pd_handle* h, const CUtensorMap& tmA, const CUtensorMap& tmB, const SkinnyArgs& g, int ranks, cudaStream_t stream) {
    if (!(h->skinny_smem_configured & NG)) {
        cudaError_t e = cudaFuncSetAttribute(pd_gemm_skinny_kernel<NG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             Cfg<NG>::SMEM_BYTES);
        if (e != cudaSuccess) PD_FAIL(h, PD_ERR_DEVICE, "cudaFuncSetAttribute(smem=%d): %s", Cfg<NG>::SMEM_BYTES, cudaGetErrorString(e));
        h->skinny_smem_configured |= NG;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ranks, pd_cdiv(g.N, Cfg<NG>::BN), 1);
    cfg.blockDim = dim3(Cfg<NG>::NUM_THREADS, 1, 1);
    cfg.dynamicSmemBytes = Cfg<NG>::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = ranks; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, pd_gemm_skinny_kernel<NG>, tmA, tmB, g);
    PD_CHECK_LAUNCH(h, "pd_gemm_skinny_kernel");
    return PD_OK;
}

}  // namespace

// Shapes and operands pd_gemm_skinny_kernel takes: M <= 64 rows, A K-major and B MN-major ([K][N], the weight as stored),
// both TMA-addressable (16-byte aligned, row strides multiples of 4 floats), N, K >= 8, an fp32 C that is stored, not
// accumulated, with no fused ELU backward, and at most 16 K splits in the general kernel's split rule.
bool pd_gemm_skinny_ok(const pd_handle* h, int M, int N, int K, const void* A, long lda, int a_mn, const void* B, long ldb,
                       int b_mn, const PdEpilogue& e) {
    int kbs;
    return M >= 1 && M <= BM && N >= 8 && K >= 8 && !a_mn && b_mn && (lda % 4) == 0 && (ldb % 4) == 0 &&
           (((uintptr_t)A) & 15) == 0 && (((uintptr_t)B) & 15) == 0 && !e.accumulate && !e.c_f16 && !e.dact &&
           skinny_splits(h, M, N, K, &kbs) <= MAX_SPLITS;
}

int pd_gemm_skinny_launch(pd_handle* h, int M, int N, int K, const float* A, long lda, const float* B, long ldb,
                          const PdEpilogue& epi, cudaStream_t stream) {
    PD_REQUIRE(h, pd_gemm_skinny_ok(h, M, N, K, A, lda, 0, B, ldb, 1, epi),
               "pd_gemm_skinny: needs 1 <= M <= 64, N, K >= 8, 16-byte aligned A / B with lda, ldb %% 4 == 0, a stored "
               "fp32 C and at most %d K splits (got M %d N %d K %d lda %ld ldb %ld)", MAX_SPLITS, M, N, K, lda, ldb);
    CUtensorMap tmA, tmB;
    int rc = make_map(h, &tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
    if (!rc) rc = make_map(h, &tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 32, BK);
    if (rc) return rc;
    SkinnyArgs g;
    g.M = M; g.N = N; g.epi = epi;
    g.kb_total = pd_cdiv(K, BK);
    g.splits = skinny_splits(h, M, N, K, &g.kb_per_split);
    g.spc = g.splits > MAX_RANKS ? 2 : 1;
    const int ranks = pd_cdiv(g.splits, g.spc);
    // 128-column slabs when 64-column ones would need more CTAs than SMs (a cluster waits for room on one GPC)
    if ((long)pd_cdiv(N, 64) * ranks > h->num_sms) return launch<4>(h, tmA, tmB, g, ranks, stream);
    return launch<2>(h, tmA, tmB, g, ranks, stream);
}

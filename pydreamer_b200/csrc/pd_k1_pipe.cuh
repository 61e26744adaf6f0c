// pd_k1_pipe.cuh — building blocks shared by the two persistent RSSM kernels (pd_rssm_fwd3.cu: posterior unroll,
// pd_rssm_bptt.cu: its back-propagation through time).
//
//   * CTA = 8 consumer warps + 1 producer warp.  The producer streams operands with TMA (cp.async.bulk.tensor.2d, 128-byte
//     swizzle) into a shared-memory ring guarded by full / empty mbarriers; a stage = one 64-wide k-block of up to MAXT
//     16-row weight tiles (fp16) plus the activation / gradient boxes of that k-block.
//   * WEIGHT tiles of the next phase are requested BEFORE the grid barrier that separates two phases (they do not depend on
//     it); only the activation boxes wait for the barrier, so a phase starts with its weights already in shared memory.
//   * contractions run on the legacy tensor path (mma.sync): out[rows, batch] = W[rows, K] . X[batch, K]^T with the weight
//     rows on the MMA's M side (swap-AB: the batch is only 50..64 rows).
//   * grid-wide barriers: one atomic + one polled word in L2 (cooperative launch guarantees co-residency).
#pragma once
#include "pd_common.cuh"
#include <cuda_fp16.h>

namespace k1 {

constexpr int NCW = 8;                         // consumer warps
constexpr int NCT = 32 * NCW;                  // consumer threads
constexpr int NT = NCT + 32;                   // + producer warp
constexpr int BROWS = 64;                      // batch rows staged per box (B*I <= 64)
constexpr int KB = 64;                         // contraction elements per stage
constexpr int A_TILE = 16 * 128;               // one weight tile: 16 rows x 64 halfs
constexpr int X_BOX = BROWS * 128;             // one activation box: 64 rows x 128 bytes
constexpr int NSTAGE = 4;

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0, spins = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(s_u32(bar)), "r"(parity) : "memory");
        if (!done && ++spins > (1u << 26)) __trap();            // a broken pipeline must not hang the GPU
    }
}
__device__ __forceinline__ void tma_box(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(s_u32(dst)), "l"((uint64_t)map), "r"(s_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_box3(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(s_u32(dst)), "l"((uint64_t)map), "r"(s_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t h_lo(uint32_t v) { return __float_as_uint(__half2float(__ushort_as_half((unsigned short)(v & 0xffffu)))); }
__device__ __forceinline__ uint32_t h_hi(uint32_t v) { return __float_as_uint(__half2float(__ushort_as_half((unsigned short)(v >> 16)))); }
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }

// Sum over the 256 consumer threads (result valid in all of them); sh: >= 8 floats.
__device__ __forceinline__ float cons_sum(float v, float* sh) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    v = pd_warp_sum(v);
    cons_sync();
    if (lane == 0) sh[w] = v;
    cons_sync();
    float r = lane < NCW ? sh[lane] : 0.f;
    return pd_warp_sum(r);
}

// Grid-wide barrier among the consumer threads of all CTAs (monotonic counter, cleared by the host before the launch).
__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& epoch) {
    cons_sync();
    epoch += 1;
    if (threadIdx.x == 0) {
        const unsigned target = epoch * gridDim.x;
        // release-arrive / acquire-poll: the bar.sync above orders the CTA's writes before this thread's release (cumulative
        // at gpu scope), the bar.sync below hands what the acquire observed to the rest of the CTA
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
        unsigned spins = 0;
        while (ld_acquire(ctr) < target) {
            if (++spins > (1u << 24)) __trap();                 // ~10 s: a lost CTA must not hang the device
        }
    }
    cons_sync();
}
// Producer side: wait until barrier number `epoch` has completed, then make what the other CTAs published through the
// generic proxy visible to this thread's TMA (async proxy) reads.
__device__ __forceinline__ void producer_wait_barrier(const unsigned* ctr, unsigned epoch) {
    const unsigned target = epoch * gridDim.x;
    unsigned spins = 0;
    while (ld_acquire(ctr) < target) {
        if (++spins > (1u << 24)) __trap();
    }
    __threadfence();
    asm volatile("fence.proxy.async;" ::: "memory");
}

// Stage layout: MAXT weight tiles, then XB activation boxes (X_BOX bytes apart).
template <int MAXT, int XB>
struct Ring {                       // both sides count stages identically: slot = n % NSTAGE, parity = (n / NSTAGE) & 1
    static constexpr int STAGE_BYTES = MAXT * A_TILE + XB * X_BOX;
    static constexpr int BYTES = NSTAGE * STAGE_BYTES;
    uint8_t* smem;
    uint64_t* full;
    uint64_t* empty;
    uint32_t n;
    __device__ __forceinline__ uint8_t* stage(uint32_t i) const { return smem + (i % NSTAGE) * STAGE_BYTES; }
    __device__ __forceinline__ uint8_t* xbase(uint32_t i) const { return stage(i) + MAXT * A_TILE; }
    __device__ void init(uint8_t* base, uint64_t* bars) {
        smem = base; full = bars; empty = bars + NSTAGE; n = 0;
        if (threadIdx.x == 0) {
            for (int i = 0; i < NSTAGE; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, NCW); }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
};

// One contraction job of this CTA for one phase: `ntile` weight tiles (tile i = rows [row0[i], row0[i] + 16) of wmap[i]),
// `nkb` k-blocks of 64 starting at contraction index kcol0.  Activation operand: fp16 (xf16: one box of xrows x 64 halfs per
// k-block) or fp32 (two boxes of xrows x 32 floats); a second operand (nx == 2) is staged only for k-blocks that reach
// x2_from — below it the two operands are identical and the first is reused.
template <int MAXT>
struct Job {
    const CUtensorMap* wmap[MAXT];
    int row0[MAXT];
    int ntile;
    const CUtensorMap* xmap[2];
    int nx, xrow0, xrows, xf16;
    int kcol0, nkb, x2_from;
    // Grouped weight boxes (ngop > 0): the SAME ntile tiles fetched by a few larger TMA operations instead of one 2 KB box per
    // tile — op o fills tiles gdst[o].. from rows grow[o].. of gmap[o]; g3d[o]: a 3-D map (k, row within gate, gate) whose box
    // spans all gates (a TMA operation costs about the same for a small box as for a large one).  produce() reads wmap / row0
    // only when ngop == 0: a job with grouped boxes may leave them unset (jobs B and C of pd_rssm_fwd3.cu do).
    int ngop;
    const CUtensorMap* gmap[3];
    int grow[3], gdst[3], g3d[3];
};
template <int MAXT>
__device__ __forceinline__ bool job_needs_x2(const Job<MAXT>& j, int kb) { return j.nx == 2 && j.kcol0 + (kb + 1) * KB > j.x2_from; }
template <int MAXT>
__device__ __forceinline__ uint32_t job_bytes(const Job<MAXT>& j, int kb) {
    const uint32_t xb = (uint32_t)j.xrows * 128u * (j.xf16 ? 1u : 2u);
    return (uint32_t)j.ntile * A_TILE + xb * (job_needs_x2(j, kb) ? 2u : 1u);
}

// Producer: weights of the first stages are requested before the grid barrier `wait_epoch` (0 = nothing to wait for),
// activation boxes after it.
template <int MAXT, int XB>
__device__ void produce(Ring<MAXT, XB>& ring, const Job<MAXT>& j, const unsigned* ctr, unsigned wait_epoch, int xrow_off = 0) {
    const int npre = j.nkb < NSTAGE ? j.nkb : NSTAGE;
    auto weights = [&](int kb) {
        const uint32_t n = ring.n + kb;
        mbar_wait(ring.empty + n % NSTAGE, ((n / NSTAGE) & 1) ^ 1);
        mbar_expect_tx(ring.full + n % NSTAGE, job_bytes(j, kb));
        uint8_t* st = ring.stage(n);
        if (j.ngop > 0) {
            for (int o = 0; o < j.ngop; ++o) {
                if (j.g3d[o]) tma_box3(j.gmap[o], ring.full + n % NSTAGE, st + j.gdst[o] * A_TILE, j.kcol0 + kb * KB, j.grow[o], 0);
                else          tma_box(j.gmap[o], ring.full + n % NSTAGE, st + j.gdst[o] * A_TILE, j.kcol0 + kb * KB, j.grow[o]);
            }
            return;
        }
        for (int i = 0; i < j.ntile; ++i) tma_box(j.wmap[i], ring.full + n % NSTAGE, st + i * A_TILE, j.kcol0 + kb * KB, j.row0[i]);
    };
    auto xboxes = [&](int kb) {
        const uint32_t n = ring.n + kb;
        uint8_t* st = ring.xbase(n);
        uint64_t* bar = ring.full + n % NSTAGE;
        const int kf = j.kcol0 + kb * KB;                           // contraction index of this k-block
        const bool x2 = job_needs_x2(j, kb);
        const int xr = j.xrow0 + xrow_off;                          // xrow_off: the same job over another block of batch rows
        if (j.xf16) {
            tma_box(j.xmap[0], bar, st, kf, xr);
            if (x2) tma_box(j.xmap[1], bar, st + X_BOX, kf, xr);
        } else {
            tma_box(j.xmap[0], bar, st, kf, xr);
            tma_box(j.xmap[0], bar, st + X_BOX, kf + 32, xr);
            if (x2) {
                tma_box(j.xmap[1], bar, st + 2 * X_BOX, kf, xr);
                tma_box(j.xmap[1], bar, st + 3 * X_BOX, kf + 32, xr);
            }
        }
    };
    for (int kb = 0; kb < npre; ++kb) weights(kb);
    if (wait_epoch) producer_wait_barrier(ctr, wait_epoch);
    for (int kb = 0; kb < npre; ++kb) xboxes(kb);
    for (int kb = npre; kb < j.nkb; ++kb) { weights(kb); xboxes(kb); }
    ring.n += j.nkb;
}

// Consumer, fp32 (tf32) activation operand: this warp accumulates TW weight tiles (tile0 ..) x NW8 n8-tiles of batch rows
// (n8_0 ..) over all k-blocks of the job; xsel = which operand its tiles contract with.  Warps without work pass
// active = false (they still walk the ring).  acc[i][j][4]: mma C fragment of (tile i, n8-tile j): rows g, g+8 of the tile,
// batch columns 2t, 2t+1 of the n8-tile.  Weight fragments: ldmatrix of the fp16 tile, unpacked to tf32 (exact) — the low
// halves carry the even k of a k16 step, the high halves the odd k, so one ldmatrix feeds two m16n8k8 MMAs whose B
// fragments are the matching even / odd columns of the fp32 box.
template <int TW, int NW8, int MAXT, int XB>
__device__ void consume_tf32(Ring<MAXT, XB>& ring, const Job<MAXT>& j, int tile0, int n8_0, int xsel, bool active,
                             float (&acc)[TW][NW8][4]) {
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
        for (int jn = 0; jn < NW8; ++jn)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][jn][e] = 0.f;
    for (int kb = 0; kb < j.nkb; ++kb) {
        const uint32_t n = ring.n + kb;
        mbar_wait(ring.full + n % NSTAGE, (n / NSTAGE) & 1);
        if (active) {
            const uint8_t* st = ring.stage(n);
            const uint8_t* xb = ring.xbase(n) + ((xsel && job_needs_x2(j, kb)) ? 2 * X_BOX : 0);
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {                    // four k16 steps of the 64-wide block
                uint32_t a[TW][4];
#pragma unroll
                for (int i = 0; i < TW; ++i) {
                    const int r = lane & 15;
                    ldsm_x4(s_u32(st + (tile0 + i) * A_TILE + r * 128 + (((ks * 2 + (lane >> 4)) ^ (r & 7)) << 4)), a[i][0],
                            a[i][1], a[i][2], a[i][3]);
                }
                const uint8_t* box = xb + (ks >> 1) * X_BOX;    // two k16 steps per 32-float box
                const int kk0 = (ks & 1) * 16;
#pragma unroll
                for (int jn = 0; jn < NW8; ++jn) {
                    const int row = (n8_0 + jn) * 8 + g;
                    const uint8_t* rp = box + row * 128;
                    const float2 fa = *reinterpret_cast<const float2*>(rp + ((((kk0 + 2 * t) >> 2) ^ (row & 7)) << 4) + ((2 * t) & 3) * 4);
                    const float2 fb = *reinterpret_cast<const float2*>(rp + ((((kk0 + 2 * t + 8) >> 2) ^ (row & 7)) << 4) + ((2 * t) & 3) * 4);
#pragma unroll
                    for (int i = 0; i < TW; ++i) {
                        mma_tf32(acc[i][jn], h_lo(a[i][0]), h_lo(a[i][1]), h_lo(a[i][2]), h_lo(a[i][3]), __float_as_uint(fa.x),
                                 __float_as_uint(fb.x));
                        mma_tf32(acc[i][jn], h_hi(a[i][0]), h_hi(a[i][1]), h_hi(a[i][2]), h_hi(a[i][3]), __float_as_uint(fa.y),
                                 __float_as_uint(fb.y));
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(ring.empty + n % NSTAGE);
    }
    ring.n += j.nkb;
}

// Consumer, fp16 activation operand (one 64-half box per k-block): m16n8k16, both operands by ldmatrix.  The warp's n8-tiles
// come in PAIRS (n8_0 even, NW8 even): one ldmatrix.x4 of the activation box feeds two n8-tiles.
template <int TW, int NW8, int MAXT, int XB>
__device__ void consume_f16(Ring<MAXT, XB>& ring, const Job<MAXT>& j, int tile0, int n8_0, bool active, float (&acc)[TW][NW8][4]) {
    static_assert(NW8 % 2 == 0, "n8-tiles are consumed in pairs");
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
        for (int jn = 0; jn < NW8; ++jn)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][jn][e] = 0.f;
    for (int kb = 0; kb < j.nkb; ++kb) {
        const uint32_t n = ring.n + kb;
        mbar_wait(ring.full + n % NSTAGE, (n / NSTAGE) & 1);
        if (active) {
            const uint8_t* st = ring.stage(n);
            const uint8_t* xb = ring.xbase(n);
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                uint32_t a[TW][4];
#pragma unroll
                for (int i = 0; i < TW; ++i) {
                    const int r = lane & 15;
                    ldsm_x4(s_u32(st + (tile0 + i) * A_TILE + r * 128 + (((ks * 2 + (lane >> 4)) ^ (r & 7)) << 4)), a[i][0],
                            a[i][1], a[i][2], a[i][3]);
                }
#pragma unroll
                for (int jp = 0; jp < NW8 / 2; ++jp) {
                    uint32_t b0, b1, b2, b3;
                    const int nrow = (n8_0 + jp * 2 + (lane >> 4)) * 8 + (lane & 7);
                    ldsm_x4(s_u32(xb + nrow * 128 + (((ks * 2 + ((lane >> 3) & 1)) ^ (nrow & 7)) << 4)), b0, b1, b2, b3);
#pragma unroll
                    for (int i = 0; i < TW; ++i) {
                        mma_f16(acc[i][jp * 2], a[i], b0, b1);
                        mma_f16(acc[i][jp * 2 + 1], a[i], b2, b3);
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(ring.empty + n % NSTAGE);
    }
    ring.n += j.nkb;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// row-major [rows, K] matrix as a 2-D tensor map, boxes of 128 bytes x box_rows, 128-byte swizzle, zero OOB fill
inline int make_map(pd_handle* h, const char* who, CUtensorMap* tm, const void* base, long rows, int K, int box_rows, bool f16,
                    long ld = 0) {                     // ld: row stride in elements (0: K, a dense matrix)
    cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)(ld ? ld : K) * (f16 ? 2 : 4)};
    cuuint32_t box[2] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = ((EncodeTiledFn)h->encode_tiled)(tm, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                                                   (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) PD_FAIL(h, PD_ERR_ARG, "%s: cuTensorMapEncodeTiled failed (%d) for [%ld, %d]", who, (int)r, rows, K);
    return PD_OK;
}

// [gates * rows_per_gate, K] fp16 weight matrix as a 3-D map (k, row within gate, gate): one box {64 halfs, box_rows, gates}
// lands in shared memory gate after gate — the tiles of all gates for one block of rows in ONE TMA operation.
inline int make_map3g(pd_handle* h, const char* who, CUtensorMap* tm, const void* base, long rows_per_gate, int K, int gates,
                      int box_rows) {
    cuuint64_t gdim[3] = {(cuuint64_t)K, (cuuint64_t)rows_per_gate, (cuuint64_t)gates};
    cuuint64_t gstride[2] = {(cuuint64_t)K * 2, (cuuint64_t)rows_per_gate * K * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)box_rows, (cuuint32_t)gates};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = ((EncodeTiledFn)h->encode_tiled)(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void*)base, gdim, gstride, box, estr,
                                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) PD_FAIL(h, PD_ERR_ARG, "%s: cuTensorMapEncodeTiled(3-D gates) failed (%d) for [%d x %ld, %d]", who, (int)r,
                                   gates, rows_per_gate, K);
    return PD_OK;
}

}  // namespace k1

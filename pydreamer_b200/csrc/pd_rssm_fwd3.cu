// pd_rssm_fwd3.cu — the posterior unroll of the RSSM as ONE persistent cooperative kernel (pd_rssm_unroll_fwd), third
// generation: TMA-staged operands, producer warp, weight prefetch across grid barriers, k-split recurrent contraction.
//
// Reference semantics: pydreamer/models/rssm.py:21-78 (RSSMCore.forward time loop) and :125-153 (RSSMCell.forward:
// z_mlp + a_mlp -> in_norm -> ELU -> GRUCell -> post_mlp_h + post_mlp_e -> post_norm -> ELU -> post_mlp ->
// OneHotCategoricalStraightThrough sample).  Same contract (inputs, saved tensors, sampled indices) as the first-generation
// kernel of round 1 (cp.async row staging, every CTA re-reading the whole activation operand; git history), which it replaces.
//
// Per timestep, five dependent phases separated by grid barriers (pd_k1_pipe.cuh):
//   A   batch-row owners      : x1 = mask * gather(W_z^T, idx_{t-1}) + b_z + aa_t ; LayerNorm + ELU -> za          (z is one-hot)
//   B   hidden-unit owners    : gi = za . W_ih^T (K = Hd) ; gh = sum of the k-slice partials of phase C ; GRU gates -> h'
//   C   (row group, k slice)  : partials of gh_{t+1} = h' . W_hh^T and y2 = h' . W_ph^T over a quarter of K = D each:
//                               every CTA stages 64 x D/4 of h' instead of 64 x D (r02 ncu of the first generation: the
//                               re-read activation operand was 3x the weight stream); the partials are summed by their
//                               consumers (unit owners in B, row owners in C'), which costs no extra barrier
//   C'  batch-row owners      : y2 = sum of partials + b_ph + ea_t ; LayerNorm + ELU -> pin
//   D   latent-group owners   : logits of group g for a quarter of the batch rows = pin . W_pm^T ; softmax ; argmax(p / q)
// Weights are fp16, activations fp16 (za, h', pin: the same 10 mantissa bits as the TF32 chain), accumulation fp32.
// All contractions run on mma.sync m16n8k16 with ldmatrix fragments (consume_f16, pd_k1_pipe.cuh): the weight rows are the
// MMA's M side (16-row tiles), the batch rows its N side, accumulators in registers.
//
// Stacked GRU (layers = L, 2..4; rnn.py:40-67): phase B runs once per layer, with a grid barrier after each, so a step has
// L - 1 more dependent phases.  Layer 0 contracts za with its W_ih; layer l > 0 the fp16 h' that layer l - 1 just wrote to
// h16 (its D/L columns, a strided TMA map) with its own W_ih.  Phase C is unchanged: it contracts h' with the block-diagonal
// [3D, D] W_hh the host assembles (each unit's row holds its layer's weights in its layer's columns and zeros elsewhere), so
// every unit's partial sums cover only its own layer.  The previous h of a unit comes from hin (global) instead of the
// shared-memory copy the single cell keeps.
//
// Batch rows beyond one 64-row MMA operand (IWAE: BI = B x iwae_samples, world.py:60-68 repeats every sequence I times) run in
// the MULTI instantiation: phases B and C repeat their contraction and epilogue per block of 64 rows, phase D takes 64 rows
// per pass with all eight warps, and the row owners of A / C' stride over the rows by the grid size.
#include "pd_k1_pipe.cuh"

namespace {
using namespace k1;

constexpr int MAXT = 16;                       // phase C: 3 gates x 4 tiles of W_hh rows + 2 tiles of W_ph rows = 14 of the
                                               // 16 box slots
typedef Ring<MAXT, 1> RingF;
typedef Job<MAXT> JobF;
constexpr int OFF_BAR = RingF::BYTES;
constexpr int OFF_SH = OFF_BAR + 128;                       // 64 floats: block reductions
constexpr int MAXG = 256;                                   // latent groups the kernel takes (phase A keeps one class per group)
constexpr int OFF_SIDX = OFF_SH + 256;                      // MAXG ints: sampled classes of one row
constexpr int HB = 256;                                     // batch rows the MULTI instantiation takes (4 blocks of BROWS)
constexpr int OFF_HC = OFF_SIDX + MAXG * 4;                 // [16][BROWS or HB] floats: masked h of my units (input of the next step)
constexpr int OFF_PART = OFF_HC + 16 * HB * 4;              // [2][1024] floats: phase A gather halves
constexpr int OFF_LOG = OFF_PART + 2 * 1024 * 4;            // [16 or 64][32] floats: phase D logits of my rows
constexpr int OFF_GI = OFF_LOG + 64 * 32 * 4;               // [48][65] floats: phase B gi of my units (for the gate math)
constexpr int SMEM_BYTES = OFF_GI + 48 * 65 * 4;
constexpr int KSPLIT = 4;

struct FwdMaps {
    CUtensorMap wpm;                           // fp16 W_pm, box {64 halfs, 16 rows} (phase D when C <= 16)
    CUtensorMap za, h;                         // fp16 activations [BI, K], box {64 halfs, 64 rows}
    CUtensorMap pin16;                         // fp16 [BI, Hd], box {64 halfs, 16 rows}
    CUtensorMap pin64;                         // the same matrix, box {64 halfs, 64 rows} (MULTI phase D)
    // grouped weight boxes: all three gates of a row block in one 3-D box, the 32 consecutive rows of W_ph / W_pm in one 2-D box
    CUtensorMap wih3;                          // W_ih as (k, unit, gate): box {64 halfs, 16 units, 3 gates} = tiles 0..2 of phase B
    CUtensorMap whh3;                          // W_hh as (k, unit, gate): box {64 halfs, 64 units, 3 gates} = tiles 0..11 of phase C
    CUtensorMap wph32, wpm32;                  // box {64 halfs, 32 rows} = tiles 12, 13 of phase C / the two class tiles of phase D
    CUtensorMap hl[3];                         // stacked GRU: h16 columns of layer l - 1 ([BI, D/L] at ld D), input of layer l's phase B
    CUtensorMap wih3l[3];                      // stacked GRU: W_ih of layer l as (k, unit, gate), box {64 halfs, 16 units, 3 gates}
};

// LayerNorm + ELU of one row held as v[4] per consumer thread (features tid + 256 i); writes fp32 (fp16-representable) and
// fp16 copies, mean / rstd.  Same formulas as ln_elu_fwd_kernel (pd_rowwise.cu).
__device__ void ln_elu_row(float (&v)[4], int N, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                           float* yrow, __half* y16row, float* mean_out, float* rstd_out, float* sh) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) s += (threadIdx.x + NCT * i < N) ? v[i] : 0.f;
    const float mean = cons_sum(s, sh) / (float)N;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float d = (threadIdx.x + NCT * i < N) ? v[i] - mean : 0.f;
        q += d * d;
    }
    const float var = cons_sum(q, sh) / (float)N;
    const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = threadIdx.x + NCT * i;
        if (c < N) {
            const __half hv = __float2half_rn(pd_elu((v[i] - mean) * rstd * gamma[c] + beta[c]));
            yrow[c] = __half2float(hv);
            y16row[c] = hv;
        }
    }
    if (threadIdx.x == 0) { *mean_out = mean; *rstd_out = rstd; }
}

template <bool MULTI>
__global__ void __launch_bounds__(NT, 1) rssm_unroll_fwd3_kernel(const pd_rssm_fwd_args a, const __grid_constant__ FwdMaps maps,
                                                                 const int KS) {
    constexpr int HS = MULTI ? HB : BROWS;                  // row stride of hcs
    constexpr int DR = MULTI ? 64 : 16;                     // batch rows of one phase-D pass
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    float* sh = (float*)(smem + OFF_SH);
    int* sidx = (int*)(smem + OFF_SIDX);
    float* hcs = (float*)(smem + OFF_HC);                   // hcs[r * HS + b]
    float* part = (float*)(smem + OFF_PART);                // [2][Hd]
    float* lgs = (float*)(smem + OFF_LOG);                  // lgs[rb * 32 + class]
    float* gis = (float*)(smem + OFF_GI);                   // gis[(gate * 16 + r) * 65 + b]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool producer = warp == NCW;
    const int P = gridDim.x, c = blockIdx.x;
    const int T = a.T, BI = a.BI, D = a.D, Hd = a.Hd, G = a.G, C = a.C, Z = G * C, F = D + Z, D3 = 3 * D;
    const int Bq = BI / a.I;                                // sequences (rows of aa / ea per timestep)
    const int L = a.layers > 1 ? a.layers : 1, Dl = D / L;  // GRU layers, units per layer
    const __half* wzT = (const __half*)a.ws_wzT16;          // [Z][Hd], transposed z_mlp weight (written by the host)
    __half* za16 = (__half*)a.ws_za16;
    __half* h16 = (__half*)a.ws_h16;
    __half* pin16 = (__half*)a.ws_pin16;

    RingF ring;
    ring.init(smem, (uint64_t*)(smem + OFF_BAR));

    // ---- static ownership
    // B: my hidden units of layer l are [l Dl + u4_0, l Dl + u4_1)
    const int u4_0 = (int)((long)c * Dl / P), u4_1 = (int)((long)(c + 1) * Dl / P), nu = u4_1 - u4_0;
    const int RG = P / KS, rg = c / KS, ks = c % KS;                                                    // C: row group x k slice
    const bool inC = rg < RG;
    const int u6_0 = (int)((long)rg * D / RG), u6_1 = inC ? (int)((long)(rg + 1) * D / RG) : u6_0;     // C: gh rows (units)
    const int f6_0 = (int)((long)rg * Hd / RG), f6_1 = inC ? (int)((long)(rg + 1) * Hd / RG) : f6_0;   // C: y2 features
    const int kslice = D / KS;
    const int R = max(1, min(4, P / G));                                                                 // D: CTAs per group
    const int RB = (BI + R - 1) / R;                                                                     // rows per such CTA
    const bool inD = c < G * R;
    const int g9 = c / R, sub9 = c % R, b9_0 = sub9 * RB, b9_1 = min(BI, b9_0 + RB);
    const int NBB = MULTI ? (BI + BROWS - 1) / BROWS : 1;                                                // blocks of batch rows
    const int NDC = !inD ? 0 : (MULTI ? max(0, (b9_1 - b9_0 + DR - 1) / DR) : 1);                        // phase-D passes
    const int ASTEP = MULTI ? P : (1 << 30);                                                             // row owners' stride

    for (int o = tid; o < nu * BI; o += NT) hcs[(o % nu) * HS + o / nu] = __ldcg(a.hin + (long)(o / nu) * D + u4_0 + o % nu);
    __syncthreads();

    // weight tiles come in grouped boxes (FwdMaps); phase D takes one box per 16-row tile unless its C classes fill two tiles.
    // Jobs B and C always set ngop > 0 and leave wmap / row0 unset: produce() does not read them then.
    auto job_b = [&](int l) {                                       // phase B of GRU layer l
        const CUtensorMap* xm = l == 0 ? &maps.za : &maps.hl[l - 1];
        JobF j; j.ntile = nu > 0 ? 3 : 0; j.nx = 1; j.xmap[0] = xm; j.xmap[1] = xm; j.xrow0 = 0; j.xrows = BROWS; j.xf16 = 1;
        j.kcol0 = 0; j.nkb = j.ntile ? ((l == 0 ? Hd : Dl) + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        j.ngop = 1; j.gmap[0] = l == 0 ? &maps.wih3 : &maps.wih3l[l - 1]; j.grow[0] = u4_0; j.gdst[0] = 0; j.g3d[0] = 1;
        return j;
    };
    auto job_c = [&]() {
        JobF j; j.ntile = inC ? 14 : 0; j.nx = 1; j.xmap[0] = &maps.h; j.xmap[1] = &maps.h; j.xrow0 = 0; j.xrows = BROWS; j.xf16 = 1;
        j.kcol0 = ks * kslice; j.nkb = j.ntile ? (kslice + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        j.ngop = 2;                                                     // tile = gate * 4 + i for W_hh, 12 + i for W_ph
        j.gmap[0] = &maps.whh3; j.grow[0] = u6_0; j.gdst[0] = 0; j.g3d[0] = 1;
        j.gmap[1] = &maps.wph32; j.grow[1] = f6_0; j.gdst[1] = 12; j.g3d[1] = 0;
        return j;
    };
    auto job_d = [&]() {
        JobF j; j.ntile = inD ? (C + 15) / 16 : 0; j.nx = 1; j.xmap[0] = MULTI ? &maps.pin64 : &maps.pin16; j.xmap[1] = j.xmap[0];
        j.xrow0 = b9_0; j.xrows = DR;
        j.xf16 = 1; j.kcol0 = 0; j.nkb = j.ntile ? (Hd + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        for (int i = 0; i < MAXT; ++i) { j.wmap[i] = &maps.wpm; j.row0[i] = g9 * C + 16 * i; }
        j.ngop = j.ntile == 2 ? 1 : 0; j.gmap[0] = &maps.wpm32; j.grow[0] = g9 * C; j.gdst[0] = 0; j.g3d[0] = 0;
        return j;
    };

    // ================================================= producer warp =================================================
    if (producer) {
        if (lane == 0) {
            unsigned epoch = 0;
            // prologue: barrier 1 publishes h16 = fp16(h_0); then the phase-C job computes gh_0 partials; barrier 2
            // (a further block of batch rows / pass of phase D is the same job with the activation box shifted)
            { const JobF j = job_c(); if (j.nkb) for (int bb = 0; bb < NBB; ++bb) produce(ring, j, a.ws_barrier, 1, bb * BROWS); }
            epoch = 2;
            for (int t = 0; t < T; ++t) {
                // barriers of a step: after A (1), after B of layer l (2 + l), after C (2 + L), after C' (3 + L), after D
                // (4 + L, not on the last step)
                for (int l = 0; l < L; ++l) {
                    const JobF j = job_b(l);
                    if (j.nkb) for (int bb = 0; bb < NBB; ++bb) produce(ring, j, a.ws_barrier, epoch + 1 + l, bb * BROWS);
                }
                { const JobF j = job_c(); if (j.nkb) for (int bb = 0; bb < NBB; ++bb) produce(ring, j, a.ws_barrier, epoch + 1 + L, bb * BROWS); }
                { const JobF j = job_d(); if (j.nkb) for (int rc = 0; rc < NDC; ++rc) produce(ring, j, a.ws_barrier, epoch + 3 + L, rc * DR); }
                epoch += 4 + L;
            }
        }
        return;
    }

    // ================================================= consumer warps =================================================
    unsigned epoch = 0;
    // phase C: partial products of my rows over my k slice -> global (gh partials only when want_gh, y2 partials when want_y2)
    auto phase_c = [&](bool want_gh, bool want_y2) {
        const JobF j = job_c();
        if (j.nkb == 0) return;
        // warp w < 7 takes weight tiles 2w, 2w + 1 (tile = gate * 4 + i for W_hh, 12 + i for W_ph) x all 64 batch rows
        const bool act = warp < 7;
        for (int bb = 0; bb < NBB; ++bb) {
            float acc[2][8][4];
            consume_f16<2, 8>(ring, j, 2 * warp, 0, act, acc);
            if (!act) continue;
            const int g = lane >> 2, tq = lane & 3;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int slot = 2 * warp + i;
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int rr = g + 8 * hr;
                    float* dst = nullptr;                       // element b of this row goes to dst[b * bstride]: partial
                    long bstride = 0;                           // planes [ks][b][row]
                    if (slot < 12) {
                        const int gate = slot >> 2, u = u6_0 + (slot & 3) * 16 + rr;
                        if (want_gh && u < u6_1) { dst = a.ws_ghpart + (long)ks * BI * D3 + (long)gate * D + u; bstride = D3; }
                    } else {
                        const int f = f6_0 + (slot - 12) * 16 + rr;
                        if (want_y2 && f < f6_1) { dst = a.ws_y2part + (long)ks * BI * Hd + f; bstride = Hd; }
                    }
                    if (!dst) continue;
#pragma unroll
                    for (int jn = 0; jn < 8; ++jn)
#pragma unroll
                        for (int x = 0; x < 2; ++x) {
                            const int b = bb * BROWS + jn * 8 + 2 * tq + x;
                            if (b < BI) dst[(long)b * bstride] = acc[i][jn][2 * hr + x];
                        }
                }
            }
        }
    };

    // ---- prologue: fp16 h_0 for the TMA reads of the first recurrent product
    for (long i = (long)c * NCT + tid; i < (long)BI * D; i += (long)P * NCT) h16[i] = __float2half_rn(__ldcg(a.hin + i));
    grid_barrier(a.ws_barrier, epoch);                                          // (p1)
    phase_c(true, false);                                                       // gh_0 = h_0 . W_hh^T (raw; bias and mask at use)
    grid_barrier(a.ws_barrier, epoch);                                          // (p2)

    for (int t = 0; t < T; ++t) {
        // ---- phase A (CTA b < BI): x1 = mask * gather(WzT, idx_{t-1}) + b_z + aa_t ; LayerNorm + ELU -> za
        for (int b = c; b < BI; b += ASTEP) {
            const long row = (long)t * BI + b;
            float v[4];
            if (MULTI && b != c) cons_sync();                             // sidx / part of my previous row are free again
            if (t > 0) {
                const float m = a.mask[row];
                for (int gg = tid; gg < G; gg += NCT) sidx[gg] = __ldcg(a.idx + ((long)(t - 1) * BI + b) * G + gg);
                float pa[4];                                              // bias + action term, in flight during the gather
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int f = tid + NCT * i;
                    pa[i] = f < Hd ? a.b_z[f] + a.aa[((long)t * Bq + b / a.I) * Hd + f] : 0.f;
                }
                cons_sync();
                {   // gather-sum of G rows of WzT: thread = (8 features, half of the groups), 16-byte loads, all independent
                    const int fg = tid & 127, gh = tid >> 7;
                    if (fg * 8 < Hd) {
                        float s8[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) s8[e] = 0.f;
                        const int g0 = gh * ((G + 1) / 2), g1 = min(G, g0 + (G + 1) / 2);
#pragma unroll 4
                        for (int gg = g0; gg < g1; ++gg) {
                            const uint4 w = *(const uint4*)(wzT + (long)(gg * C + sidx[gg]) * Hd + fg * 8);
                            const __half2* h2 = (const __half2*)&w;
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const float2 f2 = __half22float2(h2[e]);
                                s8[2 * e] += f2.x; s8[2 * e + 1] += f2.y;
                            }
                        }
#pragma unroll
                        for (int e = 0; e < 8; ++e) part[gh * Hd + fg * 8 + e] = s8[e];
                    }
                }
                cons_sync();
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int f = tid + NCT * i;
                    v[i] = 0.f;
                    if (f < Hd) {
                        v[i] = m * (part[f] + part[Hd + f]) + pa[i];
                        a.x1[row * Hd + f] = v[i];
                    }
                }
                for (int jz = tid; jz < Z; jz += NCT) a.zin[row * Z + jz] = (sidx[jz / C] == jz % C) ? m : 0.f;
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int f = tid + NCT * i;
                    v[i] = f < Hd ? __ldcg(a.x1 + row * Hd + f) : 0.f;
                }
            }
            ln_elu_row(v, Hd, a.ln1_g, a.ln1_b, a.eps, a.za + row * Hd, za16 + (long)b * Hd, a.m1 + row, a.r1 + row, sh);
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (1) za complete

        // ---- phase B (hidden-unit owners), once per GRU layer: gi = x . W_ih^T (x = za, or layer l - 1's h'), GRU gate math,
        //      h' -> feat / hin[t+1] / h16
        for (int l = 0; l < L; ++l) {
            const JobF j = job_b(l);
            const int uoff = l * Dl;                                    // first unit of the layer
            const float* b_ih = l == 0 ? a.b_ih : a.b_ih_l[l - 1];
            const float* b_hh = l == 0 ? a.b_hh : a.b_hh_l[l - 1];
            if (j.nkb > 0) {
              for (int bb = 0; bb < NBB; ++bb) {
                if (MULTI && bb > 0) cons_sync();                          // gis of the previous block has been read
                // warps 0..3: the three gate tiles x two n8-tiles (16 batch rows) each
                float acc[3][2][4];
                const bool act = warp < 4;
                consume_f16<3, 2>(ring, j, 0, 2 * warp, act, acc);
                if (act) {
                    const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                    for (int i = 0; i < 3; ++i)
#pragma unroll
                        for (int jn = 0; jn < 2; ++jn)
#pragma unroll
                            for (int x = 0; x < 4; ++x)
                                gis[(i * 16 + g + 8 * (x >> 1)) * 65 + (2 * warp + jn) * 8 + 2 * tq + (x & 1)] = acc[i][jn][x];
                }
                cons_sync();
                // gate math: one (unit, batch row) per thread iteration, unit fastest (coalesced global accesses)
                const int nb = MULTI ? min(BROWS, BI - bb * BROWS) : BI;
                // (the k-slice partials of up to four (unit, row) pairs are requested before any of them is used: the loop is
                //  bound by the latency of those L2 reads, and the stores below would otherwise order them pair after pair)
                for (int o0 = tid; o0 < nu * nb; o0 += 4 * NCT) {
                    float gh[4][3];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int o = o0 + q * NCT;
                        gh[q][0] = gh[q][1] = gh[q][2] = 0.f;
                        if (o < nu * nb) {
                            const int u = uoff + u4_0 + o % nu, b = bb * BROWS + o / nu;
                            for (int k = 0; k < KS; ++k) {                  // threads run over u: coalesced
                                const float* gp = a.ws_ghpart + ((long)k * BI + b) * D3 + u;
                                gh[q][0] += __ldcg(gp); gh[q][1] += __ldcg(gp + D); gh[q][2] += __ldcg(gp + 2 * D);
                            }
                        }
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int o = o0 + q * NCT;
                        if (o >= nu * nb) break;
                        const int r = o % nu, bl = o / nu, b = bb * BROWS + bl, ul = u4_0 + r, u = uoff + ul;
                        const long row = (long)t * BI + b;
                        const float m = t > 0 ? a.mask[row] : 1.f;              // h_0 arrives already masked
                        const float mn = t + 1 < T ? a.mask[row + BI] : 0.f;
                        const float ghr = m * gh[q][0] + b_hh[ul];
                        const float ghu = m * gh[q][1] + b_hh[Dl + ul];
                        const float ghn = m * gh[q][2] + b_hh[2 * Dl + ul];
                        const float rg_ = pd_sigmoid(gis[(0 * 16 + r) * 65 + bl] + b_ih[ul] + ghr);
                        const float ug_ = pd_sigmoid(gis[(1 * 16 + r) * 65 + bl] + b_ih[Dl + ul] + ghu);
                        const float ng_ = tanhf(gis[(2 * 16 + r) * 65 + bl] + b_ih[2 * Dl + ul] + rg_ * ghn);
                        const float hp = L == 1 ? hcs[r * HS + b] : __ldcg(a.hin + row * D + u);
                        const __half hh = __float2half_rn((1.f - ug_) * ng_ + ug_ * hp);
                        const float hn = __half2float(hh);
                        a.feat[row * F + u] = hn;
                        h16[(long)b * D + u] = hh;
                        hcs[r * HS + b] = hn * mn;
                        if (t + 1 < T) a.hin[(row + BI) * D + u] = hn * mn;
                        float* gt = a.gates + (((long)l * T + t) * BI + b) * 4 * Dl;        // [L, T, BI, 4 Dl]
                        gt[ul] = rg_; gt[Dl + ul] = ug_; gt[2 * Dl + ul] = ng_; gt[3 * Dl + ul] = ghn;
                    }
                }
              }
            }
            grid_barrier(a.ws_barrier, epoch);                                  // (2 + l) h' of layer l complete
        }

        // ---- phase C: partials of y2 = h' . W_ph^T and of gh_{t+1} = h' . W_hh^T
        phase_c(t + 1 < T, true);
        grid_barrier(a.ws_barrier, epoch);                                      // (2 + L) partials complete

        // ---- phase C' (CTA b < BI): y2 = partial sums + b_ph + ea_t ; LayerNorm + ELU -> pin
        for (int b = c; b < BI; b += ASTEP) {
            const long row = (long)t * BI + b;
            float v[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = tid + NCT * i;
                v[i] = 0.f;
                if (f < Hd) {
                    float s = a.b_ph[f] + (a.ea ? a.ea[((long)t * Bq + b / a.I) * Hd + f] : 0.f);
                    for (int k = 0; k < KS; ++k) s += __ldcg(a.ws_y2part + ((long)k * BI + b) * Hd + f);
                    v[i] = s;
                    a.y2[row * Hd + f] = s;
                }
            }
            ln_elu_row(v, Hd, a.ln2_g, a.ln2_b, a.eps, a.pin + row * Hd, pin16 + (long)b * Hd, a.m2 + row, a.r2 + row, sh);
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (3 + L) pin complete

        // ---- phase D (latent-group owners): logits of group g for my rows, softmax, argmax(p / q) -> post, idx, z
        for (int rc = 0; rc < NDC; ++rc) {
            const JobF j = job_d();
            float acc[1][2][4];
            if (MULTI && rc > 0) cons_sync();                                   // lgs of the previous pass has been read
            // warp = 16 classes of the group x two n8-tiles of batch rows: 16 rows per pass need warps 0 and 1, 64 rows all eight
            const int ctile = MULTI ? (warp & 1) : warp, n8_0 = MULTI ? (warp >> 1) * 2 : 0;
            const bool act = (MULTI || warp < 2) && ctile * 16 < C;
            consume_f16<1, 2>(ring, j, ctile, n8_0, act, acc);
            if (act) {
                const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                for (int jn = 0; jn < 2; ++jn)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int cls = 16 * ctile + g + 8 * (e >> 1), rb = (n8_0 + jn) * 8 + 2 * tq + (e & 1);
                        if (cls < C) lgs[rb * 32 + cls] = acc[0][jn][e];
                    }
            }
            cons_sync();
            const float pbias = lane < C ? a.b_pm[g9 * C + lane] : 0.f;
            for (int rb = warp; rb < min(DR, b9_1 - b9_0 - rc * DR); rb += NCW) {
                const int b = b9_0 + rc * DR + rb;
                const long row = (long)t * BI + b;
                const bool valid = lane < C;
                const float q = valid ? a.noise[row * Z + g9 * C + lane] : 1.f;
                float l = 0.f;
                if (valid) {
                    l = lgs[rb * 32 + lane] + pbias;
                    a.post[row * Z + g9 * C + lane] = l;
                }
                // same arithmetic as cat_sample_kernel (pd_rowwise.cu): logits - logsumexp, softmax, argmax(p / q)
                const float mx = pd_warp_max(valid ? l : -INFINITY);
                const float e = valid ? expf(l - mx) : 0.f;
                const float lse = mx + logf(pd_warp_sum(e));
                const float ln = valid ? l - lse : -INFINITY;
                const float mx2 = pd_warp_max(ln);
                const float e2 = valid ? expf(ln - mx2) : 0.f;
                const float p = e2 / pd_warp_sum(e2);
                float val = valid ? p / q : -INFINITY;
                int k = lane;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float ov = __shfl_xor_sync(0xffffffffu, val, o);
                    const int ok = __shfl_xor_sync(0xffffffffu, k, o);
                    if (ov > val || (ov == val && ok < k)) { val = ov; k = ok; }
                }
                if (valid) a.feat[row * F + D + g9 * C + lane] = (lane == k) ? 1.f : 0.f;
                if (lane == 0) a.idx[row * G + g9] = k;
            }
        }
        if (t + 1 < T) grid_barrier(a.ws_barrier, epoch);                       // (4 + L) idx_t complete
    }
}

}  // namespace

extern "C" int pd_rssm_unroll_fwd(pd_handle* h, const pd_rssm_fwd_args* a, void* stream) {
    if (!h || !a) return PD_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    PdDeviceGuard guard(h);
    constexpr size_t SMEM_REQ = (size_t)SMEM_BYTES + 1024;
    if (!h->k1_configured) {
        if (cudaFuncSetAttribute(rssm_unroll_fwd3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_REQ) != cudaSuccess ||
            cudaFuncSetAttribute(rssm_unroll_fwd3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_REQ) != cudaSuccess)
            PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_fwd: cannot reserve %d bytes of shared memory", (int)SMEM_REQ);
        int per_sm = 0, per_sm_m = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rssm_unroll_fwd3_kernel<false>, NT, SMEM_REQ);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_m, rssm_unroll_fwd3_kernel<true>, NT, SMEM_REQ);
        h->k1_ctas = (per_sm > 0 && per_sm_m > 0) ? h->num_sms : 0;             // one CTA per SM
        h->k1_configured = 1;
    }
    const int P = h->k1_ctas;
    PD_REQUIRE(h, P > 0, "pd_rssm_unroll_fwd: kernel does not fit an SM");
    const int Z = a->G * a->C;
    const int L = a->layers > 1 ? a->layers : 1;
    const int Dl = a->D / L;
    bool layers_ok = a->layers >= 0 && a->layers <= 4 && a->D % L == 0 && Dl % 8 == 0;
    for (int l = 1; l < L; ++l) layers_ok = layers_ok && a->w_ih16_l[l - 1] && a->b_ih_l[l - 1] && a->b_hh_l[l - 1];
    const int KS = (a->D % (KSPLIT * KB) == 0 && P >= KSPLIT) ? KSPLIT : 1;
    const int RG = P / KS;
    const int R = P / a->G < 4 ? (P / a->G < 1 ? 1 : P / a->G) : 4;
    // one block of batch rows: the single-block kernel; up to four (IWAE): the MULTI instantiation
    const bool multi = !(a->BI <= BROWS && a->BI <= P && (a->BI + R - 1) / R <= 16);
    const bool ok = a->T >= 1 && a->BI >= 1 && a->BI <= HB && a->I >= 1 && a->BI % a->I == 0 &&
                    a->Hd <= 4 * NCT && a->Hd % 8 == 0 && a->D % 8 == 0 && a->C >= 1 && a->C <= 32 && a->G >= 1 && a->G <= P && a->G <= MAXG &&
                    layers_ok && (Dl + P - 1) / P <= 16 && (a->D + RG - 1) / RG <= 64 &&
                    (a->Hd + RG - 1) / RG <= 32 && Z >= 1 && a->ws_ghpart && a->ws_y2part && a->ws_wzT16;
    if (!ok)
        PD_FAIL(h, PD_ERR_UNSUPPORTED, "pd_rssm_unroll_fwd: shape T=%d BI=%d D=%d Hd=%d G=%d C=%d layers=%d outside the kernel's limits",
                a->T, a->BI, a->D, a->Hd, a->G, a->C, a->layers);
    FwdMaps maps;
    memset(&maps, 0, sizeof(maps));
    const char* who = "pd_rssm_unroll_fwd";
    int rc = make_map(h, who, &maps.wpm, a->w_pm16, Z, a->Hd, 16, true);
    if (!rc) rc = make_map(h, who, &maps.za, a->ws_za16, a->BI, a->Hd, BROWS, true);
    if (!rc) rc = make_map(h, who, &maps.h, a->ws_h16, a->BI, a->D, BROWS, true);
    if (!rc) rc = make_map(h, who, &maps.pin16, a->ws_pin16, a->BI, a->Hd, 16, true);
    if (!rc) rc = make_map(h, who, &maps.pin64, a->ws_pin16, a->BI, a->Hd, BROWS, true);
    if (!rc) rc = make_map3g(h, who, &maps.wih3, a->w_ih16, Dl, a->Hd, 3, 16);
    for (int l = 1; l < L && !rc; ++l) {
        rc = make_map(h, who, &maps.hl[l - 1], (const __half*)a->ws_h16 + (long)(l - 1) * Dl, a->BI, Dl, BROWS, true, a->D);
        if (!rc) rc = make_map3g(h, who, &maps.wih3l[l - 1], a->w_ih16_l[l - 1], Dl, Dl, 3, 16);
    }
    if (!rc) rc = make_map3g(h, who, &maps.whh3, a->w_hh16, a->D, a->D, 3, 64);
    if (!rc) rc = make_map(h, who, &maps.wph32, a->w_ph16, a->Hd, a->D, 32, true);
    if (!rc) rc = make_map(h, who, &maps.wpm32, a->w_pm16, Z, a->Hd, 32, true);
    if (rc) return rc;
    if (cudaMemsetAsync(a->ws_barrier, 0, 16 * sizeof(unsigned), s) != cudaSuccess)
        PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_fwd: memset failed");
    pd_rssm_fwd_args args = *a;
    int ksv = KS;
    void* kargs[] = {(void*)&args, (void*)&maps, (void*)&ksv};
    const void* fn = multi ? (const void*)rssm_unroll_fwd3_kernel<true> : (const void*)rssm_unroll_fwd3_kernel<false>;
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(P), dim3(NT), kargs, SMEM_REQ, s);
    if (e != cudaSuccess) PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_fwd: %s", cudaGetErrorString(e));
    PD_CHECK_LAUNCH(h, "pd_rssm_unroll_fwd");
    return PD_OK;
}

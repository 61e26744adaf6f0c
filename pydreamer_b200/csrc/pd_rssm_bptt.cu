// pd_rssm_bptt.cu — back-propagation through time of the RSSM posterior unroll as ONE persistent cooperative kernel
// (pd_rssm_unroll_bwd).
//
// Reference semantics: autograd of pydreamer/models/rssm.py:21-78 (time loop) and :125-153 (RSSMCell.forward:
// z_mlp + a_mlp -> in_norm -> ELU -> GRUCell (rnn.py:60-67 -> nn.GRUCell) -> post_mlp_h + post_mlp_e -> post_norm -> ELU ->
// post_mlp -> straight-through one-hot sample), seeded by the gradients of the losses w.r.t. features / posterior logits.
// It replaces, per timestep, the launch chain  cat_st_bwd -> gemm -> ln_elu_bwd -> gemm -> gru_bwd -> gemm x2 -> ln_elu_bwd
// -> gemm  of pydreamer_b200/dreamer.py (_wm_backward) and writes exactly the tensors that chain writes (dpost, dy2, dgi, dgh,
// dx1: the operands of the batched weight-gradient GEMMs that follow) plus the LayerNorm / bias gradients it accumulates.
//
// Structure (one CTA per SM, 132 on an H100, cooperative launch):
//   * 8 consumer warps + 1 producer warp.  The producer streams operands with TMA (cp.async.bulk.tensor.2d, 128-byte
//     swizzle) into a 4-stage shared-memory ring guarded by full / empty mbarriers; a stage = one 64-wide k-block of up to
//     six 16-row weight tiles (fp16) and up to four 64-row x 32-float boxes of the gradient operand (fp32).
//     WEIGHT tiles of the next phase are requested BEFORE the grid barrier that separates the phases (they do not depend
//     on it); only the gradient boxes wait for the barrier, so a phase starts with its weights already in shared memory.
//   * contractions: out[rows, batch] = W^T[rows, K] . X[batch, K]^T on the legacy tensor path
//     (mma.sync.m16n8k8 tf32): weight fragments come from fp16 tiles (ldmatrix, exact fp16 -> tf32 unpack), the gradient
//     operand stays fp32 / tf32-rounded — gradients need fp32's exponent range, so fp16 operands are not an option here,
//     and both operands carry 10 mantissa bits exactly like the TF32 tensor-core GEMMs of the launch chain.
//   * per timestep six dependent phases, separated by grid barriers (one atomic + one polled word in L2):
//       P9+P1  latent-group owners : dz_{t} = dx1_{t+1} W_z (kept in smem) -> straight-through softmax backward + KL term -> dpost_t
//       P2     (row-group, k-slice): dpin = dpost_t W_pm          partial sums over 4 k-slices -> global
//       P3     batch-row owners    : LayerNorm+ELU backward (post_norm)  -> dy2_t, accumulates dgamma / dbeta / db
//       P4     hidden-unit owners  : dh = dy2_t W_ph + dfeat_h + carry ; GRU gate backward -> dgi_t, dgh_t (dh*u kept in smem)
//       P6/7   (row-group, k-slice): dh_{t-1} partials = dgh_t W_hh ; dza partials = dgi_t W_ih   (K = 3D split in 4)
//       P8     batch-row owners    : LayerNorm+ELU backward (in_norm)    -> dx1_t
//     K-split partial sums are added by their consumers (row owners / unit owners), which costs no extra barrier.
#include "pd_k1_pipe.cuh"

namespace {
using namespace k1;

constexpr int MAXT = 6;                        // weight tiles (16 rows) per stage: 4 of W_hh^T + 2 of W_ih^T in phase P6/7
typedef Ring<MAXT, 4> RingB;                   // + up to four 64-row x 32-float boxes of the gradient operand (fp32): 44 KB
typedef Job<MAXT> JobB;
constexpr int OFF_BAR = RingB::BYTES;                       // full[NSTAGE], empty[NSTAGE]
constexpr int OFF_SH = OFF_BAR + 128;                       // 64 floats: block reductions
constexpr int OFF_DHC = OFF_SH + 256;                       // [16][BROWS] floats: dh*u of my hidden units (carry to t-1)
constexpr int OFF_DZ = OFF_DHC + 16 * BROWS * 4;            // [16][32] floats: dzin of my (rows, latent group)
constexpr int SMEM_BYTES = OFF_DZ + 16 * 32 * 4;
constexpr int KSPLIT = 4;

struct BwdMaps {
    CUtensorMap wpmT, wphT, whhT, wihT, wzT;   // fp16 [rows][K], box {64 halfs, 16 rows}, SWIZZLE_128B
    CUtensorMap dpost, dy2, dgh, dgi, dx1;     // fp32 [(T*BI)][K], box {32 floats, 64 rows}, SWIZZLE_128B
    CUtensorMap dx1_16;                        // same tensor, box {32 floats, 16 rows}
};

__device__ __forceinline__ float rnd(float x, int on) { return on ? pd_tf32(x) : x; }

__global__ void __launch_bounds__(NT, 1) rssm_unroll_bwd_kernel(const pd_rssm_bwd_args a, const __grid_constant__ BwdMaps maps) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    float* sh = (float*)(smem + OFF_SH);
    float* dhc = (float*)(smem + OFF_DHC);                  // dhc[r * BROWS + b]
    float* dzs = (float*)(smem + OFF_DZ);                   // dzs[rb * 32 + class]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool producer = warp == NCW;
    const int P = gridDim.x, c = blockIdx.x;
    const int T = a.T, BI = a.BI, D = a.D, Hd = a.Hd, G = a.G, C = a.C, Z = G * C, F = D + Z, D3 = 3 * D;
    const int rnd_on = a.round_out;

    RingB ring;
    ring.init(smem, (uint64_t*)(smem + OFF_BAR));
    for (int i = tid; i < 16 * BROWS; i += NT) dhc[i] = 0.f;
    for (int i = tid; i < 16 * 32; i += NT) dzs[i] = 0.f;
    __syncthreads();

    // ---- static ownership
    // k-split phases: CTA = (row group rg, k slice ks); KS2 for P2 (K = Z), KS6 for P6/7 (K = 3D)
    const int KS2 = a.ks2, KS6 = a.ks6;
    const int RG2 = P / KS2, RG6 = P / KS6;
    const int rg2 = c / KS2, ks2 = c % KS2, rg6 = c / KS6, ks6 = c % KS6;
    const bool in2 = rg2 < RG2, in6 = rg6 < RG6;
    const int f2_0 = (int)((long)rg2 * Hd / RG2), f2_1 = (int)((long)(rg2 + 1) * Hd / RG2);          // P2: dpin features
    const int u6_0 = (int)((long)rg6 * D / RG6), u6_1 = (int)((long)(rg6 + 1) * D / RG6);            // P6: dh rows (units)
    const int f6_0 = (int)((long)rg6 * Hd / RG6), f6_1 = (int)((long)(rg6 + 1) * Hd / RG6);          // P7: dza features
    const int u4_0 = (int)((long)c * D / P), u4_1 = (int)((long)(c + 1) * D / P), nu4 = u4_1 - u4_0;  // P4: my hidden units
    const int R = max(1, min(4, P / G));                                                               // P9/P1: CTAs per group
    const int RB = (BI + R - 1) / R;                                                                   // rows per such CTA (<= 16)
    const bool in9 = c < G * R;
    const int g9 = c / R, sub9 = c % R, b9_0 = sub9 * RB, b9_1 = min(BI, b9_0 + RB);
    const int nt2 = in2 ? (f2_1 - f2_0 + 15) / 16 : 0;
    const int nt6h = in6 ? (u6_1 - u6_0 + 15) / 16 : 0, nt6z = in6 ? (f6_1 - f6_0 + 15) / 16 : 0;
    const int kslice2 = Z / KS2, kslice6 = D3 / KS6;

    auto job_p2 = [&](int t) {
        JobB j; j.ngop = 0; j.xf16 = 0; j.ntile = nt2; j.nx = 1; j.xmap[0] = &maps.dpost; j.xmap[1] = &maps.dpost; j.xrow0 = t * BI; j.xrows = BROWS;
        j.kcol0 = ks2 * kslice2; j.nkb = nt2 ? (kslice2 + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        for (int i = 0; i < MAXT; ++i) { j.wmap[i] = &maps.wpmT; j.row0[i] = f2_0 + 16 * i; }
        return j;
    };
    auto job_p4 = [&](int t) {
        JobB j; j.ngop = 0; j.xf16 = 0; j.ntile = nu4 > 0 ? 1 : 0; j.nx = 1; j.xmap[0] = &maps.dy2; j.xmap[1] = &maps.dy2; j.xrow0 = t * BI; j.xrows = BROWS;
        j.kcol0 = 0; j.nkb = j.ntile ? (Hd + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        for (int i = 0; i < MAXT; ++i) { j.wmap[i] = &maps.wphT; j.row0[i] = u4_0; }
        return j;
    };
    auto job_p6 = [&](int t) {
        JobB j; j.ngop = 0; j.xf16 = 0; j.ntile = (nt6h || nt6z) ? 6 : 0; j.nx = 2; j.xmap[0] = &maps.dgh; j.xmap[1] = &maps.dgi; j.xrow0 = t * BI; j.xrows = BROWS;
        j.kcol0 = ks6 * kslice6; j.nkb = j.ntile ? (kslice6 + KB - 1) / KB : 0; j.x2_from = 2 * D;   // dgi == dgh for the r, u gates
        for (int i = 0; i < 4; ++i) { j.wmap[i] = &maps.whhT; j.row0[i] = u6_0 + 16 * i; }
        for (int i = 0; i < 2; ++i) { j.wmap[4 + i] = &maps.wihT; j.row0[4 + i] = f6_0 + 16 * i; }
        return j;
    };
    auto job_p9 = [&](int t) {
        JobB j; j.ngop = 0; j.xf16 = 0; j.ntile = in9 ? (C + 15) / 16 : 0; j.nx = 1; j.xmap[0] = &maps.dx1_16; j.xmap[1] = &maps.dx1_16;
        j.xrow0 = t * BI + b9_0; j.xrows = 16;
        j.kcol0 = 0; j.nkb = j.ntile ? (Hd + KB - 1) / KB : 0; j.x2_from = 1 << 30;
        for (int i = 0; i < MAXT; ++i) { j.wmap[i] = &maps.wzT; j.row0[i] = g9 * C + 16 * i; }
        return j;
    };

    // ================================================= producer warp =================================================
    if (producer) {
        if (lane == 0) {
            unsigned epoch = 0;
            for (int t = T - 1; t >= 0; --t) {
                // barriers of a step, in order: after P1 (1), after P2 (2), after P3 (3), after P4 (4), after P6/7 (5), after P8 (6)
                { const JobB j = job_p2(t); if (j.nkb) produce(ring, j, a.ws_barrier, epoch + 1); }
                { const JobB j = job_p4(t); if (j.nkb) produce(ring, j, a.ws_barrier, epoch + 3); }
                { const JobB j = job_p6(t); if (j.nkb) produce(ring, j, a.ws_barrier, epoch + 4); }
                if (t > 0) { const JobB j = job_p9(t); if (j.nkb) produce(ring, j, a.ws_barrier, epoch + 6); }
                epoch += 6;
            }
        }
        return;
    }

    // ================================================= consumer warps =================================================
    unsigned epoch = 0;
    // LayerNorm / bias gradient accumulators of the batch-row owners (4 features per thread), kept over all timesteps
    float ag2[4] = {0, 0, 0, 0}, ab2[4] = {0, 0, 0, 0}, ax2[4] = {0, 0, 0, 0};
    float ag1[4] = {0, 0, 0, 0}, ab1[4] = {0, 0, 0, 0}, ax1[4] = {0, 0, 0, 0};

    // LayerNorm+ELU backward of one row held 4 features per thread (same formulas as ln_elu_bwd_row_kernel, pd_rowwise.cu)
    auto ln_bwd_row = [&](const float (&dyv)[4], const float* xrow, const float* yrow, const float* gamma, float mean, float rstd,
                          float* dxrow, float (&ag)[4], float (&ab)[4], float (&ax)[4]) {
        float gg[4], xh[4], dxh[4], s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = tid + NCT * i;
            if (f < Hd) {
                gg[i] = dyv[i] * pd_elu_grad_from_out(yrow[f]);
                xh[i] = (xrow[f] - mean) * rstd;
                dxh[i] = gg[i] * gamma[f];
                s1 += dxh[i]; s2 += dxh[i] * xh[i];
            } else { gg[i] = xh[i] = dxh[i] = 0.f; }
        }
        const float c1 = cons_sum(s1, sh) / (float)Hd;
        const float c2 = cons_sum(s2, sh) / (float)Hd;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = tid + NCT * i;
            if (f < Hd) {
                const float d = rstd * (dxh[i] - c1 - xh[i] * c2);
                dxrow[f] = rnd(d, rnd_on);
                ag[i] += gg[i] * xh[i]; ab[i] += gg[i]; ax[i] += d;
            }
        }
    };

    for (int t = T - 1; t >= 0; --t) {
        const bool nxt = t + 1 < T;
        // ---------------- P1 (latent-group owners): straight-through softmax backward + KL term -> dpost_t
        if (in9) {
            for (int rb = warp; rb < b9_1 - b9_0; rb += NCW) {
                const int b = b9_0 + rb;
                const long row = (long)t * BI + b;
                const bool valid = lane < C;
                const long off = (long)g9 * C + lane;
                const float l = valid ? a.post[row * Z + off] : 0.f;
                // group softmax exactly as cat_st_bwd_kernel / cat_sample_kernel (pd_rowwise.cu)
                const float mx = pd_warp_max(valid ? l : -INFINITY);
                const float e = valid ? expf(l - mx) : 0.f;
                const float lse = mx + logf(pd_warp_sum(e));
                const float ln = valid ? l - lse : -INFINITY;
                const float mx2 = pd_warp_max(ln);
                const float e2 = valid ? expf(ln - mx2) : 0.f;
                const float p = e2 / pd_warp_sum(e2);
                float dz = 0.f;
                if (valid) {
                    dz = a.dfeat[row * F + D + off];
                    if (nxt) dz += dzs[rb * 32 + lane] * a.mask[row + BI];
                }
                const float s = pd_warp_sum(valid ? p * dz : 0.f);
                if (valid) {
                    float d = p * (dz - s);
                    d += a.kl_weight * a.w[row] * a.dpost_u[row * Z + off];
                    a.dpost[row * Z + off] = rnd(d, rnd_on);
                }
            }
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (1) dpost_t complete

        // ---------------- P2 (row group x k slice): dpin partials = dpost_t . W_pm
        {
            const JobB j = job_p2(t);
            float acc[2][1][4];
            const bool act = warp * 8 < BI;
            consume_tf32<2, 1>(ring, j, 0, warp, 0, act && j.nkb > 0, acc);
            if (act && j.nkb > 0) {
                const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int f = f2_0 + 16 * i + g + 8 * (e >> 1), b = warp * 8 + 2 * tq + (e & 1);
                        if (f < f2_1 && b < BI) a.ws_part2[((long)ks2 * BI + b) * Hd + f] = acc[i][0][e];
                    }
            }
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (2) dpin partials complete

        // ---------------- P3 (batch-row owners): post_norm LayerNorm+ELU backward -> dy2_t
        if (c < BI) {
            const int b = c;
            const long row = (long)t * BI + b;
            float dyv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = tid + NCT * i;
                float s = 0.f;
                if (f < Hd)
                    for (int k = 0; k < KS2; ++k) s += __ldcg(a.ws_part2 + ((long)k * BI + b) * Hd + f);
                dyv[i] = s;
            }
            ln_bwd_row(dyv, a.y2 + row * Hd, a.pin + row * Hd, a.ln2_g, a.m2[row], a.r2[row], a.dy2 + row * Hd, ag2, ab2, ax2);
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (3) dy2_t complete

        // ---------------- P4 (hidden-unit owners): dh = dy2_t . W_ph + dfeat_h + carry ; GRU gate backward -> dgi_t, dgh_t
        {
            const JobB j = job_p4(t);
            float acc[1][1][4];
            const bool act = warp * 8 < BI;
            consume_tf32<1, 1>(ring, j, 0, warp, 0, act && j.nkb > 0, acc);
            if (act && j.nkb > 0) {
                const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = g + 8 * (e >> 1), b = warp * 8 + 2 * tq + (e & 1), u = u4_0 + r;
                    if (r < nu4 && b < BI) {
                        const long row = (long)t * BI + b;
                        float dh = acc[0][0][e] + a.dfeat[row * F + u];
                        if (nxt) {
                            float carry = dhc[r * BROWS + b];
                            for (int k = 0; k < KS6; ++k) carry += __ldcg(a.ws_part6 + ((long)k * BI + b) * D + u);
                            dh += carry * a.mask[row + BI];
                        }
                        const float* gt = a.gates + row * 4 * D;
                        const float rg = gt[u], ug = gt[D + u], ng = gt[2 * D + u], ghn = gt[3 * D + u];
                        const float hp = a.hin[row * D + u];
                        const float dn_pre = dh * (1.f - ug) * (1.f - ng * ng);
                        const float du_pre = dh * (hp - ng) * ug * (1.f - ug);
                        const float dr_pre = dn_pre * ghn * rg * (1.f - rg);
                        float* gi = a.dgi + row * D3;
                        float* gh = a.dgh + row * D3;
                        const float v0 = rnd(dr_pre, rnd_on), v1 = rnd(du_pre, rnd_on);
                        gi[u] = v0; gi[D + u] = v1; gi[2 * D + u] = rnd(dn_pre, rnd_on);
                        gh[u] = v0; gh[D + u] = v1; gh[2 * D + u] = rnd(dn_pre * rg, rnd_on);
                        dhc[r * BROWS + b] = dh * ug;
                    }
                }
            }
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (4) dgi_t, dgh_t complete

        // ---------------- P6/7 (row group x k slice): dh_{t-1} partials = dgh_t . W_hh ; dza partials = dgi_t . W_ih
        {
            const JobB j = job_p6(t);
            float acc[2][4][4];
            // warps 0..5: tile pair (warp % 3) x batch half (warp / 3); tile pairs 0,1 = W_hh^T rows, pair 2 = W_ih^T rows
            const int pair = warp % 3, half = warp / 3;
            const bool act = warp < 6 && j.nkb > 0 && half * 32 < BI;
            consume_tf32<2, 4>(ring, j, 2 * pair, 4 * half, pair == 2 ? 1 : 0, act, acc);
            if (act) {
                const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int jn = 0; jn < 4; ++jn)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int r = 16 * (2 * pair + i) + g + 8 * (e >> 1), b = (4 * half + jn) * 8 + 2 * tq + (e & 1);
                            if (b >= BI) continue;
                            if (pair < 2) {
                                const int u = u6_0 + r;
                                if (u < u6_1) a.ws_part6[((long)ks6 * BI + b) * D + u] = acc[i][jn][e];
                            } else {
                                const int f = f6_0 + r - 64;
                                if (f < f6_1) a.ws_part7[((long)ks6 * BI + b) * Hd + f] = acc[i][jn][e];
                            }
                        }
            }
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (5) partials complete

        // ---------------- P8 (batch-row owners): in_norm LayerNorm+ELU backward -> dx1_t
        if (c < BI) {
            const int b = c;
            const long row = (long)t * BI + b;
            float dyv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int f = tid + NCT * i;
                float s = 0.f;
                if (f < Hd)
                    for (int k = 0; k < KS6; ++k) s += __ldcg(a.ws_part7 + ((long)k * BI + b) * Hd + f);
                dyv[i] = s;
            }
            ln_bwd_row(dyv, a.x1 + row * Hd, a.za + row * Hd, a.ln1_g, a.m1[row], a.r1[row], a.dx1 + row * Hd, ag1, ab1, ax1);
        }
        grid_barrier(a.ws_barrier, epoch);                                      // (6) dx1_t complete

        // ---------------- P9 (latent-group owners): dz of my (rows, group) = dx1_t . W_z, kept in smem for P1 of step t-1
        if (t > 0) {
            const JobB j = job_p9(t);
            float acc[1][1][4];
            // warps 0..3: class half (warp & 1) x row octet (warp >> 1)
            const bool act = warp < 4 && j.nkb > 0 && (warp & 1) * 16 < C && (warp >> 1) * 8 < b9_1 - b9_0;
            consume_tf32<1, 1>(ring, j, warp & 1, warp >> 1, 0, act, acc);
            if (act) {
                const int g = lane >> 2, tq = lane & 3;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int cls = 16 * (warp & 1) + g + 8 * (e >> 1), rb = (warp >> 1) * 8 + 2 * tq + (e & 1);
                    if (cls < C && rb < 16) dzs[rb * 32 + cls] = acc[0][0][e];
                }
            }
            cons_sync();
        }
    }

    // ---- the LayerNorm / bias gradients, added in a fixed order: each batch-row owner writes its six [Hd] accumulators to
    // row c of a workspace, and after a grid barrier the grid adds rows c = 0..BI-1 in order into g_*.  The rows live in
    // ws_part2 (quantities 0-3) and ws_part7 (4-5): both are dead once the last P8 has read ws_part7 before barrier (6).
    auto part = [&](int q, int b) {
        return q < 4 ? a.ws_part2 + ((long)q * BI + b) * Hd : a.ws_part7 + ((long)(q - 4) * BI + b) * Hd;
    };
    if (c < BI) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = tid + NCT * i;
            if (f < Hd) {
                part(0, c)[f] = ag2[i]; part(1, c)[f] = ab2[i]; part(2, c)[f] = ax2[i];
                part(3, c)[f] = ag1[i]; part(4, c)[f] = ab1[i]; part(5, c)[f] = ax1[i];
            }
        }
    }
    grid_barrier(a.ws_barrier, epoch);                                          // (7) every owner's partials written
    float* const gout[6] = {a.g_ln2_g, a.g_ln2_b, a.g_b_ph, a.g_ln1_g, a.g_ln1_b, a.g_b_z};
    for (int e = c * NCT + tid; e < 6 * Hd; e += P * NCT) {
        const int q = e / Hd, f = e - q * Hd;
        float s = 0.f;
        for (int b = 0; b < BI; ++b) s += __ldcg(part(q, b) + f);
        gout[q][f] += s;
    }
}

}  // namespace

extern "C" int pd_rssm_unroll_bwd(pd_handle* h, const pd_rssm_bwd_args* a_in, void* stream) {
    if (!h || !a_in) return PD_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    PdDeviceGuard guard(h);
    constexpr size_t SMEM_REQ = (size_t)SMEM_BYTES + 1024;
    if (!h->k1b_configured) {
        if (cudaFuncSetAttribute(rssm_unroll_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_REQ) != cudaSuccess)
            PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_bwd: cannot reserve %d bytes of shared memory", (int)SMEM_REQ);
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rssm_unroll_bwd_kernel, NT, SMEM_REQ);
        h->k1b_ctas = per_sm > 0 ? h->num_sms : 0;
        h->k1b_configured = 1;
    }
    const int P = h->k1b_ctas;
    PD_REQUIRE(h, P > 0, "pd_rssm_unroll_bwd: kernel does not fit an SM");
    pd_rssm_bwd_args a = *a_in;
    const int Z = a.G * a.C, D3 = 3 * a.D;
    // k-split factors: slices must be whole 64-wide k-blocks
    a.ks2 = (Z % (KSPLIT * KB) == 0 && P >= KSPLIT) ? KSPLIT : 1;
    a.ks6 = (D3 % (KSPLIT * KB) == 0 && P >= KSPLIT) ? KSPLIT : 1;
    const int RG2 = P / a.ks2, RG6 = P / a.ks6;
    const int R = P / a.G < 4 ? (P / a.G < 1 ? 1 : P / a.G) : 4;
    const bool ok = a.T >= 1 && a.BI >= 1 && a.BI <= BROWS && a.BI <= P && a.Hd <= 4 * NCT && a.Hd % 4 == 0 && a.D % 4 == 0 &&
                    Z % 4 == 0 && a.C >= 1 && a.C <= 32 && a.G >= 1 && a.G <= P && (a.BI + R - 1) / R <= 16 &&
                    (a.D + P - 1) / P <= 16 && (a.Hd + RG2 - 1) / RG2 <= 32 && (a.D + RG6 - 1) / RG6 <= 64 &&
                    (a.Hd + RG6 - 1) / RG6 <= 32 && a.Hd % 8 == 0 && D3 % 8 == 0 && Z % 8 == 0;
    if (!ok)
        PD_FAIL(h, PD_ERR_UNSUPPORTED, "pd_rssm_unroll_bwd: shape T=%d BI=%d D=%d Hd=%d G=%d C=%d outside the kernel's limits",
                a.T, a.BI, a.D, a.Hd, a.G, a.C);
    BwdMaps maps;
    memset(&maps, 0, sizeof(maps));
    const long rows = (long)a.T * a.BI;
    const char* who = "pd_rssm_unroll_bwd";
    int rc = make_map(h, who, &maps.wpmT, a.w_pmT16, a.Hd, Z, 16, true);
    if (!rc) rc = make_map(h, who, &maps.wphT, a.w_phT16, a.D, a.Hd, 16, true);
    if (!rc) rc = make_map(h, who, &maps.whhT, a.w_hhT16, a.D, D3, 16, true);
    if (!rc) rc = make_map(h, who, &maps.wihT, a.w_ihT16, a.Hd, D3, 16, true);
    if (!rc) rc = make_map(h, who, &maps.wzT, a.w_zT16, Z, a.Hd, 16, true);
    if (!rc) rc = make_map(h, who, &maps.dpost, a.dpost, rows, Z, BROWS, false);
    if (!rc) rc = make_map(h, who, &maps.dy2, a.dy2, rows, a.Hd, BROWS, false);
    if (!rc) rc = make_map(h, who, &maps.dgh, a.dgh, rows, D3, BROWS, false);
    if (!rc) rc = make_map(h, who, &maps.dgi, a.dgi, rows, D3, BROWS, false);
    if (!rc) rc = make_map(h, who, &maps.dx1, a.dx1, rows, a.Hd, BROWS, false);
    if (!rc) rc = make_map(h, who, &maps.dx1_16, a.dx1, rows, a.Hd, 16, false);
    if (rc) return rc;
    if (cudaMemsetAsync(a.ws_barrier, 0, 16 * sizeof(unsigned), s) != cudaSuccess)
        PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_bwd: memset failed");
    void* kargs[] = {(void*)&a, (void*)&maps};
    cudaError_t e = cudaLaunchCooperativeKernel((const void*)rssm_unroll_bwd_kernel, dim3(P), dim3(NT), kargs, SMEM_REQ, s);
    if (e != cudaSuccess) PD_FAIL(h, PD_ERR_LAUNCH, "pd_rssm_unroll_bwd: %s", cudaGetErrorString(e));
    PD_CHECK_LAUNCH(h, "pd_rssm_unroll_bwd");
    return PD_OK;
}

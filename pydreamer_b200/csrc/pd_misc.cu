// pd_misc.cu — small pointwise kernels, loss heads, world-model loss assembly, actor-critic
// (GAE scan, actor/critic losses) and the fused optimizer.  All HBM- or latency-bound.
#include "pd_common.cuh"
#include <cuda_fp16.h>

namespace {

inline int grid_for(long total, int block, int num_sms) {
    long g = (total + block - 1) / block;
    long cap = (long)num_sms * 32;
    if (g < 1) g = 1;
    return (int)(g < cap ? g : cap);
}
#define GRID_STRIDE(i, n) for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (long)gridDim.x * blockDim.x)

__global__ void round_copy_kernel(const float* __restrict__ s, float* __restrict__ d, long n, int r) {
    GRID_STRIDE(i, n) d[i] = pd_round_if(s[i], r);
}
__global__ void pad_cols_kernel(long M, int C, int Cp, const float* __restrict__ s, long lds, float* __restrict__ d,
                                long ldd, int r) {
    GRID_STRIDE(i, M * Cp) {
        long m = i / Cp; int c = (int)(i % Cp);
        d[m * ldd + c] = c < C ? pd_round_if(s[m * lds + c], r) : 0.f;
    }
}
__global__ void mask_rows_kernel(long M, int N, const float* __restrict__ x, long ldx, const float* __restrict__ mask,
                                 float* __restrict__ o, long ldo, int r) {
    GRID_STRIDE(i, M * N) {
        long m = i / N; int c = (int)(i % N);
        o[m * ldo + c] = pd_round_if(x[m * ldx + c] * mask[m], r);
    }
}
__global__ void rowscale_kernel(long M, long N, float* __restrict__ x, long ldx, const float* __restrict__ sc, int div,
                                float alpha, int r) {
    GRID_STRIDE(i, M * N) {
        long m = i / N; long c = i % N;
        x[m * ldx + c] = pd_round_if(x[m * ldx + c] * (alpha * sc[m / div]), r);
    }
}
__global__ void group_sum_kernel(long R, int I, int W, const float* __restrict__ x, long ldx, float* __restrict__ o,
                                 long ldo, int r) {
    GRID_STRIDE(i, R * W) {
        long row = i / W; int c = (int)(i % W);
        float acc = 0.f;
        for (int k = 0; k < I; ++k) acc += x[(row * I + k) * ldx + c];
        o[row * ldo + c] = pd_round_if(acc, r);
    }
}
__global__ void to_half_kernel(long M, long N, const float* __restrict__ s, long lds, __half* __restrict__ d, long ldd) {
    GRID_STRIDE(i, M * N) {
        long m = i / N, c = i % N;
        d[m * ldd + c] = __float2half_rn(s[m * lds + c]);
    }
}
// dst[n][m] = half(src[m][n]): 32x32 tiles through shared memory (both sides coalesced)
__global__ void transpose_to_half_kernel(int M, int N, const float* __restrict__ s, long lds, __half* __restrict__ d, long ldd) {
    __shared__ float tile[32][33];
    const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int m = m0 + r, n = n0 + threadIdx.x;
        tile[r][threadIdx.x] = (m < M && n < N) ? s[(long)m * lds + n] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int n = n0 + r, m = m0 + threadIdx.x;
        if (n < N && m < M) d[(long)n * ldd + m] = __float2half_rn(tile[threadIdx.x][r]);
    }
}
__global__ void fill_kernel(float* x, long n, float v) { GRID_STRIDE(i, n) x[i] = v; }
__global__ void reset_mask_kernel(int T, int B, int I, const uint8_t* __restrict__ reset, float* __restrict__ mask) {
    GRID_STRIDE(i, (long)T * B * I) {
        long tb = i / I;
        mask[i] = reset[tb] ? 0.f : 1.f;
    }
}
// out[c] += sum_rows x[r, c] ; blockDim (32, 8); partials of the blocks of one column group are added in blockIdx.y order
// by the last of them (pd_last_block)
__global__ void colsum_kernel(long M, int N, const float* __restrict__ x, long ldx, float* out, float* ws, unsigned* tickets) {
    const int c = blockIdx.x * 32 + threadIdx.x;
    float acc = 0.f;
    if (c < N)
        for (long r = (long)blockIdx.y * blockDim.y + threadIdx.y; r < M; r += (long)gridDim.y * blockDim.y)
            acc += x[r * ldx + c];
    __shared__ float sh[8][33];
    sh[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    float* part = ws + (long)blockIdx.x * gridDim.y * 32 + threadIdx.x;
    if (threadIdx.y == 0) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += sh[i][threadIdx.x];
        part[blockIdx.y * 32] = s;
    }
    if (pd_last_block(tickets + blockIdx.x, gridDim.y) && threadIdx.y == 0 && c < N) {
        float s = 0.f;
        for (unsigned b = 0; b < gridDim.y; ++b) s += __ldcg(part + b * 32);
        out[c] += s;
    }
}

__global__ void scalar_head_loss_kernel(long M, int kind, const float* __restrict__ y, const float* __restrict__ target,
                                        int div, float* __restrict__ loss, float* __restrict__ dy,
                                        float* __restrict__ rec) {
    GRID_STRIDE(i, M) {
        float yy = y[i], t = target[i / div];
        if (kind == 0) {
            float d = t - yy;
            loss[i] = 0.5f * d * d;
            dy[i] = -d;
            if (rec) rec[i] = yy;
        } else {
            // -Bernoulli(logits=y).log_prob(t) = BCEWithLogits = max(y,0) - y t + log1p(exp(-|y|))
            loss[i] = fmaxf(yy, 0.f) - yy * t + log1pf(expf(-fabsf(yy)));
            float s = pd_sigmoid(yy);
            dy[i] = s - t;
            if (rec) rec[i] = s;
        }
    }
}

// One warp per row: lane l sums the columns l, l + 32, ... in turn, then the lanes are added by a fixed xor tree, so the
// loss of a row does not depend on scheduling.
__global__ void vec_head_loss_kernel(long M, int K, const float* __restrict__ y, long ldy, const float* __restrict__ target,
                                     long ldt, int div, float* __restrict__ loss, float* __restrict__ dy, long lddy) {
    const int lane = threadIdx.x & 31;
    const long warps = (long)gridDim.x * (blockDim.x >> 5);
    for (long m = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); m < M; m += warps) {
        const float* yr = y + m * ldy;
        const float* tr = target + (m / div) * ldt;
        float s = 0.f;
        for (int k = lane; k < K; k += 32) {
            const float d = yr[k] - tr[k];
            dy[m * lddy + k] = d;
            s += d * d;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) loss[m] = 0.5f * s;
    }
}

// One warp per row, as vec_head_loss_kernel: lane l takes the columns l, l + 32, ... in turn and the lanes meet in a fixed
// xor tree (every lane ends with the same sums).  The target bucket compares (t - s_k)^2 rounded as torch computes it
// (a subtraction and a multiplication, no FMA contraction); a lane keeps its first minimum and the tree prefers the lower
// index on equal distances, so k* is the first index of the minimum, as torch.argmin returns.
__global__ void support_head_kernel(long M, int S, const float* __restrict__ y, long ldy, const float* __restrict__ sup,
                                    const float* __restrict__ target, int div, float* __restrict__ rec,
                                    float* __restrict__ loss, float* __restrict__ dy, long lddy, int* __restrict__ idx) {
    const int lane = threadIdx.x & 31;
    const long warps = (long)gridDim.x * (blockDim.x >> 5);
    for (long m = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); m < M; m += warps) {
        const float* yr = y + m * ldy;
        float mx = -INFINITY;
        for (int k = lane; k < S; k += 32) mx = fmaxf(mx, yr[k]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float z = 0.f, zs = 0.f;
        for (int k = lane; k < S; k += 32) {
            const float e = expf(yr[k] - mx);
            z += e;
            zs += e * sup[k];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            z += __shfl_xor_sync(0xffffffffu, z, o);
            zs += __shfl_xor_sync(0xffffffffu, zs, o);
        }
        if (rec && lane == 0) rec[m] = zs / z;
        if (!target) continue;
        const float t = target[m / div];
        float bd = 0.f;
        int bk = -1;
        for (int k = lane; k < S; k += 32) {
            const float d = __fsub_rn(t, sup[k]);
            const float q = __fmul_rn(d, d);
            if (bk < 0 || q < bd) { bd = q; bk = k; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(0xffffffffu, bd, o);
            const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
            if (ok >= 0 && (bk < 0 || od < bd || (od == bd && ok < bk))) { bd = od; bk = ok; }
        }
        bk = __shfl_sync(0xffffffffu, bk, 0);
        const float inv = 1.f / z;
        for (int k = lane; k < S; k += 32) dy[m * lddy + k] = expf(yr[k] - mx) * inv - (k == bk ? 1.f : 0.f);
        if (lane == 0) {
            loss[m] = (mx + logf(z)) - yr[bk];
            if (idx) idx[m] = bk;
        }
    }
}

__device__ __forceinline__ float neg_logavgexp_neg(const float* v, int I, int stride) {
    // -logavgexp(-v) over I entries (functions.py:97-102); exact passthrough for I == 1
    if (I == 1) return v[0];
    float mx = -INFINITY;
    for (int i = 0; i < I; ++i) mx = fmaxf(mx, -v[i * stride]);
    float s = 0.f;
    for (int i = 0; i < I; ++i) s += expf(-v[i * stride] - mx);
    return -(mx + logf(s) - logf((float)I));
}

__global__ void wm_loss_kernel(int TB, int I, float kl_weight, float w_img, float w_rew, float w_term,
                               const float* __restrict__ l_img, const float* __restrict__ l_rew,
                               const float* __restrict__ l_term, const float* __restrict__ l_kl,
                               const float* __restrict__ kl_exact, const float* __restrict__ ent_prior,
                               const float* __restrict__ ent_post, const float* __restrict__ l_vec, float w_vec,
                               float* __restrict__ w, float* __restrict__ tb) {
    GRID_STRIDE(r, TB) {
        const long b = r * I;
        float mx = -INFINITY;
        for (int i = 0; i < I; ++i) {
            const float li = l_img ? l_img[b + i] : 0.f;
            float L = kl_weight * l_kl[b + i] + w_img * li + w_rew * l_rew[b + i] + w_term * l_term[b + i];
            if (l_vec) L += w_vec * l_vec[b + i];
            w[b + i] = L;
            mx = fmaxf(mx, -L);
        }
        float loss;
        if (I == 1) {
            loss = w[b];
            w[b] = 1.f / (float)TB;
        } else {
            float s = 0.f;
            for (int i = 0; i < I; ++i) s += expf(-w[b + i] - mx);
            float lse = mx + logf(s);
            loss = -(lse - logf((float)I));
            for (int i = 0; i < I; ++i) w[b + i] = expf(-w[b + i] - lse) / (float)TB;
        }
        float ep = 0.f, eq = 0.f;
        for (int i = 0; i < I; ++i) { ep += ent_prior[b + i]; eq += ent_post[b + i]; }
        float* o = tb + r * 8;
        o[0] = loss;
        o[1] = l_img ? neg_logavgexp_neg(l_img + b, I, 1) : 0.f;
        o[2] = neg_logavgexp_neg(l_rew + b, I, 1);
        o[3] = neg_logavgexp_neg(l_term + b, I, 1);
        o[4] = neg_logavgexp_neg(kl_exact + b, I, 1);
        o[5] = ep / (float)I;
        o[6] = eq / (float)I;
        o[7] = l_vec ? neg_logavgexp_neg(l_vec + b, I, 1) : 0.f;
    }
}

// out[c] = mean_rows x[r,c], N <= 32, single block of 1024 threads (32 x 32)
__global__ void colmean_kernel(long M, int N, const float* __restrict__ x, float* __restrict__ out) {
    __shared__ float sh[32][33];
    int c = threadIdx.x, ry = threadIdx.y;
    float acc = 0.f;
    if (c < N) for (long r = ry; r < M; r += 32) acc += x[r * N + c];
    sh[ry][c] = acc;
    __syncthreads();
    if (ry == 0 && c < N) {
        float s = 0.f;
        for (int i = 0; i < 32; ++i) s += sh[i][c];
        out[c] = s / (float)M;
    }
}

// ------------------------------------------------------------------ actor-critic
// The loss sums in a fixed order: thread q < NQ of every block holds the block's partial q; the partials go to row
// blockIdx.x of the stream's scratch area and the last block adds them up (a double atomicAdd would add them in arrival
// order): thread t sums rows t, t + blockDim.x, ... in turn, then the warps and the block reduce in a fixed pattern.
template <int NQ>
__device__ __forceinline__ void sums_flush(double v, double* ws, unsigned* ticket, double* sums) {
    __shared__ double red[NQ][32];
    if (threadIdx.x < NQ) ws[(long)blockIdx.x * NQ + threadIdx.x] = v;
    if (!pd_last_block(ticket, gridDim.x)) return;
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        double s = 0;
        for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) s += __ldcg(ws + (long)b * NQ + q);
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[q][wp] = s;
    }
    __syncthreads();
    if (threadIdx.x < NQ) {
        double s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
        sums[threadIdx.x] += s;
    }
}

// Block-wide fixed-order sums of the NQ per-thread values vals[q], then sums_flush.
template <int NQ>
__device__ __forceinline__ void block_sums_flush(const double* vals, double* ws, unsigned* ticket, double* sums) {
    __shared__ double shd[NQ][8];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        double x = vals[q];
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) shd[q][wp] = x;
    }
    __syncthreads();
    double x = 0;
    if (threadIdx.x < NQ)
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) x += shd[threadIdx.x][i];
    sums_flush<NQ>(x, ws, ticket, sums);
}

constexpr int MAXJ = 128;
// The per-column recursion of a2c.py:88-116 over J = H + 1 rows of column m: GAE(lambda) from the target critic's values
// vt, the rewards rew[1:] and the terminals tm[1:] (values in [0, 1], held by the caller), the reality weight
// exp(cumsum(log(1 - tm[:-1]))) (a terminal of 1 gives log 0 = -inf: weight 0 there and after), and the critic loss
// 0.5 (target - v)^2 weight with dv = -(target - v) weight coef.  STORE writes adv, agae, target and weight (and reads
// the targets back from `target`); without it the targets stay in a local array.
// s += {sum loss, sum v[0], sum v[:-1], sum rew[1:], sum rew[1:]^2}.
template <bool STORE>
__device__ __forceinline__ void gae_column(int H, int Md, int m, float gamma, float lambda, const float* __restrict__ vt,
                                           const float* __restrict__ v, const float* __restrict__ rew, const float* tm,
                                           float coef, float* __restrict__ adv, float* __restrict__ agae,
                                           float* __restrict__ target, float* __restrict__ weight, float* __restrict__ dv,
                                           double (&s)[5]) {
    float tg[STORE ? 1 : MAXJ];
    float ag = 0.f;
    // reversed scan (a2c.py:94-101)
    for (int j = H - 1; j >= 0; --j) {
        float v0 = vt[(long)j * Md + m], v1 = vt[(long)(j + 1) * Md + m];
        float r1 = rew[(long)(j + 1) * Md + m];
        float a = -v0 + r1 + gamma * (1.0f - tm[j + 1]) * v1;
        ag = (j == H - 1) ? a : a + lambda * gamma * (1.0f - tm[j + 1]) * ag;
        if (STORE) {
            adv[(long)j * Md + m] = a;
            agae[(long)j * Md + m] = ag;
            target[(long)j * Md + m] = ag + v0;
        } else {
            tg[j] = ag + v0;
        }
        s[3] += r1; s[4] += (double)r1 * r1;
    }
    float cs = 0.f;
    for (int j = 0; j < H; ++j) {
        cs += logf(1.0f - tm[j]);                 // (1-terminal0).log().cumsum(0).exp()  a2c.py:108
        float w = expf(cs);
        if (STORE) weight[(long)j * Md + m] = w;
        float val = v[(long)j * Md + m];
        float d = (STORE ? target[(long)j * Md + m] : tg[j]) - val;
        s[0] += 0.5 * (double)d * d * w;
        dv[(long)j * Md + m] = -d * w * coef;
        s[2] += val;
        if (j == 0) s[1] += val;
    }
}

__global__ void gae_critic_kernel(int H, int Md, float gamma, float lambda, const float* __restrict__ vt,
                                  const float* __restrict__ v, const float* __restrict__ rew,
                                  const float* __restrict__ tl, float* __restrict__ term, float* __restrict__ adv,
                                  float* __restrict__ agae, float* __restrict__ target, float* __restrict__ weight,
                                  float* __restrict__ dv, double* sums, double* ws, unsigned* ticket) {
    double s[5] = {0, 0, 0, 0, 0};               // {loss, v0[0], v0, r1, r1^2}
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m < Md) {
        float tm[MAXJ];
        const int J = H + 1;
        for (int j = 0; j < J; ++j) { tm[j] = pd_sigmoid(tl[(long)j * Md + m]); term[(long)j * Md + m] = tm[j]; }
        const float inv = 1.f / ((float)H * (float)Md);
        gae_column<true>(H, Md, m, gamma, lambda, vt, v, rew, tm, inv, adv, agae, target, weight, dv, s);
    }
    block_sums_flush<5>(s, ws, ticket, sums);
}

// The same recursion over observed rewards and 0/1 terminals (the world model's auxiliary critic, dreamer.py:347-365):
// T = H + 1 rows of B columns, dv = scale * d loss / d v; sums[2] += {sum loss, sum v[:-1]}.
__global__ void gae_critic_obs_kernel(int H, int Md, float gamma, float lambda, const float* __restrict__ vt,
                                      const float* __restrict__ v, const float* __restrict__ rew,
                                      const float* __restrict__ term, float scale, float* __restrict__ dv, double* sums,
                                      double* ws, unsigned* ticket) {
    double s[5] = {0, 0, 0, 0, 0};
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m < Md) {
        float tm[MAXJ];
        for (int j = 0; j <= H; ++j) tm[j] = term[(long)j * Md + m];
        const float coef = scale / ((float)H * (float)Md);
        gae_column<false>(H, Md, m, gamma, lambda, vt, v, rew, tm, coef, nullptr, nullptr, nullptr, nullptr, dv, s);
    }
    const double vals[2] = {s[0], s[2]};
    block_sums_flush<2>(vals, ws, ticket, sums);
}

__global__ void __launch_bounds__(256)
actor_loss_onehot_kernel(long rows, int A, float eta, const float* __restrict__ logits, long ldl,
                         const float* __restrict__ actions, long lda, const float* __restrict__ agae,
                         const float* __restrict__ weight, float* __restrict__ dlogits, long lddl, double* sums,
                         double* ws, unsigned* ticket) {
    __shared__ double shd[2][8];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    long row = (long)blockIdx.x * 8 + wp;
    double s_loss = 0, s_ent = 0;
    if (row < rows) {
        bool valid = lane < A;
        float l = valid ? logits[row * ldl + lane] : 0.f;
        float mx = pd_warp_max(valid ? l : -INFINITY);
        float e = valid ? expf(l - mx) : 0.f;
        float lse = mx + logf(pd_warp_sum(e));
        float lp = valid ? l - lse : 0.f;
        float p = valid ? expf(lp) : 0.f;
        float a = valid ? actions[row * lda + lane] : -INFINITY;
        // OneHotCategorical.log_prob: index = argmax(value)
        float best = a; int k = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best, o);
            int ok = __shfl_xor_sync(0xffffffffu, k, o);
            if (ob > best || (ob == best && ok < k)) { best = ob; k = ok; }
        }
        float lpa = __shfl_sync(0xffffffffu, lp, k);
        float ent = -pd_warp_sum(valid ? p * lp : 0.f);
        float ag = agae[row], w = weight[row];
        float inv = 1.f / (float)rows;
        if (valid) {
            float oh = lane == k ? 1.f : 0.f;
            dlogits[row * lddl + lane] = w * inv * (-ag * (oh - p) + eta * p * (lp + ent));
        }
        if (lane == 0) { s_loss = (double)((-lpa * ag - eta * ent) * w); s_ent = ent; }
    }
    if (lane == 0) { shd[0][wp] = s_loss; shd[1][wp] = s_ent; }
    __syncthreads();
    double x = 0;
    if (threadIdx.x < 2)
        for (int i = 0; i < 8; ++i) x += shd[threadIdx.x][i];
    sums_flush<2>(x, ws, ticket, sums);
}

// The two Gaussian policies on out[rows, 2A] = (m, s) raw.  NT = false: tanh_normal (functions.py:69-78), the base
// Normal(5 tanh(m/5), softplus(s) + 0.1) under a TanhTransform, log_prob through atanh of the clamped action, entropy of
// the base distribution.  NT = true: normal_tanh (functions.py:59-66, min_std 0.01, max_std 1), Normal(tanh(m),
// sigmoid(s) + 0.01) with no transform, so the action is unbounded and the entropy is the Normal's own.
template <bool NT>
__global__ void actor_loss_gaussian_kernel(long rows, int A, float eta, const float* __restrict__ out, long ldo,
                                           const float* __restrict__ actions, long lda,
                                           const float* __restrict__ agae, const float* __restrict__ weight,
                                           float* __restrict__ dout, long lddo, double* sums, double* ws,
                                           unsigned* ticket) {
    __shared__ double shd[2][8];
    const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
    double s_loss = 0, s_ent = 0;
    if (row < rows) {
        const float ag = agae[row], w = weight[row], inv = 1.f / (float)rows;
        float lp = 0.f, ent = 0.f;
        const float eps = 1.1920928955078125e-07f;
        for (int i = 0; i < A; ++i) {
            float m_ = out[row * ldo + i], s_ = out[row * ldo + A + i];
            if constexpr (NT) {
                float mu = tanhf(m_);
                float sg = pd_sigmoid(s_);
                float sd = sg + 0.01f;
                float zc = (actions[row * lda + i] - mu) / sd;
                float lsd = logf(sd);
                lp += -0.5f * zc * zc - lsd - 0.9189385332046727f;
                ent += 0.5f + 0.9189385332046727f + lsd;
                dout[row * lddo + i] = w * inv * (-ag * (zc / sd)) * (1.f - mu * mu);
                dout[row * lddo + A + i] = w * inv * (-ag * ((zc * zc - 1.f) / sd) - eta / sd) * (sg * (1.f - sg));
            } else {
                float th = tanhf(m_ / 5.f);
                float mu = 5.f * th;
                float sd = pd_softplus(s_) + 0.1f;
                float y = fminf(fmaxf(actions[row * lda + i], -1.f + eps), 1.f - eps);
                float x = atanhf(y);
                float zc = (x - mu) / sd;
                // Normal.log_prob - TanhTransform.log_abs_det_jacobian
                float lpn = -0.5f * zc * zc - logf(sd) - 0.9189385332046727f;
                float ladj = 2.f * (0.6931471805599453f - x - pd_softplus(-2.f * x));
                lp += lpn - ladj;
                ent += 0.5f + 0.9189385332046727f + logf(sd);
                float dlp_dmu = zc / sd;
                float dlp_dsd = (zc * zc - 1.f) / sd;
                dout[row * lddo + i] = w * inv * (-ag * dlp_dmu) * (1.f - th * th);
                dout[row * lddo + A + i] = w * inv * (-ag * dlp_dsd - eta / sd) * pd_sigmoid(s_);
            }
        }
        s_loss = (double)((-lp * ag - eta * ent) * w);
        s_ent = ent;
    }
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        s_loss += __shfl_xor_sync(0xffffffffu, s_loss, o);
        s_ent += __shfl_xor_sync(0xffffffffu, s_ent, o);
    }
    if (lane == 0) { shd[0][wp] = s_loss; shd[1][wp] = s_ent; }
    __syncthreads();
    double x = 0;
    if (threadIdx.x < 2)
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) x += shd[threadIdx.x][i];
    sums_flush<2>(x, ws, ticket, sums);
}

template <bool NT>
__global__ void gaussian_sample_kernel(long rows, int A, const float* __restrict__ out, long ldo,
                                       const float* __restrict__ eps, float* __restrict__ action, long lda) {
    GRID_STRIDE(i, rows * A) {
        long r = i / A; int c = (int)(i % A);
        if constexpr (NT) {
            float sd = pd_sigmoid(out[r * ldo + A + c]) + 0.01f;
            action[r * lda + c] = tanhf(out[r * ldo + c]) + sd * eps[i];
        } else {
            float mu = 5.f * tanhf(out[r * ldo + c] / 5.f);
            float sd = pd_softplus(out[r * ldo + A + c]) + 0.1f;
            action[r * lda + c] = tanhf(mu + sd * eps[i]);
        }
    }
}

// ------------------------------------------------------------------ optimizer
// Sum of squares in a FIXED summation order (block partials to a workspace, then one block adds them up): data-parallel
// replicas compute the clip coefficient from bit-identical all-reduced gradients and must get bit-identical norms, or the
// replicas drift apart by an ulp per clipped step (an atomicAdd over blocks sums in arrival order).
__global__ void sumsq_partial_kernel(const float* __restrict__ x, long n, float* __restrict__ partial) {
    __shared__ float sh[33];
    float acc = 0.f;
    GRID_STRIDE(i, n) { float v = x[i]; acc += v * v; }
    float s = pd_block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}
__global__ void sumsq_final_kernel(const float* __restrict__ partial, int np, float* out) {
    __shared__ float sh[33];
    float acc = 0.f;
    for (int i = threadIdx.x; i < np; i += blockDim.x) acc += partial[i];
    float s = pd_block_sum(acc, sh);
    if (threadIdx.x == 0) *out += s;
}
__global__ void clip_scale_kernel(float* __restrict__ x, long n, const float* __restrict__ sumsq, float max_norm,
                                  float* norm_out) {
    const float norm = sqrtf(*sumsq);
    float coef = max_norm / (norm + 1e-6f);
    coef = coef > 1.f ? 1.f : coef;
    GRID_STRIDE(i, n) x[i] *= coef;
    if (blockIdx.x == 0 && threadIdx.x == 0 && norm_out) *norm_out = norm;
}
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, long n, float lr, float b1, float b2, float eps, float wd,
                             const int32_t* __restrict__ step) {
    const double st = (double)(*step);
    const float bc1 = (float)(1.0 - pow((double)b1, st));
    const float bc2s = (float)sqrt(1.0 - pow((double)b2, st));
    const float step_size = lr / bc1;
    GRID_STRIDE(i, n) {
        float gi = g[i];
        float pi = p[i] * (1.f - lr * wd);
        float mi = m[i] + (gi - m[i]) * (1.f - b1);
        float vi = v[i] * b2 + (1.f - b2) * gi * gi;
        float denom = sqrtf(vi) / bc2s + eps;
        p[i] = pi - step_size * (mi / denom);
        m[i] = mi;
        v[i] = vi;
    }
}
__global__ void inc_kernel(int32_t* c) { *c += 1; }
// out[m, :] = W[idx[m], :]   (a Linear without bias applied to one-hot rows is a row gather of its transposed weight)
__global__ void gather_rows_kernel(long M, int N, const int32_t* __restrict__ idx, const float* __restrict__ W, long ldw,
                                   float* __restrict__ out, long ldo) {
    const int n4 = N >> 2;
    GRID_STRIDE(i, M * n4) {
        const long m = i / n4;
        const int c = (int)(i % n4) * 4;
        *reinterpret_cast<float4*>(out + m * ldo + c) = __ldg(reinterpret_cast<const float4*>(W + (long)idx[m] * ldw + c));
    }
}
// x *= alpha * (*scale), exact (no operand rounding); a factor of exactly 1 leaves x untouched, so the launch exits
// without touching memory (the usual loss.backward() hands over grad_output == 1)
__global__ void scale_by_kernel(float* __restrict__ x, long n, const float* __restrict__ scale, float alpha) {
    const float f = alpha * (scale ? *scale : 1.f);
    if (f == 1.f) return;
    GRID_STRIDE(i, n) x[i] *= f;
}

}  // namespace

extern "C" {

#define S(stream) ((cudaStream_t)(stream))

int pd_round_copy(pd_handle* h, const float* src, float* dst, long n, int round_out, void* stream) {
    round_copy_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(src, dst, n, round_out && h->round_ops);
    PD_CHECK_LAUNCH(h, "round_copy");
    return PD_OK;
}
int pd_pad_cols(pd_handle* h, long M, int C, int Cp, const float* src, long lds, float* dst, long ldd, void* stream) {
    pad_cols_kernel<<<grid_for(M * Cp, 256, h->num_sms), 256, 0, S(stream)>>>(M, C, Cp, src, lds, dst, ldd, h->round_ops);
    PD_CHECK_LAUNCH(h, "pad_cols");
    return PD_OK;
}
int pd_mask_rows(pd_handle* h, int M, int N, const float* x, long ldx, const float* mask, float* out, long ldo,
                 void* stream) {
    mask_rows_kernel<<<grid_for((long)M * N, 256, h->num_sms), 256, 0, S(stream)>>>(M, N, x, ldx, mask, out, ldo, h->round_ops);
    PD_CHECK_LAUNCH(h, "mask_rows");
    return PD_OK;
}
int pd_rowscale(pd_handle* h, long M, long N, float* x, long ldx, const float* scale, int scale_div, float alpha,
                void* stream) {
    rowscale_kernel<<<grid_for(M * N, 256, h->num_sms), 256, 0, S(stream)>>>(M, N, x, ldx, scale, scale_div > 0 ? scale_div : 1, alpha, h->round_ops);
    PD_CHECK_LAUNCH(h, "rowscale");
    return PD_OK;
}
int pd_group_sum(pd_handle* h, long R, int I, int W, const float* x, long ldx, float* out, long ldo, void* stream) {
    group_sum_kernel<<<grid_for(R * W, 256, h->num_sms), 256, 0, S(stream)>>>(R, I, W, x, ldx, out, ldo, h->round_ops);
    PD_CHECK_LAUNCH(h, "group_sum");
    return PD_OK;
}
int pd_colsum(pd_handle* h, long M, int N, const float* x, long ldx, float* out, void* stream) {
    dim3 block(32, 8);
    long gy = (M + 63) / 64;
    long cap = (long)h->num_sms * 8 / ((N + 31) / 32);
    if (cap < 1) cap = 1;
    if (gy > cap) gy = cap;
    dim3 grid((N + 31) / 32, (unsigned)gy);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), (long)grid.x * grid.y * 32, (int)grid.x, &ws, &tk);
    if (rc) return rc;
    colsum_kernel<<<grid, block, 0, S(stream)>>>(M, N, x, ldx, out, ws, tk);
    PD_CHECK_LAUNCH(h, "colsum");
    return PD_OK;
}
int pd_to_half(pd_handle* h, long M, long N, const float* src, long lds, void* dst, long ldd, void* stream) {
    to_half_kernel<<<grid_for(M * N, 256, h->num_sms), 256, 0, S(stream)>>>(M, N, src, lds, (__half*)dst, ldd);
    PD_CHECK_LAUNCH(h, "to_half");
    return PD_OK;
}
int pd_transpose_to_half(pd_handle* h, int M, int N, const float* src, long lds, void* dst, long ldd, void* stream) {
    dim3 grid((N + 31) / 32, (M + 31) / 32), block(32, 8);
    transpose_to_half_kernel<<<grid, block, 0, S(stream)>>>(M, N, src, lds, (__half*)dst, ldd);
    PD_CHECK_LAUNCH(h, "transpose_to_half");
    return PD_OK;
}
int pd_fill(pd_handle* h, float* x, long n, float v, void* stream) {
    fill_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(x, n, v);
    PD_CHECK_LAUNCH(h, "fill");
    return PD_OK;
}
int pd_reset_mask(pd_handle* h, int T, int B, int I, const uint8_t* reset, float* mask, void* stream) {
    reset_mask_kernel<<<grid_for((long)T * B * I, 256, h->num_sms), 256, 0, S(stream)>>>(T, B, I, reset, mask);
    PD_CHECK_LAUNCH(h, "reset_mask");
    return PD_OK;
}
int pd_scalar_head_loss(pd_handle* h, long M, int kind, const float* y, const float* target, int tgt_div, float* loss,
                        float* dy, float* rec, void* stream) {
    scalar_head_loss_kernel<<<grid_for(M, 256, h->num_sms), 256, 0, S(stream)>>>(M, kind, y, target, tgt_div > 0 ? tgt_div : 1, loss, dy, rec);
    PD_CHECK_LAUNCH(h, "scalar_head_loss");
    return PD_OK;
}
int pd_vec_head_loss(pd_handle* h, long M, int K, const float* y, long ldy, const float* target, long ldt, int tgt_div,
                     float* loss, float* dy, long lddy, void* stream) {
    PD_REQUIRE(h, M >= 0 && K >= 1 && K <= PD_VEC_HEAD_MAX_K && ldy >= K && ldt >= K && lddy >= K && tgt_div >= 1,
               "pd_vec_head_loss: K=%d (1..%d), ldy=%ld ldt=%ld lddy=%ld (>= K), tgt_div=%d (>= 1) unsupported", K,
               PD_VEC_HEAD_MAX_K, ldy, ldt, lddy, tgt_div);
    if (M == 0) return PD_OK;
    vec_head_loss_kernel<<<grid_for(M, 8, h->num_sms), 256, 0, S(stream)>>>(M, K, y, ldy, target, ldt, tgt_div, loss, dy, lddy);
    PD_CHECK_LAUNCH(h, "vec_head_loss");
    return PD_OK;
}
int pd_support_head(pd_handle* h, long M, int S, const float* y, long ldy, const float* support, const float* target,
                    int tgt_div, float* rec, float* loss, float* dy, long lddy, int* idx, void* stream) {
    PD_REQUIRE(h, M >= 0 && S >= 2 && S <= PD_SUPPORT_MAX && ldy >= S && tgt_div >= 1 && y && support,
               "pd_support_head: S=%d (2..%d), ldy=%ld (>= S), tgt_div=%d (>= 1) unsupported", S, PD_SUPPORT_MAX, ldy,
               tgt_div);
    PD_REQUIRE(h, target ? (loss && dy && lddy >= S) : (rec != nullptr),
               "pd_support_head: a target needs loss and dy (lddy=%ld >= S), no target needs rec", lddy);
    if (M == 0) return PD_OK;
    support_head_kernel<<<grid_for(M, 8, h->num_sms), 256, 0, S(stream)>>>(M, S, y, ldy, support, target, tgt_div, rec,
                                                                           loss, dy, lddy, idx);
    PD_CHECK_LAUNCH(h, "support_head");
    return PD_OK;
}
int pd_wm_loss(pd_handle* h, int TB, int I, float kl_weight, float w_img, float w_rew, float w_term, const float* l_img,
               const float* l_rew, const float* l_term, const float* l_kl, const float* kl_exact,
               const float* ent_prior, const float* ent_post, const float* l_vec, float w_vec, float* w, float* tb,
               void* stream) {
    wm_loss_kernel<<<grid_for(TB, 128, h->num_sms), 128, 0, S(stream)>>>(TB, I, kl_weight, w_img, w_rew, w_term, l_img, l_rew, l_term, l_kl, kl_exact, ent_prior, ent_post, l_vec, w_vec, w, tb);
    PD_CHECK_LAUNCH(h, "wm_loss");
    return PD_OK;
}
int pd_colmean(pd_handle* h, long M, int N, const float* x, float* out, void* stream) {
    PD_REQUIRE(h, N >= 1 && N <= 32, "pd_colmean: N=%d unsupported", N);
    colmean_kernel<<<1, dim3(32, 32), 0, S(stream)>>>(M, N, x, out);
    PD_CHECK_LAUNCH(h, "colmean");
    return PD_OK;
}
int pd_gae_critic(pd_handle* h, int H, int Md, float gamma, float lambda, const float* vt, const float* v,
                  const float* rew, const float* term_logit, float* term, float* adv, float* agae, float* target,
                  float* weight, float* dv, double* sums, void* stream) {
    PD_REQUIRE(h, H >= 1 && H + 1 <= MAXJ, "pd_gae_critic: H=%d unsupported (<%d)", H, MAXJ);
    const int grid = pd_cdiv(Md, 128);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), 2L * grid * 5, 1, &ws, &tk);          // grid x 5 doubles
    if (rc) return rc;
    gae_critic_kernel<<<grid, 128, 0, S(stream)>>>(H, Md, gamma, lambda, vt, v, rew, term_logit, term, adv, agae, target, weight, dv, sums,
                                                   (double*)ws, tk);
    PD_CHECK_LAUNCH(h, "gae_critic");
    return PD_OK;
}
int pd_gae_critic_obs(pd_handle* h, int T, int B, float gamma, float lambda, const float* vt, const float* v,
                      const float* rew, const float* term, float scale, float* dv, double* sums, void* stream) {
    PD_REQUIRE(h, T >= 2 && T <= MAXJ && B >= 1 && vt && v && rew && term && dv && sums,
               "pd_gae_critic_obs: T=%d (2..%d), B=%d (>= 1) unsupported or a NULL pointer", T, MAXJ, B);
    const int grid = pd_cdiv(B, 128);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), 2L * grid * 2, 1, &ws, &tk);          // grid x 2 doubles
    if (rc) return rc;
    gae_critic_obs_kernel<<<grid, 128, 0, S(stream)>>>(T - 1, B, gamma, lambda, vt, v, rew, term, scale, dv, sums,
                                                       (double*)ws, tk);
    PD_CHECK_LAUNCH(h, "gae_critic_obs");
    return PD_OK;
}
int pd_actor_loss_onehot(pd_handle* h, long rows, int A, float eta, const float* logits, long ldl, const float* actions,
                         long lda, const float* agae, const float* weight, float* dlogits, long lddl, double* sums,
                         void* stream) {
    PD_REQUIRE(h, A >= 1 && A <= 32, "pd_actor_loss_onehot: A=%d unsupported (<=32)", A);
    const int grid = pd_cdiv(rows, 8);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), 2L * grid * 2, 1, &ws, &tk);          // grid x 2 doubles
    if (rc) return rc;
    actor_loss_onehot_kernel<<<grid, 256, 0, S(stream)>>>(rows, A, eta, logits, ldl, actions, lda, agae, weight, dlogits, lddl, sums,
                                                          (double*)ws, tk);
    PD_CHECK_LAUNCH(h, "actor_loss_onehot");
    return PD_OK;
}
int pd_actor_loss_tanh_normal(pd_handle* h, long rows, int A, float eta, const float* out, long ldo,
                              const float* actions, long lda, const float* agae, const float* weight, float* dout,
                              long lddo, double* sums, void* stream) {
    const int grid = pd_cdiv(rows, 256);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), 2L * grid * 2, 1, &ws, &tk);          // grid x 2 doubles
    if (rc) return rc;
    actor_loss_gaussian_kernel<false><<<grid, 256, 0, S(stream)>>>(rows, A, eta, out, ldo, actions, lda, agae, weight, dout,
                                                                   lddo, sums, (double*)ws, tk);
    PD_CHECK_LAUNCH(h, "actor_loss_tanh_normal");
    return PD_OK;
}
int pd_tanh_normal_sample(pd_handle* h, long rows, int A, const float* out, long ldo, const float* eps, float* action,
                          long lda, void* stream) {
    gaussian_sample_kernel<false><<<grid_for(rows * A, 256, h->num_sms), 256, 0, S(stream)>>>(rows, A, out, ldo, eps, action,
                                                                                              lda);
    PD_CHECK_LAUNCH(h, "tanh_normal_sample");
    return PD_OK;
}
int pd_actor_loss_normal_tanh(pd_handle* h, long rows, int A, float eta, const float* out, long ldo,
                              const float* actions, long lda, const float* agae, const float* weight, float* dout,
                              long lddo, double* sums, void* stream) {
    PD_REQUIRE(h, rows >= 0 && A >= 1 && ldo >= 2L * A && lda >= A && lddo >= 2L * A,
               "pd_actor_loss_normal_tanh: rows=%ld (>= 0), A=%d (>= 1), ldo=%ld / lddo=%ld (>= 2A), lda=%ld (>= A) "
               "unsupported", rows, A, ldo, lddo, lda);
    if (rows == 0) return PD_OK;
    const int grid = pd_cdiv(rows, 256);
    float* ws;
    unsigned* tk;
    int rc = pd_scratch(h, S(stream), 2L * grid * 2, 1, &ws, &tk);          // grid x 2 doubles
    if (rc) return rc;
    actor_loss_gaussian_kernel<true><<<grid, 256, 0, S(stream)>>>(rows, A, eta, out, ldo, actions, lda, agae, weight, dout,
                                                                  lddo, sums, (double*)ws, tk);
    PD_CHECK_LAUNCH(h, "actor_loss_normal_tanh");
    return PD_OK;
}
int pd_normal_tanh_sample(pd_handle* h, long rows, int A, const float* out, long ldo, const float* eps, float* action,
                          long lda, void* stream) {
    PD_REQUIRE(h, rows >= 0 && A >= 1 && ldo >= 2L * A && lda >= A,
               "pd_normal_tanh_sample: rows=%ld (>= 0), A=%d (>= 1), ldo=%ld (>= 2A), lda=%ld (>= A) unsupported",
               rows, A, ldo, lda);
    if (rows == 0) return PD_OK;
    gaussian_sample_kernel<true><<<grid_for(rows * A, 256, h->num_sms), 256, 0, S(stream)>>>(rows, A, out, ldo, eps, action,
                                                                                             lda);
    PD_CHECK_LAUNCH(h, "normal_tanh_sample");
    return PD_OK;
}
int pd_sumsq(pd_handle* h, const float* x, long n, float* out, float* ws, void* stream) {
    PD_REQUIRE(h, ws, "pd_sumsq: workspace of pd_sumsq_ws_floats() floats required");
    int grid = grid_for(n, 256, h->num_sms);
    if (grid > 4 * h->num_sms) grid = 4 * h->num_sms;
    sumsq_partial_kernel<<<grid, 256, 0, S(stream)>>>(x, n, ws);
    PD_CHECK_LAUNCH(h, "sumsq_partial");
    sumsq_final_kernel<<<1, 256, 0, S(stream)>>>(ws, grid, out);
    PD_CHECK_LAUNCH(h, "sumsq_final");
    return PD_OK;
}
int pd_sumsq_ws_floats(const pd_handle* h) { return h ? 4 * h->num_sms : 0; }
int pd_clip_scale(pd_handle* h, float* x, long n, const float* sumsq, float max_norm, float* norm_out, void* stream) {
    clip_scale_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(x, n, sumsq, max_norm, norm_out);
    PD_CHECK_LAUNCH(h, "clip_scale");
    return PD_OK;
}
int pd_adamw(pd_handle* h, float* p, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2,
             float eps, float wd, const int32_t* step, void* stream) {
    adamw_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps, wd, step);
    PD_CHECK_LAUNCH(h, "adamw");
    return PD_OK;
}
int pd_scale_by(pd_handle* h, float* x, long n, const float* scale, float alpha, void* stream) {
    scale_by_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(x, n, scale, alpha);
    PD_CHECK_LAUNCH(h, "scale_by");
    return PD_OK;
}
int pd_gather_rows(pd_handle* h, long M, int N, const int32_t* idx, const float* W, long ldw, float* out, long ldo,
                   void* stream) {
    PD_REQUIRE(h, (N % 4) == 0 && (ldw % 4) == 0 && (ldo % 4) == 0 && ((((uintptr_t)W) | ((uintptr_t)out)) & 15) == 0,
               "pd_gather_rows: N, ldw, ldo must be multiples of 4 and the buffers 16-byte aligned");
    gather_rows_kernel<<<grid_for(M * (N / 4), 256, h->num_sms), 256, 0, S(stream)>>>(M, N, idx, W, ldw, out, ldo);
    PD_CHECK_LAUNCH(h, "gather_rows");
    return PD_OK;
}
int pd_inc(pd_handle* h, int32_t* counter, void* stream) {
    inc_kernel<<<1, 1, 0, S(stream)>>>(counter);
    PD_CHECK_LAUNCH(h, "inc");
    return PD_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ replay preprocessing on the device (SURVEY.md §8f N3)
namespace {
// image uint8 (T*B, H, W, C) -> fp32 (T*B, C, H, W) = x / 255 - 0.5   (preprocessing.py:21-29 to_image)
__global__ void image_u8_to_f32_kernel(long NB, int H, int W, int C, const uint8_t* __restrict__ src, float* __restrict__ dst) {
    const long plane = (long)H * W;
    GRID_STRIDE(i, NB * C * plane) {
        long n = i / (C * plane);
        long r = i - n * C * plane;
        int c = (int)(r / plane);
        long yx = r - (long)c * plane;
        dst[i] = __fdiv_rn((float)src[(n * plane + yx) * C + c], 255.0f) - 0.5f;
    }
}
// action index (int64) -> one-hot fp32 (preprocessing.py:135-138 to_onehot); reward -> tanh clip (functions.py:153-160)
__global__ void onehot_i64_kernel(long rows, int A, const long long* __restrict__ idx, float* __restrict__ out) {
    GRID_STRIDE(i, rows * A) {
        long r = i / A; int c = (int)(i - r * A);
        out[i] = (idx[r] == c) ? 1.f : 0.f;
    }
}
__global__ void tanh_kernel(long n, const float* __restrict__ x, float* __restrict__ y) {
    GRID_STRIDE(i, n) y[i] = tanhf(x[i]);
}
}  // namespace

extern "C" {
int pd_image_u8_to_f32(pd_handle* h, long NB, int H, int W, int C, const uint8_t* src, float* dst, void* stream) {
    image_u8_to_f32_kernel<<<grid_for(NB * C * H * W, 256, h->num_sms), 256, 0, S(stream)>>>(NB, H, W, C, src, dst);
    PD_CHECK_LAUNCH(h, "image_u8_to_f32");
    return PD_OK;
}
int pd_onehot_i64(pd_handle* h, long rows, int A, const int64_t* idx, float* out, void* stream) {
    onehot_i64_kernel<<<grid_for(rows * A, 256, h->num_sms), 256, 0, S(stream)>>>(rows, A, (const long long*)idx, out);
    PD_CHECK_LAUNCH(h, "onehot_i64");
    return PD_OK;
}
int pd_tanh(pd_handle* h, long n, const float* x, float* y, void* stream) {
    tanh_kernel<<<grid_for(n, 256, h->num_sms), 256, 0, S(stream)>>>(n, x, y);
    PD_CHECK_LAUNCH(h, "tanh");
    return PD_OK;
}
}

// pd_rowwise.cu — row-structured kernels of the RSSM / MLP path:
//   LayerNorm+ELU (fwd/bwd), GRU cell gates (fwd/bwd), categorical straight-through sampling
//   (fwd/bwd), KL(post||prior) with balancing.  All are HBM/latency-bound: one warp owns a row
//   (or a 32-class group), lanes stride the contiguous dimension so every global access is a
//   coalesced 128 B line, reductions are warp shuffles.
#include "pd_common.cuh"
#include <cuda_fp16.h>

namespace {

// ------------------------------------------------------------------ LayerNorm + ELU forward
template <int MAXV>
__global__ void __launch_bounds__(128)
ln_elu_fwd_kernel(int M, int N, const float* __restrict__ x, long ldx, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float eps, float* __restrict__ y, long ldy,
                  float* __restrict__ mean_out, float* __restrict__ rstd_out, int round_out, __half* __restrict__ y16,
                  long ldy16) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= M) return;
    const float* xr = x + (long)row * ldx;
    float v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        int c = lane + 32 * i;
        v[i] = c < N ? xr[c] : 0.f;
        s += v[i];
    }
    const float mean = pd_warp_sum(s) / (float)N;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        int c = lane + 32 * i;
        float d = c < N ? v[i] - mean : 0.f;
        q += d * d;
    }
    const float var = pd_warp_sum(q) / (float)N;
    const float rstd = 1.0f / sqrtf(var + eps);
    float* yr = y + (long)row * ldy;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        int c = lane + 32 * i;
        if (c < N) {
            float t = pd_round_if(pd_elu((v[i] - mean) * rstd * gamma[c] + beta[c]), round_out);
            yr[c] = t;
            if (y16) y16[(long)row * ldy16 + c] = __float2half_rn(t);
        }
    }
    if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
}

// ------------------------------------------------------------------ LayerNorm + ELU backward
template <int MAXV>
__global__ void __launch_bounds__(128)
ln_elu_bwd_kernel(int M, int N, const float* __restrict__ dy, long lddy, const float* __restrict__ x, long ldx,
                  const float* __restrict__ y, long ldy, const float* __restrict__ gamma,
                  const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float* __restrict__ dx,
                  long lddx, float* dgamma, float* dbeta, float* dbias, int round_out, float* ws, unsigned* tickets) {
    __shared__ float sh[3][32 * MAXV];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x; c < 32 * MAXV; c += 128) { sh[0][c] = 0.f; sh[1][c] = 0.f; sh[2][c] = 0.f; }
    __syncthreads();
    float pg[MAXV], pb[MAXV], px[MAXV], gam[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        pg[i] = pb[i] = px[i] = 0.f;
        int c = lane + 32 * i;
        gam[i] = c < N ? gamma[c] : 0.f;
    }
    for (int row = blockIdx.x * 4 + warp; row < M; row += gridDim.x * 4) {
        const float mean = mean_in[row], rstd = rstd_in[row];
        const float* xr = x + (long)row * ldx;
        const float* yr = y + (long)row * ldy;
        const float* dyr = dy + (long)row * lddy;
        float xh[MAXV], dxh[MAXV];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            int c = lane + 32 * i;
            if (c < N) {
                float g = dyr[c] * pd_elu_grad_from_out(yr[c]);
                xh[i] = (xr[c] - mean) * rstd;
                pg[i] += g * xh[i];
                pb[i] += g;
                dxh[i] = g * gam[i];
                s1 += dxh[i];
                s2 += dxh[i] * xh[i];
            } else { xh[i] = 0.f; dxh[i] = 0.f; }
        }
        const float c1 = pd_warp_sum(s1) / (float)N;
        const float c2 = pd_warp_sum(s2) / (float)N;
        float* dxr = dx + (long)row * lddx;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            int c = lane + 32 * i;
            if (c < N) {
                float d = rstd * (dxh[i] - c1 - xh[i] * c2);
                px[i] += d;
                dxr[c] = pd_round_if(d, round_out);
            }
        }
    }
    // parameter gradients in a fixed order: the four warps in turn into shared memory, the block's partials to
    // ws[block][3][N], the last block adds them up in block order
    for (int w = 0; w < 4; ++w) {
        if (warp == w) {
#pragma unroll
            for (int i = 0; i < MAXV; ++i) {
                sh[0][lane + 32 * i] += pg[i];
                sh[1][lane + 32 * i] += pb[i];
                sh[2][lane + 32 * i] += px[i];
            }
        }
        __syncthreads();
    }
    float* part = ws + (long)blockIdx.x * 3 * N;
    for (int c = threadIdx.x; c < N; c += 128) {
        part[c] = sh[0][c]; part[N + c] = sh[1][c]; part[2 * N + c] = sh[2][c];
    }
    if (pd_last_block(tickets, gridDim.x)) {
        for (int c = threadIdx.x; c < N; c += 128) {
            float g = 0.f, b = 0.f, d = 0.f;
            for (unsigned k = 0; k < gridDim.x; ++k) {
                const float* p = ws + (long)k * 3 * N;
                g += __ldcg(p + c); b += __ldcg(p + N + c); d += __ldcg(p + 2 * N + c);
            }
            dgamma[c] += g; dbeta[c] += b;
            if (dbias) dbias[c] += d;
        }
    }
}

// ------------------------------------------------------------------ LayerNorm + ELU, few rows (one RSSM timestep)
// With M = B*I = 50 rows a warp-per-row kernel exposes only 50 warps of parallelism and a long per-lane dependency
// chain; here a whole 256-thread block owns a row (<= 4 elements per thread, two block reductions).
__global__ void __launch_bounds__(256)
ln_elu_fwd_row_kernel(int N, const float* __restrict__ x, long ldx, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float eps, float* __restrict__ y, long ldy,
                      float* __restrict__ mean_out, float* __restrict__ rstd_out, int round_out, __half* __restrict__ y16,
                      long ldy16) {
    __shared__ float sh[33];
    const int row = blockIdx.x, t = threadIdx.x;
    const float* xr = x + (long)row * ldx;
    float v[4], s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { int c = t + 256 * i; v[i] = c < N ? xr[c] : 0.f; s += v[i]; }
    const float mean = pd_block_sum(s, sh) / (float)N;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { int c = t + 256 * i; float d = c < N ? v[i] - mean : 0.f; q += d * d; }
    const float rstd = 1.0f / sqrtf(pd_block_sum(q, sh) / (float)N + eps);
    float* yr = y + (long)row * ldy;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int c = t + 256 * i;
        if (c < N) {
            float t = pd_round_if(pd_elu((v[i] - mean) * rstd * gamma[c] + beta[c]), round_out);
            yr[c] = t;
            if (y16) y16[(long)row * ldy16 + c] = __float2half_rn(t);
        }
    }
    if (t == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
}

__global__ void __launch_bounds__(256)
ln_elu_bwd_row_kernel(int N, const float* __restrict__ dy, long lddy, const float* __restrict__ x, long ldx,
                      const float* __restrict__ y, long ldy, const float* __restrict__ gamma,
                      const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float* __restrict__ dx,
                      long lddx, float* dgamma, float* dbeta, float* dbias, int round_out, float* ws,
                      unsigned* tickets) {
    __shared__ float sh[33];
    const int row = blockIdx.x, t = threadIdx.x;
    const float mean = mean_in[row], rstd = rstd_in[row];
    float g[4], xh[4], dxh[4], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int c = t + 256 * i;
        if (c < N) {
            g[i] = dy[(long)row * lddy + c] * pd_elu_grad_from_out(y[(long)row * ldy + c]);
            xh[i] = (x[(long)row * ldx + c] - mean) * rstd;
            dxh[i] = g[i] * gamma[c];
            s1 += dxh[i]; s2 += dxh[i] * xh[i];
        } else { g[i] = xh[i] = dxh[i] = 0.f; }
    }
    const float c1 = pd_block_sum(s1, sh) / (float)N;
    const float c2 = pd_block_sum(s2, sh) / (float)N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int c = t + 256 * i;
        if (c < N) {
            float d = rstd * (dxh[i] - c1 - xh[i] * c2);
            dx[(long)row * lddx + c] = pd_round_if(d, round_out);
            float* part = ws + (long)row * 3 * N;            // this row's parameter-gradient terms
            part[c] = g[i] * xh[i]; part[N + c] = g[i]; part[2 * N + c] = d;
        }
    }
    if (pd_last_block(tickets, gridDim.x)) {                 // the last row block adds all rows' terms in row order
        for (int c = t; c < N; c += 256) {
            float sg = 0.f, sb = 0.f, sd = 0.f;
            for (unsigned r = 0; r < gridDim.x; ++r) {
                const float* p = ws + (long)r * 3 * N;
                sg += __ldcg(p + c); sb += __ldcg(p + N + c); sd += __ldcg(p + 2 * N + c);
            }
            dgamma[c] += sg; dbeta[c] += sb;
            if (dbias) dbias[c] += sd;
        }
    }
}

// ------------------------------------------------------------------ GRU gates
__global__ void gru_fwd_kernel(int M, int D, const float* __restrict__ gi, long ldgi, const float* __restrict__ gh,
                               long ldgh, const float* __restrict__ hprev, long ldh, float* __restrict__ hout,
                               long ldho, float* __restrict__ hmask, long ldhm, const float* __restrict__ mask_next,
                               float* __restrict__ gates, int round_out, __half* __restrict__ h16, long ldh16) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)M * D) return;
    int m = (int)(idx / D), j = (int)(idx % D);
    const float* gim = gi + (long)m * ldgi;
    const float* ghm = gh + (long)m * ldgh;
    float r = pd_sigmoid(gim[j] + ghm[j]);
    float u = pd_sigmoid(gim[D + j] + ghm[D + j]);
    float ghn = ghm[2 * D + j];
    float n = tanhf(gim[2 * D + j] + r * ghn);
    float hp = hprev[(long)m * ldh + j];
    float hn = pd_round_if((1.f - u) * n + u * hp, round_out);
    hout[(long)m * ldho + j] = hn;
    if (h16) h16[(long)m * ldh16 + j] = __float2half_rn(hn);
    if (hmask) hmask[(long)m * ldhm + j] = hn * mask_next[m];
    if (gates) {
        float* g = gates + (long)m * 4 * D;
        g[j] = r; g[D + j] = u; g[2 * D + j] = n; g[3 * D + j] = ghn;
    }
}

__global__ void gru_bwd_kernel(int M, int D, const float* __restrict__ dh_a, long ldda, const float* __restrict__ dh_b,
                               long lddb, const float* __restrict__ mask_b, const float* __restrict__ gates,
                               const float* __restrict__ hprev, long ldh, float* __restrict__ dgi, long lddgi,
                               float* __restrict__ dgh, long lddgh, float* __restrict__ dh_carry, long lddc,
                               int round_out) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)M * D) return;
    int m = (int)(idx / D), j = (int)(idx % D);
    float dh = 0.f;
    if (dh_a) dh += dh_a[(long)m * ldda + j];
    if (dh_b) dh += dh_b[(long)m * lddb + j] * (mask_b ? mask_b[m] : 1.f);
    const float* g = gates + (long)m * 4 * D;
    float r = g[j], u = g[D + j], n = g[2 * D + j], ghn = g[3 * D + j];
    float hp = hprev[(long)m * ldh + j];
    float dn_pre = dh * (1.f - u) * (1.f - n * n);
    float du_pre = dh * (hp - n) * u * (1.f - u);
    float dr_pre = dn_pre * ghn * r * (1.f - r);
    float* a = dgi + (long)m * lddgi;
    float* b = dgh + (long)m * lddgh;
    a[j] = pd_round_if(dr_pre, round_out);
    a[D + j] = pd_round_if(du_pre, round_out);
    a[2 * D + j] = pd_round_if(dn_pre, round_out);
    b[j] = a[j];
    b[D + j] = a[D + j];
    b[2 * D + j] = pd_round_if(dn_pre * r, round_out);
    dh_carry[(long)m * lddc + j] = dh * u;
}

// ------------------------------------------------------------------ categorical sampling
// One warp per (row, group); lane = class.  Arithmetic follows torch's CUDA path:
// logits - logsumexp, softmax of that, argmax(p / q).
__device__ __forceinline__ void group_softmax(float l, bool valid, float& ln, float& p) {
    float mx = pd_warp_max(valid ? l : -INFINITY);
    float e = valid ? expf(l - mx) : 0.f;
    float lse = mx + logf(pd_warp_sum(e));
    ln = valid ? l - lse : -INFINITY;
    float mx2 = pd_warp_max(ln);
    float e2 = valid ? expf(ln - mx2) : 0.f;
    p = e2 / pd_warp_sum(e2);
}

__global__ void __launch_bounds__(256)
cat_sample_kernel(long groups, int G, int C, const float* __restrict__ logits, long ldl,
                  const float* __restrict__ noise, long ldn, float* __restrict__ z, long ldz,
                  float* __restrict__ zmask, long ldzm, const float* __restrict__ mask_next,
                  int32_t* __restrict__ idx, __half* __restrict__ z16, long ldz16) {
    const int lane = threadIdx.x & 31;
    long gid = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (gid >= groups) return;
    long m = gid / G;
    int g = (int)(gid % G);
    bool valid = lane < C;
    float l = valid ? logits[m * ldl + (long)g * C + lane] : 0.f;
    float ln, p;
    group_softmax(l, valid, ln, p);
    float q = valid ? noise[m * ldn + (long)g * C + lane] : 1.f;
    float val = valid ? p / q : -INFINITY;
    int k = lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, val, o);
        int ok = __shfl_xor_sync(0xffffffffu, k, o);
        if (ov > val || (ov == val && ok < k)) { val = ov; k = ok; }
    }
    if (valid) {
        float zz = (lane == k) ? 1.f : 0.f;
        z[m * ldz + (long)g * C + lane] = zz;
        if (z16) z16[m * ldz16 + (long)g * C + lane] = __float2half_rn(zz);
        if (zmask) zmask[m * ldzm + (long)g * C + lane] = zz * mask_next[m];
    }
    if (idx && lane == 0) idx[m * G + g] = k;
}

__global__ void __launch_bounds__(256)
cat_st_bwd_kernel(long groups, int G, int C, const float* __restrict__ logits, long ldl,
                  const float* __restrict__ dz_a, long ldda, const float* __restrict__ dz_b, long lddb,
                  const float* __restrict__ mask_b, const float* __restrict__ extra, long ldex,
                  const float* __restrict__ rowscale, float alpha, float* __restrict__ dlogits, long lddl,
                  int round_out) {
    const int lane = threadIdx.x & 31;
    long gid = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (gid >= groups) return;
    long m = gid / G;
    int g = (int)(gid % G);
    bool valid = lane < C;
    long off = (long)g * C + lane;
    float l = valid ? logits[m * ldl + off] : 0.f;
    float ln, p;
    group_softmax(l, valid, ln, p);
    float dz = 0.f;
    if (valid) {
        if (dz_a) dz += dz_a[m * ldda + off];
        if (dz_b) dz += dz_b[m * lddb + off] * (mask_b ? mask_b[m] : 1.f);
    }
    float s = pd_warp_sum(valid ? p * dz : 0.f);
    if (valid) {
        float d = p * (dz - s);
        if (extra) d += alpha * (rowscale ? rowscale[m] : 1.f) * extra[m * ldex + off];
        dlogits[m * lddl + off] = pd_round_if(d, round_out);
    }
}

// ------------------------------------------------------------------ KL(post || prior)
// One block per row, one warp per group (G <= 32), lane = class (C <= 32).
__global__ void kl_kernel(int M, int G, int C, const float* __restrict__ post, long ldpo,
                          const float* __restrict__ prior, long ldpr, const int32_t* __restrict__ idx, int mode,
                          float wpost, float wprior, float* __restrict__ loss_kl, float* __restrict__ kl_exact,
                          float* __restrict__ ent_post, float* __restrict__ ent_prior, float* __restrict__ dpost,
                          long lddpo, float* __restrict__ dprior, long lddpr) {
    __shared__ float sh[4][32];
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int m = blockIdx.x;
    bool valid = lane < C;
    long off = (long)g * C + lane;
    float lp, p, lq, q;
    group_softmax(valid ? post[(long)m * ldpo + off] : 0.f, valid, lp, p);
    group_softmax(valid ? prior[(long)m * ldpr + off] : 0.f, valid, lq, q);
    // torch: kl = sum p*(lp-lq) with p==0 -> 0 ; entropy = -sum p*clamp(lp, finfo.min)
    float t = (valid && p > 0.f) ? p * (lp - lq) : 0.f;
    float kl = pd_warp_sum(t);
    float hp = -pd_warp_sum(valid ? p * fmaxf(lp, -3.4028234663852886e38f) : 0.f);
    float hq = -pd_warp_sum(valid ? q * fmaxf(lq, -3.4028234663852886e38f) : 0.f);
    float lk = kl;
    if (mode == 0) {
        if (valid) {
            dpost[(long)m * lddpo + off] = wpost * p * ((lp - lq) - kl);
            dprior[(long)m * lddpr + off] = wprior * (q - p);
        }
    } else {
        int k = idx[(long)m * G + g];
        float sel = pd_warp_sum((valid && lane == k) ? (lp - lq) : 0.f);
        lk = sel;
        if (valid) {
            float oh = lane == k ? 1.f : 0.f;
            dpost[(long)m * lddpo + off] = oh - p;
            dprior[(long)m * lddpr + off] = q - oh;
        }
    }
    if (lane == 0) { sh[0][g] = lk; sh[1][g] = kl; sh[2][g] = hp; sh[3][g] = hq; }
    __syncthreads();
    if (g == 0) {
        float a = lane < G ? sh[0][lane] : 0.f, b = lane < G ? sh[1][lane] : 0.f;
        float c = lane < G ? sh[2][lane] : 0.f, d = lane < G ? sh[3][lane] : 0.f;
        a = pd_warp_sum(a); b = pd_warp_sum(b); c = pd_warp_sum(c); d = pd_warp_sum(d);
        if (lane == 0) { loss_kl[m] = a; kl_exact[m] = b; ent_post[m] = c; ent_prior[m] = d; }
    }
}

}  // namespace

extern "C" {

int pd_ln_elu_fwd(pd_handle* h, int M, int N, const float* x, long ldx, const float* gamma, const float* beta,
                  float eps, float* y, long ldy, float* mean, float* rstd, void* y16, long ldy16, void* stream) {
    PD_REQUIRE(h, N >= 1 && N <= 1024, "pd_ln_elu_fwd: N=%d unsupported (1..1024)", N);
    cudaStream_t s = (cudaStream_t)stream;
    if (M <= 256) {
        ln_elu_fwd_row_kernel<<<M, 256, 0, s>>>(N, x, ldx, gamma, beta, eps, y, ldy, mean, rstd, h->round_ops, (__half*)y16, ldy16);
        PD_CHECK_LAUNCH(h, "ln_elu_fwd_row");
        return PD_OK;
    }
    int grid = pd_cdiv(M, 4);
    if (N <= 416) ln_elu_fwd_kernel<13><<<grid, 128, 0, s>>>(M, N, x, ldx, gamma, beta, eps, y, ldy, mean, rstd, h->round_ops, (__half*)y16, ldy16);
    else          ln_elu_fwd_kernel<32><<<grid, 128, 0, s>>>(M, N, x, ldx, gamma, beta, eps, y, ldy, mean, rstd, h->round_ops, (__half*)y16, ldy16);
    PD_CHECK_LAUNCH(h, "ln_elu_fwd");
    return PD_OK;
}

int pd_ln_elu_bwd(pd_handle* h, int M, int N, const float* dy, long lddy, const float* x, long ldx, const float* y,
                  long ldy, const float* gamma, const float* mean, const float* rstd, float* dx, long lddx,
                  float* dgamma, float* dbeta, float* dbias, void* stream) {
    PD_REQUIRE(h, N >= 1 && N <= 1024, "pd_ln_elu_bwd: N=%d unsupported (1..1024)", N);
    cudaStream_t s = (cudaStream_t)stream;
    float* ws;
    unsigned* tk;
    if (M <= 256) {
        int rc = pd_scratch(h, s, (long)M * 3 * N, 1, &ws, &tk);
        if (rc) return rc;
        ln_elu_bwd_row_kernel<<<M, 256, 0, s>>>(N, dy, lddy, x, ldx, y, ldy, gamma, mean, rstd, dx, lddx, dgamma, dbeta,
                                               dbias, h->round_ops, ws, tk);
        PD_CHECK_LAUNCH(h, "ln_elu_bwd_row");
        return PD_OK;
    }
    int grid = pd_cdiv(M, 4);
    int cap = 2 * h->num_sms;
    if (grid > cap) grid = cap;
    int rc = pd_scratch(h, s, (long)grid * 3 * N, 1, &ws, &tk);
    if (rc) return rc;
    if (N <= 416) ln_elu_bwd_kernel<13><<<grid, 128, 0, s>>>(M, N, dy, lddy, x, ldx, y, ldy, gamma, mean, rstd, dx, lddx, dgamma, dbeta, dbias, h->round_ops, ws, tk);
    else          ln_elu_bwd_kernel<32><<<grid, 128, 0, s>>>(M, N, dy, lddy, x, ldx, y, ldy, gamma, mean, rstd, dx, lddx, dgamma, dbeta, dbias, h->round_ops, ws, tk);
    PD_CHECK_LAUNCH(h, "ln_elu_bwd");
    return PD_OK;
}

int pd_gru_fwd(pd_handle* h, int M, int D, const float* gi, long ldgi, const float* gh, long ldgh, const float* hprev,
               long ldh, float* hout, long ldho, float* hmask, long ldhm, const float* mask_next, float* gates,
               void* h16, long ldh16, void* stream) {
    PD_REQUIRE(h, !hmask || mask_next, "pd_gru_fwd: hmask needs mask_next");
    long n = (long)M * D;
    gru_fwd_kernel<<<pd_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(M, D, gi, ldgi, gh, ldgh, hprev, ldh, hout, ldho,
                                                                    hmask, ldhm, mask_next, gates, h->round_ops,
                                                                    (__half*)h16, ldh16);
    PD_CHECK_LAUNCH(h, "gru_fwd");
    return PD_OK;
}

int pd_gru_bwd(pd_handle* h, int M, int D, const float* dh_a, long ldda, const float* dh_b, long lddb,
               const float* mask_b, const float* gates, const float* hprev, long ldh, float* dgi, long lddgi,
               float* dgh, long lddgh, float* dh_carry, long lddc, void* stream) {
    long n = (long)M * D;
    gru_bwd_kernel<<<pd_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(M, D, dh_a, ldda, dh_b, lddb, mask_b, gates, hprev,
                                                                    ldh, dgi, lddgi, dgh, lddgh, dh_carry, lddc,
                                                                    h->round_ops);
    PD_CHECK_LAUNCH(h, "gru_bwd");
    return PD_OK;
}

int pd_cat_sample(pd_handle* h, int M, int G, int C, const float* logits, long ldl, const float* noise, long ldn,
                  float* z, long ldz, float* zmask, long ldzm, const float* mask_next, int32_t* idx, void* z16, long ldz16,
                  void* stream) {
    PD_REQUIRE(h, C >= 1 && C <= 32, "pd_cat_sample: C=%d unsupported (<=32)", C);
    PD_REQUIRE(h, !zmask || mask_next, "pd_cat_sample: zmask needs mask_next");
    long groups = (long)M * G;
    cat_sample_kernel<<<pd_cdiv(groups, 8), 256, 0, (cudaStream_t)stream>>>(groups, G, C, logits, ldl, noise, ldn, z, ldz,
                                                                          zmask, ldzm, mask_next, idx, (__half*)z16,
                                                                          ldz16);
    PD_CHECK_LAUNCH(h, "cat_sample");
    return PD_OK;
}

int pd_cat_st_bwd(pd_handle* h, int M, int G, int C, const float* logits, long ldl, const float* dz_a, long ldda,
                  const float* dz_b, long lddb, const float* mask_b, const float* extra, long ldex,
                  const float* rowscale, float alpha, float* dlogits, long lddl, void* stream) {
    PD_REQUIRE(h, C >= 1 && C <= 32, "pd_cat_st_bwd: C=%d unsupported (<=32)", C);
    long groups = (long)M * G;
    cat_st_bwd_kernel<<<pd_cdiv(groups, 8), 256, 0, (cudaStream_t)stream>>>(groups, G, C, logits, ldl, dz_a, ldda, dz_b,
                                                                          lddb, mask_b, extra, ldex, rowscale, alpha,
                                                                          dlogits, lddl, h->round_ops);
    PD_CHECK_LAUNCH(h, "cat_st_bwd");
    return PD_OK;
}

int pd_kl(pd_handle* h, int M, int G, int C, const float* post, long ldpo, const float* prior, long ldpr,
          const int32_t* idx, int mode, float balance, float* loss_kl, float* kl_exact, float* ent_post,
          float* ent_prior, float* dpost, long lddpo, float* dprior, long lddpr, void* stream) {
    PD_REQUIRE(h, C >= 1 && C <= 32 && G >= 1 && G <= 32, "pd_kl: G=%d C=%d unsupported (<=32)", G, C);
    PD_REQUIRE(h, mode == 0 || idx, "pd_kl: mode 1 needs idx");
    float wpost = balance < 0.f ? 1.f : 1.f - balance;
    float wprior = balance < 0.f ? 1.f : balance;
    kl_kernel<<<M, 32 * G, 0, (cudaStream_t)stream>>>(M, G, C, post, ldpo, prior, ldpr, idx, mode, wpost, wprior, loss_kl,
                                                     kl_exact, ent_post, ent_prior, dpost, lddpo, dprior, lddpr);
    PD_CHECK_LAUNCH(h, "kl");
    return PD_OK;
}

}  // extern "C"

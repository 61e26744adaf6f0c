// pd_conv.cu — data movement for the stride-2 conv encoder / transposed-conv decoder
// (encoders.py:72-96, decoders.py:111-180).  The contractions themselves run on pd_gemm;
// these kernels build its operands (im2col) and fold its outputs (col2im), with bias, ELU,
// the image MSE loss and layout permutes fused in.  All HBM-bound: thread <-> one output
// element with the channel index fastest so that global accesses coalesce.
#include "pd_common.cuh"
#include <cuda_fp16.h>

namespace {

__global__ void im2col_kernel(long total, int Hout, int Wout, int Cc, int k, int korder,
                              const float* __restrict__ in, long sN, long sY, long sX, long sC,
                              float* __restrict__ col, long ldcol, int round_out) {
    const int KK = k * k * Cc;
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        long row = idx / KK;
        int kidx = (int)(idx % KK);
        int ox = (int)(row % Wout);
        long t = row / Wout;
        int oy = (int)(t % Hout);
        long n = t / Hout;
        int c, kh, kw;
        if (korder == 0) { c = kidx % Cc; int r = kidx / Cc; kw = r % k; kh = r / k; }
        else             { kw = kidx % k; int r = kidx / k; kh = r % k; c = r / k; }
        float v = in[n * sN + (long)(2 * oy + kh) * sY + (long)(2 * ox + kw) * sX + (long)c * sC];
        col[row * ldcol + kidx] = pd_round_if(v, round_out);
    }
}

// Planar (NCHW-like, sX == 1) input: one thread moves the k contiguous x-taps of one (row, channel, kh): the first
// conv layer (image NCHW) and the last deconv layer's backward (error image NCHW).
template <int K_>
__global__ void im2col_planar_kernel(long total, int Hout, int Wout, int Cc, int korder, const float* __restrict__ in,
                                     long sN, long sY, long sC, float* __restrict__ col, long ldcol, int round_out) {
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        int kh = (int)(idx % K_);
        long t = idx / K_;
        int c = (int)(t % Cc);
        long row = t / Cc;
        int ox = (int)(row % Wout);
        long t2 = row / Wout;
        int oy = (int)(t2 % Hout);
        long n = t2 / Hout;
        const float* src = in + n * sN + (long)c * sC + (long)(2 * oy + kh) * sY + 2 * ox;
        float v[K_];
#pragma unroll
        for (int j = 0; j < K_; j += 2) {                       // 2*ox is even: 8-byte aligned pairs
            const float2 p = *reinterpret_cast<const float2*>(src + j);
            v[j] = pd_round_if(p.x, round_out); v[j + 1] = pd_round_if(p.y, round_out);
        }
        float* dst = col + row * ldcol;
        if (korder == 1) {
#pragma unroll
            for (int j = 0; j < K_; ++j) dst[(c * K_ + kh) * K_ + j] = v[j];
        } else {
#pragma unroll
            for (int j = 0; j < K_; ++j) dst[(kh * K_ + j) * Cc + c] = v[j];
        }
    }
}

// NHWC fast path: one thread moves 4 consecutive channels (16 B) of one tap.
__global__ void __launch_bounds__(256)
im2col_v4_kernel(long total4, int Hout, int Wout, int C4, int k, const float* __restrict__ in,
                 long sN, long sY, long sX, float* __restrict__ col, long ldcol, int round_out) {
    // 4 independent 16-byte moves per thread per iteration (loads issued before the stores) keep enough bytes in flight
    // to approach HBM bandwidth; consecutive threads take consecutive 16-byte chunks.
    const int KK4 = k * k * C4;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long base = (long)blockIdx.x * blockDim.x + threadIdx.x; base < total4; base += 4 * stride) {
        float4 v[4];
        long dsto[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const long idx = base + u * stride;
            dsto[u] = -1;
            if (idx < total4) {
                long row = idx / KK4;
                int kidx = (int)(idx - row * KK4);
                int c4 = kidx % C4;
                int r = kidx / C4;
                int kw = r % k, kh = r / k;
                int ox = (int)(row % Wout);
                long t = row / Wout;
                int oy = (int)(t % Hout);
                long n = t / Hout;
                v[u] = __ldg(reinterpret_cast<const float4*>(in + n * sN + (long)(2 * oy + kh) * sY +
                                                             (long)(2 * ox + kw) * sX + c4 * 4));
                dsto[u] = row * ldcol + (long)kidx * 4;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (dsto[u] >= 0) {
                float4 w = v[u];
                if (round_out) { w.x = pd_tf32(w.x); w.y = pd_tf32(w.y); w.z = pd_tf32(w.z); w.w = pd_tf32(w.w); }
                *reinterpret_cast<float4*>(col + dsto[u]) = w;
            }
        }
    }
}

// four consecutive channels of a column-matrix row as float4 (fp32 or fp16 storage)
__device__ __forceinline__ float4 ld_col4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld_col4(const __half* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float ld_col1(const float* p) { return *p; }
__device__ __forceinline__ float ld_col1(const __half* p) { return __half2float(*p); }

template <typename TC>
__global__ void col2im_v4_kernel(long total4, int Hin, int Win, int Hout, int Wout, int C4, int k,
                                 const TC* __restrict__ col, long ldcol, const float* __restrict__ bias, int act,
                                 int round_out, float* __restrict__ out, long sN, long sY, long sX) {
    const int Cc = C4 * 4;
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total4; idx += (long)gridDim.x * blockDim.x) {
        int c4 = (int)(idx % C4);
        long t = idx / C4;
        int x = (int)(t % Wout);
        t /= Wout;
        int y = (int)(t % Hout);
        long n = t / Hout;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 tap[9];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int kh = (y & 1) + 2 * a;
            const int iy = (y - kh) >> 1;
            const bool oky = kh < k && iy >= 0 && iy < Hin;
#pragma unroll
            for (int bq = 0; bq < 3; ++bq) {
                const int kw = (x & 1) + 2 * bq;
                const int ix = (x - kw) >> 1;
                tap[a * 3 + bq] = (oky && kw < k && ix >= 0 && ix < Win)
                    ? ld_col4(col + ((n * Hin + iy) * Win + ix) * ldcol + (long)(kh * k + kw) * Cc + c4 * 4)
                    : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) { acc.x += tap[i].x; acc.y += tap[i].y; acc.z += tap[i].z; acc.w += tap[i].w; }
        if (bias) {
            const float4 b = *reinterpret_cast<const float4*>(bias + c4 * 4);
            acc.x += b.x; acc.y += b.y; acc.z += b.z; acc.w += b.w;
        }
        if (act == PD_ACT_ELU) { acc.x = pd_elu(acc.x); acc.y = pd_elu(acc.y); acc.z = pd_elu(acc.z); acc.w = pd_elu(acc.w); }
        if (round_out) { acc.x = pd_tf32(acc.x); acc.y = pd_tf32(acc.y); acc.z = pd_tf32(acc.z); acc.w = pd_tf32(acc.w); }
        *reinterpret_cast<float4*>(out + n * sN + (long)y * sY + (long)x * sX + c4 * 4) = acc;
    }
}

// Conv2d input gradient folded back from its column form AND taken through the ELU of the layer below in one pass
// (encoders.py:80-90 backward): out = fold(col) * elu'(dact), dbias[c] += sum over pixels — what pd_col2im followed by
// pd_bias_act_bwd do in two passes over the gradient image.  out / dact: contiguous NHWC.  192 threads per block and
// 192 % (Cc / 4) == 0: a thread keeps its channel quad over the grid-stride loop, so the bias sums stay in registers.
__global__ void __launch_bounds__(192) col2im_actbwd_kernel(long total4, int Hin, int Win, int Hout, int Wout, int C4, int k,
                                                           const float* __restrict__ col, long ldcol,
                                                           const float* __restrict__ dact, int round_out,
                                                           float* __restrict__ out, float* dbias, float* ws,
                                                           unsigned* tickets) {
    const int Cc = C4 * 4;
    const int c4 = threadIdx.x % C4;
    float4 bs = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total4; idx += (long)gridDim.x * blockDim.x) {
        long t = idx / C4;
        const long pix = t;
        int x = (int)(t % Wout);
        t /= Wout;
        int y = (int)(t % Hout);
        long n = t / Hout;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 tap[9];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int kh = (y & 1) + 2 * a;
            const int iy = (y - kh) >> 1;
            const bool oky = kh < k && iy >= 0 && iy < Hin;
#pragma unroll
            for (int bq = 0; bq < 3; ++bq) {
                const int kw = (x & 1) + 2 * bq;
                const int ix = (x - kw) >> 1;
                tap[a * 3 + bq] = (oky && kw < k && ix >= 0 && ix < Win)
                    ? ld_col4(col + ((n * Hin + iy) * Win + ix) * ldcol + (long)(kh * k + kw) * Cc + c4 * 4)
                    : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        const float4 yv = *reinterpret_cast<const float4*>(dact + pix * Cc + c4 * 4);
#pragma unroll
        for (int i = 0; i < 9; ++i) { acc.x += tap[i].x; acc.y += tap[i].y; acc.z += tap[i].z; acc.w += tap[i].w; }
        acc.x *= pd_elu_grad_from_out(yv.x); acc.y *= pd_elu_grad_from_out(yv.y);
        acc.z *= pd_elu_grad_from_out(yv.z); acc.w *= pd_elu_grad_from_out(yv.w);
        bs.x += acc.x; bs.y += acc.y; bs.z += acc.z; bs.w += acc.w;
        if (round_out) { acc.x = pd_tf32(acc.x); acc.y = pd_tf32(acc.y); acc.z = pd_tf32(acc.z); acc.w = pd_tf32(acc.w); }
        *reinterpret_cast<float4*>(out + pix * Cc + c4 * 4) = acc;
    }
    if (!dbias) return;
    __shared__ float4 sh[192];
    sh[threadIdx.x] = bs;
    __syncthreads();
    if (threadIdx.x < C4) {                    // block partials -> ws[block][Cc]; the last block adds them in block order
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int m = threadIdx.x; m < 192; m += C4) { s4.x += sh[m].x; s4.y += sh[m].y; s4.z += sh[m].z; s4.w += sh[m].w; }
        *reinterpret_cast<float4*>(ws + (long)blockIdx.x * Cc + c4 * 4) = s4;
    }
    if (pd_last_block(tickets, gridDim.x)) {
        for (int c = threadIdx.x; c < Cc; c += blockDim.x) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(ws + (long)b * Cc + c);
            dbias[c] += s;
        }
    }
}

__device__ __forceinline__ float col2im_gather(const float* __restrict__ col, long ldcol, long n, int y, int x, int c,
                                               int Hin, int Win, int Cc, int k) {
    float acc = 0.f;
    for (int kh = y & 1; kh < k; kh += 2) {
        int iy = (y - kh) >> 1;
        if (iy < 0) break;
        if (iy >= Hin) continue;
        for (int kw = x & 1; kw < k; kw += 2) {
            int ix = (x - kw) >> 1;
            if (ix < 0) break;
            if (ix >= Win) continue;
            acc += col[((n * Hin + iy) * Win + ix) * ldcol + (long)(kh * k + kw) * Cc + c];
        }
    }
    return acc;
}

__global__ void col2im_kernel(long total, int Hin, int Win, int Hout, int Wout, int Cc, int k,
                              const float* __restrict__ col, long ldcol, const float* __restrict__ bias, int act,
                              int round_out, float* __restrict__ out, long sN, long sY, long sX, long sC) {
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        int c = (int)(idx % Cc);
        long t = idx / Cc;
        int x = (int)(t % Wout);
        t /= Wout;
        int y = (int)(t % Hout);
        long n = t / Hout;
        float v = col2im_gather(col, ldcol, n, y, x, c, Hin, Win, Cc, k);
        if (bias) v += bias[c];
        if (act == PD_ACT_ELU) v = pd_elu(v);
        out[n * sN + (long)y * sY + (long)x * sX + (long)c * sC] = pd_round_if(v, round_out);
    }
}

// One block per decoded image: NCHW traversal (x fastest) for coalesced dec/target/diff access.  A thread folds ALL
// channels of its output pixel in one pass over the (pixel, tap) pieces of the column matrix (Cc <= 4: the decoder's
// last layer has 1 or 3), so every 32-byte sector of `col` is fetched once instead of once per channel
// (r02 ncu: 3.15 GB of DRAM reads for a 0.97 GB column matrix with the channel-outer loop).
template <int CMAX, typename TC>
__global__ void __launch_bounds__(256)
col2im_imgloss_kernel(int Hin, int Win, int Hout, int Wout, int Cc, int k, const TC* __restrict__ col, long ldcol,
                      const float* __restrict__ bias, const float* __restrict__ target, int tgt_div,
                      float* __restrict__ dec, float* __restrict__ diff, float* __restrict__ loss,
                      float* __restrict__ csum) {
    __shared__ float sh[33];
    const long n = blockIdx.x;
    const int plane = Hout * Wout;
    const int per = Cc * plane;
    const float* tg = target + (n / tgt_div) * (long)per;
    float acc = 0.f;
    float cacc[CMAX], bv[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c) { cacc[c] = 0.f; bv[c] = c < Cc ? bias[c] : 0.f; }
    for (int i = threadIdx.x; i < plane; i += blockDim.x) {
        const int x = i % Wout;
        const int y = i / Wout;
        float v[CMAX];
#pragma unroll
        for (int c = 0; c < CMAX; ++c) v[c] = 0.f;
        for (int kh = y & 1; kh < k; kh += 2) {                 // same tap order as col2im_gather (bit-identical sums)
            const int iy = (y - kh) >> 1;
            if (iy < 0) break;
            if (iy >= Hin) continue;
            for (int kw = x & 1; kw < k; kw += 2) {
                const int ix = (x - kw) >> 1;
                if (ix < 0) break;
                if (ix >= Win) continue;
                const TC* p = col + ((n * Hin + iy) * Win + ix) * ldcol + (long)(kh * k + kw) * Cc;
#pragma unroll
                for (int c = 0; c < CMAX; ++c)
                    if (c < Cc) v[c] += ld_col1(p + c);
            }
        }
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
            if (c < Cc) {
                const float o = v[c] + bv[c];
                const float d = o - tg[c * plane + i];
                dec[n * per + c * plane + i] = o;
                diff[n * per + c * plane + i] = d;
                acc += d * d;
                cacc[c] += d;
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CMAX; ++c) {
        const float cs = pd_block_sum(cacc[c], sh);             // uniform trip count: every thread takes part
        if (c < Cc && threadIdx.x == 0) csum[n * Cc + c] = cs;
    }
    float s = pd_block_sum(acc, sh);
    if (threadIdx.x == 0) loss[n] = 0.5f * s;
}

// dy <- dy * act'(y);  db[c] += sum_rows.  blockDim = (32, 8): a warp owns 32 consecutive columns; the blocks of one
// column group (blockIdx.x) write their partials to ws and the last of them adds them to db in blockIdx.y order.
__global__ void bias_act_bwd_kernel(long M, int N, float* __restrict__ dy, long lddy, const float* __restrict__ y,
                                    long ldy, int act, float* db, int round_out, float* ws, unsigned* tickets) {
    const int c = blockIdx.x * 32 + threadIdx.x;
    float acc = 0.f;
    if (c < N) {
        for (long r = (long)blockIdx.y * blockDim.y + threadIdx.y; r < M; r += (long)gridDim.y * blockDim.y) {
            float g = dy[r * lddy + c];
            if (act == PD_ACT_ELU) {
                g *= pd_elu_grad_from_out(y[r * ldy + c]);
                dy[r * lddy + c] = pd_round_if(g, round_out);
            }
            acc += g;
        }
    }
    if (!db) return;
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
        db[c] += s;
    }
}

struct Perm4 { int d[4]; long so[4]; long si[4]; };   // d: dims of `in`; so[a] / si[a]: stride in `out` / `in` of in-axis a

__global__ void permute4_kernel(long total, Perm4 p, const float* __restrict__ in, float* __restrict__ out,
                                int accumulate, int round_out) {
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        long t = idx;
        int i3 = (int)(t % p.d[3]); t /= p.d[3];
        int i2 = (int)(t % p.d[2]); t /= p.d[2];
        int i1 = (int)(t % p.d[1]); t /= p.d[1];
        int i0 = (int)t;
        long o = i0 * p.so[0] + i1 * p.so[1] + i2 * p.so[2] + i3 * p.so[3];
        float v = in[i0 * p.si[0] + i1 * p.si[1] + i2 * p.si[2] + i3 * p.si[3]];
        if (accumulate) out[o] += v;
        else out[o] = pd_round_if(v, round_out);
    }
}

inline int grid_for(long total, int block, int num_sms) {
    long g = (total + block - 1) / block;
    long cap = (long)num_sms * 32;
    return (int)(g < cap ? g : cap);
}

}  // namespace

extern "C" {

int pd_im2col(pd_handle* h, int NB, int Hin, int Win, int Cc, int k, int korder, const float* in, long sN, long sY,
              long sX, long sC, float* col, long ldcol, int round_out, void* stream) {
    PD_REQUIRE(h, Hin >= k && Win >= k, "pd_im2col: input %dx%d smaller than kernel %d", Hin, Win, k);
    int Hout = (Hin - k) / 2 + 1, Wout = (Win - k) / 2 + 1;
    long total = (long)NB * Hout * Wout * k * k * Cc;
    const bool v4 = korder == 0 && sC == 1 && (Cc % 4) == 0 && (sN % 4) == 0 && (sY % 4) == 0 && (sX % 4) == 0 &&
                    (ldcol % 4) == 0 && ((((uintptr_t)in) | ((uintptr_t)col)) & 15) == 0;
    if (v4) {
        im2col_v4_kernel<<<grid_for(total / 16 + 1, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
            total / 4, Hout, Wout, Cc / 4, k, in, sN, sY, sX, col, ldcol, round_out && h->round_ops);
        PD_CHECK_LAUNCH(h, "im2col_v4");
        return PD_OK;
    }
    const bool planar = sX == 1 && (k == 4 || k == 6) && (sN % 2) == 0 && (sY % 2) == 0 && (sC % 2) == 0 &&
                        ((((uintptr_t)in)) & 7) == 0;
    if (planar) {
        long tp = total / k;
        if (k == 4)
            im2col_planar_kernel<4><<<grid_for(tp, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
                tp, Hout, Wout, Cc, korder, in, sN, sY, sC, col, ldcol, round_out && h->round_ops);
        else
            im2col_planar_kernel<6><<<grid_for(tp, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
                tp, Hout, Wout, Cc, korder, in, sN, sY, sC, col, ldcol, round_out && h->round_ops);
        PD_CHECK_LAUNCH(h, "im2col_planar");
        return PD_OK;
    }
    im2col_kernel<<<grid_for(total, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
        total, Hout, Wout, Cc, k, korder, in, sN, sY, sX, sC, col, ldcol, round_out && h->round_ops);
    PD_CHECK_LAUNCH(h, "im2col");
    return PD_OK;
}

int pd_col2im(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k, const float* col, long ldcol,
              const float* bias, int act, int round_out, float* out, long sN, long sY, long sX, long sC,
              void* stream) {
    return pd_col2im_t(h, NB, Hin, Win, Hout, Wout, Cc, k, col, ldcol, 0, bias, act, round_out, out, sN, sY, sX, sC, stream);
}

int pd_col2im_t(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k, const void* colv, long ldcol,
                int col_f16, const float* bias, int act, int round_out, float* out, long sN, long sY, long sX, long sC,
                void* stream) {
    long total = (long)NB * Hout * Wout * Cc;
    if (col_f16) {
        const __half* colh = (const __half*)colv;
        PD_REQUIRE(h, sC == 1 && (Cc % 4) == 0 && (sN % 4) == 0 && (sY % 4) == 0 && (sX % 4) == 0 && (ldcol % 4) == 0 &&
                       ((((uintptr_t)out) & 15) == 0) && ((((uintptr_t)colh) & 7) == 0) && (!bias || (((uintptr_t)bias) & 15) == 0),
                   "pd_col2im: the fp16 column matrix path needs channel counts / strides that are multiples of 4");
        col2im_v4_kernel<__half><<<grid_for(total / 4, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
            total / 4, Hin, Win, Hout, Wout, Cc / 4, k, colh, ldcol, bias, act, round_out && h->round_ops, out, sN, sY, sX);
        PD_CHECK_LAUNCH(h, "col2im_v4(f16)");
        return PD_OK;
    }
    const float* col = (const float*)colv;
    const bool v4 = sC == 1 && (Cc % 4) == 0 && (sN % 4) == 0 && (sY % 4) == 0 && (sX % 4) == 0 && (ldcol % 4) == 0 &&
                    ((((uintptr_t)out) | ((uintptr_t)col)) & 15) == 0 && (!bias || (((uintptr_t)bias) & 15) == 0);
    if (v4) {
        col2im_v4_kernel<float><<<grid_for(total / 4, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
            total / 4, Hin, Win, Hout, Wout, Cc / 4, k, col, ldcol, bias, act, round_out && h->round_ops, out, sN, sY, sX);
        PD_CHECK_LAUNCH(h, "col2im_v4");
        return PD_OK;
    }
    col2im_kernel<<<grid_for(total, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(
        total, Hin, Win, Hout, Wout, Cc, k, col, ldcol, bias, act, round_out && h->round_ops, out, sN, sY, sX, sC);
    PD_CHECK_LAUNCH(h, "col2im");
    return PD_OK;
}

int pd_col2im_actbwd(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k, const float* col, long ldcol,
                     const float* dact, float* dbias, float* out, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, col && dact && out && Cc >= 1 && k >= 1 && k <= 6, "pd_col2im_actbwd: bad arguments");
    PD_REQUIRE(h, Hout >= (Hin - 1) * 2 + k && Wout >= (Win - 1) * 2 + k, "pd_col2im_actbwd: output smaller than the fold");
    const long total = (long)NB * Hout * Wout * Cc;
    const bool fused = (Cc % 4) == 0 && (192 % (Cc / 4)) == 0 && (ldcol % 4) == 0 &&
                       ((((uintptr_t)out) | ((uintptr_t)col) | ((uintptr_t)dact)) & 15) == 0;
    if (!fused) {
        int rc = pd_col2im(h, NB, Hin, Win, Hout, Wout, Cc, k, col, ldcol, nullptr, PD_ACT_NONE, 0, out, (long)Hout * Wout * Cc,
                           (long)Wout * Cc, Cc, 1, stream);
        if (rc) return rc;
        return pd_bias_act_bwd(h, (long)NB * Hout * Wout, Cc, out, Cc, dact, Cc, PD_ACT_ELU, dbias, stream);
    }
    int grid = grid_for(total / 4, 192, h->num_sms);
    float* ws = nullptr;
    unsigned* tk = nullptr;
    if (dbias) {
        if ((long)grid * Cc > PD_SCRATCH_FLOATS) grid = (int)(PD_SCRATCH_FLOATS / Cc);   // grid-stride loop: any grid works
        int rc = pd_scratch(h, (cudaStream_t)stream, (long)grid * Cc, 1, &ws, &tk);
        if (rc) return rc;
    }
    col2im_actbwd_kernel<<<grid, 192, 0, (cudaStream_t)stream>>>(
        total / 4, Hin, Win, Hout, Wout, Cc / 4, k, col, ldcol, dact, h->round_ops, out, dbias, ws, tk);
    PD_CHECK_LAUNCH(h, "col2im_actbwd");
    return PD_OK;
}

int pd_col2im_imgloss(pd_handle* h, int NB, int Hin, int Win, int Cc, int k, const float* col, long ldcol,
                      const float* bias, const float* target, int tgt_div, float* dec, float* diff, float* loss,
                      float* csum, void* stream) {
    return pd_col2im_imgloss_t(h, NB, Hin, Win, Cc, k, col, ldcol, 0, bias, target, tgt_div, dec, diff, loss, csum, stream);
}

int pd_col2im_imgloss_t(pd_handle* h, int NB, int Hin, int Win, int Cc, int k, const void* col, long ldcol, int col_f16,
                        const float* bias, const float* target, int tgt_div, float* dec, float* diff, float* loss,
                        float* csum, void* stream) {
    int Hout = (Hin - 1) * 2 + k, Wout = (Win - 1) * 2 + k;
    PD_REQUIRE(h, Cc >= 1 && Cc <= 16, "pd_col2im_imgloss: %d image channels (1..16 supported)", Cc);
    const int div = tgt_div > 0 ? tgt_div : 1;
    cudaStream_t s = (cudaStream_t)stream;
#define PD_IMGLOSS(CM, TC) col2im_imgloss_kernel<CM, TC><<<NB, 256, 0, s>>>(Hin, Win, Hout, Wout, Cc, k, (const TC*)col, ldcol, bias, target, div, dec, diff, loss, csum)
    if (col_f16) {
        if (Cc <= 4) PD_IMGLOSS(4, __half); else if (Cc <= 8) PD_IMGLOSS(8, __half); else PD_IMGLOSS(16, __half);
    } else {
        if (Cc <= 4) PD_IMGLOSS(4, float); else if (Cc <= 8) PD_IMGLOSS(8, float); else PD_IMGLOSS(16, float);
    }
#undef PD_IMGLOSS
    PD_CHECK_LAUNCH(h, "col2im_imgloss");
    return PD_OK;
}

int pd_bias_act_bwd(pd_handle* h, long M, int N, float* dy, long lddy, const float* y, long ldy, int act, float* db,
                    void* stream) {
    dim3 block(32, 8);
    long gy = (M + 63) / 64;
    long cap = (long)h->num_sms * 8 / ((N + 31) / 32);
    if (cap < 1) cap = 1;
    if (gy > cap) gy = cap;
    dim3 grid((N + 31) / 32, (unsigned)gy);
    float* ws = nullptr;
    unsigned* tk = nullptr;
    if (db) {
        int rc = pd_scratch(h, (cudaStream_t)stream, (long)grid.x * grid.y * 32, (int)grid.x, &ws, &tk);
        if (rc) return rc;
    }
    bias_act_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(M, N, dy, lddy, y, ldy, act, db, h->round_ops, ws, tk);
    PD_CHECK_LAUNCH(h, "bias_act_bwd");
    return PD_OK;
}

int pd_permute4(pd_handle* h, const float* in, float* out, const int* dims, const int* perm, const long* in_strides,
                int accumulate, int round_out, void* stream) {
    // out axis j takes in axis perm[j]; out is contiguous in its own (permuted) shape.
    Perm4 p;
    long ostride[4];
    long s = 1;
    for (int j = 3; j >= 0; --j) { ostride[j] = s; s *= dims[perm[j]]; }
    for (int a = 0; a < 4; ++a) p.d[a] = dims[a];
    for (int j = 0; j < 4; ++j) p.so[perm[j]] = ostride[j];
    {
        long st = 1;
        for (int a = 3; a >= 0; --a) { p.si[a] = in_strides ? in_strides[a] : st; st *= dims[a]; }
    }
    long total = (long)dims[0] * dims[1] * dims[2] * dims[3];
    permute4_kernel<<<grid_for(total, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(total, p, in, out, accumulate,
                                                                                      round_out && h->round_ops);
    PD_CHECK_LAUNCH(h, "permute4");
    return PD_OK;
}

}  // extern "C"

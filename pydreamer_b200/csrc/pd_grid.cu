// pd_grid.cu — the categorical grid-image front end (dense image encoder / CatImageDecoder, encoders.py:99-125,
// decoders.py:183-254, preprocessing.py:10-19): the one-hot conversion of category ids, the encoder input rows with the
// reward / terminal planes, and the categorical image loss with its gradient seed and decoded image.
#include "pd_common.cuh"

namespace {

inline int grid_blocks(long total, int block, int num_sms) {
    long g = (total + block - 1) / block;
    long cap = (long)num_sms * 32;
    if (g < 1) g = 1;
    return (int)(g < cap ? g : cap);
}
#define GRID_LOOP(i, n) for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (long)gridDim.x * blockDim.x)

// out (NB, C, P) = onehot(ids (NB, P)); an id outside [0, C) fills its pixel's C channels with NaN.
template <typename T>
__global__ void image_ids_onehot_kernel(long NB, int C, int P, const T* __restrict__ ids, float* __restrict__ out) {
    const long plane = (long)C * P;
    GRID_LOOP(i, NB * plane) {
        const long n = i / plane;
        const int r = (int)(i - n * plane);
        const int c = r / P, p = r - c * P;
        const long long id = (long long)ids[n * P + p];
        out[i] = (id < 0 || id >= C) ? __int_as_float(0x7fc00000) : (id == c ? 1.f : 0.f);
    }
}

// out[n, :] = [image[n] (C*P) | reward[n] x P | terminal[n] x P], row pitch ldo.
__global__ void grid_enc_input_kernel(long NB, int CP, int P, const float* __restrict__ image,
                                      const float* __restrict__ reward, const float* __restrict__ terminal,
                                      float* __restrict__ out, long ldo) {
    const int W = CP + 2 * P;
    GRID_LOOP(i, NB * W) {
        const long n = i / W;
        const int j = (int)(i - n * W);
        out[n * ldo + j] = j < CP ? image[n * CP + j] : (j < CP + P ? reward[n] : terminal[n]);
    }
}

// One warp per group of `div` rows sharing a target image.  Lane l takes the pixels l, l + 32, ... in turn; per pixel the
// channel loops run in index order.  A row's loss is the lane's pixel sum in that order, then a fixed xor tree across the
// lanes, so every result is bit-identical run to run.
__global__ void cat_image_loss_kernel(long groups, int div, int C, int P, const float* __restrict__ y, long ldy,
                                      const float* __restrict__ target, long ldt, float min_prob, float* __restrict__ loss,
                                      float* __restrict__ dy, long lddy, float* __restrict__ rec) {
    const int lane = threadIdx.x & 31;
    const long warps = (long)gridDim.x * (blockDim.x >> 5);
    const float ninf = -__int_as_float(0x7f800000);
    const float mix = 1.f - min_prob, unif = min_prob / (float)C;
    for (long g = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < groups; g += warps) {
        const float* t = target + g * ldt;
        float* rg = rec ? rec + g * (long)C * P : nullptr;
        if (rg)
            for (int p = lane; p < P; p += 32)
                for (int c = 0; c < C; ++c) rg[(long)c * P + p] = ninf;
        for (int i = 0; i < div; ++i) {
            const long m = g * div + i;
            const float* yr = y + m * ldy;
            float s = 0.f;
            for (int p = lane; p < P; p += 32) {
                // target class: the first maximum over the channels, NaN above everything (torch.argmax)
                int k = 0;
                float best = t[p];
                float mx = yr[p];
                for (int c = 1; c < C; ++c) {
                    const float v = t[(long)c * P + p];
                    if (!isnan(best) && (v > best || isnan(v))) { best = v; k = c; }
                    mx = fmaxf(mx, yr[(long)c * P + p]);
                }
                float se = 0.f;
                for (int c = 0; c < C; ++c) se += expf(yr[(long)c * P + p] - mx);
                const float lse = mx + logf(se);
                const float yk = yr[(long)k * P + p];
                float l, coef;
                if (min_prob == 0.f) {
                    l = lse - yk;
                    coef = 1.f;
                } else {                   // -log((1 - m) softmax(y)_k + m / C)
                    const float pk = expf(yk - mx) / se;
                    const float q = mix * pk + unif;
                    l = -logf(q);
                    coef = mix * pk / q;
                }
                s += l;
                if (dy) {
                    float* dr = dy + m * lddy;
                    for (int c = 0; c < C; ++c) {
                        const float pc = expf(yr[(long)c * P + p] - lse);
                        dr[(long)c * P + p] = coef * (pc - (c == k ? 1.f : 0.f));
                    }
                }
                if (rg) {                  // rec_c = logsumexp over the group's rows of (y_c - lse)
                    for (int c = 0; c < C; ++c) {
                        const float a = rg[(long)c * P + p], b = yr[(long)c * P + p] - lse;
                        const float hi = fmaxf(a, b);
                        rg[(long)c * P + p] = hi == ninf ? b : hi + logf(expf(a - hi) + expf(b - hi));
                    }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0 && loss) loss[m] = s;
        }
        if (rg)                            // normalise over the channels again
            for (int p = lane; p < P; p += 32) {
                float mx = rg[p];
                for (int c = 1; c < C; ++c) mx = fmaxf(mx, rg[(long)c * P + p]);
                float se = 0.f;
                for (int c = 0; c < C; ++c) se += expf(rg[(long)c * P + p] - mx);
                const float lse = mx + logf(se);
                for (int c = 0; c < C; ++c) rg[(long)c * P + p] -= lse;
            }
    }
}

}  // namespace

extern "C" {

#define S(stream) ((cudaStream_t)(stream))

int pd_image_ids_onehot(pd_handle* h, long NB, int C, int P, const void* ids, int id_bytes, float* out, void* stream) {
    PD_REQUIRE(h, NB >= 0 && C >= 1 && P >= 1 && (id_bytes == 1 || id_bytes == 4 || id_bytes == 8) && ids && out,
               "pd_image_ids_onehot: NB=%ld C=%d P=%d id_bytes=%d (1, 4 or 8) unsupported", NB, C, P, id_bytes);
    if (NB == 0) return PD_OK;
    const long n = NB * C * P;
    const int grid = grid_blocks(n, 256, h->num_sms);
    if (id_bytes == 1)
        image_ids_onehot_kernel<<<grid, 256, 0, S(stream)>>>(NB, C, P, (const uint8_t*)ids, out);
    else if (id_bytes == 4)
        image_ids_onehot_kernel<<<grid, 256, 0, S(stream)>>>(NB, C, P, (const int32_t*)ids, out);
    else
        image_ids_onehot_kernel<<<grid, 256, 0, S(stream)>>>(NB, C, P, (const long long*)ids, out);
    PD_CHECK_LAUNCH(h, "image_ids_onehot");
    return PD_OK;
}

int pd_grid_enc_input(pd_handle* h, long NB, int C, int P, const float* image, const float* reward, const float* terminal,
                      float* out, long ldo, void* stream) {
    PD_REQUIRE(h, NB >= 0 && C >= 1 && P >= 1 && ldo >= (long)(C + 2) * P && image && reward && terminal && out,
               "pd_grid_enc_input: NB=%ld C=%d P=%d ldo=%ld (>= (C+2)P) unsupported", NB, C, P, ldo);
    if (NB == 0) return PD_OK;
    const long n = NB * (C + 2) * (long)P;
    grid_enc_input_kernel<<<grid_blocks(n, 256, h->num_sms), 256, 0, S(stream)>>>(NB, C * P, P, image, reward, terminal,
                                                                                   out, ldo);
    PD_CHECK_LAUNCH(h, "grid_enc_input");
    return PD_OK;
}

int pd_cat_image_loss(pd_handle* h, long M, int C, int P, const float* y, long ldy, const float* target, long ldt,
                      int tgt_div, float min_prob, float* loss, float* dy, long lddy, float* rec, void* stream) {
    PD_REQUIRE(h, M >= 0 && C >= 2 && C <= PD_CAT_IMAGE_MAX_C && P >= 1 && P <= PD_CAT_IMAGE_MAX_P && tgt_div >= 1 &&
                      M % tgt_div == 0 && ldy >= (long)C * P && ldt >= (long)C * P && (!dy || lddy >= (long)C * P) &&
                      min_prob >= 0.f && min_prob < 1.f && y && target,
               "pd_cat_image_loss: M=%ld C=%d (2..%d) P=%d (1..%d) tgt_div=%d (divides M) ldy=%ld ldt=%ld lddy=%ld (>= C*P) "
               "min_prob=%g ([0, 1)) unsupported", M, C, PD_CAT_IMAGE_MAX_C, P, PD_CAT_IMAGE_MAX_P, tgt_div, ldy, ldt, lddy,
               (double)min_prob);
    if (M == 0) return PD_OK;
    const long groups = M / tgt_div;
    cat_image_loss_kernel<<<grid_blocks(groups, 8, h->num_sms), 256, 0, S(stream)>>>(groups, tgt_div, C, P, y, ldy, target,
                                                                                      ldt, min_prob, loss, dy, lddy, rec);
    PD_CHECK_LAUNCH(h, "cat_image_loss");
    return PD_OK;
}

}  // extern "C"

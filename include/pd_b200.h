/*
 * pd_b200.h — C ABI of libpd_b200.so: hand-written sm_90a kernels behind the PyDreamer
 * world-model training step + imagination rollout (BASELINE.json north_star; SURVEY.md §8).
 *
 * The reference (jurgisp/pydreamer) has no FFI: its boundary is the Python class
 * pydreamer.models.Dreamer (pydreamer/models/dreamer.py:19).  These entry points are the
 * arithmetic that class performs, one per fused device op; pydreamer_b200/dreamer.py composes
 * them behind the reference's Dreamer API.  Each declaration cites the reference lines whose
 * math it replaces.
 *
 * Conventions (SURVEY.md §8 b2):
 *   - plain pointers/sizes only; every pointer is a DEVICE pointer to fp32 unless noted;
 *   - `ld*` are row strides in ELEMENTS, so callers can pass views into concatenated buffers;
 *   - never allocates device memory, never synchronises, enqueues on `stream` (a cudaStream_t);
 *   - returns 0 on success, a negative PD_ERR_* otherwise; pd_last_error() gives the message;
 *   - one handle per (process, device); a handle is not re-entrant.
 */
#ifndef PD_B200_H
#define PD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pd_handle pd_handle;

#define PD_OK 0
#define PD_ERR_ARG (-1)
#define PD_ERR_LAUNCH (-2)
#define PD_ERR_DEVICE (-3)
#define PD_ERR_UNSUPPORTED (-4)

#define PD_ACT_NONE 0
#define PD_ACT_ELU 1

#define PD_GEMM_TC 0      /* TMA-fed tensor-core (mma.sync tf32 / fp16) kernel (default, the product path) */
#define PD_GEMM_SIMT 1    /* plain fp32 CUDA-core tile kernel: validation arm for the tests  */
#define PD_GEMM_C_ZEROED 1 /* pd_gemm flags bit */
#define PD_GEMM_C_F16 2    /* pd_gemm flags bit: C is an fp16 matrix (ldc in halfs); not with accumulate / residual */

/* ---- lifetime ---------------------------------------------------------------------------- */
/* A handle allocates 8 scratch areas of 16 MB on its device for the fixed-order gradient reductions, one per stream it
 * launches on, bound to a stream at its first reduction and kept for the handle's lifetime.  Reductions on a ninth stream
 * fail with PD_ERR_UNSUPPORTED: use one handle per set of at most eight streams. */
int pd_create(int device_ordinal, pd_handle** out);
void pd_destroy(pd_handle* h);
const char* pd_last_error(const pd_handle* h);
const char* pd_version(void);
int pd_set_gemm_impl(pd_handle* h, int impl);
long pd_launch_count(const pd_handle* h); /* kernels enqueued through this handle so far */
/* 1 (default): kernels that produce tensor-core operands round them to TF32 (rna) so the MMA's
 * operand truncation is exact; 0: keep full fp32 outputs (used by exactness tests). */
int pd_set_round_operands(pd_handle* h, int on);

/* ---- dense contraction ------------------------------------------------------------------- */
/* C[M,N] (=|+=) sum_k A(m,k) * B(n,k)  [+ bias[n]] [+ R[m / r_div, n]] -> act -> (tf32 round)
 *   a_mn = 0: A stored [M][K] (K contiguous, row stride lda); a_mn = 1: A stored [K][M] (M contiguous).
 *   b_mn = 0: B stored [N][K] (nn.Linear weight layout);      b_mn = 1: B stored [K][N].
 *   accumulate = 1: adds into C (split-K partials are summed in a fixed order; bias/R/act must be off).
 * Replaces every nn.Linear / nn.GRUCell matmul and the conv/deconv contractions:
 * common.py:47-55, rssm.py:103-116,138-146, rnn.py:60-67, encoders.py:80-90, decoders.py:128-155.
 * round_out rounds C to tf32 only while pd_set_round_operands is on (as every producer of this ABI does).
 * flags: PD_GEMM_C_ZEROED = the caller has already cleared C (accepted; the kernel never needs to clear C itself);
 *        PD_GEMM_C_F16 = C points to an fp16 matrix (the deconvolution column matrices of the decoder forward: they are
 *        written once and read once, in fp16 they cost half the HBM traffic; decoders.py:149-155); not with accumulate
 *        or a residual (PD_ERR_ARG).
 * TMA constraints (tensor-core impl): lda/ldb multiples of 4 elements, base pointers 16-byte aligned. */
int pd_gemm(pd_handle* h, int M, int N, int K,
            const float* A, long lda, int a_mn,
            const float* B, long ldb, int b_mn,
            float* C, long ldc,
            const float* bias, const float* R, long ldr, int r_div,
            int act, int round_out, int accumulate, int flags, void* stream);

/* Forward-only contraction with fp16 operands (mma.sync f16, fp32 accumulate / output): same 10-bit mantissa as
 * TF32 at twice the tensor rate and half the operand bytes.  Used where no gradient flows through the GEMM (the
 * imagination rollout and the heads evaluated on dreamed features, dreamer.py:188-216, a2c.py:88,112).
 * A: [M][K] fp16, B: [N][K] fp16 (both K-major, ld % 8 == 0), C fp32. */
int pd_gemm_f16(pd_handle* h, int M, int N, int K, const void* A, long lda, const void* B, long ldb,
                float* C, long ldc, const float* bias, const float* R, long ldr, int r_div,
                int act, int round_out, void* stream);
/* Few-row contraction against a weight in its stored orientation (weight-streaming kernel, split-K summed in a fixed order
 * inside a thread-block cluster): C[M,N] = sum_k A[m][k] * B[k][n] [+ bias[n]] [+ R[m / r_div, n]] -> act -> (tf32
 * round).  pd_gemm takes this kernel for every call it accepts with a_mn = 0, b_mn = 1 and no accumulate / fp16 C; the
 * BPTT input gradients of the posterior unroll (rssm.py:103-116 backward, M = B*I rows) are such calls.
 * It splits K where pd_gemm's tensor-core kernel does and adds the same partial sums in the same order, so both give the
 * same bits.  Accepts 1 <= M <= 64, N >= 8, K >= 8, A and B 16-byte aligned with lda, ldb multiples of 4, and shapes that
 * kernel splits at most 16 ways; anything else is PD_ERR_ARG before any launch.  C is written outright (no pre-clear);
 * any ldc. */
int pd_gemm_skinny(pd_handle* h, int M, int N, int K, const float* A, long lda, const float* B, long ldb,
                   float* C, long ldc, const float* bias, const float* R, long ldr, int r_div,
                   int act, int round_out, void* stream);
/* Implicit-GEMM convolution contractions: one operand is gathered on the fly from an NHWC fp32 tensor X[NB,H,W,C] by TMA
 * im2col-mode loads (k x k taps, stride 2, no padding; P,Q = (H-k)/2+1) instead of a materialised im2col matrix.
 *   mode 1: Cmat[NB*P*Q, odim] = im2col(X) * O        O: [odim][k*k*C] (o_mn=0) or [k*k*C][odim] (o_mn=1)
 *           -> Conv2d forward (encoders.py:80-88) and ConvTranspose2d input gradient
 *   mode 2: Cmat[k*k*cpad, odim] += im2col(X)^T * O   O: [NB*P*Q][odim]; rows (tap, channel) with channels padded to 32
 *           -> ConvTranspose2d weight gradient
 *   mode 3: Cmat[odim, k*k*cpad] += O^T * im2col(X)   O: [NB*P*Q][odim]
 *           -> Conv2d weight gradient */
int pd_conv_gemm(pd_handle* h, int mode, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo, int o_mn,
                 int odim, float* Cmat, long ldc, const float* bias, int act, int round_out, int accumulate, void* stream);
/* dst(fp16)[m, n] = src(fp32)[m, n] */
int pd_to_half(pd_handle* h, long M, long N, const float* src, long lds, void* dst, long ldd, void* stream);

/* ---- LayerNorm(eps, biased var, affine) + ELU -------------------------------------------- */
/* y = ELU(LN(x)); saves per-row mean / rstd.  common.py:45-51, rssm.py:105,110,115,139-140,144-145.
 * 1 <= N <= 1024, otherwise PD_ERR_ARG before any launch. */
int pd_ln_elu_fwd(pd_handle* h, int M, int N, const float* x, long ldx,
                  const float* gamma, const float* beta, float eps,
                  float* y, long ldy, float* mean, float* rstd,
                  void* y16 /* optional fp16 copy of y (operand of a forward-only pd_gemm_f16) */, long ldy16, void* stream);
/* dx from dy; ACCUMULATES (+=) dgamma, dbeta and (optional) dbias (= column sums of dx, the grad of the
 * bias of the Linear that produced x), summed in a fixed order.  1 <= N <= 1024, otherwise PD_ERR_ARG. */
int pd_ln_elu_bwd(pd_handle* h, int M, int N, const float* dy, long lddy,
                  const float* x, long ldx, const float* y, long ldy,
                  const float* gamma, const float* mean, const float* rstd,
                  float* dx, long lddx, float* dgamma, float* dbeta, float* dbias, void* stream);

/* ---- GRU cell pointwise (torch.nn.GRUCell gate order r|u|n) -------------------------------- */
/* rnn.py:48-49,60-67 -> nn.GRUCell: r=s(gi_r+gh_r) u=s(gi_u+gh_u) n=tanh(gi_n+r*gh_n) h'=(1-u)n+u*h.
 * gates[M,4,D] (optional) saves r,u,n,gh_n.  hmask (optional): also writes h' * mask_next[m] (the next step's
 * reset-masked input, rssm.py:134). */
int pd_gru_fwd(pd_handle* h, int M, int D, const float* gi, long ldgi, const float* gh, long ldgh,
               const float* hprev, long ldh, float* hout, long ldho,
               float* hmask, long ldhm, const float* mask_next,
               float* gates, void* h16 /* optional fp16 copy of h' */, long ldh16, void* stream);
/* dh_out = dh_a + dh_b * mask_b (either optional);  outputs dgi[M,3D], dgh[M,3D] and dh_carry = dh_out*u. */
int pd_gru_bwd(pd_handle* h, int M, int D, const float* dh_a, long ldda, const float* dh_b, long lddb,
               const float* mask_b, const float* gates, const float* hprev, long ldh,
               float* dgi, long lddgi, float* dgh, long lddgh, float* dh_carry, long lddc,
               void* stream);

/* ---- categorical straight-through latent -------------------------------------------------- */
/* logits[M, G*C] -> per (m,g): l = logits - logsumexp; p = softmax(l); k = argmax_c p_c / q_c
 * (== torch.multinomial's sampling, SURVEY.md App. D; exact ties go to the lowest class, torch.argmax's first maximum);
 * z = onehot(k).  1 <= C <= 32, otherwise PD_ERR_ARG.
 * rssm.py:147-148,178-179,195-201; a2c.py:47-48 with G = 1 for the one-hot actor.
 * zmask (optional) = z * mask_next[m]; idx (optional) int32 [M,G]. */
int pd_cat_sample(pd_handle* h, int M, int G, int C, const float* logits, long ldl,
                  const float* noise, long ldn, float* z, long ldz,
                  float* zmask, long ldzm, const float* mask_next, int32_t* idx,
                  void* z16 /* optional fp16 copy of z */, long ldz16, void* stream);
/* straight-through backward: dlogits = p * (dz - sum_c p dz) + alpha * rowscale[m] * extra;
 * dz = dz_a + dz_b * mask_b (each optional).  1 <= C <= 32, otherwise PD_ERR_ARG. */
int pd_cat_st_bwd(pd_handle* h, int M, int G, int C, const float* logits, long ldl,
                  const float* dz_a, long ldda, const float* dz_b, long lddb, const float* mask_b,
                  const float* extra, long ldex, const float* rowscale, float alpha,
                  float* dlogits, long lddl, void* stream);

/* ---- persistent RSSM posterior unroll (rssm.py:21-78 RSSMCore.forward, 125-153 RSSMCell.forward) -------------
 * ONE cooperative kernel walks all T timesteps (csrc/pd_rssm_fwd3.cu): per step { z_mlp as a gather over the sampled
 * one-hot + a_mlp term -> LayerNorm+ELU -> GRU gates -> post_mlp_h + embed term -> LayerNorm+ELU -> post_mlp ->
 * categorical sample }, with grid-wide barriers between the dependent phases instead of kernel boundaries; every CTA owns
 * a fixed slice of hidden units / features / latent groups for the whole sequence.  Operands are staged by a producer
 * warp with TMA into an mbarrier ring (weights of the next phase are prefetched across the grid barrier), contractions are
 * fp16 mma.sync with fp32 accumulation, the recurrent products over K = D are split in four k-slices.  Writes exactly the
 * buffers the chain of per-step kernels writes (the backward reads them).
 * Caller prepares: hin[0] / zin[0] (masked in_state), x1[0] (pre-norm input of step 0 incl. bias and action term),
 * aa / ea (action and embed projections hoisted over T), fp16 weight copies incl. the TRANSPOSED z_mlp weight ws_wzT16
 * (pd_transpose_to_half).  Limits (P = #CTAs = #SMs; KS = 4 when D % 256 == 0, else 1): BI <= 256 and a multiple of I
 * (rows beyond 64 are taken in blocks of 64), Hd <= 1024, C <= 32, G <= min(P, 256), D <= 16 * P, D and Hd multiples of 8,
 * ceil(D / (P / KS)) <= 64 and ceil(Hd / (P / KS)) <= 32; otherwise PD_ERR_UNSUPPORTED before any launch (use the chain). */
typedef struct pd_rssm_fwd_args {
    int T, BI, I, D, Hd, G, C;                 /* rows BI = B*I; Z = G*C; feat row pitch F = D + Z */
    const void *w_z16, *w_ih16, *w_hh16, *w_ph16, *w_pm16;   /* fp16 [Hd,Z] [3D,Hd] [3D,D] [Hd,D] [Z,Hd] */
    const float *b_z, *ln1_g, *ln1_b, *b_ih, *b_hh, *b_ph, *ln2_g, *ln2_b, *b_pm;
    float eps;
    const float *aa;                           /* [T*B, Hd] */
    const float *ea;                           /* [T*B, Hd] or NULL (open loop: no embed term) */
    const float *mask;                         /* [T, BI]  1 - reset */
    const float *noise;                        /* [T, BI, Z] Exp(1) */
    float *x1, *za, *m1, *r1;                  /* [T,BI,Hd] x2, [T,BI] x2 */
    float *gates;                              /* [T,BI,4D]  r,u,n,gh_n */
    float *feat;                               /* [T,BI,D+Z] h' | z */
    float *hin, *zin;                          /* [T,BI,D], [T,BI,Z] masked step inputs */
    float *y2, *pin, *m2, *r2;                 /* [T,BI,Hd] x2, [T,BI] x2 */
    float *post;                               /* [T,BI,Z] posterior logits */
    int32_t *idx;                              /* [T,BI,G] sampled classes */
    void *ws_wzT16;                            /* in: fp16 [Z,Hd] = z_mlp.weight^T (pd_transpose_to_half) */
    void *ws_za16, *ws_h16, *ws_pin16;         /* workspace fp16 [BI,Hd] [BI,D] [BI,Hd] */
    unsigned int *ws_barrier;                  /* workspace, 16 words, cleared by the call: [0] barrier counter */
    float *ws_ghpart, *ws_y2part;              /* workspace 4*BI*3D and 4*BI*Hd floats: k-slice partial sums of the recurrent products */
    /* Stacked GRU (rnn.py:40-67 GRUCellStack), appended: `layers` = L, 0 or 1 = the single cell above.  For 2 <= L <= 4 layer
     * l owns the units [l D/L, (l+1) D/L) of h; layer 0 reads za, layer l > 0 the fresh h' of layer l - 1.  w_ih16 / b_ih /
     * b_hh are then layer 0's ([3D/L, Hd], [3D/L]), w_hh16 is the block-diagonal [3D, D] of the layers' W_hh (row
     * gate * D + u holds unit u's row of its layer's W_hh in its layer's D/L columns, zeros elsewhere), the arrays below
     * hold layers 1 .. L-1, and `gates` is laid out [L, T, BI, 4D/L].  Further limits: D/L a multiple of 8,
     * D/L <= 16 * P (instead of D). */
    int layers;
    const void *w_ih16_l[3];                   /* fp16 [3D/L, D/L] of layers 1 .. L-1 */
    const float *b_ih_l[3], *b_hh_l[3];        /* [3D/L] of layers 1 .. L-1 */
} pd_rssm_fwd_args;
int pd_rssm_unroll_fwd(pd_handle* h, const pd_rssm_fwd_args* a, void* stream);

/* ---- Back-propagation through time of the posterior unroll, one persistent cooperative kernel ------------------------ */
/* Autograd of rssm.py:21-78,125-153 / rnn.py:60-67 for all T timesteps (csrc/pd_rssm_bptt.cu): per step, descending t,
 *   dz     = dfeat[t][:, D:] + mask[t+1] * (dx1[t+1] . W_z)                       straight-through sample, rssm.py:147-148
 *   dpost  = softmax'(post[t]) dz + kl_weight * w[t] * dpost_u[t]                 (+ the KL gradient of dreamer.py:328-343)
 *   dy2    = LN+ELU backward(post_norm)(dpost . W_pm)                             rssm.py:115-116
 *   dh     = dy2 . W_ph + dfeat[t][:, :D] + mask[t+1] * (dgh[t+1] . W_hh + dh[t+1] * u[t+1])
 *   dgi, dgh = GRU gate backward(dh; gates[t], hin[t])                            nn.GRUCell, gate order r|u|n
 *   dx1    = LN+ELU backward(in_norm)(dgi . W_ih)                                 rssm.py:138-140
 * Inputs are what pd_rssm_unroll_fwd (or the per-timestep chain) saved; outputs dpost, dy2, dgi, dgh, dx1 [T, BI, .] are the
 * operands of the batched weight-gradient GEMMs, tf32-rounded when round_out != 0.  LayerNorm affine and the two bias
 * gradients fed by LayerNorm inputs are ACCUMULATED (+=) into g_*, in a fixed order (each batch-row owner's partials
 * go to a row of ws_part2 / ws_part7 after their last use, and the grid adds the rows in order).  Weights come as TRANSPOSED fp16 copies (pd_transpose_to_half):
 * contraction operands carry 10 mantissa bits on both sides (fp16 weights are exact in tf32; gradients are tf32-rounded fp32),
 * like the TF32 GEMMs of the launch chain this replaces.  Limits (P = #CTAs = #SMs; R = min(4, P / G) CTAs per latent
 * group; ks2 / ks6 = 4 when Z resp. 3D is a multiple of 256, else 1): BI <= min(64, P), ceil(BI / R) <= 16, Hd <= 1024,
 * C <= 32, G <= P, D <= 16 * P, Hd, D, 3D and Z multiples of 8, ceil(Hd / (P / ks2)) <= 32, ceil(D / (P / ks6)) <= 64,
 * ceil(Hd / (P / ks6)) <= 32; otherwise PD_ERR_UNSUPPORTED before any launch (use the chain). */
typedef struct pd_rssm_bwd_args {
    int T, BI, D, Hd, G, C;
    int round_out;
    int ks2, ks6;                              /* set by the library (k-split factors) */
    float kl_weight;
    const void *w_pmT16, *w_phT16, *w_hhT16, *w_ihT16, *w_zT16;   /* fp16: [Hd,Z] [D,Hd] [D,3D] [Hd,3D] [Z,Hd] */
    const float *ln2_g, *ln1_g;                /* post_norm / in_norm weight [Hd] */
    const float *post, *pin, *y2, *m2, *r2;    /* [T,BI,Z] [T,BI,Hd] [T,BI,Hd] [T,BI] [T,BI] */
    const float *x1, *za, *m1, *r1;            /* [T,BI,Hd] [T,BI,Hd] [T,BI] [T,BI] */
    const float *gates, *hin, *mask;           /* [T,BI,4D] (r,u,n,gh_n) [T,BI,D] [T,BI] */
    const float *dfeat, *dpost_u, *w;          /* [T,BI,D+Z] seeds, [T,BI,Z] unweighted KL gradient, [T,BI] row weights */
    float *dpost, *dy2, *dgi, *dgh, *dx1;      /* out [T,BI,Z] [T,BI,Hd] [T,BI,3D] [T,BI,3D] [T,BI,Hd] */
    float *g_ln2_g, *g_ln2_b, *g_b_ph, *g_ln1_g, *g_ln1_b, *g_b_z;   /* += [Hd] each */
    float *ws_part2, *ws_part6, *ws_part7;     /* workspace [4,BI,Hd] [4,BI,D] [4,BI,Hd]; part2 + part7 also hold the 6 x [BI,Hd] g_* partials */
    unsigned int *ws_barrier;                  /* workspace, 16 words, cleared by the call */
} pd_rssm_bwd_args;
int pd_rssm_unroll_bwd(pd_handle* h, const pd_rssm_bwd_args* a, void* stream);
/* dst[n, m] (fp16) = src[m, n] (fp32): the transposed fp16 weight copies pd_rssm_unroll_bwd contracts with. */
int pd_transpose_to_half(pd_handle* h, int M, int N, const float* src, long lds, void* dst, long ldd, void* stream);

/* ---- KL(post || prior) with balancing, entropies, unweighted grads ------------------------ */
/* dreamer.py:328-343,369-379.  mode 0 (I == 1): value KL, grads (1-bal)*dKL/dpost and bal*dKL/dprior
 * (bal < 0 => plain KL, weight 1 on both: the reference's kl_balance 0.5 and 0, dreamer.py:241,334).  mode 1 (I > 1):
 * sampled log q(z) - log p(z) with idx from pd_cat_sample.  kl_exact / entropies are for metrics.
 * One block of G warps per row: 1 <= G <= 32 and 1 <= C <= 32, otherwise PD_ERR_ARG. */
int pd_kl(pd_handle* h, int M, int G, int C, const float* post, long ldpo, const float* prior, long ldpr,
          const int32_t* idx, int mode, float balance,
          float* loss_kl, float* kl_exact, float* ent_post, float* ent_prior,
          float* dpost, long lddpo, float* dprior, long lddpr, void* stream);

/* ---- convolution data movement (k x k, stride 2, no padding) ------------------------------ */
/* col[(n,oy,ox), kidx] = in[n, 2oy+kh, 2ox+kw, c]; korder 0: kidx=(kh,kw,c); 1: kidx=(c,kh,kw).
 * Input addressed by element strides (sN,sY,sX,sC) so NCHW and NHWC both work.
 * Forward operand of Conv2d (encoders.py:80-88) and backward operand of ConvTranspose2d. */
int pd_im2col(pd_handle* h, int NB, int Hin, int Win, int Cc, int k, int korder,
              const float* in, long sN, long sY, long sX, long sC,
              float* col, long ldcol, int round_out, void* stream);
/* out[n,y,x,c] = act(bias[c] + sum_{kh,kw: (y-kh)%2==0...} col[(n,(y-kh)/2,(x-kw)/2), (kh,kw,c)]).
 * Forward of ConvTranspose2d (decoders.py:149-155) and input-gradient of Conv2d. */
int pd_col2im(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k,
              const float* col, long ldcol, const float* bias, int act, int round_out,
              float* out, long sN, long sY, long sX, long sC, void* stream);
/* Last decoder layer fused with the image loss (decoders.py:163-167): dec NCHW, target NCHW of
 * image row n / tgt_div; loss[n] = 0.5*sum diff^2; diff stored NHWC for the backward gather. */
int pd_col2im_imgloss(pd_handle* h, int NB, int Hin, int Win, int Cc, int k,
                      const float* col, long ldcol, const float* bias,
                      const float* target, int tgt_div,
                      float* dec, float* diff, float* loss, float* csum /* [NB,Cc] per-image channel sums of diff */,
                      void* stream);
/* The same two folds over an fp16 (col_f16 = 1) or fp32 (0) column matrix; ldcol in elements. */
int pd_col2im_t(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k, const void* col, long ldcol,
                int col_f16, const float* bias, int act, int round_out, float* out, long sN, long sY, long sX, long sC,
                void* stream);
int pd_col2im_imgloss_t(pd_handle* h, int NB, int Hin, int Win, int Cc, int k, const void* col, long ldcol, int col_f16,
                        const float* bias, const float* target, int tgt_div, float* dec, float* diff, float* loss,
                        float* csum, void* stream);
/* dy <- dy * act'(y) in place (act from output y), db[c] += column sums of the result. */
int pd_bias_act_bwd(pd_handle* h, long M, int N, float* dy, long lddy, const float* y, long ldy,
                    int act, float* db, void* stream);
/* The ELU backward + bias gradient of the layer BELOW fused into the kernel that produces that layer's output gradient
 * (instead of a separate pd_bias_act_bwd pass over the gradient image):
 *   pd_gemm_actbwd:      C = (A B^T) .* elu'(dact) in the GEMM epilogue, then dbias[n] += sum_m C[m, n] (Linear / explicit-column deconv dX;
 *                        decoders.py:128-155 backward, autograd of nn.ELU + bias)
 *   pd_conv_gemm_actbwd: the same for pd_conv_gemm mode 1 (ConvTranspose2d input gradient gathered by TMA im2col)
 *   pd_col2im_actbwd:    out = fold(col) .* elu'(dact), dbias[c] += sum over pixels  (Conv2d input gradient; encoders.py:80-90
 *                        backward); out / dact contiguous NHWC [NB, Hout, Wout, Cc], Hout >= 2(Hin-1)+k (rows a stride-2 conv never read get 0)
 * dact is the saved forward output of the layer below (ELU derivative from the output: y > 0 ? 1 : y + 1).
 * Every bias / LayerNorm gradient and loss sum of this ABI is added in a fixed order: the same inputs give bit-identical
 * results. */
int pd_gemm_actbwd(pd_handle* h, int M, int N, int K, const float* A, long lda, int a_mn, const float* B, long ldb, int b_mn,
                   float* C, long ldc, const float* dact, long lddact, float* dbias, void* stream);
int pd_conv_gemm_actbwd(pd_handle* h, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo, int o_mn,
                        int odim, float* Cmat, long ldc, const float* dact, long lddact, float* dbias, void* stream);
int pd_col2im_actbwd(pd_handle* h, int NB, int Hin, int Win, int Hout, int Wout, int Cc, int k, const float* col, long ldcol,
                     const float* dact, float* dbias, float* out, void* stream);
/* generic 4-D permutation copy out[perm(i)] (+)= in[i];  dims (HOST int[4]) of `in`, perm[j] (HOST) = source axis of out axis j. */
int pd_permute4(pd_handle* h, const float* in, float* out, const int* dims, const int* perm,
                const long* in_strides /* HOST long[4] element strides of `in`, or NULL = contiguous */,
                int accumulate, int round_out, void* stream);

/* ---- small pointwise / reductions ---------------------------------------------------------- */
int pd_round_copy(pd_handle* h, const float* src, float* dst, long n, int round_out, void* stream);
int pd_pad_cols(pd_handle* h, long M, int C, int Cp, const float* src, long lds, float* dst, long ldd, void* stream);
int pd_mask_rows(pd_handle* h, int M, int N, const float* x, long ldx, const float* mask,
                 float* out, long ldo, void* stream);
/* x[m,:] *= alpha * scale[m / scale_div] */
int pd_rowscale(pd_handle* h, long M, long N, float* x, long ldx, const float* scale, int scale_div, float alpha, void* stream);
/* out[m, :] = W[idx[m], :]: `a_mlp` (rssm.py:104, Linear without bias) applied to a one-hot action is a row gather of the
 * transposed weight W = a_mlp.weight^T [A, Hd] (dreamer.py:197-205: the imagination rollout samples one-hot actions). */
int pd_gather_rows(pd_handle* h, long M, int N, const int32_t* idx, const float* W, long ldw, float* out, long ldo,
                   void* stream);
/* out[r, :] = sum_{i<I} x[r*I + i, :]  (undo the IWAE row expansion, rssm.py:35-41) */
int pd_group_sum(pd_handle* h, long R, int I, int W, const float* x, long ldx, float* out, long ldo, void* stream);
int pd_colsum(pd_handle* h, long M, int N, const float* x, long ldx, float* out, void* stream); /* out += */
int pd_fill(pd_handle* h, float* x, long n, float v, void* stream);
/* reset (uint8/bool [T,B]) -> mask f32 [T, B*I] = !reset   (rssm.py:41) */
int pd_reset_mask(pd_handle* h, int T, int B, int I, const uint8_t* reset, float* mask, void* stream);

/* ---- scalar-head losses (decoders.py:257-319) ---------------------------------------------- */
/* kind 0: DenseNormalDecoder  loss = 0.5 (t-y)^2, dy = (y-t);  kind 1: DenseBernoulliDecoder
 * loss = softplus(y) - t*y, dy = sigmoid(y)-t, rec = sigmoid(y).  target row = m / tgt_div. */
int pd_scalar_head_loss(pd_handle* h, long M, int kind, const float* y, const float* target, int tgt_div,
                        float* loss, float* dy, float* rec, void* stream);

/* Vector-observation head (decoders.py:290-319 DenseNormalDecoder with out_dim = K, std 1/sqrt(2 pi)):
 *   loss[m] = 0.5 * sum_k (t[k] - y[m,k])^2,   dy[m,k] = y[m,k] - t[k],   target row t = target[m / tgt_div].
 * One warp per row; each row's sum is added in a fixed order (bit-identical run to run).  y, target, dy are row-strided
 * (ld in elements).  1 <= K <= PD_VEC_HEAD_MAX_K, ld* >= K, tgt_div >= 1, otherwise PD_ERR_ARG before any launch. */
#define PD_VEC_HEAD_MAX_K 4096
int pd_vec_head_loss(pd_handle* h, long M, int K, const float* y, long ldy, const float* target, long ldt, int tgt_div,
                     float* loss, float* dy, long lddy, void* stream);

/* Categorical reward head on a support s[S] (decoders.py:322-362 DenseCategoricalSupportDecoder, common.py:77-86
 * CategoricalSupport.mean): for M rows of S logits y (row pitch ldy), p = softmax(y[m]),
 *   rec[m]  = sum_k p_k s_k                                    (the expected reward; NULL allowed when target is given)
 * and, with a target (row m reads target[m / tgt_div]):
 *   k*      = argmin_k (t - s_k)^2 in fp32, the first index on ties (to_categorical, decoders.py:349-352),
 *   loss[m] = logsumexp(y[m]) - y[m, k*],   dy[m, k] = p_k - [k == k*] (pitch lddy),   idx[m] = k* (int32, optional).
 * A NULL target is the expectation-only mode (rewards of the imagination rollout): only rec is written.  One warp per
 * row; every sum of a row is added in a fixed order.  2 <= S <= PD_SUPPORT_MAX, ldy >= S, tgt_div >= 1, with a target
 * loss, dy and lddy >= S, without one rec; otherwise PD_ERR_ARG before any launch. */
#define PD_SUPPORT_MAX 1024
int pd_support_head(pd_handle* h, long M, int S, const float* y, long ldy, const float* support, const float* target,
                    int tgt_div, float* rec, float* loss, float* dy, long lddy, int* idx, void* stream);

/* World-model loss assembly (dreamer.py:362-379, decoders.py:50-108): per (t,b) over I samples.
 * in: per-row losses [TB*I]; out: w[TB*I] = softmax_i(-L)/(TB) (grad of loss_model wrt L_tbi),
 * tb[TB,8] = {loss_model, loss_image, loss_reward, loss_terminal, loss_kl(exact), ent_prior, ent_post, loss_vecobs}.
 * l_img may be NULL (a model without an image decoder: read as 0); l_vec may be NULL (no vector observation: column 7
 * stays 0), else it enters L with weight w_vec. */
int pd_wm_loss(pd_handle* h, int TB, int I, float kl_weight, float w_img, float w_rew, float w_term,
               const float* l_img, const float* l_rew, const float* l_term, const float* l_kl,
               const float* kl_exact, const float* ent_prior, const float* ent_post,
               const float* l_vec, float w_vec, float* w, float* tb, void* stream);
/* out[c] = mean over rows of x[M,N]  (N <= 32) */
int pd_colmean(pd_handle* h, long M, int N, const float* x, float* out, void* stream);

/* ---- actor-critic (a2c.py:61-149) ---------------------------------------------------------- */
/* Column-wise GAE(lambda) scan + reality weights + critic loss/grad.  J = H+1 rows of Md columns.
 * vt = critic_target values, v = critic values, rew = reward head output, term_logit = terminal logits.
 * outputs: adv, agae, target, weight [H,Md]; dv [H,Md] = d loss_critic / d v; term [J,Md] = sigmoid;
 * sums[5] (double) += {loss_critic*HMd, sum v0[0], sum v0, sum r1, sum r1^2}.  1 <= H <= 127, otherwise PD_ERR_ARG. */
int pd_gae_critic(pd_handle* h, int H, int Md, float gamma, float lambda,
                  const float* vt, const float* v, const float* rew, const float* term_logit,
                  float* term, float* adv, float* agae, float* target, float* weight, float* dv,
                  double* sums, void* stream);
/* The same scan over observed rewards and 0/1 terminals: the world model's auxiliary critic (dreamer.py:347-365,
 * a2c.py:81-116) on T rows (H = T - 1) of B columns.  vt = critic_target values, v = critic values, rew = rewards,
 * term = terminals (each [T,B]).  dv [T-1,B] = scale * d loss_critic / d v[:-1] with
 * loss_critic = mean(0.5 (target - v[:-1])^2 weight); a terminal of 1 gives weight 0 at its row and after, never NaN.
 * sums[2] (double) += {loss_critic * (T-1) B, sum v[:-1]}, added in a fixed order (bit-identical run to run).
 * 2 <= T <= 128, B >= 1, every pointer non-NULL, otherwise PD_ERR_ARG before any launch. */
int pd_gae_critic_obs(pd_handle* h, int T, int B, float gamma, float lambda, const float* vt, const float* v,
                      const float* rew, const float* term, float scale, float* dv, double* sums, void* stream);
/* reinforce actor loss, one-hot policy (a2c.py:119-130): rows = H*Md.
 * sums[2] (double) += {sum (loss_policy - eta*ent)*w, sum ent};  dlogits = d mean(.)/d logits. */
int pd_actor_loss_onehot(pd_handle* h, long rows, int A, float eta, const float* logits, long ldl,
                         const float* actions, long lda, const float* agae, const float* weight,
                         float* dlogits, long lddl, double* sums, void* stream);
/* tanh_normal policy (functions.py:69-78): out[rows,2A] = (mean_, std_) raw, action in (-1,1). */
int pd_actor_loss_tanh_normal(pd_handle* h, long rows, int A, float eta, const float* out, long ldo,
                              const float* actions, long lda, const float* agae, const float* weight,
                              float* dout, long lddo, double* sums, void* stream);
/* a = tanh(5 tanh(m/5) + (softplus(s)+0.1) * eps)   (dreamer.py:197-200 with tanh_normal) */
int pd_tanh_normal_sample(pd_handle* h, long rows, int A, const float* out, long ldo,
                          const float* eps, float* action, long lda, void* stream);
/* normal_tanh policy (functions.py:59-66 with min_std 0.01, max_std 1; a2c.py:119-130 reinforce): out[rows,2A] = (m, s)
 * raw, mu = tanh(m), sd = sigmoid(s) + 0.01, policy Independent(Normal(mu, sd), 1) with no transform on the action.
 * sums[2] (double) += {sum (-log_prob(a) agae - eta entropy) w, sum entropy} with the Normal's entropy, added in a
 * fixed order (bit-identical run to run); dout[rows,2A] = d mean(.)/d out.
 * rows >= 0, A >= 1, ldo >= 2A, lddo >= 2A, lda >= A, otherwise PD_ERR_ARG before any launch; rows = 0 launches nothing. */
int pd_actor_loss_normal_tanh(pd_handle* h, long rows, int A, float eta, const float* out, long ldo,
                              const float* actions, long lda, const float* agae, const float* weight,
                              float* dout, long lddo, double* sums, void* stream);
/* a = tanh(m) + (sigmoid(s) + 0.01) * eps, unbounded   (dreamer.py:196-200 with normal_tanh: Normal.sample()).
 * rows >= 0, A >= 1, ldo >= 2A, lda >= A, otherwise PD_ERR_ARG before any launch; rows = 0 launches nothing. */
int pd_normal_tanh_sample(pd_handle* h, long rows, int A, const float* out, long ldo,
                          const float* eps, float* action, long lda, void* stream);

/* ---- replay preprocessing on the device (pydreamer/preprocessing.py:91-188; SURVEY.md §8f N3) ------------ */
/* uint8 image (NB,H,W,C) -> fp32 (NB,C,H,W) = x/255 - 0.5 (preprocessing.py:21-29): the batch crosses PCIe as bytes. */
int pd_image_u8_to_f32(pd_handle* h, long NB, int H, int W, int C, const uint8_t* src, float* dst, void* stream);
/* int64 action index -> one-hot fp32 (preprocessing.py:135-138) */
int pd_onehot_i64(pd_handle* h, long rows, int A, const int64_t* idx, float* out, void* stream);
/* y = tanh(x): clip_rewards 'tanh' (functions.py:153-160) */
int pd_tanh(pd_handle* h, long n, const float* x, float* y, void* stream);
/* Category ids (NB, P) of id_bytes bytes each (1: uint8, 4: int32, 8: int64) -> fp32 one-hot (NB, C, P)
 * (preprocessing.py:10-19, 105-110 with C = image_channels).  An id outside [0, C) is a malformed batch: its pixel's C
 * channels are NaN, and nothing outside `out` is written.  One thread per output element. */
int pd_image_ids_onehot(pd_handle* h, long NB, int C, int P, const void* ids, int id_bytes, float* out, void* stream);

/* ---- categorical grid images (encoders.py:14-17, 50-60, 99-125; decoders.py:183-254) --------------------------- */
/* Dense image encoder input rows with reward_input: out[n] = [image[n] (C*P floats, contiguous rows) | reward[n] x P |
 * terminal[n] x P], row pitch ldo >= (C+2) P.  One thread per output element. */
int pd_grid_enc_input(pd_handle* h, long NB, int C, int P, const float* image, const float* reward, const float* terminal,
                      float* out, long ldo, void* stream);
/* Categorical image loss (CatImageDecoder.loss / training_step) on M rows of C*P logits y in CHW order (channel stride P,
 * row pitch ldy); row m's target is row m / tgt_div of `target` (one-hot images, pitch ldt).  Per pixel:
 *   k       = argmax over c of target[c], the first maximum, NaN above everything (torch.argmax);
 *   loss    = logsumexp(y) - y[k]; with min_prob = m > 0, -log((1 - m) softmax(y)[k] + m / C);
 *   dy[c]   = d loss / d y[c] (pitch lddy; NULL: not written).
 * loss[m] (NULL: not written) = the pixel sum.  rec (optional, (M / tgt_div, C, P) contiguous): the decoded image of each
 * group of tgt_div rows, normalise(logsumexp over the group of normalise(y)) with normalise(x) = x - logsumexp_c(x).
 * One warp per group, lanes over pixels; every sum is added in a fixed order (bit-identical run to run).
 * 2 <= C <= PD_CAT_IMAGE_MAX_C, 1 <= P <= PD_CAT_IMAGE_MAX_P, tgt_div >= 1 dividing M, ld* >= C*P, 0 <= min_prob < 1,
 * otherwise PD_ERR_ARG before any launch. */
#define PD_CAT_IMAGE_MAX_C 64
#define PD_CAT_IMAGE_MAX_P 4096
int pd_cat_image_loss(pd_handle* h, long M, int C, int P, const float* y, long ldy, const float* target, long ldt,
                      int tgt_div, float min_prob, float* loss, float* dy, long lddy, float* rec, void* stream);

/* ---- optimizer (dreamer.py:60-87, train.py:193-198) ---------------------------------------- */
/* out += sum x^2 in a fixed summation order (bit-identical on every data-parallel replica); ws: pd_sumsq_ws_floats(h) floats */
int pd_sumsq(pd_handle* h, const float* x, long n, float* out /* += */, float* ws, void* stream);
int pd_sumsq_ws_floats(const pd_handle* h);
/* norm = sqrt(*sumsq); coef = min(1, max_norm/(norm+1e-6)); x *= coef; *norm_out = norm
 * (== torch.nn.utils.clip_grad_norm_). */
int pd_clip_scale(pd_handle* h, float* x, long n, const float* sumsq, float max_norm, float* norm_out, void* stream);
/* x *= alpha * (*scale) without operand rounding (scale may be NULL = 1); exits without touching memory when the factor is
 * exactly 1.  Applies the grad_output of `loss.backward(g)` (train.py:184-187, GradScaler under amp) and the 1/world of the
 * data-parallel mean to the gradient arena. */
int pd_scale_by(pd_handle* h, float* x, long n, const float* scale, float alpha, void* stream);
/* torch.optim.AdamW (decoupled wd, no amsgrad); *step is a device int32 already incremented. */
int pd_adamw(pd_handle* h, float* p, const float* g, float* m, float* v, long n,
             float lr, float beta1, float beta2, float eps, float wd, const int32_t* step, void* stream);
int pd_inc(pd_handle* h, int32_t* counter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PD_B200_H */

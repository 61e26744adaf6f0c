// pd_api.cu — handle lifetime, error reporting and the pd_gemm dispatcher of libpd_b200.so.
#include "pd_common.cuh"
#include <stdlib.h>

int pd_gemm_tc_launch(pd_handle* h, int M, int N, int K, const void* A, long lda, int a_mn, const void* B,
                      long ldb, int b_mn, const PdEpilogue& epi, cudaStream_t stream, int f16);
int pd_gemm_simt_launch(pd_handle* h, int M, int N, int K, const float* A, long lda, int a_mn, const float* B,
                        long ldb, int b_mn, const PdEpilogue& epi, cudaStream_t stream);

int pd_conv_gemm_launch(pd_handle* h, int mode, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo,
                        int o_mn, int ODIM, const PdEpilogue& epi, cudaStream_t stream);
bool pd_gemm_skinny_ok(const pd_handle* h, int M, int N, int K, const void* A, long lda, int a_mn, const void* B, long ldb,
                       int b_mn, const PdEpilogue& e);
int pd_gemm_skinny_launch(pd_handle* h, int M, int N, int K, const float* A, long lda, const float* B, long ldb,
                          const PdEpilogue& epi, cudaStream_t stream);

int pd_scratch(pd_handle* h, cudaStream_t stream, long nfloats, int ngroups, float** ws, unsigned** tickets) {
    PD_REQUIRE(h, nfloats <= PD_SCRATCH_FLOATS && ngroups <= PD_SCRATCH_TICKETS,
               "reduction needs %ld partials / %d groups, the scratch area holds %ld / %d", nfloats, ngroups, PD_SCRATCH_FLOATS,
               PD_SCRATCH_TICKETS);
    for (int i = 0; i < PD_SCRATCH_SLOTS; ++i) {
        PdScratch& sc = h->scratch[i];
        if (!sc.used) { sc.used = 1; sc.stream = stream; }
        if (sc.stream == stream) {
            *ws = sc.ws;
            *tickets = sc.tickets;
            return PD_OK;
        }
    }
    PD_FAIL(h, PD_ERR_UNSUPPORTED, "more than %d streams on one handle", PD_SCRATCH_SLOTS);
}

extern "C" {

const char* pd_version(void) { return "pd_b200 0.1 (sm_90a; TMA + mbarrier pipelines, mma.sync tf32 / fp16)"; }

int pd_create(int device_ordinal, pd_handle** out) {
    if (!out) return PD_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device_ordinal < 0 || device_ordinal >= ndev) return PD_ERR_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_ordinal) != cudaSuccess) return PD_ERR_DEVICE;
    if (prop.major != 9) return PD_ERR_UNSUPPORTED;    // sm_90a only: no fallback paths
    pd_handle* h = (pd_handle*)calloc(1, sizeof(pd_handle));
    if (!h) return PD_ERR_DEVICE;
    h->device = device_ordinal;
    h->num_sms = prop.multiProcessorCount;
    h->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    h->gemm_impl = PD_GEMM_TC;
    h->round_ops = 1;
    cudaSetDevice(device_ordinal);
    for (int i = 0; i < PD_SCRATCH_SLOTS; ++i) {
        PdScratch& sc = h->scratch[i];
        if (cudaMalloc(&sc.ws, PD_SCRATCH_FLOATS * sizeof(float)) != cudaSuccess ||
            cudaMalloc(&sc.tickets, PD_SCRATCH_TICKETS * sizeof(unsigned)) != cudaSuccess ||
            cudaMemset(sc.tickets, 0, PD_SCRATCH_TICKETS * sizeof(unsigned)) != cudaSuccess) {
            pd_destroy(h);
            return PD_ERR_DEVICE;
        }
    }
    cudaDriverEntryPointQueryResult qres;
    void* fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
        pd_destroy(h);
        return PD_ERR_DEVICE;
    }
    h->encode_tiled = fn;
    *out = h;
    return PD_OK;
}

void pd_destroy(pd_handle* h) {
    if (!h) return;
    PdDeviceGuard guard(h);
    for (int i = 0; i < PD_SCRATCH_SLOTS; ++i) {
        cudaFree(h->scratch[i].ws);
        cudaFree(h->scratch[i].tickets);
    }
    free(h);
}
const char* pd_last_error(const pd_handle* h) { return h ? h->err : "null handle"; }
long pd_launch_count(const pd_handle* h) { return h ? h->launches : 0; }

int pd_set_gemm_impl(pd_handle* h, int impl) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, impl == PD_GEMM_TC || impl == PD_GEMM_SIMT, "unknown gemm impl %d", impl);
    h->gemm_impl = impl;
    return PD_OK;
}

int pd_set_round_operands(pd_handle* h, int on) {
    if (!h) return PD_ERR_ARG;
    h->round_ops = on ? 1 : 0;
    return PD_OK;
}

int pd_gemm(pd_handle* h, int M, int N, int K, const float* A, long lda, int a_mn, const float* B, long ldb, int b_mn,
            float* C, long ldc, const float* bias, const float* R, long ldr, int r_div, int act, int round_out,
            int accumulate, int flags, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, M > 0 && N > 0 && K > 0, "pd_gemm: bad shape %d %d %d", M, N, K);
    PD_REQUIRE(h, A && B && C, "pd_gemm: null operand");
    PD_REQUIRE(h, !(accumulate && (bias || R || act)), "pd_gemm: accumulate excludes bias/residual/act");
    // R may be C itself (C += A.B^T in place, e.g. the BPTT chain's input gradients): every route's epilogue reads R[i, j]
    // after the contraction, before C[i, j] is written, and no other element's store can overtake that read (each output
    // tile is read and then stored by the CTA that owns it).  A new epilogue must keep that property.
    PdEpilogue e;
    e.C = C; e.ldc = ldc; e.bias = bias; e.R = R; e.ldr = ldr; e.r_div = r_div > 0 ? r_div : 1;
    e.act = act; e.round_out = round_out && h->round_ops; e.accumulate = accumulate;
    e.c_f16 = (flags & PD_GEMM_C_F16) ? 1 : 0;
    e.dact = nullptr; e.lddact = 0;
    PD_REQUIRE(h, !(e.c_f16 && (accumulate || R)), "pd_gemm: an fp16 output cannot accumulate or add a residual");
    // Skinny / unaligned contractions (scalar heads N=1, action inputs K=18, ...) cannot be described
    // by a TMA tensor map (16-byte strides) and have no tensor-core work to speak of: CUDA cores.
    const bool tma_ok = (lda % 4 == 0) && (ldb % 4 == 0) && ((((uintptr_t)A) & 15) == 0) &&
                        ((((uintptr_t)B) & 15) == 0) && N >= 8 && K >= 8 &&
                        (!e.c_f16 || ((ldc % 8 == 0) && !e.round_out && ((((uintptr_t)C) & 15) == 0)));
    if (h->gemm_impl == PD_GEMM_SIMT || !tma_ok)
        return pd_gemm_simt_launch(h, M, N, K, A, lda, a_mn, B, ldb, b_mn, e, (cudaStream_t)stream);
    // Few rows against a weight stored [K][N] (the BPTT chain's input gradients): stream the weight, not 128-row tiles.
    if (pd_gemm_skinny_ok(h, M, N, K, A, lda, a_mn, B, ldb, b_mn, e))
        return pd_gemm_skinny_launch(h, M, N, K, A, lda, B, ldb, e, (cudaStream_t)stream);
    return pd_gemm_tc_launch(h, M, N, K, A, lda, a_mn, B, ldb, b_mn, e, (cudaStream_t)stream, 0);
}

int pd_gemm_skinny(pd_handle* h, int M, int N, int K, const float* A, long lda, const float* B, long ldb, float* C, long ldc,
                   const float* bias, const float* R, long ldr, int r_div, int act, int round_out, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, A && B && C, "pd_gemm_skinny: null operand");
    PdEpilogue e;
    e.C = C; e.ldc = ldc; e.bias = bias; e.R = R; e.ldr = ldr; e.r_div = r_div > 0 ? r_div : 1;
    e.act = act; e.round_out = round_out && h->round_ops; e.accumulate = 0; e.c_f16 = 0;
    e.dact = nullptr; e.lddact = 0;
    return pd_gemm_skinny_launch(h, M, N, K, A, lda, B, ldb, e, (cudaStream_t)stream);
}

int pd_conv_gemm(pd_handle* h, int mode, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo, int o_mn,
                 int odim, float* Cmat, long ldc, const float* bias, int act, int round_out, int accumulate, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, mode >= 1 && mode <= 3 && X && O && Cmat, "pd_conv_gemm: bad arguments");
    PD_REQUIRE(h, (mode == 1) == (accumulate == 0), "pd_conv_gemm: mode 1 stores, modes 2/3 accumulate");
    PdEpilogue e;
    e.C = Cmat; e.ldc = ldc; e.bias = bias; e.R = nullptr; e.ldr = 0; e.r_div = 1;
    e.act = act; e.round_out = round_out && h->round_ops; e.accumulate = accumulate; e.c_f16 = 0;
    e.dact = nullptr; e.lddact = 0;
    return pd_conv_gemm_launch(h, mode, NB, H, W, C, k, X, O, ldo, o_mn, odim, e, (cudaStream_t)stream);
}

int pd_gemm_f16(pd_handle* h, int M, int N, int K, const void* A, long lda, const void* B, long ldb, float* C, long ldc,
                const float* bias, const float* R, long ldr, int r_div, int act, int round_out, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, M > 0 && N >= 8 && K >= 8, "pd_gemm_f16: bad shape %d %d %d", M, N, K);
    PD_REQUIRE(h, A && B && C, "pd_gemm_f16: null operand");
    PdEpilogue e;
    e.C = C; e.ldc = ldc; e.bias = bias; e.R = R; e.ldr = ldr; e.r_div = r_div > 0 ? r_div : 1;
    e.act = act; e.round_out = round_out && h->round_ops; e.accumulate = 0; e.c_f16 = 0;
    e.dact = nullptr; e.lddact = 0;
    return pd_gemm_tc_launch(h, M, N, K, A, lda, 0, B, ldb, 0, e, (cudaStream_t)stream, 1);
}

// Input gradient of a layer followed by the backward of the ELU that preceded it in the forward pass:
//   C = (A B^T) * elu'(dact) (tf32-rounded if round_out) in the GEMM's epilogue, then dbias[n] += sum_m C[m, n] (pd_colsum).
// Falls back to GEMM + pd_bias_act_bwd where the tensor-core epilogue cannot take it (C not TMA-addressable, SIMT arm).
int pd_gemm_actbwd(pd_handle* h, int M, int N, int K, const float* A, long lda, int a_mn, const float* B, long ldb, int b_mn,
                   float* C, long ldc, const float* dact, long lddact, float* dbias, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, M > 0 && N > 0 && K > 0 && A && B && C && dact, "pd_gemm_actbwd: bad arguments");
    const bool tma_ok = (lda % 4 == 0) && (ldb % 4 == 0) && (ldc % 4 == 0) && ((((uintptr_t)A) & 15) == 0) &&
                        ((((uintptr_t)B) & 15) == 0) && ((((uintptr_t)C) & 15) == 0) && N >= 8 && K >= 8;
    if (h->gemm_impl == PD_GEMM_SIMT || !tma_ok) {
        int rc = pd_gemm(h, M, N, K, A, lda, a_mn, B, ldb, b_mn, C, ldc, nullptr, nullptr, 0, 1, PD_ACT_NONE, 0, 0, 0, stream);
        if (rc) return rc;
        return pd_bias_act_bwd(h, M, N, C, ldc, dact, lddact, PD_ACT_ELU, dbias, stream);
    }
    PdEpilogue e;
    e.C = C; e.ldc = ldc; e.bias = nullptr; e.R = nullptr; e.ldr = 0; e.r_div = 1;
    e.act = PD_ACT_NONE; e.round_out = h->round_ops; e.accumulate = 0; e.c_f16 = 0;
    e.dact = dact; e.lddact = lddact;
    int rc = pd_gemm_tc_launch(h, M, N, K, A, lda, a_mn, B, ldb, b_mn, e, (cudaStream_t)stream, 0);
    if (rc || !dbias) return rc;
    return pd_colsum(h, M, N, C, ldc, dbias, stream);
}

// The same for the implicit-GEMM convolution form 1 (ConvTranspose2d input gradient, decoders.py:149-155 backward).
int pd_conv_gemm_actbwd(pd_handle* h, int NB, int H, int W, int C, int k, const float* X, const float* O, long ldo, int o_mn,
                        int odim, float* Cmat, long ldc, const float* dact, long lddact, float* dbias, void* stream) {
    if (!h) return PD_ERR_ARG;
    PD_REQUIRE(h, X && O && Cmat && dact, "pd_conv_gemm_actbwd: bad arguments");
    PdEpilogue e;
    e.C = Cmat; e.ldc = ldc; e.bias = nullptr; e.R = nullptr; e.ldr = 0; e.r_div = 1;
    e.act = PD_ACT_NONE; e.round_out = h->round_ops; e.accumulate = 0; e.c_f16 = 0;
    e.dact = dact; e.lddact = lddact;
    int rc = pd_conv_gemm_launch(h, 1, NB, H, W, C, k, X, O, ldo, o_mn, odim, e, (cudaStream_t)stream);
    if (rc || !dbias) return rc;
    const int P = (H - k) / 2 + 1, Q = (W - k) / 2 + 1;
    return pd_colsum(h, (long)NB * P * Q, odim, Cmat, ldc, dbias, stream);
}

}  // extern "C"

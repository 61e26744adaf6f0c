"""Kernel-level tests of the weight-streaming few-row GEMM (csrc/pd_gemm_skinny.cu, pd_gemm_skinny): C[M <= 64, N] =
A[M][K] . B[K][N] (+ bias, + residual row m // r_div, ELU, tf32 rounding), with B the weight as stored, against a FLOAT64
reference computed from the exact fp32 values the kernel reads; the route pd_gemm takes for the BPTT chain's input
gradients; run-to-run bit identity; and the host-side refusals.

Bounds follow tests/test_gemm_conv_f64_gpu.py: C_ACC * depth * U * sum_k |a_k b_k| with depth = 4 k-steps per 32-k block
of a split plus the number of splits, which are the general kernel's (tc_depth), plus the tf32 operand term for raw fp32
operands and the epilogue's additions."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_gemm_conv_f64_gpu import (ACT_ELU, C_ACC, ELU_REL, TF32_OP, U, Bufs, cdiv, check_out, operand, refused,
                                          sync, tc_depth, tma_gap)
from tests.util import CPU, DEV, Gen, f64, fp32, ops, round_out, tf32_rna  # noqa: F401

if CPU:
    pytest.skip("pd_gemm_skinny has no float32 twin: GPU only", allow_module_level=True)
pytestmark = pytest.mark.gpu

# The five per-timestep input gradients of the posterior unroll's BPTT (Dreamer._wm_backward): (name, N = in, K = out)
# at `atari` (deter 2048, hidden 1000, stoch 32 x 32) and `dmc` (deter 1024); M = B * I = 50 rows.
CHAIN = {
    "atari": [("post_mlp", 1000, 1024), ("post_mlp_h", 2048, 1000), ("gru_weight_hh", 2048, 6144),
              ("gru_weight_ih", 1000, 6144), ("z_mlp", 1024, 1000)],
    "dmc": [("post_mlp", 1000, 1024), ("post_mlp_h", 1024, 1000), ("gru_weight_hh", 1024, 3072),
            ("gru_weight_ih", 1000, 3072), ("z_mlp", 1024, 1000)],
}


def skinny_depth(N, K):
    """Length of an output element's fp32 accumulation chain: the general kernel's (tc_depth), whose K splits this kernel
    takes over."""
    return tc_depth(50, N, cdiv(K, 32))[0]


def skinny(ops, A, B, C, bias=None, R=None, r_div=1, act=0, rnd=False):
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    M, N = C.shape
    ops._ck(ops.lib.pd_gemm_skinny(ops.h, M, N, A.shape[1], p(A), A.stride(0), p(B), B.stride(0), p(C), C.stride(0),
                                   p(bias), p(R), R.stride(0) if R is not None else 0, r_div, act, int(rnd), ops._s()),
            "pd_gemm_skinny")


def case(name, M, N, K, **kw):
    return pytest.param(dict(M=M, N=N, K=K, **kw), id=name)


CASES = [case(f"m{M}", M, 200, 333, bias=True, res="rows", rnd=1) for M in (1, 7, 16, 50, 64)] + [
    case(f"atari_{n}", 50, N, K, res="rows" if n in ("post_mlp_h", "gru_weight_hh") else None, opnd="raw")
    for n, N, K in CHAIN["atari"]] + [
    # N not a multiple of the 64-column slab (N = 72: the second slab's last 32-column group lies wholly past N); the
    # smallest N and K; K not a multiple of 32 or of the rank count (9 blocks -> 5 ranks of 2 and 1)
    case("n72_partial_slab", 33, 72, 256, bias=True, act=ACT_ELU, rnd=1),
    case("n8_k8_one_block_one_rank", 5, 8, 8, bias=True),
    case("k288_uneven_ranks", 64, 130, 288, res="rows", r_div=3),
    case("k40_two_ranks_partial_block", 17, 96, 40, bias=True, res="inplace", rnd=1),
    # strided operands: rows of A / B / C padded (ldc not a multiple of 4: plain stores)
    case("strided_lda_ldb_ldc", 50, 100, 500, a_gap=12, b_gap=28, c_gap=3, bias=True, act=ACT_ELU),
]


@pytest.mark.parametrize("c", CASES)
def test_skinny_gemm_matches_float64_reference(ops, round_out, c):
    M, N, K = c["M"], c["N"], c["K"]
    g = Gen(M * 7 + N * 3 + K)
    rd = fp32 if c.get("opnd") == "raw" else tf32_rna
    A, Bm = rd(g.normal(M, K)), rd(g.normal(K, N, scale=1.0 / math.sqrt(K)))       # Bm: the weight as stored, [K][N]
    bias = fp32(g.normal(N, scale=0.5)) if c.get("bias") else None
    r_div = c.get("r_div", 1)
    R = fp32(g.normal(cdiv(M, r_div) if c.get("res") == "rows" else M, N, scale=0.5)) if c.get("res") else None
    Ad = operand(A, gap=c.get("a_gap", tma_gap(K)))
    Bd = operand(Bm, gap=c.get("b_gap", tma_gap(N)))
    bufs = Bufs()
    C = bufs.out(M, N, gap=c.get("c_gap", 4), init=R if c.get("res") == "inplace" else None)
    Rd = C if c.get("res") == "inplace" else (operand(R, gap=3) if R is not None else None)
    skinny(ops, Ad, Bd, C, None if bias is None else bias.float(), Rd, r_div, c.get("act", 0), bool(c.get("rnd")))
    bufs.check()

    ref, terms = A @ Bm, A.abs() @ Bm.abs()
    err = C_ACC * skinny_depth(N, K) * U * terms + (TF32_OP * terms if c.get("opnd") == "raw" else 0.0)
    extra = torch.zeros_like(ref)
    if bias is not None:
        ref, extra = ref + bias, extra + bias.abs()
    if R is not None:
        rr = R[torch.arange(M, device=R.device) // r_div]
        ref, extra = ref + rr, extra + rr.abs()
    err = err + 2 * U * (terms + extra)
    if c.get("act") == ACT_ELU:
        ref = F.elu(ref)
        err = err + (ELU_REL + U) * ref.abs()
    print(f"\n{M}x{N}x{K}, depth {skinny_depth(N, K)}")
    check_out("C", C, ref, err, bool(c.get("rnd")) and bool(round_out), {})


def kernels_of(fn):
    """Names of the CUDA kernels fn() launches."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        sync()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.mark.parametrize("preset", list(CHAIN))
def test_chain_input_gradients_take_the_skinny_kernel_with_the_general_kernels_bits(ops, round_out, preset):
    """pd_gemm sends each chain GEMM (a_mn 0, b_mn 1, stored, fp32 C, M = 50) to pd_gemm_skinny_kernel, writing C outright
    (no pre-clear: C starts as NaN); 65 rows keep the general tensor-core kernel.  Both split K alike (one row of output
    tiles either way), so the 50 rows equal the first 50 of the 65 bit for bit: the chain computes what it computed on the
    general kernel."""
    g = Gen(3)
    for name, N, K in CHAIN[preset]:
        A = g.normal(65, K).float()                                      # raw fp32: the chain's gradients are not rounded
        W = tf32_rna(g.normal(K, N, scale=1.0 / math.sqrt(K))).float()
        R = g.normal(65, N).float() if name in ("post_mlp_h", "gru_weight_hh") else None
        out = {}
        for M in (50, 65):
            C = torch.full((M, N), float("nan"), device=DEV)
            names = kernels_of(lambda: ops.gemm(A[:M].contiguous(), W, C, b_mn=True,
                                                res=None if R is None else R[:M].contiguous(), round_out=True))
            want, other = ("pd_gemm_skinny_kernel", "pd_gemm_tf32_kernel") if M <= 64 else ("pd_gemm_tf32_kernel", "pd_gemm_skinny_kernel")
            assert any(want in n for n in names) and not any(other in n for n in names), (name, M, names)
            assert not torch.isnan(C).any(), (name, M)
            out[M] = C
        assert torch.equal(out[50], out[65][:50]), (name, (out[50] - out[65][:50]).abs().max().item())


def test_same_inputs_give_bit_identical_outputs_run_to_run(ops):
    g = Gen(8)
    runs = []
    for name, N, K in CHAIN["atari"]:
        A, W = tf32_rna(g.normal(50, K)).float(), tf32_rna(g.normal(K, N, scale=0.02)).float()
        R = g.normal(50, N).float()
        outs = []
        for _ in range(3):
            C = torch.empty(50, N, device=DEV)
            ops.gemm(A, W, C, b_mn=True, res=R)
            sync()
            outs.append(C)
        runs.append((name, outs))
    for name, outs in runs:
        for o in outs[1:]:
            assert torch.equal(outs[0], o), name


def _raw(ops, M, N, K, lda, ldb, a_off=0, b_off=0):
    A = torch.zeros(max(M, 1) * lda + 64, device=DEV)
    B = torch.zeros(max(K, 1) * ldb + 64, device=DEV)
    C = torch.zeros(max(M, 1), max(N, 1), device=DEV)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + 4 * off)
    ops._ck(ops.lib.pd_gemm_skinny(ops.h, M, N, K, p(A, a_off), lda, p(B, b_off), ldb, p(C), C.stride(0), None, None, 0, 1, 0,
                                   0, ops._s()), "pd_gemm_skinny")


REFUSALS = {
    "m65": dict(M=65, N=64, K=64, lda=64, ldb=64),
    "m0": dict(M=0, N=64, K=64, lda=64, ldb=64),
    "n7": dict(M=50, N=7, K=64, lda=64, ldb=8),
    "k7": dict(M=50, N=64, K=7, lda=8, ldb=64),
    "lda_not_multiple_of_4": dict(M=50, N=64, K=64, lda=66, ldb=64),
    "ldb_not_multiple_of_4": dict(M=50, N=64, K=64, lda=64, ldb=65),
    "a_not_16_byte_aligned": dict(M=50, N=64, K=64, lda=64, ldb=64, a_off=1),
    "b_not_16_byte_aligned": dict(M=50, N=64, K=64, lda=64, ldb=64, b_off=2),
    # one 128-column tile and 192 k-blocks: the general kernel splits K 48 ways, more than one cluster adds up
    "more_than_16_splits": dict(M=50, N=100, K=6144, lda=6144, ldb=100),
}


@pytest.mark.parametrize("what", list(REFUSALS))
def test_shapes_past_the_limits_are_refused_before_any_launch(ops, what):
    refused(ops, lambda: _raw(ops, **REFUSALS[what]))

"""Tensor-core GEMM launches with an MN-major operand (csrc/pd_gemm_sm90.cu: the transposer warps rewrite each landed
MN-major tile into the K-major layout, then the wgmma consumers read it) at the shapes the Atari training step runs them
(T = B = 50, deter 2048, hidden 400, 64 x 64 images), plus partial k-blocks and partial 32-column groups.

The references, bounds and guard bands are those of test_gemm_conv_f64_gpu.py (its docstring explains them): float64
results from the exact fp32 values the kernel reads, each element bounded by its own error terms with the chain depth that
pick_splits gives the launch.  The split-K partial sums of these launches are added in a fixed order, so two runs on the
same inputs are bit-identical."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_gemm_conv_f64_gpu import (C_ACC, DEC_GEO, U, Bufs, case, cdiv, check_out, gemm_inputs,
                                          gemm_ref, operand, report, sync, tc_depth, tma_gap)
from tests.util import CPU, DEV, Gen, bound, ops, round_out, tf32_rna, ulp  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
ACT_ELU = 1

MN_CASES = [
    # world-model head weight gradient: dW[400, 3072] += dY^T X over the 37500 imagined states (K = H * T * B = 15 * 2500),
    # both operands MN-major; 96 tiles: not split; 400 % 32 = 16 -> the last row block takes 2-D boxes (a partial group)
    case("wgrad_400x3072_k37500_both_mn_accumulate", 400, 3072, 37500, a_mn=1, b_mn=1, acc=True, split=False),
    # hidden-layer weight gradient over the same states: 16 tiles, split 8 ways over K
    case("wgrad_400x400_k37500_both_mn_split", 400, 400, 37500, a_mn=1, b_mn=1, acc=True, split=True),
    # BPTT chain input gradient: dh[50, 2048] = dG[50, 6144] W[6144, 2048], B MN-major, one row of tiles -> skinny split
    case("bptt_dx_50x2048_k6144_b_mn_skinny", 50, 2048, 6144, b_mn=1, split=True),
    # the same with N = 1000 (1000 % 32 = 8: a partial column group in the last tile)
    case("bptt_dx_50x1000_k6144_b_mn_partial_group", 50, 1000, 6144, b_mn=1, split=True),
    # last decoder layer's input gradient fused with the ELU backward of the layer below: 2.25 M rows, B MN-major
    case("decoder_dx_actbwd_2250000x48_k108_b_mn", 2250000, 48, 108, b_mn=1, actbwd=True, split=False),
    # weight gradient with a partial last k-block (2500 % 32 = 4) and a partial column group in A (1000 % 32 = 8), split 2
    case("wgrad_1000x1024_k2500_partial_k_and_group", 1000, 1024, 2500, a_mn=1, b_mn=1, acc=True, split=True),
    # A MN-major: two k-blocks, the second 17 deep; M = 200 and N = 136: partial column groups; every epilogue term
    case("a_mn_partial_k_block_epilogue", 200, 136, 49, a_mn=1, bias=True, act=ACT_ELU, rnd=1),
    # B MN-major with one k-block of 20 rows, raw fp32 operands and a residual
    case("b_mn_single_partial_k_block_raw", 264, 72, 20, b_mn=1, opnd="raw", res="rows", rnd=1),
]


def run_gemm(ops, c, A, B, bias, R, dact, db0):
    """Launches case c on device copies of its operands; returns (C, dbias, bufs)."""
    M, N = c["M"], c["N"]
    a_mn, b_mn = c.get("a_mn", 0), c.get("b_mn", 0)
    As, Bs = A.T if a_mn else A, B.T if b_mn else B
    Ad = operand(As, gap=tma_gap(As.shape[1]))
    Bd = operand(Bs, gap=tma_gap(Bs.shape[1]))
    bufs = Bufs()
    C = bufs.out(M, N, gap=tma_gap(N), init=R if c.get("acc") else None)
    db = None
    if c.get("actbwd"):
        db = bufs.out(1, N, init=db0).view(N)
        ops.gemm_actbwd(Ad, Bd, C, dact.float(), db, a_mn=bool(a_mn), b_mn=bool(b_mn))
    else:
        resd = operand(R, gap=3) if c.get("res") == "rows" else None
        ops.gemm(Ad, Bd, C, a_mn=bool(a_mn), b_mn=bool(b_mn), bias=None if bias is None else bias.float(), res=resd,
                 r_div=c.get("r_div", 1), act=c.get("act", 0), round_out=bool(c.get("rnd")),
                 accumulate=bool(c.get("acc")))
    return C, db, bufs


@gpu
@pytest.mark.parametrize("c", MN_CASES)
def test_mn_major_gemm_matches_float64_reference(ops, round_out, c):
    M, N, K = c["M"], c["N"], c["K"]
    g = Gen(M * 5 + N * 11 + K)
    A, B, bias, R, dact = gemm_inputs(c, g)
    db0 = g.normal(N, scale=0.5).float().double() if c.get("actbwd") else None
    assert (tc_depth(M, N, cdiv(K, 32), c.get("acc", False))[1] > 1) == c.get("split", False)
    ref, err, depth = gemm_ref(c, A, B, bias, R, dact, False)
    C, db, bufs = run_gemm(ops, c, A, B, bias, R, dact, db0)
    bufs.check()
    print(f"\n{M}x{N}x{K} a_mn {c.get('a_mn', 0)} b_mn {c.get('b_mn', 0)}, depth {depth}")
    stats = {}
    if c.get("actbwd"):
        check_out("C", C, ref, err, round_out, stats)
        cref = db0 + ref.sum(0)
        cerr = err.sum(0) + (M + 1) * U * (ref.abs().sum(0) + db0.abs())
        if round_out:
            cerr = cerr + ulp(ref.abs() + err, -126, 10).sum(0)
        report("dbias", bound("dbias", db, cref, cerr))
    else:
        check_out("C", C, ref, err, bool(c.get("rnd")) and bool(round_out), stats)
    if stats:
        print(f"  references within their error of a rounding boundary: {stats}")


def decoder_mode2_inputs(g):
    """First implicit decoder layer (Dreamer._dec_geo[1]: 5x5 -> 13x13, k = 5, 192 -> 96 channels) over T*B = 2500 images:
    the output gradient (NHWC) and the saved layer input (pixels x channels), both tf32."""
    hi, ho, k, ci, co = DEC_GEO[1]
    nb = 2500
    dout = tf32_rna(g.normal(nb, ho, ho, co, scale=0.1))
    xin = tf32_rna(F.elu(g.normal(nb * hi * hi, ci)))
    return dout, xin, k


@gpu
def test_conv_mode2_decoder_weight_gradient_at_step_shape(ops):
    """conv_gemm mode 2 (both operands MN-major: im2col boxes of the output gradient, the saved input) for the first
    implicit decoder layer at the step's shape: dW[(tap, c), ci] += sum over 62500 pixels, split over K."""
    g = Gen(77)
    dout, xin, k = decoder_mode2_inputs(g)
    nb, ho, _, co = dout.shape
    ci = xin.shape[1]
    px = xin.shape[0]
    bufs = Bufs()
    gdec = bufs.out(k * k * co, ci, init=torch.zeros(k * k * co, ci, dtype=torch.float64, device=DEV))
    ops.conv_gemm(2, dout.float().contiguous(), k, xin.float().contiguous(), gdec)
    bufs.check()

    def cols(x):                                 # NHWC -> [pixels, (kh, kw, c)] of the k x k stride-2 taps
        u = F.unfold(x.permute(0, 3, 1, 2), k, stride=2)                          # [nb, c*k*k, L]
        return u.view(nb, co, k, k, -1).permute(0, 4, 2, 3, 1).reshape(px, k * k * co)

    ref = cols(dout).T @ xin
    terms = cols(dout.abs()).T @ xin.abs()
    depth, splits = tc_depth(k * k * co, ci, cdiv(px, 32), True, may_skinny=False)
    assert splits > 1
    print(f"\ndecoder mode 2 dW depth {depth} splits {splits}")
    report("dW", bound("dW", gdec, ref, C_ACC * depth * U * terms))


@gpu
def test_mn_major_split_sums_are_identical_run_to_run(ops):
    """The split-K launches above (weight gradient, skinny B MN-major, conv mode 2) give bit-identical results run to run."""
    g = Gen(31)
    A, B = tf32_rna(g.normal(37500, 400)).float(), tf32_rna(g.normal(37500, 400, scale=0.01)).float()
    A2, B2 = tf32_rna(g.normal(50, 6144)).float(), tf32_rna(g.normal(6144, 2048, scale=0.01)).float()
    dout, xin, k = decoder_mode2_inputs(g)
    dout, xin = dout.float().contiguous(), xin.float().contiguous()
    C0 = tf32_rna(g.normal(400, 400)).float()
    assert tc_depth(400, 400, cdiv(37500, 32), True)[1] > 1
    assert tc_depth(50, 2048, 6144 // 32)[1] > 1

    def once():
        out = dict(wgrad=C0.clone(), skinny=torch.empty(50, 2048, device=DEV),
                   mode2=torch.zeros(k * k * dout.shape[3], xin.shape[1], device=DEV))
        ops.gemm(A, B, out["wgrad"], a_mn=True, b_mn=True, accumulate=True)
        ops.gemm(A2, B2, out["skinny"], b_mn=True)
        ops.conv_gemm(2, dout, k, xin, out["mode2"])
        sync()
        return out

    first = once()
    for _ in range(2):
        again = once()
        for name, v in first.items():
            assert torch.equal(v, again[name]), name
    assert math.isfinite(float(first["wgrad"].abs().sum()))

"""Kernel-level tests of the dense and implicit-convolution GEMM (csrc/pd_gemm_sm90.cu), its CUDA-core arms
(csrc/pd_gemm_simt.cu: gemv_rows, wcolsum, the generic validation kernel) and the convolution folds (csrc/pd_conv.cu:
im2col, col2im, col2im_actbwd, col2im_imgloss, permute4), called directly through NativeOps on seeded random operands and
compared with a FLOAT64 reference computed from the exact fp32 / fp16 values the kernel reads.

References.  Dense GEMM: A64 @ B64^T, + bias, + residual row m // r_div, F.elu.  Convolution layers: torch.autograd over
float64 F.conv2d / F.conv_transpose2d (+ F.elu), composed layer by layer exactly as pydreamer_b200/dreamer.py composes the
kernels; the RefOps twins are never the reference.  The ELU backward from a saved output is aten.elu_backward(is_result=True),
i.e. what autograd runs for F.elu; bias gradients are autograd's (or its column sum, for the dense GEMM).

Bounds.  Every element is bounded by its own error terms, never relative to a tensor maximum:
  * fp32 accumulation: C_ACC * depth * U * sum_k |a_k b_k|, U = 2^-24.  `depth` is the length of the element's fp32
    accumulation chain in the kernel: k-steps per split plus the number of splits (tc_depth restates pick_splits), the
    whole K on the CUDA-core arms.  sum_k |a_k b_k| is the same contraction over absolute values (for a convolution, the
    same autograd over absolute values).  C_ACC = 2 allows for the tensor core's internal accumulation of the 8 (tf32) or
    16 (fp16) products of one instruction; it is an allowance, not a measured constant;
  * raw fp32 operands (not pre-rounded to tf32): + 2 * 2^-10 * sum_k |a_k b_k| for the operand precision, whether the
    hardware truncates the low 13 bits or rounds them; fp16 operands have exact products, so only the accumulation term;
  * each further fp32 addition (bias, residual, accumulate into C, the taps of a fold) adds its depth in U of its terms;
  * the epilogue ELU adds the documented 5e-7 relative error of pd_elu (pd_common.cuh:104-125); |elu'| <= 1 carries the
    input error through.
  max(err / bound) is printed per case (run pytest with -s), so the slack of each bound is visible.

Rounded outputs.  An output rounded to tf32 (round_out with set_round_operands on) must be tf32-representable and equal
tf32_rna(reference) except within its error of a rounding boundary; an fp16 output equals reference.half() with the same
allowance.  round_out of pd_gemm / pd_gemm_f16 / pd_conv_gemm is gated by set_round_operands like every other producer:
tests run with rounding off and on.

Guard bands.  Outputs are pre-filled with NaN (or with non-zero values where they accumulate) and live inside storage whose
gap columns and trailing guard band hold a sentinel that must stay untouched; strided operands are views whose gap columns
hold NaN, so a read outside the view poisons the result.

CPU dry run.  PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/ref_ops.py in place of the kernels: a
dry run of the references and bounds without a GPU (the twins do not round, and have no host-side argument checks)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import CPU, DEV, Gen, bound, f64, fp16, fp32, ops, round_out, rounded, tf32_rna, ulp  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24                                  # unit roundoff of fp32
C_ACC = 2.0                                     # tensor-core accumulation allowance per chain step (not measured)
TF32_OP = 2.0 * 2.0 ** -10                      # raw fp32 operand read as tf32: truncated or rounded low 13 bits
ELU_REL = 5e-7                                  # relative error of pd_elu's ex2.approx branch (pd_common.cuh:104-125)
P = torch.cuda.get_device_properties(0).multi_processor_count if (not CPU and torch.cuda.is_available()) else 132
NAN = float("nan")
SENT = -12345.0                                 # sentinel of gap columns and guard bands
ACT_NONE, ACT_ELU = 0, 1
SCRATCH_FLOATS, SCRATCH_TICKETS = 4 << 20, 4096  # PD_SCRATCH_FLOATS / PD_SCRATCH_TICKETS (pd_common.cuh)
ENC_GEO = ((64, 31, 3, 48), (31, 14, 48, 96), (14, 6, 96, 192), (6, 2, 192, 384))           # Dreamer._enc_geo, cd = 48
DEC_GEO = ((1, 5, 5, 1536, 192), (5, 13, 5, 192, 96), (13, 30, 6, 96, 48), (30, 64, 6, 48, 3))  # Dreamer._dec_geo
NB = 6          # images: encoder layer 1 has 1176 output pixels (10 tiles of 128, a partial last 32-pixel block)


def cdiv(a, b):
    return -(-a // b)


def pick_splits(tiles, kb_total, slots, min_kb):
    """pd_gemm_sm90.cu pick_splits, restated: the split count minimising waves x (k-blocks per unit + 6) among those whose
    partial tiles fit the 16 MB scratch area; 1 with more tiles than tickets or fewer than two splits' room."""
    maxs = min(kb_total // min_kb, (SCRATCH_FLOATS // (128 * 128)) // tiles)
    if tiles > SCRATCH_TICKETS or maxs < 2:
        return 1
    best, best_cost = 1, 1e300
    for sp in range(1, maxs + 1):
        kbs = cdiv(kb_total, sp)
        if cdiv(kb_total, kbs) != sp:
            continue
        cost = cdiv(tiles * sp, slots) * (kbs + 6.0)
        if cost < best_cost - 1e-9:
            best, best_cost = sp, cost
    return best


def tc_depth(M, N, kb_total, accumulate=False, may_skinny=True):
    """Length of an output element's fp32 accumulation chain in pd_gemm_tf32_kernel: 4 k-steps (m16n8k8 tf32 / m16n8k16
    fp16, or one wgmma k8 / k16) per 128-byte k-block of its split, then the in-order sum of the splits.  Splits as
    pd_gemm_tc_launch / pd_conv_gemm_launch pick them: accumulating launches, and (dense GEMM only) skinny ones with one
    row of tiles on at most half the SMs and >= 8 k-blocks.  Returns (depth, splits)."""
    num_m, tiles = cdiv(M, 128), cdiv(M, 128) * cdiv(N, 128)
    skinny = may_skinny and num_m == 1 and tiles * 2 <= P and kb_total >= 8
    splits = pick_splits(tiles, kb_total, P, 8 if accumulate else 4) if (accumulate or skinny) else 1
    kbs = cdiv(kb_total, splits)
    splits = cdiv(kb_total, kbs)
    return 4 * kbs + splits, splits


def simt_depth(K):
    """CUDA-core arms: the generic kernel's per-element fma chain is K long; gemv_rows (K/32 per lane + 5 shuffle levels)
    and wcolsum (rows per thread + 8 + blocks) are shorter."""
    return K + 16


# ----------------------------------------------------------------------------------------------------- buffers
class Bufs:
    """Storage for kernel outputs: the view the kernel writes (pre-filled) inside storage whose every other element (gap
    columns and a guard band after the last row) holds a sentinel that must stay untouched."""

    def __init__(self):
        self.items = []

    def out(self, rows, n, dtype=torch.float32, gap=0, off=0, init=None):
        ld = n + gap
        flat = torch.full((off + rows * ld + 512,), SENT, dtype=dtype, device=DEV)
        view = flat[off:off + rows * ld].view(rows, ld)[:, :n]
        if init is None:
            view.fill_(NAN)
        else:
            view.copy_(init.reshape(rows, n))
        keep = torch.ones(flat.numel(), dtype=torch.bool, device=DEV)
        keep[off:off + rows * ld].view(rows, ld)[:, :n] = False
        self.items.append((flat, keep, flat.clone()))
        return view

    def check(self):
        sync()
        for i, (flat, keep, before) in enumerate(self.items):
            iv = {4: torch.int32, 2: torch.int16}[flat.element_size()]
            assert torch.equal(flat.view(iv)[keep], before.view(iv)[keep]), f"output {i}: written outside its view"


def tma_gap(cols, dtype=torch.float32):
    """Gap columns that make rows of `cols` elements TMA-addressable (16-byte rows), at least 16 bytes of them."""
    q = 8 if dtype == torch.float16 else 4
    return (-cols) % q + q


def operand(v, gap=0, off=0, dtype=torch.float32):
    """The 2-D float64 v as a `dtype` view into rows of ld = cols + gap, starting `off` elements into its storage; gap
    columns and the leading elements hold NaN."""
    r, c = v.shape
    flat = torch.full((off + r * (c + gap) + 64,), NAN, dtype=dtype, device=DEV)
    view = flat[off:off + r * (c + gap)].view(r, c + gap)[:, :c]
    view.copy_(v)
    return view


def sync():
    if not CPU:
        torch.cuda.synchronize()


def report(name, ratio):
    print(f"  {name}: max err/bound {ratio:.3g}")


def check_out(name, got, ref, err, rnd, stats):
    """An output the kernel rounds to tf32 when rnd (round_out and set_round_operands both on); the float32 twins of the
    dry run never round, so there the bound widens by one tf32 ulp instead."""
    if rnd and not CPU:
        assert ((got.contiguous().view(torch.int32) & 0x1FFF) == 0).all(), f"{name}: not tf32-rounded"
        rounded(name, got, ref, err, "tf32", stats)
        report(name, bound(name, got, ref, err + ulp(torch.maximum(ref.abs(), got.double().abs()), -126, 10)))
    else:
        report(name, bound(name, got, ref, err + (ulp(ref, -126, 10) if rnd else 0.0)))


def elu_bwd_from_out(g, y):
    """Autograd's ELU backward from the saved output (alpha 1): g * (y > 0 ? 1 : y + 1)."""
    return torch.ops.aten.elu_backward(g, 1.0, 1, 1, True, y)


# ----------------------------------------------------------------------------------------------------- dense GEMM
def case(name, M, N, K, **kw):
    return pytest.param(dict(M=M, N=N, K=K, **kw), id=name)


# Each case names the branch it exists for and the condition that selects it, and declares the kernel that must run it
# (`arm`: the wgmma or the mma.sync instantiation of pd_gemm_tf32_kernel, gemv_rows, wcolsum or the generic CUDA-core
# kernel) and, where it matters, whether pick_splits splits it (`split`, for P = 132 SMs).  Operands and C have rows of
# ld % 4 == 0 (fp16: % 8) unless a case asks for another gap.
GEMM_CASES = [
    # RSSM step GEMMs (M = B*I = 50): one row of tiles, long K -> skinny split-K (pd_gemm_sm90.cu:704, num_m == 1,
    # tiles * 2 <= #SMs, >= 8 k-blocks); wgmma instantiation (both operands K-major, :552)
    case("rssm_k1024_skinny_wgmma_bias_elu", 50, 1024, 1024, arm="wgmma", split=True, bias=True, act=ACT_ELU, rnd=1),
    case("rssm_k2048_skinny_raw_residual", 50, 1536, 2048, arm="wgmma", split=True, opnd="raw", res="rows", rnd=1),
    case("rssm_k6144_skinny_partial_n", 50, 200, 6144, arm="wgmma", split=True, bias=True, rnd=1),
    # head MLPs: 2500 rows = 19 full tiles + 68 rows (cuts a 16-row wgmma store box); N = 400 leaves 16 columns in the
    # last 32-column box; no split (20 x 4 tiles)
    case("head_mlp_wgmma_partial_m_n", 2500, 400, 3072, arm="wgmma", split=False, bias=True, act=ACT_ELU, rnd=1),
    case("head_mlp_residual_rdiv50", 2500, 400, 3072, arm="wgmma", opnd="raw", res="rows", r_div=50, rnd=1),
    case("head_mlp_residual_in_place", 2500, 400, 1000, arm="wgmma", bias=True, res="inplace", act=ACT_ELU, rnd=1),
    # decoder Linear (N = 1536 = 32 * cd): raw fp32 operands; partial last k-block (K % 32 = 17; rows padded to lda = 1044)
    case("decoder_linear_raw_partial_k", 300, 1536, 1041, arm="wgmma", opnd="raw", bias=True, rnd=1),
    # mma.sync instantiation: an MN-major operand (:552).  M = 300 / N = 264: MN % 32 != 0 -> the 3-D box holds a partial
    # column group and the tiles holding it take 2-D boxes (a3_part / b3_part, :509-511, :106)
    case("mma_a_mn_partial_group", 300, 264, 100, arm="mma", a_mn=1, bias=True, act=ACT_ELU, rnd=1),
    case("mma_b_mn_partial_group_raw", 300, 264, 100, arm="mma", b_mn=1, opnd="raw", res="rows", rnd=1),
    case("mma_both_mn_rows_cut_at_32", 140, 200, 333, arm="mma", a_mn=1, b_mn=1, bias=True, rnd=1),
    # weight gradients (K = 2500 rows, both MN-major, accumulate into non-zero C): split-K with a fixed-order partial
    # sum (pick_splits, :705); 2500 % 32 != 0 -> partial last k-block; M = 400 -> a3_part
    case("wgrad_head_accumulate_splitk", 400, 1024, 2500, arm="mma", split=True, a_mn=1, b_mn=1, acc=True),
    # accumulate with more than 128 tiles: the partial tiles do not fit the scratch area -> pick_splits returns 1 (:570)
    case("wgrad_accumulate_170_tiles_no_split", 1200, 2100, 2500, arm="mma", split=False, a_mn=1, b_mn=1, acc=True),
    # actor logits (N = 18): C rows of 18 floats with ldc = 18 -> not TMA-addressable (ldc % 4 != 0, :687): the generic
    # store epilogue, without and with accumulate (atomicAdd after the split sum, :411-426: ldc = 401, 4 tiles, A [2500][18]
    # in rows of lda = 20 so that the tensor cores take it)
    case("actor_logits_generic_store", 300, 18, 400, arm="wgmma", bias=True, act=ACT_ELU, rnd=1, c_gap=0),
    case("generic_store_accumulate_split", 18, 400, 2500, arm="mma", split=True, a_mn=1, b_mn=1, acc=True, c_gap=1),
    # fp16 operands (pd_gemm_f16): skinny split and a full head, with every epilogue term
    case("f16_rssm_skinny", 50, 1024, 2048, arm="wgmma", split=True, opnd="f16", bias=True, act=ACT_ELU, rnd=1),
    case("f16_head_residual_rdiv", 2500, 400, 3072, arm="wgmma", opnd="f16", bias=True, res="rows", r_div=50, act=ACT_ELU, rnd=1),
    # fp16 C (PD_GEMM_C_F16: the decoder's column matrices): TMA store of fp16 boxes; with skinny split
    case("c_f16_columns", 700, 1200, 96, arm="wgmma", c16=True, bias=True),
    case("c_f16_skinny_split", 50, 1200, 2048, arm="wgmma", split=True, c16=True, act=ACT_ELU),
    # fused ELU backward (pd_gemm_actbwd): dX of a deconvolution / Linear; M <= 128 -> skinny split
    case("actbwd_deconv_b_mn", 900, 48, 108, arm="mma", b_mn=1, actbwd=True),
    case("actbwd_skinny_split", 100, 512, 2048, arm="wgmma", split=True, actbwd=True),
    case("actbwd_generic_store_falls_back", 200, 18, 64, arm="wgmma", actbwd=True, c_gap=1),   # ldc % 4 != 0 (pd_api.cu:150)
    # CUDA-core product paths (pd_gemm_simt.cu:129-149):
    case("scalar_head_gemv_n1", 2500, 1, 400, arm="gemv", bias=True, res="rows", r_div=50, act=ACT_ELU, rnd=1),   # N <= 4, K-major
    case("gemv_n4", 333, 4, 1000, arm="gemv", bias=True, act=ACT_ELU, rnd=1),
    # M <= 4, accumulate, both MN-major, A = the head's output gradient [K][M] with ld = M: not TMA-addressable
    case("wcolsum_m1", 1, 400, 2500, arm="wcolsum", a_mn=1, b_mn=1, acc=True, a_gap=0),
    case("wcolsum_m3", 3, 1000, 2500, arm="wcolsum", a_mn=1, b_mn=1, acc=True, a_gap=0),
    # generic SIMT via tma_ok false (pd_api.cu:111-115)
    case("simt_n_below_8", 300, 6, 400, arm="simt", bias=True, act=ACT_ELU, rnd=1),          # N < 8 (and > 4: not gemv)
    case("simt_k_below_8", 300, 400, 6, arm="simt", bias=True, rnd=1),                        # K < 8
    case("simt_lda_not_multiple_of_4", 300, 400, 18, arm="simt", a_gap=1, bias=True, rnd=1),  # lda = 19
    case("simt_a_misaligned", 300, 400, 64, arm="simt", a_off=1, a_gap=0, res="rows", rnd=1),          # A 4 bytes off a 16-byte boundary
    case("simt_b_mn_accumulate_misaligned", 200, 96, 500, arm="simt", b_mn=1, acc=True, a_off=1),
    # SIMT validation arm (set_gemm_impl(1)): the same contract on the plain kernel
    case("impl_simt_epilogue", 300, 264, 100, arm="simt", impl=1, bias=True, res="rows", r_div=3, act=ACT_ELU, rnd=1),
    case("impl_simt_accumulate_mn", 130, 200, 700, arm="simt", impl=1, a_mn=1, b_mn=1, acc=True),
    case("impl_simt_c_f16", 100, 96, 200, arm="simt", impl=1, c16=True, bias=True, act=ACT_ELU),
]


def gemm_inputs(c, g):
    M, N, K = c["M"], c["N"], c["K"]
    s = 1.0 / math.sqrt(K)                      # outputs of order 1: the ELU sees both of its branches (|x| < 0.25 too)
    opnd = c.get("opnd", "tf32")
    rd = {"tf32": lambda v: tf32_rna(v), "raw": fp32, "f16": fp16}[opnd]
    A, B = rd(g.normal(M, K, scale=1.0)), rd(g.normal(N, K, scale=s))
    bias = fp32(g.normal(N, scale=0.5)) if c.get("bias") else None
    R = None
    if c.get("res") == "rows":
        R = fp32(g.normal(cdiv(M, c.get("r_div", 1)), N, scale=0.5))
    elif c.get("res") == "inplace" or c.get("acc"):
        R = fp32(g.normal(M, N, scale=0.5))     # the residual read from C itself / the values C accumulates onto
    dact = fp32(F.elu(g.normal(M, N, scale=1.0))) if c.get("actbwd") else None
    return A, B, bias, R, dact


def dispatch(c, lda, ldb, ldc):
    """The kernel a case reaches, restating the host dispatch: pd_gemm_f16 always runs on the tensor cores; pd_gemm
    (pd_api.cu:111-116, and pd_gemm_actbwd's fallback) sends the validation arm and every call a TMA map cannot describe
    to the CUDA cores, whose product paths are gemv_rows (N <= 4, K-major, storing) and wcolsum (M <= 4, both MN-major,
    accumulating) (pd_gemm_simt.cu:129-149); the tensor-core kernel runs its wgmma instantiation when both operands are
    K-major and mma.sync otherwise (pd_gemm_sm90.cu:552)."""
    M, N, K, a_mn, b_mn, acc = c["M"], c["N"], c["K"], c.get("a_mn", 0), c.get("b_mn", 0), c.get("acc", False)
    if c.get("opnd") != "f16":
        tma_ok = lda % 4 == 0 and ldb % 4 == 0 and not c.get("a_off") and N >= 8 and K >= 8 and \
            (not c.get("c16") or ldc % 8 == 0)
        if c.get("impl", 0) == 1 or not tma_ok:
            if c.get("impl", 0) == 0 and not acc and not c.get("c16") and N <= 4 and not a_mn and not b_mn:
                return "gemv"
            if c.get("impl", 0) == 0 and acc and M <= 4 and a_mn and b_mn:
                return "wcolsum"
            return "simt"
    return "mma" if (a_mn or b_mn) else "wgmma"


def gemm_ref(c, A, B, bias, R, dact, simt):
    """float64 result, its bound before any output rounding, and the chain depth used."""
    M, N, K = c["M"], c["N"], c["K"]
    opnd = c.get("opnd", "tf32")
    kb = cdiv(K, 64 if opnd == "f16" else 32)
    depth = simt_depth(K) if simt else tc_depth(M, N, kb, c.get("acc", False))[0]
    ref = A @ B.T
    terms = A.abs() @ B.abs().T
    err = C_ACC * depth * U * terms
    if opnd == "raw" and not simt:
        err = err + TF32_OP * terms
    extra = torch.zeros_like(ref)
    if bias is not None:
        ref, extra = ref + bias, extra + bias.abs()
    if R is not None and not c.get("acc"):
        rr = R[torch.arange(M, device=R.device) // c.get("r_div", 1)] if c.get("res") == "rows" else R
        ref, extra = ref + rr, extra + rr.abs()
    err = err + 2 * U * (terms + extra)         # the bias and residual additions
    if c.get("acc"):
        ref = R + ref
        err = err + U * (ref.abs() + R.abs())   # one addition into C (TMA reduce-add / atomicAdd / +=)
    if c.get("act") == ACT_ELU:
        ref = F.elu(ref)
        err = err + (ELU_REL + U) * ref.abs()
    if dact is not None:
        g = ref
        ref = elu_bwd_from_out(g, dact)
        err = err * (dact.clamp(max=0) + 1) + 2 * U * (g.abs() * (dact.clamp(max=0) + 1))
    return ref, err, depth


@gpu
@pytest.mark.parametrize("c", GEMM_CASES)
def test_gemm_matches_float64_reference(ops, round_out, c):
    M, N, K = c["M"], c["N"], c["K"]
    g = Gen(M * 7 + N * 3 + K)
    A, B, bias, R, dact = gemm_inputs(c, g)
    f16 = c.get("opnd") == "f16"
    dt = torch.float16 if f16 else torch.float32
    a_mn, b_mn = c.get("a_mn", 0), c.get("b_mn", 0)
    As, Bs = A.T if a_mn else A, B.T if b_mn else B
    Ad = operand(As, gap=c.get("a_gap", tma_gap(As.shape[1], dt)), off=c.get("a_off", 0), dtype=dt)
    Bd = operand(Bs, gap=tma_gap(Bs.shape[1], dt), dtype=dt)
    cdt = torch.float16 if c.get("c16") else torch.float32
    c_gap = c.get("c_gap", tma_gap(N, cdt))
    arm = dispatch(c, Ad.stride(0), Bd.stride(0), N + c_gap)
    assert arm == c["arm"], f"the case reaches {arm}, not the {c['arm']} kernel it exists for"
    simt = arm in ("gemv", "wcolsum", "simt")
    if "split" in c:
        assert (tc_depth(M, N, cdiv(K, 64 if f16 else 32), c.get("acc", False))[1] > 1) == c["split"]
    ref, err, depth = gemm_ref(c, A, B, bias, R, dact, simt)
    bufs = Bufs()
    C = bufs.out(M, N, dtype=cdt, gap=c_gap,
                 init=R if (c.get("acc") or c.get("res") == "inplace") else None)
    biasd = None if bias is None else bias.float()
    resd = None
    if c.get("res") == "rows":
        resd = operand(R, gap=3)
    elif c.get("res") == "inplace":
        resd = C
    if c.get("actbwd"):
        db0 = fp32(g.normal(N, scale=0.5))
        db = bufs.out(1, N, init=db0).view(N)

    def call():
        if c.get("actbwd"):
            ops.gemm_actbwd(Ad, Bd, C, dact.float(), db, a_mn=bool(a_mn), b_mn=bool(b_mn))
        elif f16:
            ops.gemm_f16(Ad, Bd, C, bias=biasd, res=resd, r_div=c.get("r_div", 1), act=c.get("act", 0),
                         round_out=bool(c.get("rnd")))
        else:
            ops.gemm(Ad, Bd, C, a_mn=bool(a_mn), b_mn=bool(b_mn), bias=biasd, res=resd, r_div=c.get("r_div", 1),
                     act=c.get("act", 0), round_out=bool(c.get("rnd")), accumulate=bool(c.get("acc")))

    ops.set_gemm_impl(c.get("impl", 0))
    try:
        call()
    finally:
        ops.set_gemm_impl(0)
    bufs.check()
    stats = {}
    print(f"\n{M}x{N}x{K} {arm}, depth {depth}")
    if c.get("c16"):
        if CPU:
            report("C", bound("C", C, ref, err + ulp(ref, -14, 10)))
        else:
            rounded("C", C, ref, err, "fp16", stats)
            report("C", bound("C", C, ref, err + ulp(torch.maximum(ref.abs(), C.double().abs()), -14, 10)))
    elif c.get("actbwd"):
        check_out("C", C, ref, err, round_out, stats)
        # dbias += column sums of C (pd_colsum of the stored C, or bias_act_bwd's sums of the unrounded values)
        cref = db0 + ref.sum(0)
        cerr = err.sum(0) + (M + 1) * U * (ref.abs().sum(0) + db0.abs())
        if round_out:
            cerr = cerr + ulp(ref.abs() + err, -126, 10).sum(0)
        report("dbias", bound("dbias", db, cref, cerr))
    else:
        check_out("C", C, ref, err, bool(c.get("rnd")) and bool(round_out), stats)
    if stats:
        print(f"  references within their error of a rounding boundary: {stats}")


@gpu
@pytest.mark.parametrize("which", ["gemm", "gemm_f16", "conv_gemm"])
def test_round_out_follows_set_round_operands(ops, round_out, which):
    """round_out = 1 rounds the GEMM output to tf32 only while set_round_operands is on, as for every producer
    (pd_b200.h: 0 keeps full fp32 outputs); with it off the output keeps its low mantissa bits."""
    g = Gen(11)
    if which == "conv_gemm":
        X = tf32_rna(g.normal(2, 14, 14, 96))
        w = tf32_rna(g.normal(192, 4, 4, 96, scale=0.05))
        C = torch.full((2 * 36, 192), NAN, device=DEV)
        ops.conv_gemm(1, X.float().contiguous(), 4, w.reshape(192, -1).float().contiguous(), C, round_out=True)
        ref = F.conv2d(X.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1).reshape(72, 192)
        terms = F.conv2d(X.abs().permute(0, 3, 1, 2), w.abs().permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1).reshape(72, 192)
        depth = tc_depth(72, 192, 16 * 3, may_skinny=False)[0]
    else:
        dt = torch.float16 if which == "gemm_f16" else torch.float32
        rd = fp16 if which == "gemm_f16" else tf32_rna
        A, B = rd(g.normal(300, 512)), rd(g.normal(256, 512, scale=0.05))
        C = torch.full((300, 256), NAN, device=DEV)
        getattr(ops, which)(A.to(dt), B.to(dt), C, round_out=True)
        ref, terms = A @ B.T, A.abs() @ B.abs().T
        depth = tc_depth(300, 256, cdiv(512, 64 if dt == torch.float16 else 32))[0]
    sync()
    err = C_ACC * depth * U * terms
    check_out(which, C, ref, err, bool(round_out), {})
    if not CPU and not round_out:
        assert ((C.view(torch.int32) & 0x1FFF) != 0).any(), f"{which}: output tf32-rounded with rounding off"


# ----------------------------------------------------------------------------------------------------- convolutions
def conv_case(li, implicit):
    return pytest.param(li, implicit, id=f"layer{li}-{'implicit' if implicit else 'explicit'}")


def nchw(x):
    return x.permute(0, 3, 1, 2)


def nhwc_rows(x):                               # NCHW float64 -> (pixels, channels) rows
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def image(g):
    """NB preprocessed images (uint8 / 255 - 0.5, preprocessing.py:21-29): fp32 values a tf32 operand cannot hold, in the
    NHWC index order; the product stores them NCHW (obs["image"]) and gathers them through the [n,y,x,c] view."""
    return fp32(torch.floor(g.rand(NB, 64, 64, 3) * 256).clamp(max=255) / 255 - 0.5)


def image_view(x):
    """The NCHW fp32 image as the [n,y,x,c] view Dreamer hands to im2col (dreamer.py:928-932: sX = 1 -> the planar
    k = 4 gather with korder 1, pd_conv.cu:383-389)."""
    return nchw(x).float().contiguous().permute(0, 2, 3, 1)


def image_operand(x, round_out):
    """The image values the layer-0 GEMM reads: im2col rounds them to tf32 while rounding is on (the float32 twin never
    does), and the tensor cores read raw fp32 ones with 10 mantissa bits; returns them and the operand-precision share."""
    if round_out and not CPU:
        return tf32_rna(x), 0.0
    return x, TF32_OP


ENC_FWD = [conv_case(0, False)] + [conv_case(li, imp) for li in (1, 2, 3) for imp in (False, True)]


@gpu
@pytest.mark.parametrize("li,implicit", ENC_FWD)
def test_encoder_layer_forward_matches_conv2d(ops, round_out, li, implicit):
    """dreamer.py:928-943: implicit conv_gemm mode 1 (layers 2-4), or im2col + gemm, with bias + ELU + round_out.  Layer 1
    gathers the NCHW image through its [n,y,x,c] view with korder 1 (the planar k = 4 kernel), matching the NCHW-ordered
    nn.Conv2d weight; the others take NHWC activations, korder 0 and the weight regrouped (Cout,Cin,kh,kw) ->
    (Cout,(kh,kw,Cin)) by permute4 as Dreamer._prepare_weights does (dreamer.py:563-571).  Against
    F.elu(F.conv2d(x, w, b, stride=2))."""
    hin, hout, ci, co = ENC_GEO[li]
    g = Gen(100 + li)
    x = image(g) if li == 0 else tf32_rna(g.normal(NB, hin, hin, ci))         # NHWC order; layers 2-4: rounded activations
    w = tf32_rna(g.uniform(co, ci, 4, 4, bound=1 / math.sqrt(16 * ci)))        # nn.Conv2d layout
    b = fp32(g.uniform(co, bound=0.5))
    px = NB * hout * hout
    bufs = Bufs()
    act = bufs.out(px, co)
    x4 = image_view(x) if li == 0 else x.float().contiguous()
    if li == 0:
        Wg = w.float().reshape(co, -1)                                        # (c,kh,kw) order == im2col korder 1
    else:
        Wg = torch.empty(co, 4, 4, ci, device=DEV)
        ops.permute4(w.float().contiguous(), Wg, (0, 2, 3, 1))
        Wg = Wg.view(co, 16 * ci)
    if implicit:
        ops.conv_gemm(1, x4, 4, Wg, act, bias=b.float(), act=ACT_ELU, round_out=True)
        depth = tc_depth(px, co, 16 * cdiv(ci, 32), may_skinny=False)[0]
    else:
        col = bufs.out(px, 16 * ci)
        ops.im2col(x4, 4, 1 if li == 0 else 0, col, round_out=True)
        ops.gemm(col, Wg, act, bias=b.float(), act=ACT_ELU, round_out=True)
        depth = tc_depth(px, co, cdiv(16 * ci, 32))[0]
    bufs.check()
    x, op_err = image_operand(x, round_out) if li == 0 else (x, 0.0)
    pre = nhwc_rows(F.conv2d(nchw(x), w, b, stride=2))
    terms = nhwc_rows(F.conv2d(nchw(x).abs(), w.abs(), b.abs(), stride=2))
    ref = F.elu(pre)
    err = (C_ACC * (depth + 1) * U + op_err) * terms + (ELU_REL + U) * ref.abs()
    print(f"\nencoder layer {li} {'implicit' if implicit else 'explicit'} depth {depth}")
    check_out("act", act, ref, err, bool(round_out), {})


ENC_BWD = [conv_case(0, False)] + [conv_case(li, imp) for li in (1, 2, 3) for imp in (False, True)]


@gpu
@pytest.mark.parametrize("li,implicit", ENC_BWD)
def test_encoder_layer_backward_matches_autograd(ops, round_out, li, implicit):
    """dreamer.py:1318-1334: the weight gradient by conv_gemm mode 3 into the 32-channel-padded layout (or gemm over the
    saved im2col matrix), the column gradient gemm(da, W), col2im_actbwd through the ELU of the layer below (with its bias
    gradient; layer 1's 31-wide input has a last row / column the conv never reads) and permute4 of the weight gradient
    back into the nn.Conv2d layout.  Layer 1 (dreamer.py:1331) has no input gradient: its weight gradient is a gemm over
    the korder-1 column matrix of the image, accumulated straight into the nn.Conv2d weight's gradient, whose
    (Cin,kh,kw)-major rows need no permute4.  Against float64 autograd of F.conv2d and F.elu."""
    hin, hout, ci, co = ENC_GEO[li]
    g = Gen(200 + li)
    px = NB * hout * hout
    a_prev = image(g) if li == 0 else tf32_rna(F.elu(g.normal(NB, hin, hin, ci)))   # the image / layer li-1's saved output
    w = tf32_rna(g.uniform(co, ci, 4, 4, bound=1 / math.sqrt(16 * ci)))
    da = tf32_rna(g.normal(px, co, scale=0.1))                                 # gradient at layer li's pre-activation
    db0 = fp32(g.normal(ci, scale=0.1))

    def grads(a, wt, d):
        a = nchw(a).clone().requires_grad_(True)
        wt = wt.clone().requires_grad_(True)
        bb = torch.zeros(co, dtype=f64, device=DEV, requires_grad=True)
        y = F.conv2d(a, wt, bb, stride=2)
        (y * nchw(d.view(NB, hout, hout, co))).sum().backward()
        return a.grad.permute(0, 2, 3, 1), wt.grad, bb.grad

    if li == 0:
        g0 = fp32(g.normal(co, ci * 16, scale=0.1))                            # the gradient accumulates onto these
        bufs = Bufs()
        col = bufs.out(px, 16 * ci)
        ops.im2col(image_view(a_prev), 4, 1, col, round_out=True)
        gW = bufs.out(co, 16 * ci, init=g0)
        ops.gemm(da.float().contiguous(), col, gW, a_mn=True, b_mn=True, accumulate=True)
        bufs.check()
        xr, op_err = image_operand(a_prev, round_out)
        _, gwt, _ = grads(xr, w, da)
        _, twt, _ = grads(xr.abs(), w.abs(), da.abs())
        ref, twt = g0 + gwt.reshape(co, -1), twt.reshape(co, -1)
        dw_depth = tc_depth(co, 16 * ci, cdiv(px, 32), True)[0]
        print(f"\nencoder layer 0 backward dW depth {dw_depth}")
        report("dW", bound("dW", gW, ref, (C_ACC * dw_depth * U + op_err) * twt + U * (ref.abs() + g0.abs())))
        return
    cpad = cdiv(ci, 32) * 32 if implicit else ci
    bufs = Bufs()
    gw = bufs.out(co, 16 * cpad, init=torch.zeros(co, 16 * cpad, dtype=f64, device=DEV))
    a4, dad = a_prev.float().contiguous(), da.float().contiguous()
    Wg = torch.empty(co, 4, 4, ci, device=DEV)
    ops.permute4(w.float().contiguous(), Wg, (0, 2, 3, 1))
    Wg = Wg.view(co, 16 * ci)
    if implicit:
        ops.conv_gemm(3, a4, 4, dad, gw)
        dw_depth = tc_depth(co, 16 * cpad, cdiv(px, 32), True, may_skinny=False)[0]
    else:
        col = bufs.out(px, 16 * ci)
        ops.im2col(a4, 4, 0, col, round_out=True)
        ops.gemm(dad, col, gw, a_mn=True, b_mn=True, accumulate=True)
        dw_depth = tc_depth(co, 16 * ci, cdiv(px, 32), True)[0]
    dcol = bufs.out(px, 16 * ci)
    ops.gemm(dad, Wg, dcol, b_mn=True)
    dprev = torch.full((NB, hin, hin, ci), NAN, device=DEV)
    db = bufs.out(1, ci, init=db0).view(ci)
    ops.col2im_actbwd(dcol, hout, hout, 4, a4, db, dprev)
    gW = torch.full((co, ci, 4, 4), NAN, device=DEV)
    ops.permute4(gw.view(co, 4, 4, cpad)[..., :ci], gW, (0, 3, 1, 2))
    bufs.check()

    ga, gwt, _ = grads(a_prev, w, da)
    ta, twt, _ = grads(a_prev.abs(), w.abs(), da.abs())                        # the same sums over absolute values
    print(f"\nencoder layer {li} backward {'implicit' if implicit else 'explicit'} dW depth {dw_depth}")
    report("dW", bound("dW", gW, gwt, C_ACC * dw_depth * U * twt))
    # input gradient: gemm (K = co, not rounded) -> fold of <= 4 taps -> * elu'(a_prev) -> tf32 when rounding is on
    dx_depth = tc_depth(px, 16 * ci, cdiv(co, 32))[0]
    dref = elu_bwd_from_out(ga, a_prev)
    e = a_prev.clamp(max=0) + 1
    derr = C_ACC * (dx_depth + 4) * U * ta * e + 2 * U * ga.abs() * e
    check_out("dx", dprev, dref, derr, bool(round_out), {})
    # bias gradient of layer li-1: autograd of its bias = the sum of dref over pixels
    bref = db0 + dref.sum((0, 1, 2))
    berr = derr.sum((0, 1, 2)) + (NB * hin * hin + 1) * U * (dref.abs().sum((0, 1, 2)) + db0.abs())
    report("dbias", bound("dbias", db, bref, berr))


@gpu
@pytest.mark.parametrize("Cc", [20, 48])
def test_col2im_actbwd_fused_and_composed_match_autograd(ops, round_out, Cc):
    """pd_col2im_actbwd on the 31-wide encoder input: Cc = 48 takes the fused kernel, Cc = 20 the composed fallback
    (192 % (Cc / 4) != 0: col2im + bias_act_bwd, pd_conv.cu:443-449).  The fold is the adjoint of F.unfold, taken by
    autograd; rows / columns the unfold never reads get zero gradient."""
    Hin, Hout, k = 14, 31, 4
    g = Gen(Cc)
    col = fp32(g.normal(NB * Hin * Hin, k * k * Cc))
    dact = tf32_rna(F.elu(g.normal(NB, Hout, Hout, Cc)))
    db0 = fp32(g.normal(Cc, scale=0.1))
    out = torch.full((NB, Hout, Hout, Cc), NAN, device=DEV)
    bufs = Bufs()
    db = bufs.out(1, Cc, init=db0).view(Cc)
    ops.col2im_actbwd(col.float(), Hin, Hin, k, dact.float().contiguous(), db, out)
    bufs.check()

    def fold(c):
        X = torch.zeros(NB, Cc, Hout, Hout, dtype=f64, device=DEV, requires_grad=True)
        u = F.unfold(X, k, stride=2)                                          # (NB, (c,kh,kw), L)
        u = u.view(NB, Cc, k, k, -1).permute(0, 4, 2, 3, 1).reshape(NB * Hin * Hin, k * k * Cc)
        (u * c).sum().backward()
        return X.grad.permute(0, 2, 3, 1)

    f, fa = fold(col), fold(col.abs())
    ref = elu_bwd_from_out(f, dact)
    e = dact.clamp(max=0) + 1
    err = 4 * U * fa * e + 2 * U * f.abs() * e
    check_out("dx", out, ref, err, bool(round_out), {})
    bref = db0 + ref.sum((0, 1, 2))
    report("dbias", bound("dbias", db, bref, err.sum((0, 1, 2)) + (NB * Hout * Hout + 1) * U * (ref.abs().sum((0, 1, 2)) + db0.abs())))


DEC_FWD = [pytest.param(li, c16, id=f"layer{li}-{'f16' if c16 else 'f32'}cols") for li in range(4) for c16 in (False, True)]


@gpu
@pytest.mark.parametrize("li,c16", DEC_FWD)
def test_decoder_layer_forward_matches_conv_transpose2d(ops, round_out, li, c16):
    """dreamer.py:1115-1127: gemm of the layer input with the (kh,kw,Cout)-major weight (permute4 of the ConvTranspose2d
    weight, dreamer.py:573-579) into an fp32 or fp16 column matrix, then col2im (+ bias, ELU, round_out) or, for the last
    layer, col2im_imgloss against a target shared by tgt_div = 2 rows.  Layers 0-2 fold with col2im_v4; the last layer
    writes the NCHW image through the scalar col2im.  Against F.conv_transpose2d (+ F.elu) and 0.5 * sum diff^2."""
    hi, ho, k, ci, co = DEC_GEO[li]
    g = Gen(300 + li)
    N = NB
    x = tf32_rna(F.elu(g.normal(N * hi * hi, ci))) if li else tf32_rna(g.normal(N, ci))
    w = tf32_rna(g.uniform(ci, co, k, k, bound=1 / math.sqrt(ci)))           # nn.ConvTranspose2d layout
    b = fp32(g.uniform(co, bound=0.5))
    ncol = k * k * co
    bufs = Bufs()
    cols = bufs.out(N * hi * hi, ncol, dtype=torch.float16 if c16 else torch.float32)
    Wg = torch.empty(k, k, co, ci, device=DEV)
    ops.permute4(w.float().contiguous(), Wg, (2, 3, 1, 0))
    ops.gemm(x.float().contiguous(), Wg.view(ncol, ci), cols)
    xin = nchw(x.view(N, hi, hi, ci))
    pre = F.conv_transpose2d(xin, w, b, stride=2)                            # (N, co, ho, ho)
    terms = F.conv_transpose2d(xin.abs(), w.abs(), b.abs(), stride=2)
    gdepth = tc_depth(N * hi * hi, ncol, cdiv(ci, 32))[0]
    if c16 and (ncol % 8 or CPU):
        gdepth = max(gdepth, simt_depth(ci))    # fp16 C without 16-byte rows: the CUDA-core kernel writes it
    taps = cdiv(k, 2) ** 2
    err = C_ACC * (gdepth + taps + 1) * U * terms
    if c16:
        err = err + 2.0 ** -11 * terms + taps * 2.0 ** -25                   # each column element rounded to fp16
    stats = {}
    print(f"\ndecoder layer {li} forward {'fp16' if c16 else 'fp32'} columns, gemm depth {gdepth}")
    if c16:
        cref = (x @ Wg.double().view(ncol, ci).T)
        cerr = C_ACC * gdepth * U * (x.abs() @ Wg.double().view(ncol, ci).abs().T)
        if CPU:
            report("cols", bound("cols", cols, cref, cerr + ulp(cref, -14, 10)))
        else:
            rounded("cols", cols, cref, cerr, "fp16", stats)
    if li < 3:
        out = bufs.out(N * ho * ho, co).view(N, ho, ho, co)
        ops.col2im(cols, hi, hi, k, b.float(), ACT_ELU, out, round_out=True)
        bufs.check()
        ref = F.elu(pre).permute(0, 2, 3, 1)
        check_out("out", out, ref, err.permute(0, 2, 3, 1) + (ELU_REL + U) * ref.abs(), bool(round_out), stats)
        return
    # last layer: the image itself (scalar col2im into the NCHW image, no ELU, no rounding; fp32 columns only, as
    # Dreamer._cols_dtype keeps them for k*k*3 columns) and the fused image loss
    if not c16:
        img = torch.full((N, co, ho, ho), NAN, device=DEV)
        ops.col2im(cols, hi, hi, k, b.float(), ACT_NONE, img.permute(0, 2, 3, 1), round_out=False)
        sync()
        report("image", bound("image", img, pre, err))
    tgt = fp32(g.normal(N // 2, co, ho, ho, scale=0.5))
    dec, diff = torch.full((N, co, ho, ho), NAN, device=DEV), torch.full((N, co, ho, ho), NAN, device=DEV)
    loss, csum = bufs.out(1, N).view(N), bufs.out(N, co)
    ops.col2im_imgloss(cols, N, hi, hi, co, k, b.float(), tgt.float(), 2, dec, diff, loss, csum)
    bufs.check()
    imgloss_check(pre, err, tgt, 2, dec, diff, loss, csum)


def imgloss_check(pre, err, tgt, tdiv, dec, diff, loss, csum):
    N = pre.shape[0]
    d = pre - tgt[torch.arange(N, device=pre.device) // tdiv]
    derr = err + U * d.abs()
    report("dec", bound("dec", dec, pre, err))
    report("diff", bound("diff", diff, d, derr))
    plane = pre[0].numel()
    lref = 0.5 * (d * d).sum((1, 2, 3))
    lerr = (d.abs() * derr + 0.5 * derr * derr).sum((1, 2, 3)) + (plane + 2) * U * lref
    report("loss", bound("loss", loss, lref, lerr))
    report("csum", bound("csum", csum, d.sum((2, 3)), derr.sum((2, 3)) + plane * U * d.abs().sum((2, 3))))


@gpu
@pytest.mark.parametrize("Cc", [3, 6, 12])
@pytest.mark.parametrize("c16", [False, True], ids=["f32cols", "f16cols"])
def test_col2im_imgloss_channel_blocks_match_float64(ops, Cc, c16):
    """col2im_imgloss_kernel<CMAX> for CMAX 4 / 8 / 16 (Cc = 3 / 6 / 12) over fp32 and fp16 column matrices, tgt_div = 3:
    the fold is F.conv_transpose2d with a one-hot weight (column (kh,kw,c) of pixel (n,iy,ix) lands on output channel c)."""
    hi, k, N = 13, 6, 6
    ho = 2 * (hi - 1) + k
    g = Gen(Cc + 50 * c16)
    col64 = g.normal(N * hi * hi, k * k * Cc, scale=0.3)
    col64 = fp16(col64) if c16 else fp32(col64)
    b = fp32(g.normal(Cc, scale=0.5))
    tgt = fp32(g.normal(N // 3, Cc, ho, ho, scale=0.5))
    colv = col64.to(torch.float16 if c16 else torch.float32)
    dec, diff = torch.full((N, Cc, ho, ho), NAN, device=DEV), torch.full((N, Cc, ho, ho), NAN, device=DEV)
    bufs = Bufs()
    loss, csum = bufs.out(1, N).view(N), bufs.out(N, Cc)
    ops.col2im_imgloss(colv, N, hi, hi, Cc, k, b.float(), tgt.float(), 3, dec, diff, loss, csum)
    bufs.check()
    # column (kh, kw, c) as a ConvTranspose2d over k*k*Cc input channels with a one-hot weight
    wid = torch.zeros(k * k * Cc, Cc, k, k, dtype=f64, device=DEV)
    for kh in range(k):
        for kw in range(k):
            for c in range(Cc):
                wid[(kh * k + kw) * Cc + c, c, kh, kw] = 1.0
    xin = nchw(col64.view(N, hi, hi, k * k * Cc))
    pre = F.conv_transpose2d(xin, wid, b, stride=2)
    terms = F.conv_transpose2d(xin.abs(), wid, b.abs(), stride=2)
    imgloss_check(pre, 10 * U * terms, tgt, 3, dec, diff, loss, csum)


DEC_BWD = [conv_case(li, False) for li in (0, 3)] + [conv_case(li, imp) for li in (1, 2) for imp in (False, True)]


@gpu
@pytest.mark.parametrize("li,implicit", DEC_BWD)
def test_decoder_layer_backward_matches_autograd(ops, round_out, li, implicit):
    """dreamer.py:1178-1206: layers 2-3 (PD_B200_IMPLICIT_CONV) by conv_gemm mode 2 into the 32-channel-padded weight
    gradient and conv_gemm_actbwd (o_mn = True) for the input gradient through the ELU of the layer below; otherwise
    im2col (the identity on layer 1's 5x5 input; k = 6 planar on the last layer's NCHW image gradient) + an accumulating
    gemm + gemm_actbwd (or, layer 1, gemm with round_out); then permute4 back to (Cin, Cout, kh, kw).  Against float64
    autograd of F.conv_transpose2d and F.elu."""
    hi, ho, k, ci, co = DEC_GEO[li]
    g = Gen(400 + li)
    N = NB
    pxi = N * hi * hi
    xin = tf32_rna(F.elu(g.normal(pxi, ci))) if li else tf32_rna(g.normal(pxi, ci))   # the saved layer input (ELU output)
    w = tf32_rna(g.uniform(ci, co, k, k, bound=1 / math.sqrt(ci)))
    dout = tf32_rna(g.normal(N, ho, ho, co, scale=0.1))                                  # NHWC gradient at the output
    db0 = fp32(g.normal(ci, scale=0.1))
    copad = cdiv(co, 32) * 32 if implicit else co
    bufs = Bufs()
    Wg = torch.empty(k, k, co, ci, device=DEV)
    ops.permute4(w.float().contiguous(), Wg, (2, 3, 1, 0))
    Wg = Wg.view(k * k * co, ci)
    gdec = bufs.out(k * k * copad, ci, init=torch.zeros(k * k * copad, ci, dtype=f64, device=DEV))
    dxin = bufs.out(pxi, ci)
    db = bufs.out(1, ci, init=db0).view(ci)
    xd = xin.float().contiguous()
    if li == 3:                                  # the image gradient is NCHW; dout4 is its [n,y,x,c] view (sX = 1: planar)
        dimg = nchw(dout).float().contiguous()
        dout4 = dimg.permute(0, 2, 3, 1)
    else:
        dout4 = dout.float().contiguous()
    if implicit:
        ops.conv_gemm(2, dout4, k, xd, gdec)
        ops.conv_gemm_actbwd(dout4, k, Wg, dxin, xd, db, o_mn=True)
        dw_depth = tc_depth(k * k * copad, ci, cdiv(pxi, 32), True, may_skinny=False)[0]
        dx_depth = tc_depth(pxi, ci, k * k * cdiv(co, 32), may_skinny=False)[0]
    else:
        if li == 0:
            dcols = dout4.reshape(N, k * k * co)
        else:
            dcols = bufs.out(pxi, k * k * co)
            ops.im2col(dout4, k, 0, dcols, round_out=True)
        ops.gemm(dcols, xd, gdec, a_mn=True, b_mn=True, accumulate=True)
        if li > 0:
            ops.gemm_actbwd(dcols, Wg, dxin, xd, db, b_mn=True)
        else:
            ops.gemm(dcols, Wg, dxin, b_mn=True, round_out=True)
        # (layer 1: K = NB images < 8 -> the CUDA-core kernel takes the weight gradient)
        dw_depth = simt_depth(pxi) if pxi < 8 else tc_depth(k * k * co, ci, cdiv(pxi, 32), True)[0]
        dx_depth = tc_depth(pxi, ci, cdiv(k * k * co, 32))[0]
    gW = torch.full((ci, co, k, k), NAN, device=DEV)
    ops.permute4(gdec.view(k, k, copad, ci)[:, :, :co], gW, (3, 2, 0, 1))
    bufs.check()

    def grads(x, wt, d):
        x = nchw(x.view(N, hi, hi, ci)).clone().requires_grad_(True)
        wt = wt.clone().requires_grad_(True)
        (F.conv_transpose2d(x, wt, stride=2) * nchw(d)).sum().backward()
        return x.grad.permute(0, 2, 3, 1).reshape(pxi, ci), wt.grad

    gx, gwt = grads(xin, w, dout)
    tx, twt = grads(xin.abs(), w.abs(), dout.abs())
    print(f"\ndecoder layer {li} backward {'implicit' if implicit else 'explicit'} dW depth {dw_depth} dX depth {dx_depth}")
    report("dW", bound("dW", gW, gwt, C_ACC * dw_depth * U * twt))
    err = C_ACC * dx_depth * U * tx
    if li == 0:
        check_out("dx", dxin, gx, err, bool(round_out), {})
        return
    dref = elu_bwd_from_out(gx, xin)
    e = xin.clamp(max=0) + 1
    derr = err * e + 2 * U * gx.abs() * e
    check_out("dx", dxin, dref, derr, bool(round_out), {})
    bref = db0 + dref.sum(0)
    berr = derr.sum(0) + (pxi + 1) * U * (dref.abs().sum(0) + db0.abs())
    if round_out:
        berr = berr + ulp(dref.abs() + derr, -126, 10).sum(0)               # pd_colsum adds the stored (rounded) C
    report("dbias", bound("dbias", db, bref, berr))


# ----------------------------------------------------------------------------------------------------- refusals
def refused(ops, call):
    """A call the host code must refuse with PD_ERR_ARG before launching anything."""
    if CPU:
        pytest.skip("host-side argument checks and launch counts of the native library")
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        call()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a refused call launched a kernel"


def _conv_gemm_raw(ops, mode, X, k, O, Cmat, accumulate):
    import ctypes
    NB_, H, W, C = X.shape
    rc = ops.lib.pd_conv_gemm(ops.h, mode, NB_, H, W, C, k, ctypes.c_void_p(X.data_ptr()), ctypes.c_void_p(O.data_ptr()),
                              O.stride(0), 0, Cmat.shape[1], ctypes.c_void_p(Cmat.data_ptr()), Cmat.stride(0), None, 0, 0,
                              int(accumulate), ops._s())
    ops._ck(rc, "pd_conv_gemm")


REFUSALS = {
    # pd_gemm_f16 reads K-major operands only (the ABI has no MN-major flag) and needs 16-byte rows: ld % 8 == 0
    "f16_lda_not_multiple_of_8": lambda o, z: o.gemm_f16(z(64, 68, torch.float16)[:, :64], z(64, 64, torch.float16),
                                                         z(64, 64)),
    "f16_ldb_not_multiple_of_8": lambda o, z: o.gemm_f16(z(64, 64, torch.float16), z(64, 68, torch.float16)[:, :64],
                                                         z(64, 64)),
    "f16_c_accumulate": lambda o, z: o.gemm(z(64, 64), z(64, 64), z(64, 64, torch.float16), accumulate=True),
    "f16_c_residual": lambda o, z: o.gemm(z(64, 64), z(64, 64), z(64, 64, torch.float16), res=z(64, 64)),
    "conv_gemm_channels_not_multiple_of_4": lambda o, z: o.conv_gemm(1, z(2, 14, 14, 6).contiguous(), 4, z(32, 96),
                                                                      z(72, 32)),
    "conv_gemm_mode1_accumulate": lambda o, z: _conv_gemm_raw(o, 1, z(2, 14, 14, 32), 4, z(32, 512), z(72, 32), True),
    "conv_gemm_mode3_store": lambda o, z: _conv_gemm_raw(o, 3, z(2, 14, 14, 32), 4, z(72, 32), z(32, 512), False),
    "gemm_accumulate_with_bias": lambda o, z: o.gemm(z(64, 64), z(64, 64), z(64, 64), bias=z(64), accumulate=True),
    "gemm_accumulate_with_elu": lambda o, z: o.gemm(z(64, 64), z(64, 64), z(64, 64), act=ACT_ELU, accumulate=True),
}


@gpu
@pytest.mark.parametrize("what", list(REFUSALS))
def test_invalid_calls_are_refused_before_any_launch(ops, what):
    def z(*shape):
        dt = shape[-1] if isinstance(shape[-1], torch.dtype) else torch.float32
        return torch.zeros(*(shape[:-1] if isinstance(shape[-1], torch.dtype) else shape), device=DEV, dtype=dt)

    refused(ops, lambda: REFUSALS[what](ops, z))


@gpu
def test_actbwd_with_c_not_tma_addressable_takes_the_composed_path(ops):
    """pd_gemm_actbwd with ldc % 4 != 0 cannot use the fused epilogue (it needs a TMA-addressable fp32 C): it composes
    pd_gemm + pd_bias_act_bwd (pd_api.cu:150-156): two launches, and the result is checked by the matrix case
    actbwd_generic_store_falls_back."""
    if CPU:
        pytest.skip("launch counts of the native library")
    g = Gen(5)
    A, B, dact = tf32_rna(g.normal(200, 64)).float(), tf32_rna(g.normal(18, 64)).float(), F.elu(g.normal(200, 18)).float()
    C = torch.zeros(200, 19, device=DEV)[:, :18]
    db = torch.zeros(18, device=DEV)
    n0 = ops.launch_count()
    ops.gemm_actbwd(A, B, C, dact, db)
    torch.cuda.synchronize()
    assert ops.launch_count() - n0 == 2


# ----------------------------------------------------------------------------------------------------- determinism
@gpu
def test_split_sums_are_identical_run_to_run(ops):
    """The split-K partial sums of conv_gemm modes 2 / 3 and of the skinny dense GEMM, and col2im_actbwd's bias gradient,
    are added in a fixed order: the same inputs give bit-identical results on every run."""
    g = Gen(9)
    X = tf32_rna(g.normal(NB, 31, 31, 48)).float().contiguous()
    D1 = tf32_rna(g.normal(NB * 196, 96)).float()                              # encoder layer 1: 1176 pixels
    Xd = tf32_rna(g.normal(NB, 30, 30, 48)).float().contiguous()
    Xi = tf32_rna(g.normal(NB * 169, 96)).float()                              # decoder layer 2: 1014 pixels
    A, B = tf32_rna(g.normal(50, 6144)).float(), tf32_rna(g.normal(2048, 6144, scale=0.01)).float()
    col, dact = g.normal(NB * 196, 16 * 48).float(), F.elu(g.normal(NB, 31, 31, 48)).float().contiguous()
    assert tc_depth(96, 16 * 64, cdiv(NB * 196, 32), True, may_skinny=False)[1] > 1
    assert tc_depth(36 * 64, 96, cdiv(NB * 169, 32), True, may_skinny=False)[1] > 1
    assert tc_depth(50, 2048, 6144 // 32)[1] > 1

    def once():
        out = dict(m3=torch.zeros(96, 16 * 64, device=DEV), m2=torch.zeros(36 * 64, 96, device=DEV),
                   skinny=torch.empty(50, 2048, device=DEV), db=torch.zeros(48, device=DEV))
        ops.conv_gemm(3, X, 4, D1, out["m3"])
        ops.conv_gemm(2, Xd, 6, Xi, out["m2"])
        ops.gemm(A, B, out["skinny"])
        ops.col2im_actbwd(col, 14, 14, 4, dact, out["db"], torch.empty(NB, 31, 31, 48, device=DEV))
        sync()
        return out

    first = once()
    for _ in range(3):
        again = once()
        for k, v in first.items():
            assert torch.equal(v, again[k]), k


def test_pick_splits_restatement_selects_the_documented_branches():
    """The split counts tc_depth derives (and the cases above rely on) for P = 132 SMs: skinny RSSM step GEMMs split,
    a weight gradient with few tiles splits, one with more than 128 tiles does not, a 20-tile head does not."""
    global P
    saved, P = P, 132
    try:
        assert tc_depth(50, 1024, 32)[1] > 1                                   # skinny (num_m = 1, 8 tiles)
        assert tc_depth(2500, 400, 96)[1] == 1                                 # 80 tiles, not accumulating
        assert tc_depth(400, 1024, cdiv(2500, 32), True)[1] > 1                # 32 tiles: split-K
        assert tc_depth(1200, 2100, cdiv(2500, 32), True)[1] == 1              # 170 tiles: the partials do not fit
    finally:
        P = saved

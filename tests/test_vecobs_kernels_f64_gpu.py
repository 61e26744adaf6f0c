"""Kernel-level tests of what the vector-observation path adds: pd_vec_head_loss, the vecobs / image-less operands of
pd_wm_loss, and the GEMMs of the vecobs MLPs and of W_pe's column slices at the `minecraft` (K = 27) and `vectorenv`
(K = 4) shapes, against float64 references computed from the kernel's own fp32 inputs (conventions of
tests/test_rowwise_misc_f64_gpu.py and tests/test_gemm_conv_f64_gpu.py: per-element bounds in U = 2^-24, NaN-filled outputs
inside sentinel guard bands).

PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/ref_ops.py and oracle/vecobs_ops.py in place of the
kernels."""
import ctypes
import math

import pytest
import torch

from tests.test_gemm_conv_f64_gpu import Bufs as GemmBufs
from tests.test_gemm_conv_f64_gpu import check_out, dispatch, gemm_ref, operand, refused
from tests.test_rowwise_misc_f64_gpu import Bufs, f32, nlae
from tests.util import CPU, DEV, Gen, bound, f64, fp32, ops, round_out, tf32_rna  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24
MAX_K = 4096                                    # PD_VEC_HEAD_MAX_K (include/pd_b200.h)


@pytest.fixture(scope="module")
def ops(request):                               # noqa: F811  (tests.util's fixture, with the vecobs twins on the CPU)
    """NativeOps on cuda:0 (the float32 VecRefOps twin under PD_TEST_DEV=cpu); puts the handle back to its defaults after."""
    if CPU:
        from oracle.vecobs_ops import VecRefOps

        yield VecRefOps("cpu")
        return
    o = request.getfixturevalue("native_ops")
    yield o
    o.set_round_operands(True)
    o.set_gemm_impl(0)


# ----------------------------------------------------------------------------------------------------- pd_vec_head_loss
@gpu
@pytest.mark.parametrize("gap", [0, 5])
@pytest.mark.parametrize("div", [1, 3])
@pytest.mark.parametrize("K", [1, 4, 27, 32, 33, MAX_K])
def test_vec_head_loss_against_float64_autograd(ops, K, div, gap):
    M = (37 if K == MAX_K else 1001) * div
    g = Gen(K * 10 + div + gap)
    y, t = fp32(g.normal(M, K, scale=2.0)), fp32(g.normal(M // div, K))
    B = Bufs()
    loss, dy = B.out("loss", (M,)), B.out("dy", (M, K), gap=gap)
    yd = y.float()
    if gap:                                     # strided input rows: the gap columns hold NaN
        yv = torch.full((M, K + gap), float("nan"), device=DEV)
        yv[:, :K] = yd
        yd = yv[:, :K]
    ops.vec_head_loss(yd, f32(t), div, loss, dy)
    B.check()
    tt = t.repeat_interleave(div, 0)
    yg = y.clone().requires_grad_(True)
    std = 1 / math.sqrt(2 * math.pi)            # decoders.py:290-305: -Independent(Normal(y, std)).log_prob(t) * std^2
    lr = -torch.distributions.Independent(torch.distributions.Normal(yg, std), 1).log_prob(tt) * std ** 2
    lr.sum().backward()
    d = tt - y
    # each squared difference: the subtraction and the square (2 U), then a chain of ceil(K/32) + 5 additions
    El = (3 + math.ceil(K / 32) + 5) * U * 0.5 * (d * d).sum(-1) + 1e-12 * K
    bound("loss", loss, lr.detach(), El)
    bound("dy", dy, yg.grad, U * d.abs())


@gpu
def test_vec_head_loss_is_bit_identical_run_to_run(ops):
    g = Gen(5)
    M, K = 4096, 27
    y, t = f32(g.normal(M, K)), f32(g.normal(M, K))
    outs = []
    for _ in range(3):
        loss, dy = torch.empty(M, device=DEV), torch.empty(M, K, device=DEV)
        ops.vec_head_loss(y, t, 1, loss, dy)
        outs.append((loss, dy))
    for loss, dy in outs[1:]:
        assert torch.equal(loss, outs[0][0]) and torch.equal(dy, outs[0][1])


@gpu
@pytest.mark.parametrize("what", ["K0", "K_above_max", "ld_below_K", "tgt_div0"])
def test_vec_head_loss_refusals_launch_nothing(ops, what):
    z = lambda *s: torch.zeros(*s, device=DEV)
    buf = z(8 * 32)

    def raw(K, ldy):                                # the C entry point itself: ops.vec_head_loss derives ld from views
        p = ctypes.c_void_p(buf.data_ptr())
        ops._ck(ops.lib.pd_vec_head_loss(ops.h, 8, K, p, ldy, p, K, 1, p, p, K, ops._s()), "pd_vec_head_loss")

    calls = {
        "K0": lambda: ops.vec_head_loss(z(8, 0), z(8, 0), 1, z(8), z(8, 0)),
        "K_above_max": lambda: ops.vec_head_loss(z(8, MAX_K + 1), z(8, MAX_K + 1), 1, z(8), z(8, MAX_K + 1)),
        "ld_below_K": lambda: raw(27, 20),
        "tgt_div0": lambda: ops.vec_head_loss(z(8, 4), z(8, 4), 0, z(8), z(8, 4)),
    }
    refused(ops, calls[what])


# ----------------------------------------------------------------------------------------------------- pd_wm_loss
@gpu
@pytest.mark.parametrize("img", [True, False], ids=["image", "no_image"])
@pytest.mark.parametrize("vec", [True, False], ids=["vecobs", "no_vecobs"])
@pytest.mark.parametrize("I", [1, 4])
def test_wm_loss_with_vecobs_and_without_image(ops, I, vec, img):
    TB = 133
    N = TB * I
    g = Gen(I * 4 + 2 * vec + img)
    ls = [fp32(g.rand(N) * s) for s in (1e3, 2.0, 5.0, 50.0, 30.0, 10.0, 10.0, 300.0)]
    l_img, l_rew, l_term, l_kl, kl_exact, ent_prior, ent_post, l_vec = ls
    kw, wi, wr, wt, wv = 0.1, 1.0, 1.0, 5.0, 2.0
    B = Bufs()
    w, tb = B.out("w", (N,)), B.out("tb", (TB, 8))
    ops.wm_loss(TB, I, kw, wi, wr, wt, f32(l_img) if img else None, *(f32(v) for v in ls[1:7]), w, tb,
                **(dict(l_vec=f32(l_vec), w_vec=wv) if vec else {}))
    B.check()
    img_ = l_img if img else torch.zeros_like(l_img)
    terms = [kw * l_kl, wi * img_, wr * l_rew, wt * l_term] + ([wv * l_vec] if vec else [])
    Lg = sum(terms).view(TB, I).clone().requires_grad_(True)
    lm = nlae(Lg, I)
    lm.mean().backward()
    L = Lg.detach()
    EL = (len(terms) + 1) * U * sum(t.abs() for t in terms).view(TB, I)
    spread = (L - L.amin(-1, keepdim=True)).amax(-1)
    Elae = EL.amax(-1) + (0 if I == 1 else U * (2 * L.abs().amax(-1) + 2 * spread + I + 8 + math.log(I)))
    bound("loss_model", tb[:, 0], lm.detach(), Elae + U * lm.detach().abs())
    bound("w", w, Lg.grad.reshape(-1), (Lg.grad * (2 * EL + Elae[:, None] + 8 * U + U * (L.abs() + 10))).reshape(-1) + 2.0 ** -126)
    for j, v, on in ((1, l_img, img), (7, l_vec, vec)):
        if on:
            r = nlae(v.view(TB, I), I)
            bound(f"tb[{j}]", tb[:, j], r, U * (2 * v.abs().max() + I + 8) + U * r.abs())
        else:
            assert (tb[:, j] == 0).all(), j


# ----------------------------------------------------------------------------------------------------- GEMM shapes
def gcase(name, M, N, K, lda, ldb, ldc, arm, **kw):
    return pytest.param(dict(M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, arm=arm, **kw), id=name)


R_MC, E_MC = 1536, 32 * 48 + 256                  # minecraft: T*B = 48*32 rows, embedding 1536 (image) + 256 (vecobs)
VEC_GEMMS = [
    # encoder MLP, first layer: rows of K = 27 / 4 floats are not 16-byte multiples (or K < 8) -> generic CUDA-core kernel
    gcase("enc_fwd_k27_lda27", R_MC, 400, 27, 27, 28, 400, "simt", bias=True, rnd=1),
    gcase("enc_fwd_k4_lda4", R_MC, 400, 4, 4, 4, 400, "simt", bias=True, rnd=1),
    # its weight gradient: B = the vector batch [rows][27] (MN-major, ldb = 27), C = W [400][27] with ldc = 27
    gcase("enc_wgrad_n27_ldb27_ldc27", 400, 27, R_MC, 400, 27, 27, "simt", a_mn=1, b_mn=1, acc=True),
    gcase("enc_wgrad_n4_ldb4", 400, 4, R_MC, 400, 4, 4, "simt", a_mn=1, b_mn=1, acc=True),
    # head output layer: N = 27 with ldc = 27 -> tensor cores with the generic store epilogue; N = 4 -> gemv_rows
    gcase("head_out_n27_ldc27", R_MC, 27, 400, 400, 400, 27, "wgmma", bias=True),
    gcase("head_out_n4_ldc4", R_MC, 4, 400, 400, 400, 4, "gemv", bias=True),
    # head backward: weight gradient with A = dy [rows][27] (lda = 27), input gradient with K = 27
    gcase("head_wgrad_m27_lda27", 27, 400, R_MC, 27, 400, 400, "simt", a_mn=1, b_mn=1, acc=True),
    gcase("head_wgrad_m4_lda4", 4, 400, R_MC, 4, 400, 400, "mma", a_mn=1, b_mn=1, acc=True),
    gcase("head_dx_k27_lda27", R_MC, 400, 27, 27, 400, 400, "simt", b_mn=1),
    # W_pe column slices (ldb = E = 1792): hoisted ea from the image part, then + the vecobs part through the residual
    gcase("pe_fwd_image_cols", R_MC, 1000, 1536, 1536, E_MC, 1000, "wgmma"),
    gcase("pe_fwd_vecobs_cols_residual", R_MC, 1000, 256, 256, E_MC, 1000, "wgmma", res="inplace", b_off=1536),
    # backward: dembed_vec = dea . W_pe[:, 1536:], and W_pe's gradient written into its vecobs columns (ldc = E)
    gcase("pe_dembed_vecobs_cols", R_MC, 256, 1000, 1000, E_MC, 256, "mma", b_mn=1, b_off=1536),
    gcase("pe_wgrad_vecobs_cols_ldc_E", 1000, 256, R_MC, 1000, 256, E_MC, "mma", a_mn=1, b_mn=1, acc=True, c_off=1536),
]


@gpu
@pytest.mark.parametrize("c", VEC_GEMMS)
def test_vecobs_gemm_shapes_match_float64_reference(ops, round_out, c):
    M, N, K = c["M"], c["N"], c["K"]
    a_mn, b_mn = c.get("a_mn", 0), c.get("b_mn", 0)
    arm = dispatch(c, c["lda"], c["ldb"], c["ldc"])
    assert arm == c["arm"], f"the case reaches {arm}, not the {c['arm']} kernel the model's host dispatch picks"
    g = Gen(M * 7 + N * 3 + K)
    A, Bm = tf32_rna(g.normal(M, K)), tf32_rna(g.normal(N, K, scale=1.0 / math.sqrt(K)))
    bias = fp32(g.normal(N, scale=0.5)) if c.get("bias") else None
    R = fp32(g.normal(M, N, scale=0.5)) if (c.get("acc") or c.get("res")) else None
    As, Bs = (A.T if a_mn else A), (Bm.T if b_mn else Bm)
    Ad = operand(As, gap=c["lda"] - As.shape[1])
    boff = c.get("b_off", 0)                        # a column slice of a wider matrix: the other columns hold NaN
    Bd = operand(torch.cat([torch.zeros(Bs.shape[0], boff, dtype=f64, device=DEV), Bs], 1), gap=c["ldb"] - boff - Bs.shape[1])[:, boff:]
    coff = c.get("c_off", 0)
    bufs = GemmBufs()
    Cw = bufs.out(M, coff + N, gap=c["ldc"] - coff - N, init=torch.cat([torch.full((M, coff), -7.0, dtype=f64, device=DEV),
                                                                        R if R is not None else torch.full((M, N), float("nan"), dtype=f64, device=DEV)], 1))
    C = Cw[:, coff:]
    simt = arm in ("gemv", "wcolsum", "simt")
    ref, err, depth = gemm_ref(dict(c, res="inplace" if c.get("res") else None), A, Bm, bias, R, None, simt)
    ops.gemm(Ad, Bd, C, a_mn=bool(a_mn), b_mn=bool(b_mn), bias=None if bias is None else bias.float(),
             res=C if c.get("res") else None, round_out=bool(c.get("rnd")), accumulate=bool(c.get("acc")))
    bufs.check()
    if coff:
        assert (Cw[:, :coff] == -7.0).all(), "columns left of the slice were written"
    check_out("C", C, ref, err, bool(c.get("rnd")) and bool(round_out), {})

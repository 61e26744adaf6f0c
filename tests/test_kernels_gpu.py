"""GPU parity tests: every hand-written kernel (through the C ABI) against oracle/ref_ops.py on the
same seeded inputs.  Tolerances are written next to each check:
  * tensor-core GEMM with integer-valued operands: bit-exact (tf32 holds them exactly, fp32 sums exact)
  * tensor-core GEMM with random fp32 operands:   1e-3 of the output scale (TF32 operand precision)
  * pointwise / rowwise kernels (operand rounding off): 1e-5 relative
  * categorical sample indices: bit-exact."""
import pytest
import torch

from oracle.ref_ops import RefOps

import os

pytestmark = pytest.mark.gpu
# PD_TEST_DEV=cpu runs this file with the reference table on both sides: a dry run of the test code itself
DEV = os.environ.get("PD_TEST_DEV", "cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def ints(*shape, seed=0, lo=-4, hi=5):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return torch.randint(lo, hi, shape, generator=g).float().to(DEV)


def close(a, b, rtol=1e-5, atol=1e-6, what=""):
    err = (a.double() - b.double()).abs().max().item()
    ref = b.double().abs().max().item()
    assert err <= atol + rtol * max(ref, 1e-30), f"{what}: max err {err:.3e} vs scale {ref:.3e}"


@pytest.fixture(scope="module")
def ops(request):
    if DEV == "cpu":
        yield RefOps("cpu")
        return
    native_ops = request.getfixturevalue("native_ops")
    native_ops.set_round_operands(False)
    yield native_ops
    native_ops.set_round_operands(True)
    native_ops.set_gemm_impl(0)


@pytest.fixture(scope="module")
def ref():
    return RefOps(DEV)


GEMM_SHAPES = [(128, 128, 32), (128, 128, 256), (50, 1000, 1024), (300, 6144, 1000), (130, 264, 100), (64, 48, 48),
               (257, 1000, 2048), (2500, 400, 3072), (900, 108, 48),
               # MN-major operands as 3-D TMA boxes: tiles with full 32-column groups followed by groups past the end
               (160, 96, 200),
               # partial last m-tile (the wgmma slices of 16 rows and the mma.sync slices of 32 rows cut at different rows)
               (400, 512, 96), (450, 300, 64),
               # odd k-block counts and a partial last k-block
               (1024, 512, 160), (2500, 768, 1000), (1100, 300, 136),
               # tall with one n-tile, N below the 128-column tile
               (4500, 48, 48), (5000, 108, 40), (4200, 128, 200),
               # many tiles: full waves of persistent CTAs
               (1024, 512, 256), (2500, 6144, 96), (640, 1000, 1000)]


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_exact_on_integer_operands(ops, ref, impl, a_mn, b_mn, M, N, K):
    ops.set_gemm_impl(impl)
    A = ints(K, M, seed=1) if a_mn else ints(M, K, seed=1)
    B = ints(K, N, seed=2) if b_mn else ints(N, K, seed=2)
    C = torch.full((M, N), float("nan"), device=DEV)
    Cr = torch.empty(M, N, device=DEV)
    ops.gemm(A, B, C, a_mn=a_mn, b_mn=b_mn)
    ref.gemm(A, B, Cr, a_mn=a_mn, b_mn=b_mn)
    assert torch.equal(C, Cr), f"max diff {(C - Cr).abs().max().item()}"


@pytest.mark.parametrize("impl", [1, 0])
def test_gemm_epilogue_bias_residual_elu_and_strided_views(ops, ref, impl):
    ops.set_gemm_impl(impl)
    M, N, K, I = 96, 1000, 512, 4
    big = ints(M, K + 64, seed=3)
    A = big[:, 32:32 + K]                       # strided view (lda = K+64, offset 128 B)
    B = ints(N, K, seed=4)
    bias = ints(N, seed=5)
    res = ints(M // I, N, seed=6)
    Cbig = torch.zeros(M, N + 24, device=DEV)
    C = Cbig[:, 8:8 + N]                        # ldc = N+24, 32 B offset
    Cr = torch.empty(M, N, device=DEV)
    ops.gemm(A, B, C, bias=bias, res=res, r_div=I, act=1)
    ref.gemm(A, B, Cr, bias=bias, res=res, r_div=I, act=1)
    close(C, Cr, rtol=1e-6, what="epilogue")
    assert Cbig[:, :8].abs().sum() == 0 and Cbig[:, 8 + N:].abs().sum() == 0


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("M,N,K", [(108, 48, 90000), (1000, 2048, 2500), (400, 400, 40000), (48, 48, 5000),
                                   (1, 400, 37500), (3, 48, 5000), (1024, 2048, 2500)])
def test_gemm_splitk_accumulate_both_mn_major(ops, ref, impl, M, N, K):
    """weight-gradient form: C[M,N] += sum_k A[k,m] B[k,n]"""
    ops.set_gemm_impl(impl)
    A, B = ints(K, M, seed=7, lo=-2, hi=3), ints(K, N, seed=8, lo=-2, hi=3)
    C = ints(M, N, seed=9)
    Cr = C.clone()
    ops.gemm(A, B, C, a_mn=1, b_mn=1, accumulate=True)
    ref.gemm(A, B, Cr, a_mn=1, b_mn=1, accumulate=True)
    assert torch.equal(C, Cr), f"max diff {(C - Cr).abs().max().item()}"


@pytest.mark.parametrize("impl", [1, 0])
def test_gemm_skinny_m_splitk_with_bias_and_residual(ops, ref, impl):
    """M = 50 rows (one RSSM timestep): one row of output tiles over a long K, with bias + residual."""
    ops.set_gemm_impl(impl)
    for (M, N, K, I) in [(50, 1000, 1024, 1), (50, 6144, 2048, 1), (48, 1000, 2048, 4), (50, 2048, 6144, 1)]:
        A, B, bias, res = ints(M, K, seed=1), ints(N, K, seed=2), ints(N, seed=3), ints(M // I, N, seed=4)
        big = torch.full((M, N + 40), 7.0, device=DEV)
        C = big[:, 8:8 + N]
        Cr = torch.empty(M, N, device=DEV)
        ops.gemm(A, B, C, bias=bias, res=res, r_div=I)
        ref.gemm(A, B, Cr, bias=bias, res=res, r_div=I)
        assert torch.equal(C, Cr) and (big[:, :8] == 7).all() and (big[:, 8 + N:] == 7).all()
        Bt = B.t().contiguous()                           # dX form, B MN-major, in-place residual (C += A B)
        C2 = ints(M, N, seed=5); C2r = C2.clone(); keep = C2.clone()
        ops.gemm(A, Bt, C2, b_mn=True, res=C2)
        ref.gemm(A, Bt, C2r, b_mn=True, res=keep)
        assert torch.equal(C2, C2r)


def test_gemm_tf32_error_on_random_operands(ops, native_ops):
    if DEV == "cpu":
        pytest.skip("dry run")
    ops.set_gemm_impl(0)
    M, N, K = 512, 1024, 2048
    A, B = rnd(M, K, seed=10), rnd(N, K, scale=0.05, seed=11)
    C = torch.empty(M, N, device=DEV)
    ops.gemm(A, B, C)
    exact = A.double() @ B.double().t()
    err = (C.double() - exact).abs().max().item() / exact.abs().max().item()
    bias = ((C.double() - exact) * exact.sign()).mean().item() / exact.abs().mean().item()
    print(f"tf32 gemm (raw fp32 operands): max rel err {err:.3e}, signed mean shrink {bias:.3e}")
    assert err < 2e-3
    # operands pre-rounded to tf32 (what the producers do): error drops to accumulation order only
    At = torch.empty_like(A); Bt = torch.empty_like(B)
    native_ops.set_round_operands(True)
    ops.round_copy(A, At); ops.round_copy(B, Bt)
    native_ops.set_round_operands(False)
    ops.gemm(At, Bt, C)
    exact_t = At.double() @ Bt.double().t()
    err_t = (C.double() - exact_t).abs().max().item() / exact_t.abs().max().item()
    err_r = (exact_t - exact).abs().max().item() / exact.abs().max().item()
    print(f"tf32 gemm (rna-rounded operands): vs rounded-exact {err_t:.3e}; rounding itself {err_r:.3e}")
    assert err_t < 2e-5 and err_r < 1e-3


def test_gemm_skinny_shapes_fall_to_simt(ops, ref):
    ops.set_gemm_impl(0)
    for (M, N, K) in [(2500, 1, 400), (2500, 6, 400), (777, 1000, 18), (333, 1000, 6)]:
        A, B = rnd(M, K, seed=1), rnd(N, K, seed=2)
        C, Cr = torch.empty(M, N, device=DEV), torch.empty(M, N, device=DEV)
        ops.gemm(A, B, C); ref.gemm(A, B, Cr)
        close(C, Cr, rtol=1e-5, what=f"skinny {M}x{N}x{K}")
    # N = 18 (actor logits) is wide enough for the tensor-core path: TF32 operand precision
    A, B = rnd(2500, 400, seed=1), rnd(18, 400, seed=2)
    C, Cr = torch.empty(2500, 18, device=DEV), torch.empty(2500, 18, device=DEV)
    ops.gemm(A, B, C); ref.gemm(A, B, Cr)
    close(C, Cr, rtol=2e-3, what="N=18 tf32")


@pytest.mark.parametrize("M,N", [(50, 1000), (2500, 400), (7, 1000), (1000, 33)])
def test_ln_elu_fwd_bwd(ops, ref, M, N):
    x, gamma, beta, dy = rnd(M, N, scale=2.0), rnd(N) * 0.5 + 1, rnd(N, seed=3) * 0.1, rnd(M, N, seed=5)
    out = {}
    for name, o in (("n", ops), ("r", ref)):
        y, mean, rstd = torch.empty(M, N, device=DEV), torch.empty(M, device=DEV), torch.empty(M, device=DEV)
        o.ln_elu_fwd(x, gamma, beta, 1e-3, y, mean, rstd)
        dx = torch.empty(M, N, device=DEV)
        dg, db, dbias = (torch.zeros(N, device=DEV) for _ in range(3))
        o.ln_elu_bwd(dy, x, y, gamma, mean, rstd, dx, dg, db, dbias)
        out[name] = (y, mean, rstd, dx, dg, db, dbias)
    # vs torch autograd as well
    xa = x.clone().requires_grad_(True); ga = gamma.clone().requires_grad_(True); ba = beta.clone().requires_grad_(True)
    ya = torch.nn.functional.elu(torch.nn.functional.layer_norm(xa, (N,), ga, ba, 1e-3))
    ya.backward(dy)
    close(out["n"][0], ya.detach(), 1e-5, 1e-6, "ln y vs torch")
    close(out["n"][3], xa.grad, 2e-5, 1e-6, "ln dx vs torch")
    close(out["n"][4], ga.grad, 5e-5, 1e-5, "ln dgamma vs torch")
    close(out["n"][5], ba.grad, 5e-5, 1e-5, "ln dbeta vs torch")
    for a, b, w in zip(out["n"], out["r"], ("y", "mean", "rstd", "dx", "dgamma", "dbeta", "dbias")):
        close(a, b, 5e-5, 1e-5, "ln " + w)


@pytest.mark.parametrize("M,D", [(50, 2048), (333, 64)])
def test_gru_fwd_bwd(ops, ref, M, D):
    gi, gh, hp = rnd(M, 3 * D), rnd(M, 3 * D, seed=1), torch.tanh(rnd(M, D, seed=2))
    mask = (torch.rand(M, device=DEV) > 0.3).float()
    dh_a, dh_b = rnd(M, D, seed=3), rnd(M, D, seed=4)
    res = {}
    for name, o in (("n", ops), ("r", ref)):
        hout, hm, gates = torch.empty(M, D, device=DEV), torch.empty(M, D, device=DEV), torch.empty(M, 4 * D, device=DEV)
        o.gru_fwd(gi, gh, hp, hout, hm, mask, gates)
        dgi, dgh, dc = torch.empty(M, 3 * D, device=DEV), torch.empty(M, 3 * D, device=DEV), torch.empty(M, D, device=DEV)
        o.gru_bwd(dh_a, dh_b, mask, gates, hp, dgi, dgh, dc)
        res[name] = (hout, hm, gates, dgi, dgh, dc)
    cell = torch.nn.GRUCell(8, D).to(DEV)   # formula check against torch's own fused cell
    gia, gha, hpa = gi.clone().requires_grad_(True), gh.clone().requires_grad_(True), hp.clone().requires_grad_(True)
    r = torch.sigmoid(gia[:, :D] + gha[:, :D]); u = torch.sigmoid(gia[:, D:2 * D] + gha[:, D:2 * D])
    n = torch.tanh(gia[:, 2 * D:] + r * gha[:, 2 * D:]); hy = n + u * (hpa - n)
    hy.backward(dh_a + dh_b * mask[:, None])
    close(res["n"][0], hy.detach(), 1e-5, 1e-6, "gru h")
    close(res["n"][3], gia.grad, 2e-5, 1e-6, "gru dgi")
    close(res["n"][4], gha.grad, 2e-5, 1e-6, "gru dgh")
    for a, b, w in zip(res["n"], res["r"], ("h", "hmask", "gates", "dgi", "dgh", "dcarry")):
        close(a, b, 2e-5, 1e-6, "gru " + w)


@pytest.mark.parametrize("M,G,C", [(50, 32, 32), (2500, 32, 32), (2500, 1, 18), (100, 4, 7)])
def test_cat_sample_bit_exact_and_st_bwd(ops, ref, M, G, C):
    logits = rnd(M, G * C, scale=2.0)
    noise = torch.empty(M, G * C, device=DEV).exponential_()
    mask = (torch.rand(M, device=DEV) > 0.3).float()
    res = {}
    for name, o in (("n", ops), ("r", ref)):
        z, zm = torch.empty(M, G * C, device=DEV), torch.empty(M, G * C, device=DEV)
        idx = torch.empty(M, G, dtype=torch.int32, device=DEV)
        o.cat_sample(logits, noise, G, C, z, zm, mask, idx)
        res[name] = (z, zm, idx)
    # the oracle definition: torch's own formulation
    l3 = logits.view(M, G, C)
    probs = torch.distributions.OneHotCategorical(logits=l3).probs
    k = (probs / noise.view(M, G, C)).argmax(-1)
    mism = (res["n"][2].long() != k).sum().item()
    assert mism == 0, f"{mism} / {M * G} sampled indices differ from argmax(probs/q)"
    assert torch.equal(res["n"][0], res["r"][0]) and torch.equal(res["n"][1], res["r"][1])
    dz_a, dz_b, extra, rs = rnd(M, G * C, seed=1), rnd(M, G * C, seed=2), rnd(M, G * C, seed=3), torch.rand(M, device=DEV)
    dn, dr = torch.empty(M, G * C, device=DEV), torch.empty(M, G * C, device=DEV)
    ops.cat_st_bwd(logits, G, C, dz_a, dz_b, mask, extra, rs, 0.1, dn)
    ref.cat_st_bwd(logits, G, C, dz_a, dz_b, mask, extra, rs, 0.1, dr)
    close(dn, dr, 2e-5, 1e-6, "st bwd")
    la = logits.clone().requires_grad_(True)
    pa = torch.softmax(la.view(M, G, C), -1).view(M, G * C)
    pa.backward(dz_a + dz_b * mask[:, None])
    close(dn - 0.1 * rs[:, None] * extra, la.grad, 5e-5, 1e-6, "st bwd vs autograd")


@pytest.mark.parametrize("mode", [0, 1])
def test_kl(ops, ref, mode):
    M, G, C = 300, 32, 32
    post, prior = rnd(M, G * C, scale=1.5), rnd(M, G * C, scale=1.5, seed=1)
    idx = torch.randint(0, C, (M, G), device=DEV, dtype=torch.int32)
    res = {}
    for name, o in (("n", ops), ("r", ref)):
        v = [torch.empty(M, device=DEV) for _ in range(4)] + [torch.empty(M, G * C, device=DEV) for _ in range(2)]
        o.kl(post, prior, idx, mode, 0.8, G, C, *v)
        res[name] = v
    for a, b, w in zip(res["n"], res["r"], ("loss_kl", "kl_exact", "ent_post", "ent_prior", "dpost", "dprior")):
        close(a, b, 3e-5, 1e-5, "kl " + w)
    if mode == 0:  # against torch.distributions + autograd (dreamer.py:328-339)
        import torch.distributions as D
        pa, qa = post.clone().requires_grad_(True), prior.clone().requires_grad_(True)
        d = lambda x: D.Independent(D.OneHotCategoricalStraightThrough(logits=x.view(M, G, C)), 1)
        loss = 0.2 * D.kl.kl_divergence(d(pa), d(qa.detach())) + 0.8 * D.kl.kl_divergence(d(pa.detach()), d(qa))
        loss.sum().backward()
        close(res["n"][0], loss.detach(), 3e-5, 1e-5, "kl vs torch")
        close(res["n"][4], pa.grad, 5e-5, 1e-6, "dpost vs torch")
        close(res["n"][5], qa.grad, 5e-5, 1e-6, "dprior vs torch")
        close(res["n"][2], d(post).entropy(), 3e-5, 1e-5, "entropy")


@pytest.mark.parametrize("Cin,Cout", [(5, 8), (8, 12)])       # second case takes the float4 (C % 4 == 0) paths
def test_conv_data_movement_against_torch_conv(ops, ref, Cin, Cout):
    torch.backends.cudnn.allow_tf32 = False      # the torch reference conv must be true fp32 for a 1e-5 comparison
    NB, k = 6, 4
    x = rnd(NB, Cin, 14, 14)
    w = rnd(Cout, Cin, k, k, seed=1)
    b = rnd(Cout, seed=2)
    yref = torch.nn.functional.conv2d(x, w, b, stride=2)                     # (NB,Cout,6,6)
    for korder in (0, 1):
        col = torch.empty(NB * 36, k * k * Cin, device=DEV)
        ops.im2col(x.permute(0, 2, 3, 1), k, korder, col, round_out=False)
        colr = torch.empty_like(col)
        ref.im2col(x.permute(0, 2, 3, 1), k, korder, colr)
        assert torch.equal(col, colr)
        wk = (w.permute(0, 2, 3, 1) if korder == 0 else w).reshape(Cout, -1).contiguous()
        y = torch.empty(NB * 36, Cout, device=DEV)
        ops.set_gemm_impl(1)
        ops.gemm(col, wk, y, bias=b)
        close(y.view(NB, 6, 6, Cout).permute(0, 3, 1, 2), yref, 1e-5, 1e-5, f"conv korder {korder}")
    xi = rnd(NB, 3, 16, 16, seed=9)                                           # planar input, k=6 (last deconv backward)
    c6, c6r = torch.empty(NB * 36, 108, device=DEV), torch.empty(NB * 36, 108, device=DEV)
    ops.im2col(xi.permute(0, 2, 3, 1), 6, 0, c6, round_out=False); ref.im2col(xi.permute(0, 2, 3, 1), 6, 0, c6r)
    assert torch.equal(c6, c6r)
    # transposed conv = gemm + col2im  (decoders.py:149-155)
    wt = rnd(Cout, Cin, 5, 5, seed=3)   # ConvTranspose2d weight (in=Cout, out=Cin)
    bt = rnd(Cin, seed=4)
    xin = rnd(NB, Cout, 6, 6, seed=5)
    yt = torch.nn.functional.conv_transpose2d(xin, wt, bt, stride=2)           # (NB,Cin,15,15)
    wtp = wt.permute(2, 3, 1, 0).reshape(25 * Cin, Cout).contiguous()
    cols = torch.empty(NB * 36, 25 * Cin, device=DEV)
    ops.gemm(xin.permute(0, 2, 3, 1).reshape(NB * 36, Cout).contiguous(), wtp, cols)
    out = torch.empty(NB, 15, 15, Cin, device=DEV)
    ops.col2im(cols, 6, 6, 5, bt, 0, out, round_out=False)
    close(out.permute(0, 3, 1, 2), yt, 1e-5, 1e-5, "convT via col2im")
    outr = torch.empty_like(out)
    ref.col2im(cols, 6, 6, 5, bt, 0, outr)
    close(out, outr, 1e-6, 1e-6, "col2im vs ref")
    # output extent larger than the taps reach (conv input-grad for odd sizes): zero fill + ELU
    out2, out2r = torch.empty(NB, 16, 16, Cin, device=DEV), torch.empty(NB, 16, 16, Cin, device=DEV)
    ops.col2im(cols, 6, 6, 5, None, 1, out2, round_out=False); ref.col2im(cols, 6, 6, 5, None, 1, out2r)
    close(out2, out2r, 1e-6, 1e-6, "col2im padded extent")
    # fused image loss
    tgt = rnd(NB // 2, Cin, 15, 15, seed=6)
    r = {}
    for name, o in (("n", ops), ("r", ref)):
        dec, diff = torch.empty(NB, Cin, 15, 15, device=DEV), torch.empty(NB, Cin, 15, 15, device=DEV)
        loss, cs = torch.empty(NB, device=DEV), torch.empty(NB, Cin, device=DEV)
        o.col2im_imgloss(cols, NB, 6, 6, Cin, 5, bt, tgt, 2, dec, diff, loss, cs)
        r[name] = (dec, diff, loss, cs)
    for a, b_, w_ in zip(r["n"], r["r"], ("dec", "diff", "loss", "csum")):
        close(a, b_, 2e-5, 1e-5, "imgloss " + w_)
    ops.set_gemm_impl(0)


def test_bias_act_bwd_permute_small_ops(ops, ref):
    M, N = 5000, 48
    y = torch.nn.functional.elu(rnd(M, N))
    dy = rnd(M, N, seed=1)
    a, b = dy.clone(), dy.clone()
    da, db = torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)
    ops.bias_act_bwd(a, y, 1, da); ref.bias_act_bwd(b, y, 1, db)
    close(a, b, 1e-6, 1e-7, "act bwd"); close(da, db, 1e-4, 1e-4, "bias grad")
    x = rnd(7, 5, 4, 3)
    for perm in [(0, 2, 3, 1), (2, 3, 1, 0), (0, 3, 1, 2), (3, 2, 0, 1)]:
        o1 = torch.empty([x.shape[p] for p in perm], device=DEV)
        ops.permute4(x, o1, perm)
        assert torch.equal(o1, x.permute(*perm).contiguous())
        o2 = o1.clone(); ops.permute4(x, o2, perm, accumulate=True)
        assert torch.equal(o2, 2 * o1)
    m = torch.rand(M, device=DEV)
    o1 = torch.empty(M, N, device=DEV); ops.mask_rows(dy, m, o1); close(o1, dy * m[:, None], 1e-6)
    z = dy.clone(); ops.rowscale(z, m[: M // 4], 4, 0.5); close(z, dy * 0.5 * m[: M // 4].repeat_interleave(4)[:, None], 1e-6)
    gs = torch.empty(M // 4, N, device=DEV); ops.group_sum(dy, 4, gs); close(gs, dy.view(M // 4, 4, N).sum(1), 1e-5, 1e-6)
    cs = torch.zeros(N, device=DEV); ops.colsum(dy, cs); close(cs, dy.sum(0), 1e-4, 1e-4)
    reset = torch.rand(5, 7, device=DEV) > 0.5
    mk = torch.empty(5, 21, device=DEV); ops.reset_mask(reset, 3, mk)
    assert torch.equal(mk.view(5, 7, 3), (~reset).float()[:, :, None].expand(5, 7, 3))


@pytest.mark.parametrize("I", [1, 4])
def test_losses_and_wm_loss(ops, ref, I):
    TB = 120; N = TB * I
    y, tgt = rnd(N), torch.tanh(rnd(TB, seed=1))
    tb01 = (torch.rand(TB, device=DEV) > 0.9).float()
    for kind, t in ((0, tgt), (1, tb01)):
        r = {}
        for name, o in (("n", ops), ("r", ref)):
            v = [torch.empty(N, device=DEV) for _ in range(3)]
            o.scalar_head_loss(kind, y, t, I, *v); r[name] = v
        for a, b in zip(r["n"], r["r"]):
            close(a, b, 1e-5, 1e-6, f"head loss {kind}")
    ls = [torch.rand(N, device=DEV) * s for s in (100, 1, 1, 20, 20, 100, 100)]
    r = {}
    for name, o in (("n", ops), ("r", ref)):
        w, tb = torch.empty(N, device=DEV), torch.empty(TB, 8, device=DEV)
        o.wm_loss(TB, I, 0.1, 1.0, 1.0, 1.0, *ls, w, tb)
        mean = torch.empty(8, device=DEV); o.colmean(tb, mean)
        r[name] = (w, tb, mean)
    for a, b, nm in zip(r["n"], r["r"], ("w", "tb", "mean")):
        close(a, b, 2e-5, 1e-6, "wm_loss " + nm)


def test_actor_critic_kernels(ops, ref):
    H, Md, A = 15, 700, 18
    J = H + 1
    vt, v, rew, tl = rnd(J * Md), rnd(J * Md, seed=1), rnd(J * Md, seed=2), rnd(J * Md, seed=3) - 3
    r = {}
    for name, o in (("n", ops), ("r", ref)):
        term = torch.empty(J * Md, device=DEV)
        outs = [torch.empty(H * Md, device=DEV) for _ in range(5)]
        sums = torch.zeros(8, dtype=torch.float64, device=DEV)
        o.gae_critic(H, Md, 0.99, 0.95, vt, v, rew, tl, term, *outs, sums)
        r[name] = [term] + outs + [sums]
    for a, b, nm in zip(r["n"], r["r"], ("term", "adv", "agae", "target", "weight", "dv", "sums")):
        close(a, b, 3e-5, 1e-6, "gae " + nm)
    logits = rnd(H * Md, A)
    acts = torch.nn.functional.one_hot(torch.randint(0, A, (H * Md,), device=DEV), A).float()
    ag, w = r["r"][2], r["r"][4]
    res = {}
    for name, o in (("n", ops), ("r", ref)):
        dl = torch.zeros(H * Md, A, device=DEV); s = torch.zeros(2, dtype=torch.float64, device=DEV)
        o.actor_loss_onehot(1e-3, logits, acts, ag, w, dl, s); res[name] = (dl, s)
    close(res["n"][0], res["r"][0], 3e-5, 1e-9, "actor dlogits"); close(res["n"][1], res["r"][1], 1e-5, 1e-6, "actor sums")
    # tanh_normal
    Ac = 12
    out = rnd(H * Md, 2 * Ac)
    eps = torch.randn(H * Md, Ac, device=DEV)
    an, ar = torch.empty(H * Md, Ac, device=DEV), torch.empty(H * Md, Ac, device=DEV)
    ops.tanh_normal_sample(out, eps, an); ref.tanh_normal_sample(out, eps, ar)
    close(an, ar, 1e-5, 1e-6, "tanh_normal sample")
    res = {}
    for name, o in (("n", ops), ("r", ref)):
        dl = torch.zeros(H * Md, 2 * Ac, device=DEV); s = torch.zeros(2, dtype=torch.float64, device=DEV)
        o.actor_loss_tanh_normal(1e-4, out, ar, ag, w, dl, s); res[name] = (dl, s)
    close(res["n"][0], res["r"][0], 2e-3, 1e-9, "tanh_normal dout")   # atanh near |a|->1 amplifies ulps
    close(res["n"][1], res["r"][1], 1e-4, 1e-4, "tanh_normal sums")


def test_optimizer_kernels_against_torch_adamw(ops):
    n = 1_000_003
    p0, g = rnd(n), rnd(n, scale=3.0, seed=1)
    ss = torch.zeros(1, device=DEV); ops.sumsq(g, ss)
    close(ss, (g.double() ** 2).sum().float().view(1), 1e-4, 0, "sumsq")
    gc = g.clone(); norm = torch.empty(1, device=DEV)
    ops.clip_scale(gc, ss, 200.0, norm)
    gt = g.clone().requires_grad_(False)
    pt = torch.nn.Parameter(p0.clone()); pt.grad = g.clone()
    tn = torch.nn.utils.clip_grad_norm_([pt], 200.0)
    close(norm, tn.view(1), 1e-4, 0, "norm"); close(gc, pt.grad, 1e-4, 1e-7, "clipped grad")
    opt = torch.optim.AdamW([pt], lr=3e-4, eps=1e-5)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    for it in range(3):
        opt.step()
        ops.inc(step)
        ops.adamw(p, gc, m, v, 3e-4, 0.9, 0.999, 1e-5, 0.01, step)
    close(p, pt.detach(), 1e-5, 1e-6, "adamw params after 3 steps")


@pytest.mark.parametrize("M,N,K", [(50, 1000, 1024), (2500, 400, 3072), (2500, 6144, 1000), (640, 1000, 1000), (128, 128, 64),
                                   # 2-CTA kernel, two k-chunks per TMA box: K with a partial last chunk / an odd chunk count
                                   (2500, 512, 400), (2500, 1000, 2048), (1500, 768, 328), (1024, 1024, 200)])
def test_gemm_f16_operands_exact_on_integers(ops, ref, M, N, K):
    """kind::f16 path (forward-only layers): integer operands are exact in fp16, fp32 accumulation is exact."""
    if DEV == "cpu":
        pytest.skip("dry run")
    ops.set_gemm_impl(0)
    A, B = ints(M, K, seed=1), ints(N, K, seed=2)
    bias, res = ints(N, seed=3), ints(M, N, seed=4)
    C, Cr = torch.full((M, N), float("nan"), device=DEV), torch.empty(M, N, device=DEV)
    ops.gemm_f16(A.half(), B.half(), C, bias=bias, res=res)
    ref.gemm(A, B, Cr, bias=bias, res=res)
    assert torch.equal(C, Cr), f"max diff {(C - Cr).abs().max().item()}"
    big = torch.zeros(M, K + 64, device=DEV, dtype=torch.float16)
    big[:, 8:8 + K] = A.half()
    ops.gemm_f16(big[:, 8:8 + K], B.half(), C, act=1)                  # strided fp16 view + ELU epilogue
    ref.gemm(A, B, Cr, act=1)
    close(C, Cr, 1e-6, 1e-6, "f16 strided")


def test_gemm_partial_last_k_block_fp16_and_tf32(ops, ref):
    """K-major operands (the wgmma path) with odd k-block counts and a partial last k-block, fp16 and tf32.  Bit-exact."""
    ops.set_gemm_impl(0)
    o = ops
    for M, N, K in ((2500, 512, 400), (2500, 1000, 2048), (1500, 768, 328), (2500, 6144, 1000)):      # fp16 operands
        A, B = ints(M, K, seed=1), ints(N, K, seed=2)
        bias, res = ints(N, seed=3), ints(M, N, seed=4)
        C, Cr = torch.full((M, N), float("nan"), device=DEV), torch.empty(M, N, device=DEV)
        o.gemm_f16(A.half(), B.half(), C, bias=bias, res=res)
        ref.gemm(A, B, Cr, bias=bias, res=res)
        assert torch.equal(C, Cr), f"f16 {M, N, K}: max diff {(C - Cr).abs().max().item()}"
    for M, N, K in ((1024, 512, 160), (2500, 768, 1000), (1100, 300, 136), (2500, 400, 3072)):       # tf32 operands
        A, B = ints(M, K, seed=1), ints(N, K, seed=2)
        C, Cr = torch.full((M, N), float("nan"), device=DEV), torch.empty(M, N, device=DEV)
        o.gemm(A, B, C)
        ref.gemm(A, B, Cr)
        assert torch.equal(C, Cr), f"tf32 {M, N, K}: max diff {(C - Cr).abs().max().item()}"


def test_fp16_side_outputs_of_producers(ops, ref):
    if DEV == "cpu":
        pytest.skip("dry run")
    M, N, D, G, C = 300, 1000, 256, 32, 32
    x, gamma, beta = rnd(M, N, scale=2.0), rnd(N) * 0.5 + 1, rnd(N, seed=3) * 0.1
    y, mean, rstd = torch.empty(M, N, device=DEV), torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    y16 = torch.empty(M, N, device=DEV, dtype=torch.float16)
    ops.ln_elu_fwd(x, gamma, beta, 1e-3, y, mean, rstd, y16)
    assert torch.equal(y16, y.half())
    gi, gh, hp = rnd(M, 3 * D), rnd(M, 3 * D, seed=1), torch.tanh(rnd(M, D, seed=2))
    hout, h16 = torch.empty(M, D, device=DEV), torch.empty(M, D, device=DEV, dtype=torch.float16)
    ops.gru_fwd(gi, gh, hp, hout, h16=h16)
    assert torch.equal(h16, hout.half())
    logits, noise = rnd(M, G * C, scale=2.0), torch.empty(M, G * C, device=DEV).exponential_()
    z, z16 = torch.empty(M, G * C, device=DEV), torch.empty(M, G * C, device=DEV, dtype=torch.float16)
    ops.cat_sample(logits, noise, G, C, z, z16=z16)
    assert torch.equal(z16, z.half())
    src, dst = rnd(77, 130), torch.empty(77, 130, device=DEV, dtype=torch.float16)
    ops.to_half(src, dst)
    assert torch.equal(dst, src.half())


@pytest.mark.parametrize("NB,H,C,k,odim", [(3, 14, 96, 4, 192), (2, 31, 48, 4, 96), (3, 13, 96, 5, 192), (2, 30, 48, 6, 96),
                                             (5, 6, 192, 4, 384), (7, 5, 192, 5, 1536),
                                             # >= 384 output pixels: mode 1 runs on the 2-CTA kernel (pairs of 128-pixel tiles)
                                             (9, 30, 48, 6, 96), (21, 14, 96, 4, 192), (40, 8, 192, 4, 384)])
def test_implicit_conv_gemm_tma_im2col_exact(ops, ref, NB, H, C, k, odim):
    """TMA im2col-mode operands (no materialised im2col matrix): conv forward / deconv dX (mode 1, both weight layouts),
    deconv weight gradient (mode 2) and conv weight gradient (mode 3).  Integer operands: bit-exact."""
    if DEV == "cpu":
        pytest.skip("dry run")
    ops.set_gemm_impl(0)
    P = (H - k) // 2 + 1
    pixels, K = NB * P * P, k * k * C
    cpad = (C + 31) // 32 * 32
    X = ints(NB, H, H, C, seed=1, lo=-2, hi=3)
    Wk, bias = ints(odim, K, seed=2, lo=-2, hi=3), ints(odim, seed=3)
    for o_mn, O in ((False, Wk), (True, Wk.t().contiguous())):
        C1, C1r = torch.full((pixels, odim), float("nan"), device=DEV), torch.empty(pixels, odim, device=DEV)
        ops.conv_gemm(1, X, k, O, C1, o_mn=o_mn, bias=bias, act=1)
        ref.conv_gemm(1, X, k, O, C1r, o_mn=o_mn, bias=bias, act=1)
        close(C1, C1r, 1e-6, 1e-6, f"conv_gemm mode 1 o_mn={o_mn}")
    Ot = ints(pixels, odim, seed=4, lo=-2, hi=3)
    C2, C3 = ints(k * k * cpad, odim, seed=5), ints(odim, k * k * cpad, seed=6)
    C2r, C3r = C2.clone(), C3.clone()
    ops.conv_gemm(2, X, k, Ot, C2); ref.conv_gemm(2, X, k, Ot, C2r)
    assert torch.equal(C2, C2r), f"mode 2 max diff {(C2 - C2r).abs().max().item()}"
    ops.conv_gemm(3, X, k, Ot, C3); ref.conv_gemm(3, X, k, Ot, C3r)
    assert torch.equal(C3, C3r), f"mode 3 max diff {(C3 - C3r).abs().max().item()}"


@pytest.mark.parametrize("NB,H,C,k,odim", [(9, 30, 48, 6, 96), (21, 14, 96, 4, 192), (5, 13, 96, 5, 192), (3, 31, 48, 4, 96)])
def test_implicit_conv_gemm_all_modes_with_mn_major_weights(ops, ref, NB, H, C, k, odim):
    """Mode 1 with an MN-major weight plus the fused ELU backward and bias gradient, modes 2 and 3 (K = pixels, split over
    the SMs), and tall plain GEMMs with one n-tile.  Bit-exact."""
    ops.set_gemm_impl(0)
    o = ops
    P = (H - k) // 2 + 1
    pixels, K, cpad = NB * P * P, k * k * C, (C + 31) // 32 * 32
    X = ints(NB, H, H, C, seed=1, lo=-2, hi=3)
    Wt = ints(K, odim, seed=2, lo=-2, hi=3)
    dact = ints(pixels, odim, seed=3, lo=-3, hi=3)
    res = {}
    for name, oo in (("n", o), ("r", ref)):
        Cm, db = torch.full((pixels, odim), float("nan"), device=DEV), ints(odim, seed=4).clone()
        oo.conv_gemm_actbwd(X, k, Wt, Cm, dact, db, o_mn=True)
        Ot = ints(pixels, odim, seed=5, lo=-2, hi=3)
        C2, C3 = ints(k * k * cpad, odim, seed=6), ints(odim, k * k * cpad, seed=7)
        oo.conv_gemm(2, X, k, Ot, C2); oo.conv_gemm(3, X, k, Ot, C3)
        res[name] = (Cm, db, C2, C3)
    for a, b_, w in zip(res["n"], res["r"], ("mode 1 + actbwd", "dbias", "mode 2", "mode 3")):
        assert torch.equal(a, b_), f"{w}: max diff {(a - b_).abs().max().item()}"
    for M, N, K, b_mn in ((4500, 48, 48, 0), (5000, 108, 40, 1), (4200, 128, 200, 0)):          # tall plain GEMMs
        A = ints(M, K, seed=1)
        B = ints(K, N, seed=2) if b_mn else ints(N, K, seed=2)
        bias = ints(N, seed=3)
        C, Cr = torch.full((M, N), float("nan"), device=DEV), torch.empty(M, N, device=DEV)
        o.gemm(A, B, C, b_mn=bool(b_mn), bias=bias, act=1)
        ref.gemm(A, B, Cr, b_mn=bool(b_mn), bias=bias, act=1)
        close(C, Cr, 1e-6, 1e-6, f"tall gemm {M, N, K, b_mn}")


@pytest.mark.parametrize("M,N,K,b_mn", [(900, 48, 108, 1), (300, 96, 200, 0), (257, 40, 64, 1), (2500, 192, 96, 1), (130, 18, 40, 0),
                                        (4300, 48, 108, 1), (4100, 96, 64, 0)])       # the last two: M2 instantiation
def test_gemm_with_fused_elu_backward_and_bias_gradient(ops, ref, M, N, K, b_mn):
    """pd_gemm_actbwd: C = (A B^T) * elu'(dact), dbias += column sums, in the GEMM epilogue (TMA-store staging box re-read
    column-wise) — against GEMM + bias_act_bwd of the op table.  Integer operands: bit-exact, bias sums included."""
    ops.set_gemm_impl(0)
    A = ints(M, K, seed=1, lo=-2, hi=3)
    B = ints(K, N, seed=2, lo=-2, hi=3) if b_mn else ints(N, K, seed=2, lo=-2, hi=3)
    dact = ints(M, N, seed=3, lo=-3, hi=3)                   # elu'(y) from the output: 1 for y > 0, y + 1 otherwise
    out = {}
    for name, o in (("n", ops), ("r", ref)):
        C = torch.full((M, N), float("nan"), device=DEV)
        db = ints(N, seed=4).clone()
        o.gemm_actbwd(A, B, C, dact, db, b_mn=bool(b_mn))
        out[name] = (C, db)
    assert torch.equal(out["n"][0], out["r"][0]), f"C max diff {(out['n'][0] - out['r'][0]).abs().max().item()}"
    assert torch.equal(out["n"][1], out["r"][1]), f"dbias max diff {(out['n'][1] - out['r'][1]).abs().max().item()}"


@pytest.mark.parametrize("NB,H,C,k,odim", [(3, 13, 96, 5, 192), (2, 30, 48, 6, 96), (7, 5, 192, 5, 1536),
                                             (9, 30, 48, 6, 96), (30, 13, 96, 5, 192)])      # the last two: 2-CTA kernel
def test_implicit_conv_input_gradient_with_fused_elu_backward(ops, ref, NB, H, C, k, odim):
    """pd_conv_gemm_actbwd (mode 1 + ELU backward + bias gradient in the epilogue) against the composed op-table twin."""
    ops.set_gemm_impl(0)
    P = (H - k) // 2 + 1
    pixels, K = NB * P * P, k * k * C
    X = ints(NB, H, H, C, seed=1, lo=-2, hi=3)
    Wt = ints(K, odim, seed=2, lo=-2, hi=3)                  # [K][odim]: the decoder's o_mn layout
    dact = ints(pixels, odim, seed=3, lo=-3, hi=3)
    out = {}
    for name, o in (("n", ops), ("r", ref)):
        Cm = torch.full((pixels, odim), float("nan"), device=DEV)
        db = ints(odim, seed=4).clone()
        o.conv_gemm_actbwd(X, k, Wt, Cm, dact, db, o_mn=True)
        out[name] = (Cm, db)
    assert torch.equal(out["n"][0], out["r"][0]), f"C max diff {(out['n'][0] - out['r'][0]).abs().max().item()}"
    assert torch.equal(out["n"][1], out["r"][1]), f"dbias max diff {(out['n'][1] - out['r'][1]).abs().max().item()}"


@pytest.mark.parametrize("NB,Hin,Cc,extra", [(3, 6, 48, 0), (2, 14, 96, 1), (5, 2, 192, 0), (2, 5, 20, 1), (70, 14, 48, 1), (3, 14, 4, 1)])
def test_col2im_with_fused_elu_backward_and_bias_gradient(ops, ref, NB, Hin, Cc, extra):
    """pd_col2im_actbwd (k = 4 fold of the Conv2d input gradient * elu'(saved activation), per-channel sums) against
    col2im + bias_act_bwd of the op table; Cc = 20 takes the composed fallback (192 % (Cc / 4) != 0); `extra` rows / columns
    past the fold (encoder: 31 = 2 * 13 + 4 + 1) receive zero gradient."""
    k = 4
    Hout = (Hin - 1) * 2 + k + extra                         # extra = 1: a 31-wide image whose last row / column the conv never read
    col = ints(NB * Hin * Hin, k * k * Cc, seed=1, lo=-2, hi=3)
    dact = ints(NB, Hout, Hout, Cc, seed=2, lo=-3, hi=3)
    out = {}
    for name, o in (("n", ops), ("r", ref)):
        dst = torch.full((NB, Hout, Hout, Cc), float("nan"), device=DEV)
        db = ints(Cc, seed=3).clone()
        o.col2im_actbwd(col, Hin, Hin, k, dact, db, dst)
        out[name] = (dst, db)
    assert torch.equal(out["n"][0], out["r"][0]), f"max diff {(out['n'][0] - out['r'][0]).abs().max().item()}"
    close(out["n"][1], out["r"][1], 1e-6, 1e-6, "bias gradient")


@pytest.mark.parametrize("NB,Hin,k,Cc", [(3, 5, 5, 16), (2, 13, 6, 48), (5, 4, 6, 4)])
def test_fp16_column_matrix_gemm_store_and_col2im(ops, ref, NB, Hin, k, Cc):
    """Decoder forward with fp16 column matrices: pd_gemm writes C as fp16 (PD_GEMM_C_F16) and pd_col2im / pd_col2im_imgloss
    fold it back.  Integer-valued operands keep every product and sum exact in fp16, so the native path must equal the twin
    bit for bit; random operands stay within one fp16 rounding of the fp32-column result."""
    Cin = 24
    rows = NB * Hin * Hin
    X, Wt = ints(rows, Cin, lo=-2, hi=3), ints(k * k * Cc, Cin, seed=1, lo=-2, hi=3)
    Hout = (Hin - 1) * 2 + k
    bias = ints(Cc, seed=2)
    got = {}
    for name, o in (("n", ops), ("r", ref)):
        cols = torch.zeros(rows, k * k * Cc, device=DEV, dtype=torch.float16)
        o.gemm(X, Wt, cols)
        out = torch.zeros(NB, Hout, Hout, Cc, device=DEV)
        o.col2im(cols, Hin, Hin, k, bias, 1, out, round_out=False)
        got[name] = (cols.clone(), out)
    assert torch.equal(got["n"][0], got["r"][0]), "fp16 GEMM output"
    close(got["n"][1], got["r"][1], 1e-6, 1e-6, "col2im over fp16 columns")
    # random operands against the fp32-column path
    Xr, Wr = rnd(rows, Cin), rnd(k * k * Cc, Cin, seed=1) * 0.2
    c16, c32 = torch.zeros(rows, k * k * Cc, device=DEV, dtype=torch.float16), torch.zeros(rows, k * k * Cc, device=DEV)
    ops.gemm(Xr, Wr, c16); ops.gemm(Xr, Wr, c32)
    close(c16.float(), c32, 1e-3, 1e-4, "fp16 vs fp32 columns")
    if Cc <= 16:                                            # the fused last-layer fold + image loss over fp16 columns
        tgt = rnd(NB, Cc, Hout, Hout, seed=5)
        res = {}
        for name, o in (("n", ops), ("r", ref)):
            dec, diff = torch.zeros(NB, Cc, Hout, Hout, device=DEV), torch.zeros(NB, Cc, Hout, Hout, device=DEV)
            loss, csum = torch.zeros(NB, device=DEV), torch.zeros(NB, Cc, device=DEV)
            o.col2im_imgloss(c16, NB, Hin, Hin, Cc, k, bias, tgt, 1, dec, diff, loss, csum)
            res[name] = (dec, diff, loss, csum)
        for a, b_, w in zip(res["n"], res["r"], ("dec", "diff", "loss", "csum")):
            close(a, b_, 2e-5, 1e-5, "imgloss over fp16 columns: " + w)


def test_gradient_reductions_are_identical_run_to_run(ops):
    """Bias / LayerNorm / weight gradients summed over many blocks come out bit-identical on every run (fixed summation
    order, not atomics in arrival order): the training trajectory must not depend on scheduling."""
    ops.set_gemm_impl(0)
    g = torch.Generator(device=DEV).manual_seed(5)
    r = lambda *s: torch.randn(*s, device=DEV, generator=g)
    x, y = r(40000, 96), r(40000, 96)
    xs, gamma = r(3000, 400), r(400)
    mean, rstd = xs.mean(1), xs.var(1, unbiased=False).add(1e-5).rsqrt()
    A, B = r(2500, 256), r(2500, 384)

    def once():
        out = dict(colsum=torch.zeros(96, device=DEV), db=torch.zeros(96, device=DEV), dW=torch.zeros(256, 384, device=DEV))
        ops.colsum(x, out["colsum"])
        ops.bias_act_bwd(x.clone(), y, 1, out["db"])
        for rows in (3000, 100):                                   # the many-row and the row-per-block kernels
            dg, dbt, dbi = (torch.zeros(400, device=DEV) for _ in range(3))
            ops.ln_elu_bwd(xs[:rows], xs[:rows], xs[:rows].tanh(), gamma, mean[:rows], rstd[:rows],
                           torch.empty(rows, 400, device=DEV), dg, dbt, dbi)
            out.update({f"dgamma{rows}": dg, f"dbeta{rows}": dbt, f"dbias{rows}": dbi})
        ops.gemm(A, B, out["dW"], a_mn=True, b_mn=True, accumulate=True)   # weight gradient: K = 2500 rows
        torch.cuda.synchronize()
        return out

    first = once()
    for _ in range(3):
        again = once()
        for k, v in first.items():
            assert torch.equal(v, again[k]), k


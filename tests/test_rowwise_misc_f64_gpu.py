"""Kernel-level tests of the row-wise, loss, actor-critic and optimizer kernels (csrc/pd_rowwise.cu, csrc/pd_misc.cu and
the bias / ELU backward of csrc/pd_conv.cu), called directly through NativeOps on seeded inputs and compared with a
FLOAT64 reference computed from the kernel's own fp32 inputs.

References.  Where the reference implementation uses them, the references are torch.autograd over float64
torch.nn.functional / torch.distributions expressions: F.layer_norm + F.elu, the nn.GRUCell equations,
OneHotCategorical(StraightThrough) log-prob / entropy / KL, logavgexp, clip_grad_norm_, torch.optim.AdamW(foreach=False),
and the reference's GAE / reality-weight / critic / actor-loss expressions (a2c.py:81-130, functions.py:69-78,
dreamer.py:328-343,362-379) restated here.  A gradient the kernel computes in closed form is compared with autograd,
never with another closed form.  The closed forms below (`cf_*`) only build error bounds;
test_closed_forms_match_autograd ties each of them to autograd to 1e-10 without a GPU.

Bounds.  Every element is held to a small multiple of U = 2^-24 times the float64 magnitude of the terms that produce it
(sum |terms| for a sum, the depth of the kernel's fp32 summation tree times that for a reduction, |x^|.|gamma| plus the
row terms for the LayerNorm backward), plus the documented 5e-7 relative error of the ex2.approx ELU
(pd_common.cuh:104-125).  No bound is relative to a tensor's maximum.  The reasoning sits next to each bound.

Rounded outputs.  Tests of kernels that round tensor-core operands run with round_out (set_round_operands) 0 and 1; with
1 a tf32-rounded output must equal the rounded reference except within its error of a rounding boundary.

Guard bands.  Outputs are pre-filled with NaN and followed by a sentinel guard band; strided outputs have sentinel gap
columns that must stay untouched, strided inputs are views whose gap columns hold NaN.  Accumulating outputs start from
non-zero values, so `+=` and `=` differ.

PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/ref_ops.py in place of the kernels: a dry run of the
references and bounds without a GPU."""
import math

import pytest
import torch
import torch.distributions as D
import torch.nn.functional as F

from oracle.ref_ops import RefOps
from tests.util import CPU, DEV, Gen, bound, f64, fp16, fp32, ops, round_out, rounded, ulp  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24                                  # unit roundoff of fp32
ELU_REL = 5e-7                                  # relative error of pd_elu's ex2.approx branch (pd_common.cuh:104-125)
TINY = 2.0 ** -126                              # fp32 underflow: anything below this may flush or lose bits
P = torch.cuda.get_device_properties(0).multi_processor_count if (not CPU and torch.cuda.is_available()) else 132
NAN_GUARD = -12345.0                            # sentinel of guard bands and gap columns
IDX_GUARD = -777
NAN = float("nan")


# ----------------------------------------------------------------------------------------------------- helpers
def check(name, got, ref, err, round_out, stats):
    """An output the kernel rounds to tf32 when round_out is set (the float32 twin of the dry run does not round)."""
    if round_out and not CPU:
        assert ((got.contiguous().view(torch.int32) & 0x1FFF) == 0).all(), f"{name}: not tf32-rounded"
        rounded(name, got, ref, err, "tf32", stats)
    else:
        bound(name, got, ref, err + (ulp(ref, -126, 10) if round_out else 0.0))


class Bufs:
    """Output buffers: the view the kernel writes, pre-filled (NaN by default), inside storage whose every other element
    (gap columns of a strided view and a guard band after the last row) holds a sentinel that must stay untouched."""

    def __init__(self):
        self.items = []

    def out(self, name, shape, dtype=torch.float32, gap=0, fill=NAN, init=None):
        shape = tuple(shape)
        n = shape[-1]
        rows = math.prod(shape[:-1])
        ld = n + gap
        sent = IDX_GUARD if dtype == torch.int32 else NAN_GUARD
        flat = torch.full((rows * ld + max(256, 2 * ld),), sent, dtype=dtype, device=DEV)
        view = flat[:rows * ld].view(rows, ld)[:, :n]
        if init is not None:
            view.copy_(init.reshape(rows, n))
        else:
            view.fill_(fill)
        keep = torch.ones(flat.numel(), dtype=torch.bool, device=DEV)
        keep[:rows * ld].view(rows, ld)[:, :n] = False
        self.items.append((name, flat, keep, flat.clone()))
        return view if len(shape) == 2 else view.reshape(shape)

    def check(self):
        if not CPU:
            torch.cuda.synchronize()
        for name, flat, keep, before in self.items:
            iv = {4: torch.int32, 2: torch.int16}[flat.element_size()]
            assert torch.equal(flat.view(iv)[keep], before.view(iv)[keep]), f"{name}: written outside its view"


def gapped(v, gap=5):
    """fp32 copy of the 2-D float64 v as a view into rows of ld = N + gap whose gap columns hold NaN."""
    M, N = v.shape
    buf = torch.full((M, N + gap), NAN, dtype=torch.float32, device=DEV)
    buf[:, :N] = v
    return buf[:, :N]


def f32(v):
    return v.float().contiguous()


def sync():
    if not CPU:
        torch.cuda.synchronize()


def refused(ops, call, code):
    """A call past a host-side limit fails with `code` before launching anything."""
    if CPU:
        pytest.skip("host-side argument checks of the native library (the float32 twin checks no limits)")
    with pytest.raises(RuntimeError, match=rf"failed \({code}\)"):
        call()
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------- closed forms
# Used only to build error bounds; test_closed_forms_match_autograd ties each to autograd.
def cf_ln_elu_bwd(dy, x, y, gamma, mu, r):
    eg = torch.where(y > 0, torch.ones_like(y), y + 1)
    g = dy * eg
    xh = (x - mu[:, None]) * r[:, None]
    dxh = g * gamma
    c1, c2 = dxh.mean(-1, keepdim=True), (dxh * xh).mean(-1, keepdim=True)
    return dict(eg=eg, g=g, xh=xh, dxh=dxh, c1=c1, c2=c2, dx=r[:, None] * (dxh - c1 - xh * c2))


def cf_gru_bwd(dh, r, u, n, ghn, hp):
    dn = dh * (1 - u) * (1 - n * n)
    du = dh * (hp - n) * u * (1 - u)
    dr = dn * ghn * r * (1 - r)
    return dict(dgi=torch.cat([dr, du, dn], 1), dgh=torch.cat([dr, du, dn * r], 1), carry=dh * u)


def cf_cat_st_bwd(p, dz):
    return p * (dz - (p * dz).sum(-1, keepdim=True))


def cf_kl(lp, lq, p, q, wpost, wprior):
    kl = (p * (lp - lq)).sum(-1, keepdim=True)
    return wpost * p * ((lp - lq) - kl), wprior * (q - p)


def cf_actor_onehot(lp, p, oh, ag, w, eta, rows):
    ent = -(p * lp).sum(-1, keepdim=True)
    return (w / rows)[:, None] * (-ag[:, None] * (oh - p) + eta * p * (lp + ent))


def cf_tanh_normal(m_, s_, a, ag, w, eta, rows):
    th = torch.tanh(m_ / 5)
    mu, sd = 5 * th, F.softplus(s_) + 0.1
    zc = (torch.atanh(a) - mu) / sd
    c = (w / rows)[:, None]
    return (c * (-ag[:, None] * zc / sd) * (1 - th * th),
            c * (-ag[:, None] * (zc * zc - 1) / sd - eta / sd) * torch.sigmoid(s_))


# ----------------------------------------------------------------------------------------------------- LayerNorm + ELU
LN_EPS = 1e-3
LN_BIG = 4 * (2 * P * 4) + 3      # the backward grid is capped at 2 * #SMs blocks of 4 warps: each warp loops 4-5 times
LN_M = [1, 255, 256, 257, 2500, LN_BIG]
LN_N = [1, 31, 33, 400, 416, 417, 1000, 1024]
KS = 40                           # fp32 additions an element of a LayerNorm row sum goes through: <= 32 per lane + 5
                                  # shuffle levels (warp kernels), 4 + 5 + 5 (256-thread row kernel), + the / N


def ln_inputs(M, N, seed):
    g = Gen(seed)
    x = fp32(g.normal(M, N, scale=2.0) + g.uniform(M, 1, bound=3.0))      # a row offset: the mean must come off
    return x, fp32(1 + g.normal(N, scale=0.3)), fp32(g.normal(N, scale=0.3))


def ln_fwd_ref(x, gamma, beta):
    """float64 F.layer_norm + F.elu, the statistics, and the fp32 error of computing them the kernel's way."""
    N = x.shape[1]
    var, mu = torch.var_mean(x, -1, unbiased=False)
    r = 1.0 / torch.sqrt(var + LN_EPS)
    pre = F.layer_norm(x, (N,), gamma, beta, LN_EPS)
    y = F.elu(pre)
    # mean: KS roundings of each |x| in the sum, one for / N
    e_mu = KS * U * x.abs().mean(-1) + U * mu.abs()
    # variance: d = x - mean carries the mean's error (it only adds e_mu^2 to the mean square) and one rounding; d*d one,
    # the sum KS; rstd = 1/sqrt(var + eps) halves the relative error of var + eps and adds three roundings
    d = x - mu[:, None]
    e_var = (KS + 4) * U * (d * d).mean(-1) + e_mu ** 2
    e_r = r * (0.5 * e_var / (var + LN_EPS) + 3 * U)
    xh = d * r[:, None]
    e_xh = r[:, None] * (e_mu[:, None] + U * d.abs()) + xh.abs() * (e_r / r)[:, None] + U * xh.abs()
    # pre = xh * gamma + beta: |x^|.|gamma| carries e_xh, two more roundings; ELU' <= 1 passes the error on, then the
    # ex2.approx branch's relative error, its degree-7 polynomial's 4e-10 and the rounding of x * log2(e) (|pre| U e^pre)
    e_pre = gamma.abs() * e_xh + 2 * U * ((xh * gamma).abs() + pre.abs() + beta.abs())
    e_y = e_pre + (ELU_REL + U) * y.abs() + 4e-10 + U * pre.abs() * (y + 1).clamp_min(0)
    return y, mu, r, e_y, e_mu, e_r


def ln_bwd_ref(dy, x, gamma, beta, y_in):
    """Autograd of F.elu(F.layer_norm(x)) (dx, dgamma, dbeta; dbias = column sums of dx) and the error bounds of the
    kernel's closed form evaluated in fp32 on fp32 inputs (y, mean, rstd = float64 values rounded to fp32)."""
    N = x.shape[1]
    xg, gg, bg = (v.clone().requires_grad_(True) for v in (x, gamma, beta))
    F.elu(F.layer_norm(xg, (N,), gg, bg, LN_EPS)).backward(dy)
    var, mu = torch.var_mean(x, -1, unbiased=False)
    r = 1.0 / torch.sqrt(var + LN_EPS)
    c = cf_ln_elu_bwd(dy, x, y_in, gamma, mu, r)
    eg, g, xh, dxh, c1, c2 = (c[k] for k in ("eg", "g", "xh", "dxh", "c1", "c2"))
    # inputs: y (rounded: U|y| on elu' = y + 1, plus the add), mean and rstd (rounded: U|mean|, U rstd)
    Eg = dy.abs() * U * (y_in.abs() * (y_in <= 0) + eg) + U * g.abs()
    Exh = U * (r[:, None] * (mu.abs()[:, None] + (x - mu[:, None]).abs()) + 2 * xh.abs())
    Edxh = gamma.abs() * Eg + U * dxh.abs()
    Ec1 = (Edxh.sum(-1, keepdim=True) + KS * U * dxh.abs().sum(-1, keepdim=True)) / N + U * c1.abs()
    t2 = dxh * xh
    Ec2 = ((Edxh * xh.abs() + dxh.abs() * Exh + U * t2.abs()).sum(-1, keepdim=True)
           + KS * U * t2.abs().sum(-1, keepdim=True)) / N + U * c2.abs()
    T = dxh.abs() + c1.abs() + (xh * c2).abs()
    Edx = r[:, None] * (Edxh + Ec1 + Exh * c2.abs() + xh.abs() * Ec2 + 4 * U * T) + U * c["dx"].abs()
    terms = dict(g=(g * xh, Eg * xh.abs() + g.abs() * Exh + U * (g * xh).abs()), b=(g, Eg), x=(c["dx"], Edx))
    return xg.grad, gg.grad, bg.grad, Edx, terms


def ln_col_depth(M, N):
    """Roundings of one row's term in the kernel's column sums: the 256-row kernel adds row terms in row order; the warp
    kernels add per lane over a warp's rows, then the 4 warps of a block, then the blocks of the capped grid in order."""
    if M <= 256:
        return M
    grid = min(-(-M // 4), 2 * P)
    return -(-M // (4 * grid)) + 4 + grid


@gpu
@pytest.mark.parametrize("N", LN_N)
@pytest.mark.parametrize("M", LN_M)
def test_ln_elu_fwd_bwd_against_float64_autograd(ops, round_out, M, N):
    x, gamma, beta = ln_inputs(M, N, seed=M + N)
    B = Bufs()
    y = B.out("y", (M, N), gap=3)
    y16 = B.out("y16", (M, N), dtype=torch.float16, gap=2)
    mean, rstd = B.out("mean", (M,)), B.out("rstd", (M,))
    ops.ln_elu_fwd(gapped(x), f32(gamma), f32(beta), LN_EPS, y, mean, rstd, y16)
    B.check()
    yr, mu, r, e_y, e_mu, e_r = ln_fwd_ref(x, gamma, beta)
    stats = {}
    check("y", y, yr, e_y, round_out, stats)
    # the fp16 side output is the kernel's own (rounded) fp32 y converted with round-to-nearest-even
    assert torch.equal(y16.double(), fp16(y.double())), "y16 != fp16(y)"
    bound("mean", mean, mu, e_mu)
    bound("rstd", rstd, r, e_r)

    # backward on fp32-rounded float64 forward values; dgamma / dbeta / dbias accumulate into non-zero values
    g = Gen(M * N + 1)
    dy = fp32(g.normal(M, N))
    y_in = fp32(yr)
    pre = {k: fp32(g.normal(N)) for k in ("dgamma", "dbeta", "dbias")}
    for with_bias in (True, False):
        B = Bufs()
        dx = B.out("dx", (M, N), gap=7)
        acc = {k: B.out(k, (N,), init=pre[k]) for k in ("dgamma", "dbeta", "dbias")}
        ops.ln_elu_bwd(gapped(dy), gapped(x), gapped(y_in), f32(gamma), f32(mu), f32(r), dx, acc["dgamma"],
                       acc["dbeta"], acc["dbias"] if with_bias else None)
        B.check()
        dx_ref, dg_ref, db_ref, Edx, terms = ln_bwd_ref(dy, x, gamma, beta, y_in)
        check("dx", dx, dx_ref, Edx, round_out, stats)
        # column sums: each row term's propagated error, the kernel's summation depth, the add into the pre-filled value
        depth = ln_col_depth(M, N) + 2
        for k, ref in (("dgamma", dg_ref), ("dbeta", db_ref), ("dbias", dx_ref.sum(0))):
            v, e = terms[{"dgamma": "g", "dbeta": "b", "dbias": "x"}[k]]
            lim = e.sum(0) + depth * U * v.abs().sum(0) + U * (pre[k] + ref).abs()
            if k == "dbias" and not with_bias:
                assert torch.equal(acc[k].double(), pre[k]), "dbias written although NULL"
            else:
                bound(k, acc[k], pre[k] + ref, lim)
    print("tf32 values within error of a rounding boundary", stats)


@gpu
def test_ln_elu_bwd_maxv32_identical_run_to_run(ops):
    """The MAXV = 32 backward (M = 2500 > 256, 416 < N <= 1024) adds its parameter gradients in a fixed order."""
    M, N = 2500, 1000
    x, gamma, beta = ln_inputs(M, N, seed=3)
    y, mu, r, *_ = ln_fwd_ref(x, gamma, beta)
    dy = fp32(Gen(4).normal(M, N))
    outs = []
    for _ in range(2):
        o = [torch.empty(M, N, device=DEV)] + [torch.full((N,), 0.25, device=DEV) for _ in range(3)]
        ops.ln_elu_bwd(f32(dy), f32(x), f32(y), f32(gamma), f32(mu), f32(r), *o)
        sync()
        outs.append(o)
    for a, b, n in zip(*outs, ("dx", "dgamma", "dbeta", "dbias")):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{n} differs between two identical runs"


@gpu
@pytest.mark.parametrize("N", [0, 1025])
def test_ln_elu_refuses_row_lengths_outside_1_to_1024(ops, N):
    M = 300
    x = torch.zeros(M, max(N, 1), device=DEV)
    keep = torch.full((M, max(N, 1)), NAN, device=DEV)
    st = torch.full((M,), NAN, device=DEV)
    p = lambda t: t.data_ptr()
    L, h = getattr(ops, "lib", None), getattr(ops, "h", None)
    for M_ in (M, 10):        # both launch branches
        refused(ops, lambda: ops._ck(L.pd_ln_elu_fwd(h, M_, N, p(x), x.shape[1], p(st), p(st), 1e-3, p(keep), x.shape[1],
                                                     p(st), p(st), None, 0, ops._s()), "pd_ln_elu_fwd"), -1)
        refused(ops, lambda: ops._ck(L.pd_ln_elu_bwd(h, M_, N, p(x), x.shape[1], p(x), x.shape[1], p(x), x.shape[1], p(st),
                                                     p(st), p(st), p(keep), x.shape[1], p(st), p(st), p(st), ops._s()),
                                     "pd_ln_elu_bwd"), -1)
    assert torch.isnan(keep).all() and torch.isnan(st).all(), "a refused call wrote an output"


# ----------------------------------------------------------------------------------------------------- GRU gates
GRU_CASES = [(7, 1), (5, 33), (9, 1000), (50, 2048)]     # M * D not a multiple of 256 except at D = 2048 (impossible)


def gru_inputs(M, D, seed):
    g = Gen(seed)
    gi, gh = fp32(g.normal(M, 3 * D, scale=2.0)), fp32(g.normal(M, 3 * D, scale=2.0))
    gi[0] = 30.0 * torch.sign(g.normal(3 * D))              # saturated pre-activations: sigmoid -> 0 / 1, tanh -> +-1
    if M > 1:
        gh[1] = -30.0 * torch.sign(g.normal(3 * D))
    return gi, gh, fp32(g.normal(M, D)), (g.rand(M) > 0.3).to(f64)


def gru_fwd64(gi, gh, hp):
    """The nn.GRUCell equations (gate order r | u | n), float64."""
    D = hp.shape[1]
    r = torch.sigmoid(gi[:, :D] + gh[:, :D])
    u = torch.sigmoid(gi[:, D:2 * D] + gh[:, D:2 * D])
    ghn = gh[:, 2 * D:]
    n = torch.tanh(gi[:, 2 * D:] + r * ghn)
    return r, u, n, ghn, (1 - u) * n + u * hp


@gpu
@pytest.mark.parametrize("M,D", GRU_CASES)
def test_gru_fwd_against_float64(ops, round_out, M, D):
    gi, gh, hp, mask = gru_inputs(M, D, seed=M + D)
    B = Bufs()
    hout, hmask = B.out("h", (M, D), gap=3), B.out("hmask", (M, D), gap=1)
    gates, h16 = B.out("gates", (M, 4 * D)), B.out("h16", (M, D), dtype=torch.float16, gap=2)
    ops.gru_fwd(gapped(gi, 7), gapped(gh, 3), gapped(hp, 2), hout, hmask, f32(mask), gates, h16)
    B.check()
    r, u, n, ghn, h = gru_fwd64(gi, gh, hp)
    s = lambda v, j: v[:, j * D:(j + 1) * D]
    # sigmoid: the pre-activation sum rounds (U|x|, times sigmoid' = s(1-s)); expf 2 ulp, 1 + e and the division one each
    E_r = 4 * U * r + U * (s(gi, 0) + s(gh, 0)).abs() * r * (1 - r)
    E_u = 4 * U * u + U * (s(gi, 1) + s(gh, 1)).abs() * u * (1 - u)
    # tanh: its argument carries |gh_n| E_r and two roundings; tanh' <= 1 - n^2; tanhf 2 ulp
    arg = s(gi, 2) + r * ghn
    E_n = (1 - n * n) * (ghn.abs() * E_r + U * ((r * ghn).abs() + arg.abs())) + 3 * U * n.abs()
    E_h = (n - hp).abs() * E_u + (1 - u) * E_n + 4 * U * (((1 - u) * n).abs() + (u * hp).abs()) + U * u * n.abs()
    gt = gates.view(M, 4, D)
    bound("r", gt[:, 0], r, E_r)
    bound("u", gt[:, 1], u, E_u)
    bound("n", gt[:, 2], n, E_n)
    assert torch.equal(gt[:, 3].double(), ghn), "gates[3] != gh_n"
    stats = {}
    check("h", hout, h, E_h, round_out, stats)
    assert torch.equal(h16.double(), fp16(hout.double())), "h16 != fp16(h')"
    assert torch.equal(hmask.double(), hout.double() * mask[:, None]), "hmask != h' * mask_next"
    assert ((gt[0, 1] == 0) | (gt[0, 1] == 1)).any() or CPU, "the +-30 row does not saturate the update gate"


GRU_BWD_OPTS = ["all", "no_dh_a", "no_dh_b", "no_mask_b"]


@gpu
@pytest.mark.parametrize("opt", GRU_BWD_OPTS)
@pytest.mark.parametrize("M,D", GRU_CASES)
def test_gru_bwd_against_float64_autograd(ops, round_out, M, D, opt):
    gi, gh, hp, mask = gru_inputs(M, D, seed=M * D)
    g = Gen(D)
    dh_a = None if opt == "no_dh_a" else fp32(g.normal(M, D))
    dh_b = None if opt == "no_dh_b" else fp32(g.normal(M, D))
    mask_b = None if opt == "no_mask_b" else mask
    # autograd of sum(dh * h') over the GRUCell equations; dh = dh_a + dh_b * mask_b
    dh = torch.zeros(M, D, dtype=f64, device=DEV)
    if dh_a is not None:
        dh = dh + dh_a
    if dh_b is not None:
        dh = dh + dh_b * (mask_b[:, None] if mask_b is not None else 1.0)
    gig, ghg, hpg = (v.clone().requires_grad_(True) for v in (gi, gh, hp))
    r, u, n, ghn, h = gru_fwd64(gig, ghg, hpg)
    (h * dh).sum().backward()
    gates = fp32(torch.stack([r, u, n, ghn], 1).detach()).reshape(M, 4 * D)
    B = Bufs()
    dgi, dgh, carry = B.out("dgi", (M, 3 * D), gap=5), B.out("dgh", (M, 3 * D), gap=3), B.out("dh_carry", (M, D), gap=1)
    ops.gru_bwd(None if dh_a is None else gapped(dh_a, 3), None if dh_b is None else gapped(dh_b, 2),
                None if mask_b is None else f32(mask_b), f32(gates), gapped(hp, 4), dgi, dgh, carry)
    B.check()
    # running error bound: +, -, * only on fp32 inputs (the gates rounded once, dh summed once), <= 16 roundings, each
    # bounded by U times the expression evaluated on absolute values with every difference turned into a sum
    gv = gates.view(M, 4, D)
    ra, ua, na, gha = gv[:, 0], gv[:, 1], gv[:, 2].abs(), gv[:, 3].abs()
    dha = torch.zeros_like(dh)
    if dh_a is not None:
        dha = dha + dh_a.abs()
    if dh_b is not None:
        dha = dha + dh_b.abs()
    dn_a = dha * (1 + ua) * (1 + na * na)
    du_a = dha * (hp.abs() + na) * ua * (1 + ua)
    dr_a = dn_a * gha * ra * (1 + ra)
    lim = lambda v: 16 * U * v
    stats = {}
    check("dgi", dgi, gig.grad, lim(torch.cat([dr_a, du_a, dn_a], 1)), round_out, stats)
    check("dgh", dgh, ghg.grad, lim(torch.cat([dr_a, du_a, dn_a * ra], 1)), round_out, stats)
    bound("dh_carry", carry, hpg.grad, lim(dha * ua))     # dh * u is never rounded


# ----------------------------------------------------------------------------------------------------- categorical
def softmax_err(l, G, C):
    """float64 log-softmax / softmax of the kernel's fp32 logits per group of C, and their fp32 error: with A = max |l| of
    the group, l - lse carries U(|l| + |lse|) and the error of lse (U |max|, expf's 2 ulp and the log of a sum of at most
    32 terms, relative errors |l - max| U): <= U (6 A + 16).  p = exp(lp - max lp) / sum doubles that and adds the
    normalisation's roundings; below 2^-126 it may underflow."""
    M = l.shape[0]
    lg = l.reshape(M, G, C)
    lp = torch.log_softmax(lg, -1)
    p = lp.exp()
    A = lg.abs().amax(-1, keepdim=True)
    Elp = U * (6 * A + 16)
    Ep = p * (2 * Elp + 12 * U) + TINY
    return lp, p, Elp.expand_as(lp), Ep


def cat_logits(M, G, C, seed):
    """Normal logits; group 0 of every row spread +-60 (most of p underflows to 0 in fp32); the last group of row 0 a tie
    of all classes, the last group of row 1 a tie of classes 1 and C - 1 (exact: equal logits, equal noise)."""
    g = Gen(seed)
    l = fp32(g.normal(M, G, C, scale=3.0))
    noise = fp32(torch.empty(M, G, C, dtype=torch.float32).exponential_(generator=g.g).double()).to(DEV)
    l[:, 0] = 60.0 * torch.sign(g.normal(M, C))
    l[0, -1] = 0.5
    noise[0, -1] = 1.0
    if M > 1 and C > 1:
        l[1, -1] = -5.0
        l[1, -1, 1] = l[1, -1, C - 1] = 4.0
        noise[1, -1, 1] = noise[1, -1, C - 1] = 0.75
    return l.reshape(M, G * C), noise.reshape(M, G * C)


CAT_C = [1, 2, 7, 17, 31, 32]
CAT_G = [1, 3, 32, 33]
CAT_M = 13                         # M * G not a multiple of 8 (the last 8-group block partial) except at G = 32


@gpu
@pytest.mark.parametrize("opt", ["all", "none"])
@pytest.mark.parametrize("G", CAT_G)
@pytest.mark.parametrize("C", CAT_C)
def test_cat_sample_is_first_argmax_of_p_over_q(ops, C, G, opt):
    M, Z = CAT_M, G * C
    l, noise = cat_logits(M, G, C, seed=C * G)
    mask = (Gen(1).rand(M) > 0.3).to(f64)
    B = Bufs()
    z = B.out("z", (M, Z), gap=3)
    zmask = B.out("zmask", (M, Z), gap=2) if opt == "all" else None
    idx = B.out("idx", (M, G), dtype=torch.int32, fill=-1) if opt == "all" else None
    z16 = B.out("z16", (M, Z), dtype=torch.float16, gap=1) if opt == "all" else None
    ops.cat_sample(gapped(l, 3), gapped(noise, 6), G, C, z, zmask, f32(mask) if zmask is not None else None, idx, z16)
    B.check()
    lp, p, _, Ep = softmax_err(l, G, C)
    ratio = p / noise.reshape(M, G, C)
    want = ratio.argmax(-1)                       # torch.argmax: the FIRST maximum
    k = z.double().reshape(M, G, C).argmax(-1)
    assert torch.equal(z.double(), F.one_hot(k, C).reshape(M, Z).to(f64)), "z is not one-hot"
    # near-ties: the fp32 p / q of two classes within their error of each other (exact ties are not near-ties)
    e = Ep / noise.reshape(M, G, C)
    top = ratio.topk(min(2, C), -1)
    near = torch.zeros(M, G, dtype=torch.bool, device=DEV)
    if C > 1:
        i0, i1 = top.indices[..., :1], top.indices[..., 1:2]
        gap_ = (top.values[..., 0] - top.values[..., 1])
        near = (gap_ > 0) & (gap_ <= (e.gather(-1, i0) + e.gather(-1, i1))[..., 0])
    wrong = (k != want) & ~near
    assert not wrong.any(), f"{int(wrong.sum())} samples differ from the first argmax of p/q away from a near-tie"
    assert int(k[0, -1]) == 0, "an exact tie of all classes must give class 0"
    if C > 1:
        assert int(k[1, -1]) == 1, "an exact tie of classes 1 and C-1 must give class 1"
    if opt == "all":
        assert torch.equal(idx.long(), k), "idx != the sampled class"
        assert torch.equal(z16.double(), z.double()), "z16 != z"
        assert torch.equal(zmask.double(), z.double() * mask[:, None]), "zmask != z * mask_next"
    print("near-ties", int(near.sum()))


CAT_BWD_OPTS = ["all", "no_dz_a", "no_dz_b", "no_mask_b", "no_extra", "no_rowscale"]


@gpu
@pytest.mark.parametrize("opt", CAT_BWD_OPTS)
@pytest.mark.parametrize("G", CAT_G)
@pytest.mark.parametrize("C", CAT_C)
def test_cat_st_bwd_against_float64_autograd(ops, round_out, C, G, opt):
    M, Z = CAT_M, G * C
    l, _ = cat_logits(M, G, C, seed=C + G)
    g = Gen(C * 7 + G)
    dz_a = None if opt == "no_dz_a" else fp32(g.normal(M, Z))
    dz_b = None if opt == "no_dz_b" else fp32(g.normal(M, Z))
    mask_b = None if opt == "no_mask_b" else (g.rand(M) > 0.3).to(f64)
    extra = None if opt == "no_extra" else fp32(g.normal(M, Z))
    rs = None if opt == "no_rowscale" else fp32(g.rand(M))
    alpha = 0.75
    dz = torch.zeros(M, Z, dtype=f64, device=DEV)
    dza = torch.zeros_like(dz)
    if dz_a is not None:
        dz, dza = dz + dz_a, dza + dz_a.abs()
    if dz_b is not None:
        dz, dza = dz + dz_b * (mask_b[:, None] if mask_b is not None else 1.0), dza + dz_b.abs()
    # autograd of sum(dz * z) over OneHotCategoricalStraightThrough (z = sample + p - p.detach()), plus the linear term
    # alpha * rowscale * extra . logits
    lg = l.clone().requires_grad_(True)
    zs = D.OneHotCategoricalStraightThrough(logits=lg.view(M, G, C)).rsample().reshape(M, Z)
    loss = (dz * zs).sum()
    ex = 0.0
    if extra is not None:
        ex = alpha * (rs[:, None] if rs is not None else 1.0) * extra
        loss = loss + (ex * lg).sum()
    loss.backward()
    B = Bufs()
    dl = B.out("dlogits", (M, Z), gap=4)
    ops.cat_st_bwd(gapped(l, 2), G, C, None if dz_a is None else gapped(dz_a, 1), None if dz_b is None else gapped(dz_b, 3),
                   None if mask_b is None else f32(mask_b), None if extra is None else gapped(extra, 2),
                   None if rs is None else f32(rs), alpha, dl)
    B.check()
    # p (dz - s), s = sum p dz over the warp: Ep carries into both; dz = dz_a + dz_b * mask two roundings; the sum 7
    _, p, _, Ep = softmax_err(l, G, C)
    dzg, dzag = dz.view(M, G, C), dza.view(M, G, C)
    s = (p * dzg).sum(-1, keepdim=True)
    Edz = 2 * U * dzag
    Es = (Ep * dzg.abs() + p * Edz).sum(-1, keepdim=True) + 7 * U * (p * dzag).sum(-1, keepdim=True)
    E = Ep * (dzg - s).abs() + p * (Edz + Es) + 2 * U * p * (dzag + s.abs())
    E = E.reshape(M, Z)
    if extra is not None:
        E = E + 4 * U * (ex.abs() + (lg.grad - ex).abs())
    stats = {}
    check("dlogits", dl, lg.grad, E + U * lg.grad.abs(), round_out, stats)


# ----------------------------------------------------------------------------------------------------- KL
KL_G = [1, 3, 17, 32]
KL_C = [2, 7, 32]
KL_MODES = [(0, -1.0), (0, 0.0), (0, 0.8), (0, 1.0), (1, None)]


def kl_ref(post, prior, G, C, mode, balance, idx):
    """torch.distributions: KL(post || prior) per row, entropies, and autograd of the loss of dreamer.py:328-343: the
    plain KL (balance < 0), (1 - b) KL(post || sg(prior)) + b KL(sg(post) || prior), or the sampled log q(z) - log p(z)."""
    M = post.shape[0]
    lp, lq = (v.reshape(M, G, C).clone().requires_grad_(True) for v in (post, prior))
    dp, dq = D.OneHotCategorical(logits=lp), D.OneHotCategorical(logits=lq)
    kl = D.kl_divergence(dp, dq)
    if mode == 1:
        z = F.one_hot(idx.long(), C).to(f64)
        loss = dp.log_prob(z) - dq.log_prob(z)
    elif balance < 0:
        loss = kl
    else:
        loss = ((1 - balance) * D.kl_divergence(dp, D.OneHotCategorical(logits=lq.detach()))
                + balance * D.kl_divergence(D.OneHotCategorical(logits=lp.detach()), dq))
    loss.sum().backward()
    return (loss.sum(-1).detach(), kl.sum(-1).detach(), dp.entropy().sum(-1).detach(), dq.entropy().sum(-1).detach(),
            lp.grad.reshape(M, G * C), lq.grad.reshape(M, G * C))


@gpu
@pytest.mark.parametrize("mode,balance", KL_MODES, ids=lambda v: str(v))
@pytest.mark.parametrize("C", KL_C)
@pytest.mark.parametrize("G", KL_G)
def test_kl_against_float64_distributions(ops, G, C, mode, balance):
    M, Z = 6, G * C
    g = Gen(G * 100 + C)
    post, prior = fp32(g.normal(M, Z, scale=2.0)), fp32(g.normal(M, Z, scale=2.0))
    post[0] = 60.0 * torch.sign(g.normal(Z))          # row 0: most of p underflows to 0 in fp32 (the p > 0 branch)
    prior[1] = -60.0 * torch.sign(g.normal(Z))
    idx = torch.randint(0, C, (M, G), generator=g.g).to(DEV)
    idx[0] = C - 1
    idx = idx.to(torch.int32)
    B = Bufs()
    outs = [B.out(n, (M,)) for n in ("loss_kl", "kl_exact", "ent_post", "ent_prior")]
    dpost, dprior = B.out("dpost", (M, Z), gap=3), B.out("dprior", (M, Z), gap=1)
    ops.kl(gapped(post, 2), gapped(prior, 5), idx if mode == 1 else None, mode, balance if mode == 0 else 0.0, G, C,
           *outs, dpost, dprior)
    B.check()
    loss, kl, hp, hq, gpo, gpr = kl_ref(post, prior, G, C, mode, balance if mode == 0 else -1.0, idx)
    lp, p, Elp, Ep = softmax_err(post, G, C)
    lq, q, Elq, Eq = softmax_err(prior, G, C)
    d = lp - lq
    # per group: sum_c p (lp - lq) over a warp (5 levels + product + difference), then the groups (5 levels)
    klg = (p * d).sum(-1)
    Eklg = (Ep * d.abs() + p * (Elp + Elq)).sum(-1) + 8 * U * (p * d.abs()).sum(-1)
    row = lambda e, v: e.sum(-1) + 7 * U * v.abs().sum(-1)
    Ent = lambda lx, x, El, Ex: row((Ex * lx.abs() + x * El).sum(-1) + 8 * U * (x * lx.abs()).sum(-1), (x * lx).sum(-1))
    bound("kl_exact", outs[1], kl, row(Eklg, klg))
    bound("ent_post", outs[2], hp, Ent(lp, p, Elp, Ep))
    bound("ent_prior", outs[3], hq, Ent(lq, q, Elq, Eq))
    if mode == 0:
        wpo, wpr = (1.0, 1.0) if balance < 0 else (1 - balance, balance)
        bound("loss_kl", outs[0], loss, row(Eklg, klg))
        E1 = wpo * (Ep * (d - klg[..., None]).abs() + p * (Elp + Elq + Eklg[..., None]) + 3 * U * p * (d.abs() + klg.abs()[..., None]))
        E2 = wpr * (Ep + Eq + 2 * U * (p + q))
    else:
        sel = d.gather(-1, idx.long()[..., None])[..., 0]
        bound("loss_kl", outs[0], loss, row(Elp[..., 0] + Elq[..., 0] + U * sel.abs(), sel))
        E1, E2 = Ep + U, Eq + U
    bound("dpost", dpost, gpo, E1.reshape(M, Z))
    bound("dprior", dprior, gpr, E2.reshape(M, Z))


# ----------------------------------------------------------------------------------------------------- heads and losses
@gpu
@pytest.mark.parametrize("div", [1, 4])
@pytest.mark.parametrize("kind", [0, 1])
def test_scalar_head_loss_against_float64_autograd(ops, kind, div):
    M = 1003 * div
    g = Gen(kind * 10 + div)
    if kind == 0:
        y, t = fp32(g.normal(M, scale=3.0)), fp32(g.normal(M // div))
    else:
        y, t = fp32(g.uniform(M, bound=80.0)), (g.rand(M // div) > 0.5).to(f64)   # |y| up to 80: exp(|y|) overflows
        y[:4] = torch.tensor([80.0, -80.0, 0.0, 17.0], dtype=f64)
    B = Bufs()
    loss, dy, rec = B.out("loss", (M,)), B.out("dy", (M,)), B.out("rec", (M,))
    ops.scalar_head_loss(kind, f32(y), f32(t), div, loss, dy, rec)
    B.check()
    tt = t.repeat_interleave(div)
    yg = y.clone().requires_grad_(True)
    if kind == 0:
        # DenseNormalDecoder: -Normal(y, 1).log_prob(t) without its constant
        lr = -D.Normal(yg, 1.0).log_prob(tt) - 0.5 * math.log(2 * math.pi)
        rec_ref = y
        El = 3 * U * (tt - y) ** 2 + U * (tt - y).abs()
        Ed = U * (tt - y).abs()
    else:
        lr = -D.Bernoulli(logits=yg).log_prob(tt)
        rec_ref = torch.sigmoid(y)
        # max(y,0) - y t + log1p(exp(-|y|)): three roundings of the terms, expf 2 + log1pf 1 ulp of the last
        l1p = torch.log1p(torch.exp(-y.abs()))
        El = 3 * U * (y.clamp_min(0) + (y * tt).abs() + lr.detach().abs()) + 4 * U * l1p
        # the float64 reference itself: torch forms log(1 + exp(-|y|)) without log1p, so a loss below ~1e-16 comes out 0
        # (the kernel's log1pf keeps it)
        El = El + 4 * 2.0 ** -53 * (1 + y.abs())
        if CPU:
            El = El + 2 * U * y.abs()        # the float32 twin's BCE cancels terms of size |y|; the kernel does not
        Ed = 4 * U * rec_ref + U * (rec_ref - tt).abs()
    lr.sum().backward()
    bound("loss", loss, lr.detach(), El)
    bound("dy", dy, yg.grad, Ed)
    bound("rec", rec, rec_ref, 4 * U * rec_ref.abs())


def nlae(v, I):
    """-logavgexp(-v) over the last dim (functions.py:97-102): logsumexp - log I, a squeeze for I == 1."""
    return v[..., 0] if I == 1 else -((-v).logsumexp(-1) - math.log(I))


@gpu
@pytest.mark.parametrize("I", [1, 2, 3, 16])
def test_wm_loss_against_float64_autograd(ops, I):
    TB = 133
    N = TB * I
    g = Gen(I)
    # per-sample losses up to 1e3: exp(-L) underflows to 0 in fp32 without the max shift
    ls = [fp32(g.rand(N) * s) for s in (1e3, 2.0, 5.0, 50.0, 30.0, 10.0, 10.0)]
    l_img, l_rew, l_term, l_kl, kl_exact, ent_prior, ent_post = ls
    kw, wi, wr, wt = 0.1, 1.0, 1.0, 5.0
    B = Bufs()
    w, tb = B.out("w", (N,)), B.out("tb", (TB, 8))
    ops.wm_loss(TB, I, kw, wi, wr, wt, *(f32(v) for v in ls), w, tb)
    B.check()
    ws = [fp32(torch.tensor(v, dtype=f64)) for v in (kw, wi, wr, wt)]
    Lg = ((ws[0] * l_kl + ws[1] * l_img + ws[2] * l_rew + ws[3] * l_term).view(TB, I)).clone().requires_grad_(True)
    lm = nlae(Lg, I)
    lm.mean().backward()                                     # w = d mean_tb(loss_model) / d L
    L = Lg.detach()
    EL = 4 * U * (ws[0] * l_kl + ws[1] * l_img + ws[2] * l_rew + ws[3] * l_term).view(TB, I)

    def Elae(v, Ev):
        # logavgexp is 1-Lipschitz in the max norm; the shift -v - max, expf (2 ulp), the sum of I terms, logf, - log I
        if I == 1:
            return Ev[..., 0]
        spread = (v - v.amin(-1, keepdim=True)).amax(-1)
        return Ev.amax(-1) + U * (2 * v.abs().amax(-1) + 2 * spread + I + 8 + math.log(I))

    bound("loss_model", tb[:, 0], lm.detach(), Elae(L, EL) + U * lm.detach().abs())
    if I == 1:
        bound("w", w, Lg.grad.reshape(-1), U * Lg.grad.abs().reshape(-1))
    else:
        # w = expf(-L - lse) / TB: the argument carries E_L, the error of lse (that of the loss) and one rounding; expf
        # 2 ulp, the division one more
        lse = (-L).logsumexp(-1, keepdim=True)
        Ew = Lg.grad * (EL + Elae(L, EL)[:, None] + U * (L + lse).abs() + 4 * U) + TINY     # far weights underflow
        bound("w", w, Lg.grad.reshape(-1), Ew.reshape(-1))
    z = torch.zeros(TB, I, dtype=f64, device=DEV)
    for j, v in ((1, l_img), (2, l_rew), (3, l_term), (4, kl_exact)):
        r = nlae(v.view(TB, I), I)
        bound(f"tb[{j}]", tb[:, j], r, Elae(v.view(TB, I), z) + U * r.abs())
    for j, v in ((5, ent_prior), (6, ent_post)):
        r = v.view(TB, I).mean(-1)
        bound(f"tb[{j}]", tb[:, j], r, (I + 1) * U * r.abs())
    assert (tb[:, 7] == 0).all()


@gpu
@pytest.mark.parametrize("N", [1, 8, 32])
@pytest.mark.parametrize("M", [1, 31, 33, 5000])
def test_colmean_against_float64(ops, M, N):
    x = fp32(Gen(M + N).normal(M, N) + 2.0)
    B = Bufs()
    out = B.out("out", (N,))
    ops.colmean(f32(x), out)
    B.check()
    # 32 threads per column add every 32nd row, thread 0 adds the 32 partials, then / M
    depth = -(-M // 32) + 32 + 2
    bound("colmean", out, x.mean(0), depth * U * x.abs().mean(0))


# ----------------------------------------------------------------------------------------------------- actor-critic
GAE_H = [1, 2, 15, 127]
GAE_MD = [1, 127, 128, 129, 2500]
GAE_GL = [(0.99, 0.0), (0.99, 0.95), (0.99, 1.0), (1.0, 0.0), (1.0, 0.95), (1.0, 1.0)]


def gae_ref(H, Md, gam, lam, vt, v, rew, term):
    """a2c.py:81-114 restated in float64 on the kernel's fp32 inputs and its own fp32 terminal probabilities, with a
    running error bound of each fp32 step; dv = d loss_critic / d value0 by autograd."""
    gam, lam = float(fp32(torch.tensor(gam))), float(fp32(torch.tensor(lam)))
    vt, v, rew, term = (t.view(H + 1, Md) for t in (vt, v, rew, term))
    t1 = term[1:]
    a = -vt[:-1] + rew[1:] + gam * (1.0 - t1) * vt[1:]
    Ea = 4 * U * (vt[:-1].abs() + rew[1:].abs() + (gam * (1.0 - t1) * vt[1:]).abs()) + U * (1.0 - t1) * vt[1:].abs()
    ag, Eag = [None] * H, [None] * H
    for j in reversed(range(H)):
        if j == H - 1:
            ag[j], Eag[j] = a[j], Ea[j]
        else:
            c = lam * gam * (1.0 - t1[j])
            ag[j] = a[j] + c * ag[j + 1]
            Eag[j] = Ea[j] + c * Eag[j + 1] + 4 * U * (a[j].abs() + (c * ag[j + 1]).abs())
    ag, Eag = torch.stack(ag), torch.stack(Eag)
    tgt = ag + vt[:-1]
    Etgt = Eag + U * (ag.abs() + vt[:-1].abs())
    # reality weight: exp(cumsum(log(1 - terminal0))); a terminal probability of exactly 1 gives log 0 = -inf, weight 0
    om = 1.0 - term[:-1]
    lg = torch.log(om)
    cs = lg.cumsum(0)
    wgt = cs.exp()
    # 1 - t rounds only below t = 1/2 (U (1 - t)); logf 1 ulp of |log|; each cumsum step U |cs|; expf 2 ulp + U |cs|
    fin = torch.where(torch.isfinite(lg), lg, torch.zeros_like(lg))
    rel = (3 * U * fin.abs() + 2 * U).cumsum(0) + U * torch.where(torch.isfinite(cs), cs, torch.zeros_like(cs)).abs().cumsum(0)
    Ew = wgt * (rel + U * cs.abs().nan_to_num(0, 0, 0) + 2 * U)
    val = v[:-1].clone().requires_grad_(True)
    loss = (0.5 * (tgt - val) ** 2 * wgt).mean()
    loss.backward()
    d = tgt - v[:-1]
    Edv = ((Etgt + U * d.abs()) * wgt + d.abs() * Ew + 4 * U * (d * wgt).abs()) / (H * Md)
    sums = torch.stack([(0.5 * d * d * wgt).sum(), v[0].sum(), v[:-1].sum(), rew[1:].sum(), (rew[1:] ** 2).sum()])
    Esums = torch.stack([(d.abs() * (Etgt + U * d.abs()) * wgt + 0.5 * d * d * Ew + 4 * U * 0.5 * d * d * wgt).sum(),
                         *(torch.zeros((), dtype=f64, device=d.device) for _ in range(4))])
    return dict(adv=(a, Ea), agae=(ag, Eag), target=(tgt, Etgt), weight=(wgt, Ew), dv=(val.grad, Edv)), sums, Esums


@gpu
@pytest.mark.parametrize("gam,lam", GAE_GL)
@pytest.mark.parametrize("Md", GAE_MD)
@pytest.mark.parametrize("H", GAE_H)
def test_gae_critic_against_float64(ops, H, Md, gam, lam):
    J = H + 1
    g = Gen(H * 1000 + Md)
    vt, v, rew = fp32(g.normal(J, Md)), fp32(g.normal(J, Md)), fp32(g.normal(J, Md))
    tl = fp32(g.normal(J, Md) - 2.0)
    # terminal logits +40 (fp32 sigmoid exactly 1: the reality weight goes through log 0) and -40 (sigmoid ~4e-18)
    sel = g.rand(J, Md)
    tl = torch.where(sel < 0.02, torch.full_like(tl, 40.0), torch.where(sel > 0.97, torch.full_like(tl, -40.0), tl))
    B = Bufs()
    term = B.out("term", (J * Md,))
    outs = {n: B.out(n, (H * Md,)) for n in ("adv", "agae", "target", "weight", "dv")}
    pre = torch.tensor([1.5, -2.0, 3.0, 4.0, -5.0, 6.0, 7.0, 8.0], dtype=f64, device=DEV)
    sums = pre.clone()
    ops.gae_critic(H, Md, gam, lam, f32(vt), f32(v), f32(rew), f32(tl), term, *outs.values(), sums)
    B.check()
    tr = torch.sigmoid(tl)
    bound("term", term.view(J, Md), tr, 4 * U * tr + TINY)
    if not CPU:
        assert (term.view(J, Md)[tl == 40.0] == 1.0).all(), "fp32 sigmoid(40) is not exactly 1"
    ref, s_ref, Es = gae_ref(H, Md, gam, lam, vt, v, rew, term.double())
    for n, (r, e) in ref.items():
        bound(n, outs[n].view(H, Md), r, e)
    if (tl[:H] == 40.0).any():
        assert (outs["weight"].view(H, Md)[(tl[:H] == 40.0).int().cumsum(0) > 0] == 0).all(), \
            "a certain terminal does not zero the reality weight of its step and all later ones"
    # the double sums: float64 additions of fp32 values (1e-12 of sum |terms| covers any order) into non-zero values
    mag = torch.stack([s_ref[0].abs(), v.abs().sum(), v.abs().sum(), rew.abs().sum(), (rew ** 2).sum()]) + 1
    if CPU:
        mag = mag * (H * Md * U * 1e12)   # the float32 twin sums in fp32, the kernel in double
    bound("sums", sums[:5], pre[:5] + s_ref, Es + 1e-12 * mag + 1e-12 * pre[:5].abs())
    assert torch.equal(sums[5:], pre[5:]), "sums past the fifth written"


@gpu
def test_gae_critic_refuses_horizon_128(ops):
    Md = 4
    z = torch.zeros(129 * Md, device=DEV)
    keep = torch.full((129 * Md,), NAN, device=DEV)
    sums = torch.zeros(5, dtype=f64, device=DEV)
    refused(ops, lambda: ops.gae_critic(128, Md, 0.99, 0.95, z, z, z, z, keep, keep, keep, keep, keep, keep, sums), -1)
    assert torch.isnan(keep).all() and (sums == 0).all()


ACT_A = [1, 2, 18, 32]
ACT_ROWS = [1, 7, 9, 24000]


@gpu
@pytest.mark.parametrize("eta", [0.0, 1e-3, 1.0])
@pytest.mark.parametrize("rows", ACT_ROWS)
@pytest.mark.parametrize("A", ACT_A)
def test_actor_loss_onehot_against_float64_autograd(ops, A, rows, eta):
    g = Gen(A * 31 + rows)
    l = fp32(g.normal(rows, A, scale=3.0))
    acts = F.one_hot(torch.randint(0, A, (rows,), generator=g.g), A).to(f64).to(DEV)
    ag, w = fp32(g.normal(rows)), fp32(g.rand(rows))
    B = Bufs()
    dl = B.out("dlogits", (rows, A), gap=3)                   # columns past A must stay untouched
    pre = torch.tensor([0.5, -1.5], dtype=f64, device=DEV)
    sums = pre.clone()
    ops.actor_loss_onehot(eta, gapped(l, 5), f32(acts), f32(ag), f32(w), dl, sums)
    B.check()
    # autograd of ((-log pi(a) * agae - eta * H) * w).mean() (a2c.py:119-130)
    lg = l.clone().requires_grad_(True)
    pi = D.OneHotCategorical(logits=lg)
    ent = pi.entropy()
    per = (-pi.log_prob(acts) * ag - fp32(torch.tensor(eta, dtype=f64)) * ent) * w
    per.mean().backward()
    lp, p, Elp, Ep = (v[:, 0] for v in softmax_err(l, 1, A))
    eta32 = float(fp32(torch.tensor(eta, dtype=f64)))
    Eent = (Ep * lp.abs() + p * Elp).sum(-1) + 7 * U * (p * lp.abs()).sum(-1)
    en = ent.detach()
    c = (w / rows)[:, None]
    E = c * (ag.abs()[:, None] * (Ep + U * (acts + p)) + eta32 * (Ep * (lp + en[:, None]).abs() + p * (Elp + Eent[:, None]))
             + 4 * U * (ag.abs()[:, None] * (acts + p) + eta32 * p * (lp.abs() + en.abs()[:, None]))) + 2 * U * lg.grad.abs()
    bound("dlogits", dl, lg.grad, E)
    lpa = (lp * acts).sum(-1)
    Erow = w * (ag.abs() * Elp[:, 0] + eta32 * Eent + 3 * U * ((lpa * ag).abs() + eta32 * en.abs()))
    bound("sums[0]", sums[0], pre[0] + per.detach().sum(), Erow.sum() + 1e-12 * (per.detach().abs().sum() + 1))
    bound("sums[1]", sums[1], pre[1] + en.sum(), Eent.sum() + 1e-12 * (en.abs().sum() + 1))


TN_A = [1, 6, 12]
TN_ROWS = [1, 45, 333]                    # not multiples of 32: the warp shuffle of the sums runs over inactive rows


def tn_inputs(rows, A, seed):
    g = Gen(seed)
    # mean logits +-50 (tanh(m/5) saturates); std logits up to 100, half of them normal: softplus on both sides of its
    # threshold 20
    out = torch.cat([fp32(g.uniform(rows, A, bound=50.0)), fp32(g.uniform(rows, A) * 55 + 45)], 1)
    out[:, A:] = torch.where(g.rand(rows, A) < 0.5, fp32(g.normal(rows, A, scale=3.0)), out[:, A:])
    return out


def tn_mu_sd(out, A):
    th = torch.tanh(out[:, :A] / 5)
    return th, 5 * th, F.softplus(out[:, A:]) + 0.1


@gpu
@pytest.mark.parametrize("rows", TN_ROWS)
@pytest.mark.parametrize("A", TN_A)
def test_tanh_normal_sample_against_float64(ops, A, rows):
    out = tn_inputs(rows, A, seed=A + rows)
    eps = fp32(Gen(rows).normal(rows, A))
    B = Bufs()
    act = B.out("action", (rows, A), gap=2)
    ops.tanh_normal_sample(gapped(out, 3), f32(eps), act)
    B.check()
    th, mu, sd = tn_mu_sd(out, A)
    a = torch.tanh(mu + sd * eps)
    # mu = 5 tanhf(m/5): 2 ulp of tanh, the / 5 and * 5; sd: log1pf(expf) 3 ulp (exact above the threshold 20), + 0.1;
    # the argument two roundings; tanh' = 1 - a^2, tanhf 2 ulp
    Emu = 5 * (3 * U * th.abs() + (1 - th * th) * U * (out[:, :A] / 5).abs()) + U * mu.abs()
    Esd = 4 * U * sd
    arg = mu + sd * eps
    bound("action", act, a, (1 - a * a) * (Emu + eps.abs() * Esd + 2 * U * ((sd * eps).abs() + arg.abs())) + 3 * U * a.abs())


@gpu
@pytest.mark.parametrize("rows", TN_ROWS)
@pytest.mark.parametrize("A", TN_A)
def test_actor_loss_tanh_normal_against_float64_autograd(ops, A, rows):
    out = tn_inputs(rows, A, seed=A * 3 + rows)
    g = Gen(A + rows * 7)
    th, mu, sd = tn_mu_sd(out, A)
    a = fp32(torch.tanh(mu + sd * g.normal(rows, A)))
    a[0, 0] = 1.0                                   # |a| == 1: the kernel clamps to 1 - 2^-23
    if A > 1:
        a[0, 1] = -1.0
    ag, w = fp32(g.normal(rows)), fp32(g.rand(rows))
    eta = 1e-3
    B = Bufs()
    dout = B.out("dout", (rows, 2 * A), gap=3)
    pre = torch.tensor([0.25, 2.0], dtype=f64, device=DEV)
    sums = pre.clone()
    ops.actor_loss_tanh_normal(eta, gapped(out, 1), gapped(a, 2), f32(ag), f32(w), dout, sums)
    B.check()
    # autograd of ((-log pi(a) * agae - eta * H) * w).mean() with pi = TransformedDistribution(Independent(Normal), Tanh)
    # and H the Normal's entropy (functions.py:69-78).  The kernel clamps actions to +-(1 - 2^-23); torch 2.11's
    # TanhTransform does not clamp (atanh(+-1) is infinite), so the reference is given the clamped action: for |a| < 1
    # that is the fp32 action itself except a = +-(1 - 2^-24), and at |a| = 1 it is the clamped float64 formula.
    ac = a.clamp(-1 + 2.0 ** -23, 1 - 2.0 ** -23)
    og = out.clone().requires_grad_(True)
    mg, sg = og[:, :A], og[:, A:]
    normal = D.Independent(D.Normal(5 * torch.tanh(mg / 5), F.softplus(sg) + 0.1), 1)
    pi = D.TransformedDistribution(normal, [D.TanhTransform()])
    eta32 = float(fp32(torch.tensor(eta, dtype=f64)))
    per = (-pi.log_prob(ac) * ag - eta32 * normal.entropy()) * w
    per.mean().backward()
    # error of zc = (atanh(a) - mu) / sd: atanhf 3 ulp of x, mu and sd as in the sample test, two roundings
    x = torch.atanh(ac)
    zc = (x - mu) / sd
    Emu = 5 * (3 * U * th.abs() + (1 - th * th) * U * (out[:, :A] / 5).abs()) + U * mu.abs()
    Esd = 4 * U * sd
    Ezc = (3 * U * x.abs() + Emu + U * (x - mu).abs()) / sd + zc.abs() * (Esd / sd + U)
    c = (w / rows)[:, None]
    # d/dmean_ = c (-ag zc / sd)(1 - th^2): 1 - th^2 carries 2|th| E_th + U absolute (th -> 1 at |m| = 50)
    E_m = c * ag.abs()[:, None] * ((Ezc / sd + zc.abs() * Esd / sd ** 2) * (1 - th * th)
                                   + zc.abs() / sd * (5 * U + 2 * U * (out[:, :A] / 5).abs()) + 4 * U * (zc / sd).abs() * (1 - th * th))
    sig = torch.sigmoid(out[:, A:])
    E_s = c * sig * (ag.abs()[:, None] * ((2 * zc.abs() * Ezc + (zc * zc + 1) * Esd / sd) / sd + 4 * U * (zc * zc + 1) / sd)
                     + eta32 * (Esd / sd ** 2 + 2 * U / sd)) + 4 * U * og.grad[:, A:].abs()
    gr = og.grad
    bound("dout mean", dout[:, :A], gr[:, :A], E_m + 2 * U * gr[:, :A].abs())
    bound("dout std", dout[:, A:], gr[:, A:], E_s)
    # per-row log-prob: |dlp/dzc| = |zc| carries Ezc, log sd carries Esd / sd, the log-det (|d/dx| <= 4) 4 E_x, a few
    # roundings of each term, and the A-term sum A roundings of the running sum
    lpn = -0.5 * zc * zc - sd.log() - 0.5 * math.log(2 * math.pi)
    ladj = 2 * (math.log(2) - x - F.softplus(-2 * x))
    lp_terms = ((zc.abs() * Ezc + Esd / sd + 6 * U * (0.5 * zc * zc + sd.log().abs() + 1 + x.abs()) + 12 * U * x.abs()).sum(-1)
                + A * U * (lpn.abs() + ladj.abs()).sum(-1))
    ent = normal.entropy().detach()
    Eent = (Esd / sd + 3 * U * (sd.log().abs() + 1.5)).sum(-1) + A * U * ent.abs()
    Erow = w * (ag.abs() * lp_terms + eta32 * Eent) + 3 * U * per.detach().abs()
    bound("sums[0]", sums[0], pre[0] + per.detach().sum(), Erow.sum() + 1e-12 * (per.detach().abs().sum() + 1))
    bound("sums[1]", sums[1], pre[1] + ent.sum(), Eent.sum() + 1e-12 * (ent.abs().sum() + 1))


# ----------------------------------------------------------------------------------------------------- optimizer
SUMSQ_N = [1, 255, 257, 4 * P * 256, 4 * P * 256 + 1, 50_000_000]


@gpu
@pytest.mark.parametrize("n", SUMSQ_N)
def test_sumsq_against_float64(ops, n):
    x = fp32(Gen(n % 1000).normal(n))
    out = torch.full((1,), 3.25, device=DEV)
    ops.sumsq(f32(x), out)
    sync()
    # partial kernel: a thread adds every (grid*256)th element, then a 256-thread block sum (10 levels); the final
    # kernel adds the <= 4 #SMs partials the same way; the square, the add into the pre-filled value
    grid = min(-(-n // 256), 32 * P, 4 * P)
    depth = -(-n // (grid * 256)) + 10 + -(-grid // 256) + 10 + 2
    ref = (x * x).sum()
    bound("sumsq", out.double()[0], 3.25 + ref, depth * U * ref + U * (3.25 + ref))


@gpu
@pytest.mark.parametrize("case", ["above", "equal", "below", "zero", "above_no_norm_out"])
def test_clip_scale_against_clip_grad_norm(ops, case):
    n = 100_003
    x = fp32(Gen(5).normal(n))
    if case == "zero":
        x = torch.zeros_like(x)
    ss = fp32((x * x).sum())                          # the kernel's input: the fp32 sum of squares
    norm = float(ss.sqrt())
    max_norm = {"above": norm / 3, "equal": norm, "below": norm * 2, "zero": 1.0, "above_no_norm_out": norm / 7}[case]
    max_norm = float(fp32(torch.tensor(max_norm, dtype=f64)))
    xb = f32(x)
    nout = torch.full((1,), NAN, device=DEV) if case != "above_no_norm_out" else None
    ops.clip_scale(xb, f32(ss.reshape(1)), max_norm, nout)
    sync()
    pg = torch.nn.Parameter(torch.zeros(n, dtype=f64, device=DEV))
    pg.grad = x.clone()
    tn = torch.nn.utils.clip_grad_norm_([pg], max_norm)
    # norm = sqrtf(fp32 sum of squares): half the input's rounding + one; coef = max_norm / (norm + 1e-6): three roundings
    # and the norm's relative error; x * coef one more
    E_norm = 1.5 * U * float(tn)
    coef = max_norm / (float(tn) + 1e-6)
    E_coef = coef * (3 * U + E_norm / (float(tn) + 1e-6))
    if nout is not None:
        bound("norm", nout.double()[0], tn, E_norm)
    if coef - E_coef >= 1:
        # below max_norm the coefficient clamps to 1: the gradient must come back bit-unchanged
        assert torch.equal(xb.view(torch.int32), f32(x).view(torch.int32)), "an unclipped gradient was changed"
    else:
        # |min(1, a) - min(1, b)| <= |a - b|: the bound holds on both sides of the clamp ("equal" sits on it)
        bound("clipped", xb, pg.grad, x.abs() * E_coef + U * pg.grad.abs())
    if case == "equal":
        assert abs(coef - 1) < 1e-6


ADAM_STEPS = [1, 2, 10, 1000, 1_000_000]


def adam_ref(p, g, m, v, step, lr, b1, b2, eps, wd):
    """torch.optim.AdamW(foreach=False) in float64, one step from state (m, v) at step - 1."""
    pt = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([pt], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    if step > 1:
        opt.state[pt] = dict(step=torch.tensor(float(step - 1), dtype=f64), exp_avg=m.clone(), exp_avg_sq=v.clone())
    pt.grad = g.clone()
    opt.step()
    st = opt.state[pt]
    return pt.detach(), st["exp_avg"], st["exp_avg_sq"]


@gpu
@pytest.mark.parametrize("step", ADAM_STEPS)
def test_adamw_against_torch_adamw_float64(ops, step):
    n = 70_001
    g_ = Gen(step % 997)
    p, g = fp32(g_.normal(n)), fp32(g_.normal(n, scale=0.5))
    g[::7] = 0.0                                          # zero gradients: only decay and the moments' own decay act
    m = fp32(g_.normal(n, scale=0.1)) if step > 1 else torch.zeros(n, dtype=f64, device=DEV)
    v = fp32(g_.rand(n) * 0.01) if step > 1 else torch.zeros(n, dtype=f64, device=DEV)
    # lr 0.1 and wd 0.5 make the order of decay and update visible (they differ by lr * wd * update = 5% of it)
    hp = dict(lr=0.1, b1=0.9, b2=0.999, eps=1e-5, wd=0.5)
    h32 = {k: float(fp32(torch.tensor(v_, dtype=f64))) for k, v_ in hp.items()}
    pk, mk, vk = f32(p), f32(m), f32(v)
    ctr = torch.full((1,), step - 1, dtype=torch.int32, device=DEV)
    ops.inc(ctr)                                          # the device step counter the kernel reads
    ops.adamw(pk, f32(g), mk, vk, h32["lr"], h32["b1"], h32["b2"], h32["eps"], h32["wd"], ctr)
    sync()
    assert int(ctr) == step
    # The kernel receives beta1 / beta2 as fp32 and forms the bias corrections in double: the reference gets the same fp32
    # values.  With the decimal betas in double instead, the float64 reference moves p by up to 3.0e-5 (step 2), 1.6e-5
    # (10), 5.3e-5 (1000), 2.2e-5 (1e6) and 4e-16 (step 1, where m and v start at 0) on these inputs (measured), mostly
    # through 1 - beta1 = 0.10000002 vs 0.1: far above the kernel's error bound below (~1e-7).
    pr, mr, vr = adam_ref(p, g, m, v, step, h32["lr"], h32["b1"], h32["b2"], h32["eps"], h32["wd"])
    b1, b2, lr, wd, eps = h32["b1"], h32["b2"], h32["lr"], h32["wd"], h32["eps"]
    Em = 3 * U * (m.abs() + (g - m).abs() * (1 - b1))
    Ev = 4 * U * vr                                       # v' = v b2 + (1 - b2) g^2: non-negative terms
    bc1, bc2s = 1 - b1 ** step, math.sqrt(1 - b2 ** step)
    sq = vr.sqrt() / bc2s
    den = sq + eps
    Eden = sq * (3 * U + U) + U * den                     # sqrt of v' (half of 4U) + 1, / bc2s (fp32-rounded) + 1, + eps
    upd = (lr / bc1) * mr / den
    Eupd = (lr / bc1) * Em / den + upd.abs() * (Eden / den + 4 * U)
    Ep = 3 * U * (p * (1 - lr * wd)).abs() + Eupd + U * pr.abs()      # lr * wd, 1 - it, p * it: three roundings
    bound("m", mk, mr, Em)
    bound("v", vk, vr, Ev)
    bound("p", pk, pr, Ep)


@gpu
def test_scale_by_unit_factor_leaves_memory_untouched_and_scales_otherwise(ops):
    n = 10_007
    x = torch.full((n,), NAN, device=DEV)
    before = x.clone()
    one = torch.ones(1, device=DEV)
    ops.scale_by(x, one, 1.0)
    ops.scale_by(x, None, 1.0)
    ops.scale_by(x, torch.full((1,), 0.5, device=DEV), 2.0)
    sync()
    assert torch.equal(x.view(torch.int32), before.view(torch.int32)), "a factor of exactly 1 touched the buffer"
    v = fp32(Gen(2).normal(n))
    xb = f32(v)
    ops.scale_by(xb, torch.full((1,), 0.3, device=DEV), 3.0)
    sync()
    ref = v * 3.0 * float(fp32(torch.tensor(0.3, dtype=f64)))
    bound("scaled", xb, ref, 2 * U * ref.abs())              # alpha * scale rounds once, x * f once


# ----------------------------------------------------------------------------------------------------- small ops
COLSUM_CASES = [(M, N) for N in (1, 31, 33) for M in (1, 63, 64, 65, 1_000_000)] + \
               [(M, 1000) for M in (1, 63, 64, 65, 100_000)]      # N = 1000: the grid.y cap (33 blocks) from M = 2112


def colsum_depth(M, N):
    gy = min(-(-M // 64), max(P * 8 // (-(-N // 32)), 1))
    return -(-M // (gy * 8)) + 8 + gy + 1


@gpu
@pytest.mark.parametrize("M,N", COLSUM_CASES)
def test_colsum_accumulates_against_float64(ops, M, N):
    x = fp32(Gen(M % 1000 + N).normal(M, N))
    pre = fp32(Gen(N).normal(N))
    B = Bufs()
    out = B.out("out", (N,), init=pre)
    ops.colsum(gapped(x, 3), out)
    B.check()
    ref = x.sum(0)
    bound("colsum", out, pre + ref, colsum_depth(M, N) * U * x.abs().sum(0) + U * (pre + ref).abs())


@gpu
@pytest.mark.parametrize("with_db", [True, False])
@pytest.mark.parametrize("act", [0, 1])
def test_bias_act_bwd_against_float64_autograd(ops, round_out, act, with_db):
    M, N = 1001, 45
    g = Gen(act)
    pre_act = fp32(g.normal(M, N))
    y = fp32(F.elu(pre_act))
    dy = fp32(g.normal(M, N))
    db0 = fp32(g.normal(N))
    B = Bufs()
    d = B.out("dy", (M, N), gap=5, init=f32(dy))          # in place
    db = B.out("db", (N,), init=db0)
    ops.bias_act_bwd(d, y.float() if act else None, act, db if with_db else None)
    B.check()
    xg = pre_act.clone().requires_grad_(True)
    (F.elu(xg) if act else xg).backward(dy)
    ref = xg.grad
    # elu' from the fp32 output: U|y| + one rounding of y + 1, one of the product
    E = dy.abs() * U * (y.abs() + 1) + U * ref.abs() if act else torch.zeros_like(ref)
    stats = {}
    if act:
        check("dy", d, ref, E, round_out, stats)
    else:
        assert torch.equal(d.double(), dy), "act NONE changed dy"
    if with_db:
        # the bias gradient sums the unrounded products
        bound("db", db, db0 + ref.sum(0), E.sum(0) + colsum_depth(M, N) * U * ref.abs().sum(0) + U * (db0 + ref.sum(0)).abs())
    else:
        assert torch.equal(db.double(), db0)


SMALL_MN = [(1, 1), (45, 37), (1001, 67)]


@gpu
@pytest.mark.parametrize("M,N", SMALL_MN)
def test_group_sum_against_float64(ops, round_out, M, N):
    I = 3
    x = fp32(Gen(M).normal(M * I, N))
    B = Bufs()
    out = B.out("out", (M, N), gap=2)
    ops.group_sum(gapped(x, 4), I, out)
    B.check()
    ref = x.view(M, I, N).sum(1)
    check("group_sum", out, ref, I * U * x.view(M, I, N).abs().sum(1), round_out, {})


@gpu
@pytest.mark.parametrize("M,N", SMALL_MN)
def test_rowscale_against_float64(ops, round_out, M, N):
    div, alpha = 3, 0.7
    g = Gen(M + 1)
    x, sc = fp32(g.normal(M, N)), fp32(g.rand(-(-M // div)) * 4)
    buf = torch.full((M, N + 3), NAN_GUARD, device=DEV)       # in place on a strided view: the gap must stay
    buf[:, :N] = x
    xb = buf[:, :N]
    ops.rowscale(xb, f32(sc), div, alpha)
    sync()
    a32 = float(fp32(torch.tensor(alpha, dtype=f64)))
    ref = x * (a32 * sc.repeat_interleave(div)[:M])[:, None]
    check("rowscale", xb, ref, 2 * U * ref.abs(), round_out, {})
    assert (buf[:, N:] == NAN_GUARD).all(), "rowscale wrote a gap column"


@gpu
@pytest.mark.parametrize("M,N", SMALL_MN)
def test_mask_rows_against_float64(ops, round_out, M, N):
    g = Gen(M + 2)
    x, mask = fp32(g.normal(M, N)), fp32(g.rand(M))
    mask[::3] = 0.0
    B = Bufs()
    out = B.out("out", (M, N), gap=1)
    ops.mask_rows(gapped(x, 2), f32(mask), out)
    B.check()
    ref = x * mask[:, None]
    check("mask_rows", out, ref, U * ref.abs(), round_out, {})


@gpu
@pytest.mark.parametrize("M,N", [(1, 4), (37, 8), (1001, 68)])
def test_gather_rows_exact(ops, M, N):
    g = Gen(N)
    W = fp32(g.normal(23, N))
    idx = torch.randint(0, 23, (M,), generator=g.g).to(torch.int32).to(DEV)
    Wb = torch.full((23, N + 4), NAN, device=DEV)
    Wb[:, :N] = W
    B = Bufs()
    out = B.out("out", (M, N), gap=4)
    ops.gather_rows(idx, Wb[:, :N], out)
    B.check()
    assert torch.equal(out.double(), W[idx.long()])


@gpu
@pytest.mark.parametrize("T,Bt,I", [(1, 1, 1), (5, 7, 3), (17, 33, 4)])
def test_reset_mask_exact(ops, T, Bt, I):
    reset = (Gen(T).rand(T, Bt) > 0.6)
    B = Bufs()
    mask = B.out("mask", (T, Bt * I))
    ops.reset_mask(reset, I, mask)
    B.check()
    assert torch.equal(mask.view(T, Bt, I), (~reset).float()[:, :, None].expand(T, Bt, I))


@gpu
@pytest.mark.parametrize("M,N", SMALL_MN + [(33, 1000)])
def test_to_half_and_transpose_to_half_exact(ops, M, N):
    x = fp32(Gen(M * N).normal(M, N, scale=100.0))
    x.view(-1)[0] = 70000.0                     # above the fp16 range: inf
    B = Bufs()
    h = B.out("h", (M, N), dtype=torch.float16, gap=3)
    ht = B.out("ht", (N, M), dtype=torch.float16, gap=5)
    ops.to_half(gapped(x, 2), h)
    ops.transpose_to_half(gapped(x, 7), ht)
    B.check()
    want = x.float().half()
    assert torch.equal(h.view(torch.int16), want.view(torch.int16)), "to_half != round-to-nearest-even fp16"
    assert torch.equal(ht.view(torch.int16), want.t().contiguous().view(torch.int16)), "transpose_to_half != fp16(x^T)"


# ----------------------------------------------------------------------------------------------------- the KL balance map
def test_kl_balance_argument_gives_the_reference_loss_gradient():
    """dreamer.py:241 of the reference turns kl_balance 0.5 into None and then uses the plain KL whenever
    `not self.kl_balance`, which also holds for 0.  The balance passed to pd_kl must give the gradient of that loss for
    every kl_balance.  Runs on the CPU with the float64 twin of pd_kl."""
    from pydreamer_b200.dreamer import kl_balance_arg

    G, C, M = 3, 5, 4
    g = torch.Generator().manual_seed(0)
    post, prior = torch.randn(M, G * C, generator=g, dtype=f64), torch.randn(M, G * C, generator=g, dtype=f64)
    for kb in (0.0, 0.5, 0.8, 1.0):
        lp, lq = (v.view(M, G, C).clone().requires_grad_(True) for v in (post, prior))
        dp, dq = D.OneHotCategorical(logits=lp), D.OneHotCategorical(logits=lq)
        bal = None if kb == 0.5 else kb                  # the reference's own mapping and branch
        if not bal:
            loss = D.kl_divergence(dp, dq)
        else:
            loss = ((1 - bal) * D.kl_divergence(dp, D.OneHotCategorical(logits=lq.detach()))
                    + bal * D.kl_divergence(D.OneHotCategorical(logits=lp.detach()), dq))
        loss.sum().backward()
        o = [torch.empty(M, dtype=f64) for _ in range(4)] + [torch.empty(M, G * C, dtype=f64) for _ in range(2)]
        RefOps("cpu").kl(post, prior, None, 0, kl_balance_arg(kb), G, C, *o)
        assert torch.allclose(o[4], lp.grad.reshape(M, -1), rtol=0, atol=1e-12), kb
        assert torch.allclose(o[5], lq.grad.reshape(M, -1), rtol=0, atol=1e-12), kb


# ----------------------------------------------------------------------------------------------------- closed forms
def test_closed_forms_match_autograd():
    """Each closed form the bounds above are built on, against torch.autograd of the float64 reference expression, to
    1e-10 of the gradient's magnitude.  Runs on the CPU: it checks the test's own algebra, not a kernel."""
    g = torch.Generator().manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=f64)
    tol = lambda ref: 1e-10 * ref.abs().max().item() + 1e-300

    # LayerNorm + ELU backward
    M, N = 5, 37
    x, gam, bet, dy = rn(M, N) * 2 + 1, 1 + 0.3 * rn(N), 0.3 * rn(N), rn(M, N)
    xg = x.clone().requires_grad_(True)
    y = F.elu(F.layer_norm(xg, (N,), gam, bet, LN_EPS))
    y.backward(dy)
    var, mu = torch.var_mean(x, -1, unbiased=False)
    c = cf_ln_elu_bwd(dy, x, y.detach(), gam, mu, 1 / torch.sqrt(var + LN_EPS))
    assert torch.allclose(c["dx"], xg.grad, rtol=0, atol=tol(xg.grad))

    # GRU gate backward
    D_ = 6
    gi, gh, hp, dh = rn(M, 3 * D_), rn(M, 3 * D_), rn(M, D_), rn(M, D_)
    gig, ghg, hpg = (v.clone().requires_grad_(True) for v in (gi, gh, hp))
    r, u, n, ghn, h = gru_fwd64(gig, ghg, hpg)
    (h * dh).sum().backward()
    c = cf_gru_bwd(dh, r.detach(), u.detach(), n.detach(), ghn.detach(), hp)
    for k, ref in (("dgi", gig.grad), ("dgh", ghg.grad), ("carry", hpg.grad)):
        assert torch.allclose(c[k], ref, rtol=0, atol=tol(ref)), k

    # straight-through categorical backward
    G, C = 3, 7
    l, dz = rn(M, G * C) * 2, rn(M, G * C)
    lg = l.clone().requires_grad_(True)
    (dz * D.OneHotCategoricalStraightThrough(logits=lg.view(M, G, C)).rsample().reshape(M, -1)).sum().backward()
    p = torch.softmax(l.view(M, G, C), -1)
    assert torch.allclose(cf_cat_st_bwd(p, dz.view(M, G, C)).reshape(M, -1), lg.grad, rtol=0, atol=tol(lg.grad))

    # KL gradients, balanced
    post, prior = rn(M, G * C), rn(M, G * C)
    _, _, _, _, gpo, gpr = kl_ref(post, prior, G, C, 0, 0.8, None)
    lp, lq = torch.log_softmax(post.view(M, G, C), -1), torch.log_softmax(prior.view(M, G, C), -1)
    a, b = cf_kl(lp, lq, lp.exp(), lq.exp(), 0.2, 0.8)
    assert torch.allclose(a.reshape(M, -1), gpo, rtol=0, atol=tol(gpo))
    assert torch.allclose(b.reshape(M, -1), gpr, rtol=0, atol=tol(gpr))

    # one-hot actor
    rows, A, eta = 9, 5, 0.3
    l = rn(rows, A)
    acts = F.one_hot(torch.randint(0, A, (rows,), generator=g), A).to(f64)
    ag, w = rn(rows), torch.rand(rows, generator=g, dtype=f64)
    lg = l.clone().requires_grad_(True)
    pi = D.OneHotCategorical(logits=lg)
    ((-pi.log_prob(acts) * ag - eta * pi.entropy()) * w).mean().backward()
    lp = torch.log_softmax(l, -1)
    ref = cf_actor_onehot(lp, lp.exp(), acts, ag, w, eta, rows)
    assert torch.allclose(ref, lg.grad, rtol=0, atol=tol(lg.grad))

    # tanh-normal actor
    out = rn(rows, 2 * A) * 3
    a = torch.tanh(rn(rows, A))
    og = out.clone().requires_grad_(True)
    normal = D.Independent(D.Normal(5 * torch.tanh(og[:, :A] / 5), F.softplus(og[:, A:]) + 0.1), 1)
    pi = D.TransformedDistribution(normal, [D.TanhTransform()])
    ((-pi.log_prob(a) * ag - eta * normal.entropy()) * w).mean().backward()
    dm, ds = cf_tanh_normal(out[:, :A], out[:, A:], a, ag, w, eta, rows)
    assert torch.allclose(torch.cat([dm, ds], 1), og.grad, rtol=0, atol=tol(og.grad))

    # critic gradient of the restated a2c.py loss
    H, Md = 4, 3
    vt, v, rew, term = rn(H + 1, Md), rn(H + 1, Md), rn(H + 1, Md), torch.sigmoid(rn(H + 1, Md))
    ref, _, _ = gae_ref(H, Md, 0.99, 0.95, vt, v, rew, term)
    tgt, wgt = ref["target"][0], ref["weight"][0]
    dv = -(tgt - v[:-1]) * wgt / (H * Md)
    assert torch.allclose(dv, ref["dv"][0], rtol=0, atol=tol(dv))

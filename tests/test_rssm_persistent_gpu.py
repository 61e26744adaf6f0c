"""Kernel-level tests of the two persistent RSSM kernels: pd_rssm_unroll_fwd (csrc/pd_rssm_fwd3.cu, the posterior unroll)
and pd_rssm_unroll_bwd (csrc/pd_rssm_bptt.cu, its back-propagation through time), called directly through NativeOps on
seeded inputs and compared with a float64 restatement of rssm.py:21-78,125-153 STEP BY STEP.

Teacher forcing: every step of the reference takes its operands from what the kernel itself saved (the sampled indices of
the previous step, x1, za, h', y2, pin, post; in the backward dpost, dy2, dgi of the same step and dx1, dgh of step t+1).
An error therefore never compounds over T, and each comparison checks ONE contraction or pointwise stage, with fp16-exact
weights and (forward) fp16-exact activations.  Tolerances, each next to its check:
  * contraction outputs: elementwise 1e-5 of sum_k |a_k| |b_k| (the |A|.|B|^T scale of that element) + 1e-6: the products
    are exact in fp32 and only the fp32 accumulation over K <= 16 * #SMs rounds; in the backward, with unrounded gradient
    operands (round_out = 0), plus 2^-10 of the same scale: mma.sync truncates an fp32 operand to tf32;
  * values the kernel rounds (fp16 za, h', pin; tf32 gradients with round_out = 1): equal to the rounded reference except
    where the reference lies within the propagated fp32 error of a rounding boundary, and never more than one ulp off;
  * LayerNorm statistics: 1e-5 relative;
  * sampled classes: exactly argmax(p / q) of the float64 softmax of the kernel's own logits, except near-ties (top two
    p / q within 1e-5 relative, counted and printed).
Every output is pre-filled with NaN (indices with -1) and followed by a sentinel guard band: an element the kernel does
not write, or a write past the last row, fails the test.

PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/ref_ops.py in place of the kernels: a dry run of the
references and tolerances without a GPU."""
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from tests.util import CPU, DEV, Gen, bound, f64, fp16, fp32, ops, rounded, ulp  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
EPS = 1e-3                                      # LayerNorm eps of the RSSM (rssm.py: nn.LayerNorm(eps=1e-3))
# The kernels own one CTA per SM; their limits are functions of that count.  Without a device the dry run uses the count
# Dreamer._persistent_*_ok assume on the reference path.
P = torch.cuda.get_device_properties(0).multi_processor_count if (not CPU and torch.cuda.is_available()) else 148
NAN_GUARD = -12345.0                            # sentinel of the guard band after each float output
IDX_GUARD = -777


# ----------------------------------------------------------------------------------------------------- helpers
def guarded(shape, dtype, fill, dev=DEV):
    """A tensor of `shape` pre-filled with `fill`, followed in memory by a sentinel guard band of at least two rows."""
    n = math.prod(shape)
    flat = torch.empty(n + max(256, 2 * shape[-1]), dtype=dtype, device=dev)
    flat[:n] = fill
    flat[n:] = IDX_GUARD if dtype == torch.int32 else NAN_GUARD
    return flat, flat[:n].view(shape)


def nan_tail(v, rows):
    """fp32 copy of the input rows v followed in memory by `rows` rows of NaN: a read past its last row poisons the result."""
    flat = torch.full((v.shape[0] + rows, v.shape[1]), float("nan"), device=v.device)
    flat[:v.shape[0]] = v
    return flat[:v.shape[0]]


def check_guards(bufs):
    for name, (flat, view) in bufs.items():
        g = flat[view.numel():]
        sentinel = IDX_GUARD if flat.dtype == torch.int32 else NAN_GUARD
        assert (g == sentinel).all(), f"{name}: written past its last row"


def contraction_tol(scale, trunc=False):
    # fp32 accumulation of exact products: 1e-5 of sum |a||b| (+1e-6 absolute); an fp32 operand that mma.sync truncates to
    # tf32 (10 mantissa bits) adds up to 2^-10 of the same scale
    return (1e-5 + (2.0 ** -10 if trunc else 0.0)) * scale + 1e-6


def group_softmax(post, G, C):
    return torch.softmax(post.reshape(post.shape[0], G, C), -1)


def dreamer_gate(kind, BI, D, Hd, G, C, ops):
    """Dreamer._persistent_rssm_ok / _persistent_bptt_ok on a stand-in holding just the state they read: whether the
    module would hand this shape to the persistent kernel."""
    from pydreamer_b200.dreamer import Dreamer

    me = SimpleNamespace(d=SimpleNamespace(D=D, Hd=Hd, G=G, C=C), _arena=torch.empty(0, device=DEV), ops=ops,
                         persistent_rssm=True, persistent_bptt=True, fp16_forward=True, _k1_wzT=torch.empty(0),
                         _k1b_w={"w": None})
    fn = Dreamer._persistent_rssm_ok if kind == "fwd" else Dreamer._persistent_bptt_ok
    return fn(me, BI)


def elu_grad_from_out(y):
    return torch.where(y > 0, torch.ones_like(y), y + 1)


def ln_stats(x):
    mu = x.mean(-1)
    r = 1.0 / torch.sqrt(x.var(-1, unbiased=False) + EPS)
    return mu, r


# ----------------------------------------------------------------------------------------------------- inputs
def make_params(D, Hd, G, C, wscale=1.0, seed=0, dev=DEV):
    """fp16-exact weights (uniform +-wscale/sqrt(fan_in), nn.Linear's init times wscale), fp32 biases and LayerNorm affine
    near their init values; all float64 on `dev`."""
    g = Gen(seed, dev="cpu")
    Z = G * C

    def lin(o, i):
        return fp16(g.uniform(o, i, bound=wscale / math.sqrt(i)))

    p = dict(Wz=lin(Hd, Z), Wih=lin(3 * D, Hd), Whh=lin(3 * D, D), Wph=lin(Hd, D), Wpm=lin(Z, Hd),
             b_z=fp32(g.uniform(Hd, bound=1 / math.sqrt(Z))), b_ih=fp32(g.uniform(3 * D, bound=1 / math.sqrt(Hd))),
             b_hh=fp32(g.uniform(3 * D, bound=1 / math.sqrt(D))), b_ph=fp32(g.uniform(Hd, bound=1 / math.sqrt(D))),
             b_pm=fp32(g.uniform(Z, bound=1 / math.sqrt(Hd))),
             ln1_g=fp32(1 + g.normal(Hd, scale=0.1)), ln1_b=fp32(g.normal(Hd, scale=0.1)),
             ln2_g=fp32(1 + g.normal(Hd, scale=0.1)), ln2_b=fp32(g.normal(Hd, scale=0.1)))
    return {k: v.to(dev) for k, v in p.items()}


def make_step_inputs(T, BI, I, D, Hd, G, C, open_loop=False, seed=1, dev=DEV):
    """aa / ea (normal), reset mask (~20% resets, every row reset at step 1), Exp(1) noise, masked h_0 (fp16-exact) and a
    masked one-hot z_0; float64 on `dev`."""
    g = Gen(seed, dev="cpu")
    B, Z = BI // I, G * C
    mask = (torch.rand(T, BI, generator=g.g) > 0.2).to(f64)
    if T > 1:
        mask[1] = 0.0
    noise = torch.empty(T, BI, Z, dtype=torch.float32).exponential_(generator=g.g).double()
    k0 = torch.randint(0, C, (BI, G), generator=g.g)
    x = dict(aa=fp32(g.normal(T * B, Hd)), ea=None if open_loop else fp32(g.normal(T * B, Hd)), mask=mask, noise=noise,
             h0=fp16(g.normal(BI, D, scale=0.5)) * mask[0, :, None],
             z0=F.one_hot(k0, C).reshape(BI, Z).to(f64) * mask[0, :, None])
    return {k: (v.to(dev) if v is not None else None) for k, v in x.items()}


def rep(v, t, B, I):
    """rows of the step-t slice of a [T*B, .] projection, repeated over the I IWAE samples of each sequence"""
    return v[t * B:(t + 1) * B].repeat_interleave(I, 0)


# ----------------------------------------------------------------------------------------------------- forward
def snapshot(bufs, keep):
    """For a call expected to be refused: the output buffers and a bitwise copy of them as they were before the call."""
    if keep is not None:
        keep["bufs"] = bufs
        keep["before"] = {n: flat.clone() for n, (flat, _) in bufs.items()}


def untouched(keep):
    for n, (flat, _) in keep["bufs"].items():
        a, b = flat.view(torch.int32), keep["before"][n].view(torch.int32)       # bitwise: NaN == NaN
        assert torch.equal(a, b), f"{n} was written by a refused call"


def run_fwd(ops, T, BI, I, D, Hd, G, C, prm, x, keep=None):
    Z, F_, B = G * C, D + G * C, BI // I
    f32 = lambda v: v.float().contiguous()
    x1_0 = fp32(x["z0"] @ prm["Wz"].t() + prm["b_z"] + rep(x["aa"], 0, B, I))
    bufs = {}

    def out(name, shape, dtype=torch.float32, fill=float("nan")):
        bufs[name] = guarded(shape, dtype, fill)
        return bufs[name][1]

    o = dict(x1=out("x1", (T, BI, Hd)), za=out("za", (T, BI, Hd)), m1=out("m1", (T, BI)), r1=out("r1", (T, BI)),
             gates=out("gates", (T, BI, 4 * D)), feat=out("feat", (T, BI, F_)), hin=out("hin", (T, BI, D)),
             zin=out("zin", (T, BI, Z)), y2=out("y2", (T, BI, Hd)), pin=out("pin", (T, BI, Hd)), m2=out("m2", (T, BI)),
             r2=out("r2", (T, BI)), post=out("post", (T, BI, Z)), idx=out("idx", (T, BI, G), torch.int32, -1))
    # caller-prepared step-0 inputs (pd_b200.h): masked h_0 / z_0 and the pre-norm input of step 0
    o["hin"][0] = f32(x["h0"]); o["zin"][0] = f32(x["z0"]); o["x1"][0] = f32(x1_0)
    w16 = {k: prm[k].to(torch.float16).contiguous() for k in ("Wz", "Wih", "Whh", "Wph", "Wpm")}
    wzT16 = torch.empty(Z, Hd, dtype=torch.float16, device=DEV)
    ops.transpose_to_half(f32(prm["Wz"]), wzT16)
    h16 = torch.float16
    snapshot(bufs, keep)
    ops.rssm_unroll_fwd(
        dict(T=T, BI=BI, I=I, D=D, Hd=Hd, G=G, C=C), EPS,
        w_z16=w16["Wz"], w_ih16=w16["Wih"], w_hh16=w16["Whh"], w_ph16=w16["Wph"], w_pm16=w16["Wpm"],
        **{k: f32(prm[k]) for k in ("b_z", "ln1_g", "ln1_b", "b_ih", "b_hh", "b_ph", "ln2_g", "ln2_b", "b_pm")},
        aa=nan_tail(x["aa"], BI), ea=None if x["ea"] is None else nan_tail(x["ea"], BI), mask=f32(x["mask"]),
        noise=f32(x["noise"]), **o,
        ws_wzT16=wzT16, ws_za16=torch.empty(BI, Hd, dtype=h16, device=DEV), ws_h16=torch.empty(BI, D, dtype=h16, device=DEV),
        ws_pin16=torch.empty(BI, Hd, dtype=h16, device=DEV), ws_barrier=torch.zeros(16, dtype=torch.int32, device=DEV),
        ws_ghpart=torch.empty(4, BI, 3 * D, device=DEV), ws_y2part=torch.empty(4, BI, Hd, device=DEV))
    if not CPU:
        torch.cuda.synchronize()
    check_guards(bufs)
    # the step-0 inputs are read, never written
    assert torch.equal(o["hin"][0].double(), x["h0"]) and torch.equal(o["zin"][0].double(), x["z0"])
    assert torch.equal(o["x1"][0].double(), x1_0)
    return o


def ln_elu_ref(x, g, b):
    """float64 LayerNorm + ELU of the kernel's fp32 rows, and the fp32 error of computing it: the mean / variance sums
    (<= 1024 terms) and the normalisation are each a few fp32 roundings of |x - mean| * rstd and of rstd * max|x|;
    1e-5 of those is > 100x that."""
    mu, r = ln_stats(x)
    xh = (x - mu[:, None]) * r[:, None]
    y = F.elu(xh * g + b)
    err = 1e-5 * (g.abs() * (xh.abs() + (r * x.abs().amax(-1))[:, None]) + b.abs()) + 1e-7
    return y, mu, r, err


def check_stats(name, got_m, got_r, x, mu, r):
    # mean: 1e-5 of the row's magnitude (a mean can cancel to ~0, so not relative to itself); rstd: 1e-5 relative
    bound(name + ".mean", got_m, mu, 1e-5 * x.abs().amax(-1) + 1e-7)
    bound(name + ".rstd", got_r, r, 1e-5 * r)


def check_fwd(o, prm, x, T, BI, I, D, Hd, G, C):
    Z, B = G * C, BI // I
    k = {n: v.double() for n, v in o.items() if n != "idx"}
    idx = o["idx"].long()
    W = {n: prm[n] for n in ("Wz", "Wih", "Whh", "Wph", "Wpm")}
    Wa = {n: v.abs() for n, v in W.items()}
    stats, ties = {}, 0
    assert ((idx >= 0) & (idx < C)).all(), "sampled class out of range"
    for t in range(T):
        m = x["mask"][t][:, None] if t > 0 else torch.ones(BI, 1, dtype=f64, device=DEV)   # h_0 / z_0 arrive masked
        aa = rep(x["aa"], t, B, I)
        if t > 0:
            # phase A: x1 = m * (one_hot(idx_{t-1}) . W_z^T) + b_z + aa (a gather-sum of G fp16 weights)
            z = F.one_hot(idx[t - 1], C).reshape(BI, Z).to(f64)
            ref = m * (z @ W["Wz"].t()) + prm["b_z"] + aa
            bound(f"x1[{t}]", k["x1"][t], ref, contraction_tol(m * (z @ Wa["Wz"].t()) + prm["b_z"].abs() + aa.abs()))
            assert torch.equal(k["zin"][t], z * m), f"zin[{t}] != one_hot(idx[{t - 1}]) * mask[{t}]"
        za, mu, r, err = ln_elu_ref(k["x1"][t], prm["ln1_g"], prm["ln1_b"])
        rounded(f"za[{t}]", k["za"][t], za, err, "fp16", stats)
        check_stats(f"ln1[{t}]", k["m1"][t], k["r1"][t], k["x1"][t], mu, r)

        # phase B: gates from the kernel's za_t, unmasked h'_{t-1} (fp16) and masked h_{t-1}
        hprev = k["feat"][t - 1][:, :D] if t > 0 else fp16(k["hin"][0])
        hp = k["hin"][t]
        gi = k["za"][t] @ W["Wih"].t() + prm["b_ih"]
        gi_s = k["za"][t].abs() @ Wa["Wih"].t() + prm["b_ih"].abs()
        gh = m * (hprev @ W["Whh"].t()) + prm["b_hh"]
        gh_s = m * (hprev.abs() @ Wa["Whh"].t()) + prm["b_hh"].abs()
        s = lambda v, j: v[:, j * D:(j + 1) * D]
        rg, ug = torch.sigmoid(s(gi, 0) + s(gh, 0)), torch.sigmoid(s(gi, 1) + s(gh, 1))
        ghn = s(gh, 2)
        ng = torch.tanh(s(gi, 2) + rg * ghn)
        # sigmoid' <= 1/4, tanh' <= 1; +1e-6 for the fp32 expf / tanhf themselves
        e_r = 0.25 * contraction_tol(s(gi_s, 0) + s(gh_s, 0)) + 1e-6
        e_u = 0.25 * contraction_tol(s(gi_s, 1) + s(gh_s, 1)) + 1e-6
        e_ghn = contraction_tol(s(gh_s, 2))
        e_n = contraction_tol(s(gi_s, 2)) + ghn.abs() * e_r + (rg + e_r) * e_ghn + 1e-6
        gt = k["gates"][t].view(BI, 4, D)
        bound(f"gate r[{t}]", gt[:, 0], rg, e_r)
        bound(f"gate u[{t}]", gt[:, 1], ug, e_u)
        bound(f"gate n[{t}]", gt[:, 2], ng, e_n)
        bound(f"gh_n[{t}]", gt[:, 3], ghn, e_ghn)
        h = (1 - ug) * ng + ug * hp
        e_h = (ng - hp).abs() * e_u + (1 - ug + e_u) * e_n + 1e-6 * (ng.abs() + hp.abs())
        rounded(f"h[{t}]", k["feat"][t][:, :D], h, e_h, "fp16", stats)
        hn = k["feat"][t][:, :D]
        if t + 1 < T:
            assert torch.equal(k["hin"][t + 1], hn * x["mask"][t + 1][:, None]), f"hin[{t + 1}] != h'_{t} * mask[{t + 1}]"

        # phases C / C': y2 = h' . W_ph^T + b_ph (+ ea)
        ea = rep(x["ea"], t, B, I) if x["ea"] is not None else torch.zeros_like(aa)
        ref = hn @ W["Wph"].t() + prm["b_ph"] + ea
        bound(f"y2[{t}]", k["y2"][t], ref, contraction_tol(hn.abs() @ Wa["Wph"].t() + prm["b_ph"].abs() + ea.abs()))
        pin, mu, r, err = ln_elu_ref(k["y2"][t], prm["ln2_g"], prm["ln2_b"])
        rounded(f"pin[{t}]", k["pin"][t], pin, err, "fp16", stats)
        check_stats(f"ln2[{t}]", k["m2"][t], k["r2"][t], k["y2"][t], mu, r)

        # phase D: posterior logits, argmax(p / q) of the float64 softmax of the kernel's logits
        ref = k["pin"][t] @ W["Wpm"].t() + prm["b_pm"]
        bound(f"post[{t}]", k["post"][t], ref, contraction_tol(k["pin"][t].abs() @ Wa["Wpm"].t() + prm["b_pm"].abs()))
        ratio = group_softmax(k["post"][t], G, C) / x["noise"][t].reshape(BI, G, C)
        want = ratio.argmax(-1)
        top = ratio.topk(2, -1).values if C > 1 else torch.cat([ratio, torch.zeros_like(ratio)], -1)
        near = (top[..., 0] - top[..., 1]) < 1e-5 * top[..., 0]
        wrong = (idx[t] != want) & ~near
        assert not wrong.any(), f"idx[{t}]: {int(wrong.sum())} samples differ from argmax(p/q) away from a near-tie"
        ties += int(near.sum())
        assert torch.equal(k["feat"][t][:, D:], F.one_hot(idx[t], C).reshape(BI, Z).to(f64)), f"feat[{t}][:, D:] != one_hot(idx)"
    print(f"near-ties {ties}; fp16 values within error of a rounding boundary:",
          {n: sum(v for k_, v in stats.items() if k_.startswith(n)) for n in ("za", "h", "pin")})


def rssm_case(name, T, BI, I, D, Hd, G, C, wscale=1.0, open_loop=False):
    return pytest.param(T, BI, I, D, Hd, G, C, wscale, open_loop, id=name)


FWD_CASES = [
    rssm_case("tiny_golden_ks1", 4, 3, 1, 64, 40, 4, 8),
    rssm_case("T1_no_recurrence", 1, 5, 1, 256, 64, 2, 32),
    rssm_case("one_row_G1", 3, 1, 1, 256, 64, 1, 32),
    rssm_case("Hd1024_ks4_iwae", 8, 16, 4, 1024, 1024, 32, 32),
    rssm_case("BI64_largest_single_block", 6, 64, 1, 2048, 1000, 32, 32),
    rssm_case("BI65_multi_C17_ks1", 5, 65, 5, 1000, 520, 16, 17),
    rssm_case("R3_RB16_single_block", 4, 48, 1, 512, 256, 40, 32),
    rssm_case("R3_RB17_multi", 4, 49, 1, 512, 256, 40, 32),
    rssm_case("atari_iwae", 4, 200, 4, 2048, 1000, 32, 32),
    rssm_case("BI256_limit", 3, 256, 1, 512, 256, 8, 24),
    rssm_case("D16P_16_units_per_cta", 4, 50, 1, 16 * P, 1024, 32, 32),
    rssm_case("G96_over_64", 4, 50, 1, 512, 128, 96, 8),
    rssm_case("G_eq_P_R1", 4, 16, 1, 512, 128, P, 2),
    rssm_case("open_loop", 4, 50, 1, 2048, 1000, 32, 32, open_loop=True),
    rssm_case("saturated_gates_4x_weights", 4, 50, 1, 1024, 512, 32, 32, wscale=4.0),
]


@gpu
@pytest.mark.parametrize("T,BI,I,D,Hd,G,C,wscale,open_loop", FWD_CASES)
def test_persistent_fwd_matches_float64_step_reference(ops, T, BI, I, D, Hd, G, C, wscale, open_loop):
    assert dreamer_gate("fwd", BI, D, Hd, G, C, ops), "Dreamer would not hand this accepted shape to the kernel"
    prm = make_params(D, Hd, G, C, wscale=wscale, seed=T + BI + D + G)
    x = make_step_inputs(T, BI, I, D, Hd, G, C, open_loop=open_loop, seed=Hd + C)
    o = run_fwd(ops, T, BI, I, D, Hd, G, C, prm, x)
    check_fwd(o, prm, x, T, BI, I, D, Hd, G, C)
    if wscale > 1:          # the case exists for the saturated regime: make sure it reaches the tails (~0% at 1x weights)
        gt = o["gates"].double().view(T, BI, 4, D)
        assert ((gt[:, :, 1] < 0.05) | (gt[:, :, 1] > 0.95)).double().mean() > 0.1
        assert (gt[:, :, 2].abs() > 0.95).double().mean() > 0.25


# ----------------------------------------------------------------------------------------------------- backward
def unroll64(prm, x, T, BI, I, D, Hd, G, C, idx=None):
    """Float64 posterior unroll without fp16 rounding (rssm.py:125-153 restated), differentiable: the saved tensors of
    the backward and, with requires_grad leaves, the graph autograd differentiates.  idx: classes to use instead of
    sampling (straight-through: z = one_hot + p - p.detach())."""
    B, Z = BI // I, G * C
    mask = x["mask"]
    S = {n: [] for n in ("x1", "za", "m1", "r1", "gates", "hin", "y2", "pin", "m2", "r2", "post", "feat", "gi", "gh", "idx")}

    def ln_elu(v, g, b):
        mu, r = ln_stats(v)
        return F.elu((v - mu[:, None]) * r[:, None] * g + b), mu, r

    h_prev, z_prev = x["h0"], x["z0"]
    for t in range(T):
        m = mask[t][:, None] if t > 0 else 1.0
        x1 = m * (z_prev @ prm["Wz"].t()) + prm["b_z"] + rep(x["aa"], t, B, I)
        hin = h_prev * m
        za, m1, r1 = ln_elu(x1, prm["ln1_g"], prm["ln1_b"])
        gi = za @ prm["Wih"].t() + prm["b_ih"]
        gh = hin @ prm["Whh"].t() + prm["b_hh"]
        rg = torch.sigmoid(gi[:, :D] + gh[:, :D])
        ug = torch.sigmoid(gi[:, D:2 * D] + gh[:, D:2 * D])
        ng = torch.tanh(gi[:, 2 * D:] + rg * gh[:, 2 * D:])
        h = (1 - ug) * ng + ug * hin
        y2 = h @ prm["Wph"].t() + prm["b_ph"] + (rep(x["ea"], t, B, I) if x["ea"] is not None else 0.0)
        pin, m2, r2 = ln_elu(y2, prm["ln2_g"], prm["ln2_b"])
        post = pin @ prm["Wpm"].t() + prm["b_pm"]
        p = group_softmax(post, G, C)
        k = idx[t] if idx is not None else (p / x["noise"][t].reshape(BI, G, C)).argmax(-1)
        z = (F.one_hot(k, C).to(f64) + p - p.detach()).reshape(BI, Z)
        for n, v in (("x1", x1), ("za", za), ("m1", m1), ("r1", r1), ("hin", hin), ("y2", y2), ("pin", pin), ("m2", m2),
                     ("r2", r2), ("post", post), ("feat", torch.cat([h, z], 1)), ("gi", gi), ("gh", gh), ("idx", k),
                     ("gates", torch.stack([rg, ug, ng, gh[:, 2 * D:]], 1).reshape(BI, 4 * D))):
            S[n].append(v)
        h_prev, z_prev = h, z
    return S


def make_seeds(T, BI, D, Z, seed=3, dev=DEV):
    g = Gen(seed, dev="cpu")
    return {k: v.to(dev) for k, v in dict(dfeat=fp32(g.normal(T, BI, D + Z, scale=0.1)),
                                          dpost_u=fp32(g.normal(T, BI, Z, scale=0.1)),
                                          w=fp32(0.5 + 0.5 * torch.rand(T, BI, generator=g.g, dtype=f64))).items()}


def ln_bwd_ref(dy, e_dy, x, y, gamma, mean, rstd):
    """LayerNorm+ELU backward (the formulas of ln_elu_bwd_row_kernel) in float64 and its error bound: e_dy (the error of
    the contraction dy) carried through d = rstd (dxh - mean(dxh) - xh mean(dxh xh)), plus 1e-5 of each fp32 term."""
    eg = elu_grad_from_out(y)
    g = dy * eg
    xh = (x - mean[:, None]) * rstd[:, None]
    dxh = g * gamma
    c1, c2 = dxh.mean(-1, keepdim=True), (dxh * xh).mean(-1, keepdim=True)
    d = rstd[:, None] * (dxh - c1 - xh * c2)
    E = e_dy * eg * gamma.abs()
    xr = rstd[:, None] * x.abs().amax(-1, keepdim=True)          # fp32 error of xh = (x - mean) * rstd is ~u * xr
    e_d = rstd[:, None] * (E + E.mean(-1, keepdim=True) + xh.abs() * (E * xh.abs()).mean(-1, keepdim=True)
                           + 1e-5 * (dxh.abs() + c1.abs() + (xh.abs() + xr) * c2.abs()))
    return d, e_d, g, xh, dict(g=(g * xh, e_dy * eg * xh.abs() + 1e-5 * g.abs() * (xh.abs() + xr)), b=(g, e_dy * eg), x=(d, e_d))


def bptt_ref(S, prm, seeds, mask, T, BI, D, Hd, G, C, kl_weight, teacher=None, trunc=False):
    """Float64 BPTT (the per-step formulas of pd_b200.h / the chain cat_st_bwd, ln_elu_bwd, gru_bwd), step by step.
    teacher: the kernel's own dpost, dy2, dgi (step t) and dgh, dx1 (step t+1) as contraction operands, so each output
    checks one stage; None: the reference's own values (a plain float64 BPTT).  Only the dh * u carry is recursed in
    float64.  Returns the outputs, their error bounds and the six LayerNorm / bias gradient sums with theirs."""
    Z = G * C
    W = {n: prm[n] for n in ("Wz", "Wih", "Whh", "Wph", "Wpm")}
    Wa = {n: v.abs() for n, v in W.items()}
    names = ("dpost", "dy2", "dgi", "dgh", "dx1")
    out = {n: [None] * T for n in names}
    err = {n: [None] * T for n in names}
    sums = {n: [0.0, 0.0, 0.0] for n in ("ln2_g", "ln2_b", "b_ph", "ln1_g", "ln1_b", "b_z")}   # value, bound, sum |terms|
    src = teacher if teacher is not None else out
    tol = lambda sc: contraction_tol(sc, trunc)
    dh_next = e_dh_next = None
    for t in reversed(range(T)):
        nxt = t + 1 < T
        mn = mask[t + 1][:, None] if nxt else None
        # dz = dfeat_z + mask_{t+1} (dx1_{t+1} . W_z); dpost = softmax'(post) dz + kl_weight w dpost_u
        dz, e_dz = seeds["dfeat"][t][:, D:].clone(), torch.zeros_like(seeds["dpost_u"][t])
        if nxt:
            dz = dz + mn * (src["dx1"][t + 1] @ W["Wz"])
            e_dz = mn * tol(src["dx1"][t + 1].abs() @ Wa["Wz"])
        p = group_softmax(S["post"][t], G, C)
        dzg, e_g = dz.view(BI, G, C), e_dz.view(BI, G, C)
        sdz = (p * dzg).sum(-1, keepdim=True)
        kl = kl_weight * seeds["w"][t][:, None] * seeds["dpost_u"][t]
        out["dpost"][t] = (p * (dzg - sdz)).reshape(BI, Z) + kl
        # |p (e - sum p e)| <= p (e + max e); 1e-5 of each fp32 term (softmax, products, the group sum)
        err["dpost"][t] = ((p * (e_g + e_g.amax(-1, keepdim=True)) + 1e-5 * p * (dzg.abs() + (p * dzg.abs()).sum(-1, keepdim=True)))
                           .reshape(BI, Z) + 1e-5 * kl.abs())
        # dy2 = LN+ELU backward (post_norm) of dpin = dpost . W_pm
        dpin = src["dpost"][t] @ W["Wpm"]
        d, e_d, _, _, gs2 = ln_bwd_ref(dpin, tol(src["dpost"][t].abs() @ Wa["Wpm"]), S["y2"][t], S["pin"][t], prm["ln2_g"],
                                       S["m2"][t], S["r2"][t])
        out["dy2"][t], err["dy2"][t] = d, e_d
        # dh = dy2 . W_ph + dfeat_h + mask_{t+1} (dgh_{t+1} . W_hh + dh_{t+1} u_{t+1}); GRU gate backward
        dh = src["dy2"][t] @ W["Wph"] + seeds["dfeat"][t][:, :D]
        e_dh = tol(src["dy2"][t].abs() @ Wa["Wph"]) + 1e-6 * dh.abs()
        if nxt:
            u1 = S["gates"][t + 1].view(BI, 4, D)[:, 1]
            dh = dh + mn * (src["dgh"][t + 1] @ W["Whh"] + dh_next * u1)
            e_dh = e_dh + mn * (tol(src["dgh"][t + 1].abs() @ Wa["Whh"]) + u1 * e_dh_next)
        gt = S["gates"][t].view(BI, 4, D)
        rg, ug, ng, ghn = gt[:, 0], gt[:, 1], gt[:, 2], gt[:, 3]
        hp = S["hin"][t]
        dn = dh * (1 - ug) * (1 - ng * ng)
        du = dh * (hp - ng) * ug * (1 - ug)
        dr = dn * ghn * rg * (1 - rg)
        e_dn = e_dh * (1 - ug) * (1 - ng * ng) + 1e-6 * dn.abs()
        e_du = e_dh * (hp - ng).abs() * ug * (1 - ug) + 1e-6 * du.abs()
        e_dr = e_dn * (ghn * rg * (1 - rg)).abs() + 1e-6 * dr.abs()
        out["dgi"][t], err["dgi"][t] = torch.cat([dr, du, dn], 1), torch.cat([e_dr, e_du, e_dn], 1)
        out["dgh"][t], err["dgh"][t] = torch.cat([dr, du, dn * rg], 1), torch.cat([e_dr, e_du, e_dn * rg + 1e-6 * (dn * rg).abs()], 1)
        dh_next, e_dh_next = dh, e_dh
        # dx1 = LN+ELU backward (in_norm) of dza = dgi . W_ih
        dza = src["dgi"][t] @ W["Wih"]
        d, e_d, _, _, gs1 = ln_bwd_ref(dza, tol(src["dgi"][t].abs() @ Wa["Wih"]), S["x1"][t], S["za"][t], prm["ln1_g"],
                                       S["m1"][t], S["r1"][t])
        out["dx1"][t], err["dx1"][t] = d, e_d
        for key, gs in (("ln2_g", gs2["g"]), ("ln2_b", gs2["b"]), ("b_ph", gs2["x"]),
                        ("ln1_g", gs1["g"]), ("ln1_b", gs1["b"]), ("b_z", gs1["x"])):
            v, e = gs
            sums[key][0] = sums[key][0] + v.sum(0)
            sums[key][1] = sums[key][1] + e.sum(0)
            sums[key][2] = sums[key][2] + v.abs().sum(0)
    return {n: torch.stack(v) for n, v in out.items()}, {n: torch.stack(v) for n, v in err.items()}, sums


def saved_fwd(T, BI, D, Hd, G, C, seed, dev=DEV):
    prm = make_params(D, Hd, G, C, seed=seed, dev=dev)
    x = make_step_inputs(T, BI, 1, D, Hd, G, C, seed=seed + 1, dev=dev)
    with torch.no_grad():
        S = unroll64(prm, x, T, BI, 1, D, Hd, G, C)
    S = {n: torch.stack(v) for n, v in S.items()}
    # what the kernel reads is fp32
    S = {n: (v if n == "idx" else fp32(v)) for n, v in S.items()}
    return prm, x, S


def run_bwd(ops, T, BI, D, Hd, G, C, prm, x, S, seeds, kl_weight, round_out, gpre, keep=None):
    Z = G * C
    f32 = lambda v: v.float().contiguous()
    bufs = {}

    def out(name, shape, fill=float("nan")):
        bufs[name] = guarded(shape, torch.float32, fill)
        return bufs[name][1]

    o = dict(dpost=out("dpost", (T, BI, Z)), dy2=out("dy2", (T, BI, Hd)), dgi=out("dgi", (T, BI, 3 * D)),
             dgh=out("dgh", (T, BI, 3 * D)), dx1=out("dx1", (T, BI, Hd)))
    g = {}
    for n in gpre:
        g[n] = out("g_" + n, (Hd,))
        g[n].copy_(gpre[n])
    wT = {}
    for name, w in (("w_pmT16", "Wpm"), ("w_phT16", "Wph"), ("w_hhT16", "Whh"), ("w_ihT16", "Wih"), ("w_zT16", "Wz")):
        wT[name] = torch.empty(prm[w].shape[1], prm[w].shape[0], dtype=torch.float16, device=DEV)
        ops.transpose_to_half(f32(prm[w]), wT[name])
    snapshot(bufs, keep)
    ops.rssm_unroll_bwd(
        dict(T=T, BI=BI, D=D, Hd=Hd, G=G, C=C), kl_weight, round_out, **wT,
        ln2_g=f32(prm["ln2_g"]), ln1_g=f32(prm["ln1_g"]),
        **{n: f32(S[n]) for n in ("post", "pin", "y2", "m2", "r2", "x1", "za", "m1", "r1", "gates", "hin")},
        mask=f32(x["mask"]), dfeat=f32(seeds["dfeat"]), dpost_u=f32(seeds["dpost_u"]), w=f32(seeds["w"]), **o,
        **{"g_" + n: g[n] for n in g},
        ws_part2=torch.empty(4, BI, Hd, device=DEV), ws_part6=torch.empty(4, BI, D, device=DEV),
        ws_part7=torch.empty(4, BI, Hd, device=DEV), ws_barrier=torch.zeros(16, dtype=torch.int32, device=DEV))
    if not CPU:
        torch.cuda.synchronize()
    check_guards(bufs)
    return o, g


def bwd_case(name, T, BI, D, Hd, G, C):
    return pytest.param(T, BI, D, Hd, G, C, id=name)


BWD_CASES = [
    bwd_case("tiny_golden", 4, 3, 64, 40, 4, 8),
    bwd_case("BI1", 3, 1, 256, 64, 2, 32),
    bwd_case("BI64_G32_RB16", 3, 64, 512, 256, 32, 32),
    bwd_case("atari", 3, 50, 2048, 1000, 32, 32),
    bwd_case("dmc_ks6_4", 3, 50, 1024, 1000, 32, 32),
    bwd_case("D1000_ks6_1", 3, 50, 1000, 512, 32, 32),
    bwd_case("Z32_ks2_1", 3, 20, 512, 512, 1, 32),
    bwd_case("Hd1024", 3, 16, 1024, 1024, 32, 32),
    bwd_case("G_eq_P_BI16", 3, 16, 512, 128, P, 2),
    bwd_case("T1", 1, 5, 256, 64, 2, 32),
]
LN_GRADS = ("ln2_g", "ln2_b", "b_ph", "ln1_g", "ln1_b", "b_z")


@gpu
@pytest.mark.parametrize("round_out", [0, 1], ids=lambda v: f"round_out{v}")
@pytest.mark.parametrize("T,BI,D,Hd,G,C", BWD_CASES)
def test_persistent_bptt_matches_float64_step_reference(ops, T, BI, D, Hd, G, C, round_out):
    assert dreamer_gate("bwd", BI, D, Hd, G, C, ops), "Dreamer would not hand this accepted shape to the kernel"
    Z = G * C
    kl_weight = 0.8
    prm, x, S = saved_fwd(T, BI, D, Hd, G, C, seed=T + BI + D + G)
    seeds = make_seeds(T, BI, D, Z)
    gen = Gen(7, dev="cpu")
    gpre = {n: fp32(gen.normal(Hd)).to(DEV) for n in LN_GRADS}         # the gradients ACCUMULATE into these
    o, g = run_bwd(ops, T, BI, D, Hd, G, C, prm, x, S, seeds, kl_weight, bool(round_out), gpre)
    k = {n: v.double() for n, v in o.items()}
    ref, err, sums = bptt_ref(S, prm, seeds, x["mask"], T, BI, D, Hd, G, C, kl_weight, teacher=k, trunc=not round_out)
    stats = {}
    for n in ("dpost", "dy2", "dgi", "dgh", "dx1"):
        if round_out and not CPU:
            # round_out = 1: the kernel stores tf32 (rna) values; the float32 twin of the dry run does not round
            assert ((o[n].view(torch.int32) & 0x1FFF) == 0).all(), f"{n}: not tf32-rounded"
            rounded(n, k[n], ref[n], err[n], "tf32", stats)
        else:
            bound(n, k[n], ref[n], err[n] + (ulp(ref[n], -126, 10) if round_out else 0.0))
    # accumulated sums over T*BI rows: the propagated error of each term, plus fp32 summation of T*BI terms
    # ((T*BI + 8) * 2^-24 of the sum of |terms|, the recursive-summation bound) and the add into the pre-filled value
    for n in LN_GRADS:
        v, e, a = sums[n]
        bound("g_" + n, g[n].double(), gpre[n] + v, e + (T * BI + 8) * 2.0 ** -24 * a + 2.0 ** -23 * (gpre[n].abs() + a))
    print(f"tf32 values within error of a rounding boundary {sum(stats.values())}")


@gpu
@pytest.mark.parametrize("T,BI,D,Hd,G,C", [c for c in BWD_CASES if c.id in ("atari", "BI64_G32_RB16", "T1")])
def test_persistent_bptt_is_identical_run_to_run(ops, T, BI, D, Hd, G, C):
    """Two launches on identical inputs and identically pre-filled g_* give bit-identical outputs, the six accumulated
    LayerNorm / bias gradients included: the batch-row owners' partials are added in row order, not in arrival order."""
    prm, x, S = saved_fwd(T, BI, D, Hd, G, C, seed=T + BI + D + G)
    seeds = make_seeds(T, BI, D, G * C)
    gpre = {n: fp32(Gen(7, dev="cpu").normal(Hd)).to(DEV) for n in LN_GRADS}
    (o1, g1), (o2, g2) = (run_bwd(ops, T, BI, D, Hd, G, C, prm, x, S, seeds, 0.8, True, gpre) for _ in range(2))
    for n in o1:
        assert torch.equal(o1[n].view(torch.int32), o2[n].view(torch.int32)), n
    for n in LN_GRADS:
        diff = int((g1[n].view(torch.int32) != g2[n].view(torch.int32)).sum())
        assert diff == 0, f"g_{n}: {diff}/{Hd} elements differ between two identical launches"


def test_bptt_reference_matches_autograd():
    """The float64 step-by-step BPTT formulas against torch.autograd over the whole unrolled float64 forward, with the
    straight-through sample on the reference's own indices (tiny golden shape, every row reset at step 1).  Runs on the
    CPU: it checks the reference, not a kernel."""
    T, BI, I, D, Hd, G, C, kl_weight = 4, 3, 1, 64, 40, 4, 8, 0.8
    Z = G * C
    prm, x, S0 = saved_fwd(T, BI, D, Hd, G, C, seed=11, dev="cpu")
    seeds = make_seeds(T, BI, D, Z, dev="cpu")
    leaves = {n: v.clone().requires_grad_(True) for n, v in prm.items()}
    S = unroll64(dict(prm, **leaves), x, T, BI, I, D, Hd, G, C, idx=S0["idx"])
    for n in ("x1", "y2", "gi", "gh", "post"):
        for v in S[n]:
            v.retain_grad()
    loss = sum((seeds["dfeat"][t] * S["feat"][t]).sum() +
               kl_weight * (seeds["w"][t][:, None] * seeds["dpost_u"][t] * S["post"][t]).sum() for t in range(T))
    loss.backward()
    saved = {n: torch.stack([v.detach() for v in S[n]]) for n in S}
    ref, _, sums = bptt_ref(saved, prm, seeds, x["mask"], T, BI, D, Hd, G, C, kl_weight)
    for n, a in dict(dpost="post", dy2="y2", dgi="gi", dgh="gh", dx1="x1").items():
        got = torch.stack([v.grad for v in S[a]])
        assert torch.allclose(ref[n], got, rtol=0, atol=1e-10 * got.abs().max().item()), n
    for n in LN_GRADS:
        assert torch.allclose(sums[n][0], leaves[n].grad, rtol=0, atol=1e-10 * leaves[n].grad.abs().max().item()), n


# ----------------------------------------------------------------------------------------------------- refusals
# Shapes just past each host-side limit: the call must fail with PD_ERR_UNSUPPORTED before launching anything, and the
# module's gate must agree (a shape the gate accepts but the kernel refuses would send Dreamer down its warning-and-fallback
# path, which turns the persistent kernel off for the rest of the process).
def _refused(fn, keep):
    if CPU:
        pytest.skip("host-side argument checks of the native library (the float32 twin checks no limits)")
    with pytest.raises(RuntimeError, match=r"failed \(-4\)"):      # PD_ERR_UNSUPPORTED
        fn()
    torch.cuda.synchronize()
    untouched(keep)
    check_guards(keep["bufs"])


@gpu
@pytest.mark.parametrize("over", [pytest.param(dict(BI=257), id="BI257"), pytest.param(dict(Hd=1032), id="Hd1032"),
                                  pytest.param(dict(C=33), id="C33"), pytest.param(dict(D=16 * P + 8), id="D16P_plus_8")])
def test_persistent_fwd_refuses_shapes_past_its_limits_before_any_launch(ops, over):
    s = dict(T=2, BI=16, I=1, D=256, Hd=64, G=2, C=8)
    s.update(over)
    T, BI, I, D, Hd, G, C = (s[k] for k in ("T", "BI", "I", "D", "Hd", "G", "C"))
    assert not dreamer_gate("fwd", BI, D, Hd, G, C, ops), "Dreamer would try the kernel and fall back with a warning"
    prm = make_params(D, Hd, G, C)
    x = make_step_inputs(T, BI, I, D, Hd, G, C)
    keep = {}
    _refused(lambda: run_fwd(ops, T, BI, I, D, Hd, G, C, prm, x, keep=keep), keep)


@gpu
@pytest.mark.parametrize("over", [pytest.param(dict(BI=65), id="BI65"), pytest.param(dict(Hd=1032), id="Hd1032"),
                                  pytest.param(dict(C=33, G=8), id="C33"), pytest.param(dict(D=16 * P + 8), id="D16P_plus_8")])
def test_persistent_bptt_refuses_shapes_past_its_limits_before_any_launch(ops, over):
    s = dict(T=2, BI=16, D=256, Hd=64, G=2, C=8)
    s.update(over)
    T, BI, D, Hd, G, C = (s[k] for k in ("T", "BI", "D", "Hd", "G", "C"))
    assert not dreamer_gate("bwd", BI, D, Hd, G, C, ops), "Dreamer would try the kernel and fall back with a warning"
    prm, x, S = saved_fwd(T, BI, D, Hd, G, C, seed=5)
    seeds = make_seeds(T, BI, D, G * C)
    gpre = {n: torch.full((Hd,), 0.5, dtype=f64, device=DEV) for n in LN_GRADS}
    keep = {}
    _refused(lambda: run_bwd(ops, T, BI, D, Hd, G, C, prm, x, S, seeds, 0.8, True, gpre, keep=keep), keep)

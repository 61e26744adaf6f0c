"""The stacked-GRU form of the persistent posterior unroll (pd_rssm_unroll_fwd with `layers` = L) step by step against a
float64 statement (oracle/gru_ops.py run in float64), its refusals, and the GEMM route of each per-layer launch of the
per-timestep chain.

Step by step: step s of the reference starts from what the kernel left after step s - 1 (its masked h, its sampled z, its
pre-norm input x1), so a sample that flips on a near-tie cannot carry into later steps.  The kernel rounds za, h' and pin to
fp16 (its tensor-core operands), as the reference does; a value within float32 error of an fp16 rounding boundary may land
one fp16 ulp away, hence the bounds below (a few fp16 ulps of O(1) values)."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.gru_ops import GruRefOps
from tests.util import Gen, f64, fp16, fp32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 1e-3


def make_case(L, T, BI, I, D, Hd, G, C, seed=0):
    g = Gen(seed, dev="cpu")
    Dl, Z, B = D // L, G * C, BI // I
    lin = lambda o, i: fp16(g.uniform(o, i, bound=1.0 / math.sqrt(i)))
    Wih = [lin(3 * Dl, Hd if l == 0 else Dl) for l in range(L)]
    Whh_l = [lin(3 * Dl, Dl) for _ in range(L)]
    Whh = torch.zeros(3 * D, D, dtype=f64)                           # the block-diagonal matrix the host assembles
    for l in range(L):
        for gate in range(3):
            Whh[gate * D + l * Dl:gate * D + (l + 1) * Dl, l * Dl:(l + 1) * Dl] = Whh_l[l][gate * Dl:(gate + 1) * Dl]
    p = dict(Wz=lin(Hd, Z), Whh=Whh, Wph=lin(Hd, D), Wpm=lin(Z, Hd), b_z=fp32(g.uniform(Hd, bound=0.3)),
             b_ph=fp32(g.uniform(Hd, bound=0.3)), b_pm=fp32(g.uniform(Z, bound=0.3)),
             ln1_g=fp32(1 + g.normal(Hd, scale=0.1)), ln1_b=fp32(g.normal(Hd, scale=0.1)),
             ln2_g=fp32(1 + g.normal(Hd, scale=0.1)), ln2_b=fp32(g.normal(Hd, scale=0.1)))
    p["Wih"], p["b_ih"] = Wih, [fp32(g.uniform(3 * Dl, bound=0.3)) for _ in range(L)]
    p["b_hh"] = [fp32(g.uniform(3 * Dl, bound=0.3)) for _ in range(L)]
    mask = (torch.rand(T, BI, generator=g.g) > 0.2).to(f64)
    if T > 1:
        mask[1] = 0.0
    k0 = torch.randint(0, C, (BI, G), generator=g.g)
    x = dict(aa=fp32(g.normal(T * B, Hd)), ea=fp32(g.normal(T * B, Hd)), mask=mask,
             noise=torch.empty(T, BI, Z, dtype=torch.float32).exponential_(generator=g.g).double(),
             h0=fp16(g.normal(BI, D, scale=0.5)) * mask[0, :, None],
             z0=F.one_hot(k0, C).reshape(BI, Z).to(f64) * mask[0, :, None])
    return p, x


def run_kernel(ops, L, T, BI, I, D, Hd, G, C, p, x, counts=None):
    Z, B = G * C, BI // I
    f32 = lambda v: v.float().contiguous().to(DEV)
    h16 = lambda v: v.to(torch.float16).contiguous().to(DEV)
    nan = lambda *shape: torch.full(shape, float("nan"), device=DEV)
    o = dict(x1=nan(T, BI, Hd), za=nan(T, BI, Hd), m1=nan(T, BI), r1=nan(T, BI), gates=nan(T, BI, 4 * D),
             feat=nan(T, BI, D + Z), hin=nan(T, BI, D), zin=nan(T, BI, Z), y2=nan(T, BI, Hd), pin=nan(T, BI, Hd),
             m2=nan(T, BI), r2=nan(T, BI), post=nan(T, BI, Z), idx=torch.full((T, BI, G), -1, dtype=torch.int32, device=DEV))
    o["hin"][0] = f32(x["h0"]); o["zin"][0] = f32(x["z0"])
    o["x1"][0] = f32(x["z0"] @ p["Wz"].t() + p["b_z"] + x["aa"][:B].repeat_interleave(I, 0))
    wzT16 = torch.empty(Z, Hd, dtype=torch.float16, device=DEV)
    ops.transpose_to_half(f32(p["Wz"]), wzT16)
    if counts is not None:
        counts["before"] = ops.launch_count()
    ops.rssm_unroll_fwd(
        dict(T=T, BI=BI, I=I, D=D, Hd=Hd, G=G, C=C, layers=L), EPS,
        w_z16=h16(p["Wz"]), w_ih16=h16(p["Wih"][0]), w_hh16=h16(p["Whh"]), w_ph16=h16(p["Wph"]), w_pm16=h16(p["Wpm"]),
        w_ih16_l=[h16(w) for w in p["Wih"][1:4]], b_ih_l=[f32(b) for b in p["b_ih"][1:4]],
        b_hh_l=[f32(b) for b in p["b_hh"][1:4]], b_z=f32(p["b_z"]), ln1_g=f32(p["ln1_g"]), ln1_b=f32(p["ln1_b"]),
        b_ih=f32(p["b_ih"][0]), b_hh=f32(p["b_hh"][0]), b_ph=f32(p["b_ph"]), ln2_g=f32(p["ln2_g"]), ln2_b=f32(p["ln2_b"]),
        b_pm=f32(p["b_pm"]), aa=f32(x["aa"]), ea=f32(x["ea"]), mask=f32(x["mask"]), noise=f32(x["noise"]), **o,
        ws_wzT16=wzT16, ws_za16=torch.empty(BI, Hd, dtype=torch.float16, device=DEV),
        ws_h16=torch.empty(BI, D, dtype=torch.float16, device=DEV),
        ws_pin16=torch.empty(BI, Hd, dtype=torch.float16, device=DEV),
        ws_barrier=torch.zeros(16, dtype=torch.int32, device=DEV), ws_ghpart=torch.empty(4, BI, 3 * D, device=DEV),
        ws_y2part=torch.empty(4, BI, Hd, device=DEV))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def reference_step(L, s, BI, I, D, Hd, G, C, p, x, k):
    """Step s in float64 from the kernel's state k after step s - 1 (its x1[s] is checked separately)."""
    Z, B = G * C, BI // I
    r = dict(x1=k["x1"][s:s + 1].double().clone(), za=torch.zeros(1, BI, Hd, dtype=f64), m1=torch.zeros(1, BI, dtype=f64),
             r1=torch.zeros(1, BI, dtype=f64), gates=torch.zeros(1, BI, 4 * D, dtype=f64),
             feat=torch.zeros(1, BI, D + Z, dtype=f64), hin=k["hin"][s:s + 1].double().clone(),
             zin=torch.zeros(1, BI, Z, dtype=f64), y2=torch.zeros(1, BI, Hd, dtype=f64), pin=torch.zeros(1, BI, Hd, dtype=f64),
             m2=torch.zeros(1, BI, dtype=f64), r2=torch.zeros(1, BI, dtype=f64), post=torch.zeros(1, BI, Z, dtype=f64),
             idx=torch.zeros(1, BI, G, dtype=torch.int64))
    GruRefOps("cpu").rssm_unroll_fwd(
        dict(T=1, BI=BI, I=I, D=D, Hd=Hd, G=G, C=C, layers=L), EPS, w_z16=p["Wz"], w_ih16=p["Wih"][0], w_hh16=p["Whh"],
        w_ph16=p["Wph"], w_pm16=p["Wpm"], w_ih16_l=p["Wih"][1:], b_ih_l=p["b_ih"][1:], b_hh_l=p["b_hh"][1:], b_z=p["b_z"],
        ln1_g=p["ln1_g"], ln1_b=p["ln1_b"], b_ih=p["b_ih"][0], b_hh=p["b_hh"][0], b_ph=p["b_ph"], ln2_g=p["ln2_g"],
        ln2_b=p["ln2_b"], b_pm=p["b_pm"], aa=x["aa"][s * B:(s + 1) * B], ea=x["ea"][s * B:(s + 1) * B],
        mask=x["mask"][s:s + 1], noise=x["noise"][s:s + 1], **r)
    return {n: v[0] for n, v in r.items()}


def close(name, got, want, tol):
    err = (got.double() - want).abs().max().item()
    assert not torch.isnan(got).any(), f"{name}: not written"
    assert err <= tol, f"{name}: max error {err:.3g} > {tol:.3g}"


@pytest.mark.parametrize("L,BI,I,D,Hd,G,C", [
    pytest.param(2, 9, 3, 256, 64, 4, 8, id="L2_BI9"),
    pytest.param(4, 16, 1, 256, 128, 8, 16, id="L4_BI16"),
    pytest.param(2, 80, 4, 512, 96, 8, 32, id="L2_BI80_multi"),
    pytest.param(4, 130, 2, 1024, 64, 16, 8, id="L4_BI130_multi"),
])
def test_stacked_unroll_matches_float64_step_by_step(native_ops, L, BI, I, D, Hd, G, C):
    T = 4
    Dl, Z, B = D // L, G * C, BI // I
    p, x = make_case(L, T, BI, I, D, Hd, G, C)
    k = run_kernel(native_ops, L, T, BI, I, D, Hd, G, C, p, x)
    gl = k["gates"].view(L, T, BI, 4 * Dl)
    flips = 0
    for s in range(T):
        if s > 0:                                                  # phase A from the kernel's own sample of step s - 1
            m = x["mask"][s][:, None]
            zprev = k["feat"][s - 1][:, D:].double()
            close(f"zin[{s}]", k["zin"][s], zprev * m, 0.0)
            x1 = m * (zprev @ p["Wz"].t()) + p["b_z"] + x["aa"][s * B:(s + 1) * B].repeat_interleave(I, 0)
            close(f"x1[{s}]", k["x1"][s], x1, 2e-3)
            close(f"hin[{s}]", k["hin"][s], k["feat"][s - 1][:, :D].double() * m, 0.0)
        r = reference_step(L, s, BI, I, D, Hd, G, C, p, x, k)
        close(f"za[{s}]", k["za"][s], r["za"], 4e-3)
        for l in range(L):
            close(f"gates[{l},{s}]", gl[l, s], r["gates"].view(L, BI, 4 * Dl)[l], 4e-3)
        close(f"h'[{s}]", k["feat"][s][:, :D], r["feat"][:, :D], 4e-3)
        close(f"y2[{s}]", k["y2"][s], r["y2"], 2e-2)
        close(f"pin[{s}]", k["pin"][s], r["pin"], 1e-2)
        close(f"post[{s}]", k["post"][s], r["post"], 2e-2)
        same = k["idx"][s].long() == r["idx"]
        flips += int((~same).sum())
    assert flips <= max(2, T * BI * G // 200), f"{flips} sampled classes differ"


@pytest.mark.parametrize("over,what", [
    (dict(L=5, D=320), "5 layers"), (dict(L=3, D=66), "22-unit layers (not a multiple of 8)"),
    (dict(L=3, D=256), "D not divisible"), (dict(drop_layer=True), "a missing layer operand")])
def test_stacked_unroll_refuses_before_any_launch(native_ops, over, what):
    L, D = over.get("L", 2), over.get("D", 256)
    BI, I, Hd, G, C, T = 8, 1, 64, 4, 8, 2
    Dl = max(D // L, 8)
    g = Gen(1, dev="cpu")
    p = dict(Wz=fp16(g.uniform(Hd, G * C)), Whh=torch.zeros(3 * D, D, dtype=f64), Wph=fp16(g.uniform(Hd, D)),
             Wpm=fp16(g.uniform(G * C, Hd)), b_z=torch.zeros(Hd, dtype=f64), b_ph=torch.zeros(Hd, dtype=f64),
             b_pm=torch.zeros(G * C, dtype=f64), ln1_g=torch.ones(Hd, dtype=f64), ln1_b=torch.zeros(Hd, dtype=f64),
             ln2_g=torch.ones(Hd, dtype=f64), ln2_b=torch.zeros(Hd, dtype=f64))
    p["Wih"] = [fp16(g.uniform(3 * Dl, Hd if l == 0 else Dl)) for l in range(L)]
    p["b_ih"] = p["b_hh"] = [torch.zeros(3 * Dl, dtype=f64) for _ in range(L)]
    if over.get("drop_layer"):
        p["Wih"] = p["Wih"][:1]
        p["b_ih"] = p["b_hh"] = p["b_ih"][:1]
    x = dict(aa=torch.zeros(T * BI, Hd, dtype=f64), ea=torch.zeros(T * BI, Hd, dtype=f64), mask=torch.ones(T, BI, dtype=f64),
             noise=torch.ones(T, BI, G * C, dtype=f64), h0=torch.zeros(BI, D, dtype=f64),
             z0=torch.zeros(BI, G * C, dtype=f64))
    counts = {}
    with pytest.raises(RuntimeError, match=r"failed \(-4\)"):             # PD_ERR_UNSUPPORTED
        run_kernel(native_ops, L, T, BI, I, D, Hd, G, C, p, x, counts)
    assert native_ops.launch_count() == counts["before"], what          # nothing launched


def _gemm(ops, impl, A, W, C, **kw):
    ops.set_gemm_impl(impl)
    try:
        ops.gemm(A, W, C, **kw)
        torch.cuda.synchronize()
    finally:
        ops.set_gemm_impl(0)
    return C.clone()


@pytest.mark.parametrize("preset", ("atari_gru2", "tiny_gru3_odd"))
def test_per_layer_launches_take_the_expected_gemm_route(native_ops, preset):
    """The per-layer GEMMs of the chain on column slices of the state rows, told apart by their bits: the CUDA-core kernel
    (forced with set_gemm_impl(GEMM_SIMT)) computes in fp32, the tensor-core routes in tf32.  At atari_gru2 (1024-unit
    layers at 16-byte offsets) the forward products and the BPTT input gradient (M = 50, the few-row route) run on the
    tensor cores: their bits differ from the CUDA-core kernel's, and the 50-row input gradient equals the first 50 rows of
    the 65-row launch of the general kernel bit for bit.  At tiny_gru3_odd (22-unit layers, 88-byte offsets) TMA cannot
    address the slices: every launch equals the CUDA-core kernel bit for bit.  The input gradient adds into its own slice
    (C and R are the same view)."""
    from pydreamer_b200.config import make_conf
    from pydreamer_b200.ops import GEMM_SIMT
    conf = make_conf(preset)
    D, L, B = conf.deter_dim, conf.gru_layers, conf.batch_size
    Dl, F_ = D // L, D + conf.stoch_dim * conf.stoch_discrete
    g = torch.Generator(device=DEV).manual_seed(0)
    feat = torch.randn(65, F_, device=DEV, generator=g)
    hin = torch.randn(65, D, device=DEV, generator=g)
    w_ih1, w_hh1 = (torch.randn(3 * Dl, Dl, device=DEV, generator=g) / math.sqrt(Dl) for _ in range(2))
    dgi = torch.randn(65, 3 * Dl, device=DEV, generator=g)
    dhp0 = torch.randn(65, D, device=DEV, generator=g)
    tc = preset == "atari_gru2"
    for name, launch in (("W_ih product", lambda impl: _gemm(native_ops, impl, feat[:B, :Dl], w_ih1,
                                                             torch.empty(B, 3 * Dl, device=DEV))),
                         ("W_hh product", lambda impl: _gemm(native_ops, impl, hin[:B, Dl:2 * Dl], w_hh1,
                                                             torch.empty(B, 3 * Dl, device=DEV)))):
        same = torch.equal(launch(0), launch(GEMM_SIMT))
        assert same != tc, (preset, name, "tensor cores" if tc else "CUDA cores")

    def input_grad(impl, M):
        dhp = dhp0[:M].clone()
        return _gemm(native_ops, impl, dgi[:M], w_ih1, dhp[:, :Dl], b_mn=True, res=dhp[:, :Dl])

    c50 = input_grad(0, B)
    assert torch.equal(c50, input_grad(GEMM_SIMT, B)) != tc, (preset, "input gradient")
    if tc:
        assert torch.equal(c50, input_grad(0, 65)[:B]), "the few-row route computes the general kernel's bits"
    ref = dhp0[:B, :Dl].double() + dgi[:B].double() @ w_ih1.double()
    assert torch.allclose(c50.double(), ref, rtol=0, atol=2e-2 * float(ref.abs().max()))

"""Kernel-level tests of the normal_tanh actor's two entry points (pd_normal_tanh_sample, pd_actor_loss_normal_tanh in
csrc/pd_misc.cu), called through NativeOps on seeded inputs and compared with FLOAT64 references computed from the
kernels' own fp32 inputs, in the style of tests/test_rowwise_misc_f64_gpu.py.

References.  The policy of functions.py:59-66 (min_std 0.01, max_std 1): Independent(Normal(tanh(m), sigmoid(s) + 0.01), 1)
with no transform on the action, sampled as mean + std * eps (dreamer.py:196-200), and the reinforce actor loss of
a2c.py:119-130, ((-log_prob(a) * agae - eta * entropy) * w).mean(), differentiated by float64 autograd through
torch.distributions.  The closed forms below only build the error bounds.

Bounds.  Every element is held to a small multiple of U = 2^-24 times the float64 magnitude of the terms that produce it;
a CUDA math function of k ulp contributes 2kU of its result (tanhf 2 ulp, expf 2 ulp, logf 1 ulp; IEEE division).  The
reasoning sits next to each bound.  Inputs cover saturated heads (|m| up to 30: tanh(m) rounds to +-1 and tanh' to 0; s
down to -40: std -> 0.01; s up to 40: std -> 1.01), actions far outside (-1, 1), zero weights and both signs of agae.

PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/normaltanh_ops.py in place of the kernels."""
import ctypes
import math

import pytest
import torch
import torch.distributions as D

from oracle.normaltanh_ops import NtRefOps
from tests.test_rowwise_misc_f64_gpu import Bufs, f32, gapped, sync
from tests.util import CPU, DEV, Gen, bound, f64, fp32

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24
TINY = 2.0 ** -126
NT_A = [1, 3, 12]
NT_ROWS = [1, 45, 333, 37_500]          # not multiples of 32 or 256: the sums' warp shuffles and blocks run past the last row
                                        # 37 500 = the DMC benchmark's H x T x B rows: 147 blocks into the fixed-order flush


@pytest.fixture(scope="module")
def ops(request):
    """NativeOps on cuda:0 (the float32 twins of oracle/normaltanh_ops.py under PD_TEST_DEV=cpu)."""
    yield NtRefOps("cpu") if CPU else request.getfixturevalue("native_ops")


def nt_inputs(rows, A, seed):
    """(m, s) raw head outputs: m uniform in +-30 with a third in +-2; s a third normal, a third at -40..-20 (sigmoid
    below 2e-9: std = 0.01 within an ulp), a third at 20..40 (std = 1.01)."""
    g = Gen(seed)
    m = torch.where(g.rand(rows, A) < 0.33, g.uniform(rows, A, bound=2.0), g.uniform(rows, A, bound=30.0))
    r = g.rand(rows, A)
    s = torch.where(r < 0.33, g.normal(rows, A, scale=2.0),
                    torch.where(r < 0.66, -30 + g.uniform(rows, A, bound=10.0), 30 + g.uniform(rows, A, bound=10.0)))
    return fp32(torch.cat([m, s], 1))


def nt_terms(out, A):
    """float64 mu, sigmoid, std and the fp32 errors of the kernel's mu = tanhf(m), sg = 1 / (1 + expf(-s)),
    sd = sg + 0.01f."""
    mu, sg = torch.tanh(out[:, :A]), torch.sigmoid(out[:, A:])
    sd = sg + 0.01
    Emu = 4 * U * mu.abs() + TINY                               # tanhf: 2 ulp
    Esg = 6 * U * sg + TINY                                     # expf 2 ulp (4U of e, times e / (1 + e) <= 1), the + 1, the /
    Esd = Esg + U * 0.01 + U * sd                               # 0.01f is 0.01 within U * 0.01; the add
    return mu, sg, sd, Emu, Esg, Esd


def nt_actions(out, A, g):
    """Actions the sampler could return, and some it could not: a fifth at +-(2..5)."""
    mu, _, sd, *_ = nt_terms(out, A)
    rows = out.shape[0]
    a = mu + sd * g.normal(rows, A)
    return fp32(torch.where(g.rand(rows, A) < 0.2, torch.sign(a) * (2 + 3 * g.rand(rows, A)), a))


@gpu
@pytest.mark.parametrize("rows", NT_ROWS)
@pytest.mark.parametrize("A", NT_A)
def test_normal_tanh_sample_against_float64(ops, A, rows):
    out = nt_inputs(rows, A, seed=A + rows)
    eps = fp32(Gen(rows + 1).normal(rows, A))
    B = Bufs()
    act = B.out("action", (rows, A), gap=2)
    ops.normal_tanh_sample(gapped(out, 3), f32(eps), act)
    B.check()
    mu, sg, sd, Emu, Esg, Esd = nt_terms(out, A)
    a = mu + sd * eps
    # sd * eps and the sum: a rounding each (one fewer when contracted to an FMA)
    bound("action", act, a, Emu + eps.abs() * Esd + U * ((sd * eps).abs() + a.abs()))
    assert float(act.abs().max()) > 1.0 or rows == 1            # unbounded: no squashing of the sample


def loss_case(rows, A, eta, seed):
    out = nt_inputs(rows, A, seed)
    g = Gen(seed + 1)
    a = nt_actions(out, A, g)
    ag = fp32(g.normal(rows) * 2)                               # both signs
    w = fp32(torch.where(g.rand(rows) < 0.15, torch.zeros(rows, dtype=f64, device=DEV), g.rand(rows)))   # zero weights
    return out, a, ag, w, float(fp32(torch.tensor(eta, dtype=f64)))


def run_loss(ops, out, a, ag, w, eta, pre=(0.25, 2.0)):
    rows, A = a.shape
    B = Bufs()
    dout = B.out("dout", (rows, 2 * A), gap=3)
    sums = torch.tensor(pre, dtype=f64, device=DEV)
    ops.actor_loss_normal_tanh(eta, gapped(out, 1), gapped(a, 2), f32(ag), f32(w), dout, sums)
    B.check()
    return dout, sums


@gpu
@pytest.mark.parametrize("eta", [0.0, 3e-3])
@pytest.mark.parametrize("rows", NT_ROWS)
@pytest.mark.parametrize("A", NT_A)
def test_actor_loss_normal_tanh_against_float64_autograd(ops, A, rows, eta):
    out, a, ag, w, eta32 = loss_case(rows, A, eta, seed=A * 3 + rows)
    pre = torch.tensor([0.25, 2.0], dtype=f64, device=DEV)
    dout, sums = run_loss(ops, out, a, ag, w, eta32)
    og = out.clone().requires_grad_(True)
    pi = D.Independent(D.Normal(torch.tanh(og[:, :A]), torch.sigmoid(og[:, A:]) + 0.01), 1)
    per = (-pi.log_prob(a) * ag - eta32 * pi.entropy()) * w
    per.mean().backward()
    gr = og.grad
    mu, sg, sd, Emu, Esg, Esd = nt_terms(out, A)
    zc = (a - mu) / sd
    # zc = (a - mu) / sd: the difference carries Emu and a rounding, the division sd's relative error and a rounding
    Ezc = (Emu + U * (a - mu).abs()) / sd + zc.abs() * (Esd / sd + U)
    c = (w / rows)[:, None]
    agc = ag.abs()[:, None]
    # d/dm = c (-ag zc / sd)(1 - mu^2): zc / sd; 1 - mu^2 carries 2|mu| Emu + mu^2 U + a rounding (absolute: at |m| = 30
    # tanh' is 4e-26 and the kernel's 1 - mu^2 is 0); inv, w * inv and the three products a rounding each
    tp = 1 - mu * mu
    E_m = c * agc * ((Ezc / sd + zc.abs() * Esd / sd ** 2) * tp + zc.abs() / sd * (2 * mu.abs() * Emu + U * (mu * mu + tp)))
    bound("dout m", dout[:, :A], gr[:, :A], E_m + 6 * U * gr[:, :A].abs())
    # d/ds = c (-ag (zc^2 - 1) / sd - eta / sd) sg (1 - sg): q = (zc^2 - 1) / sd; the inner difference; sg (1 - sg) with
    # 1 - sg absolute (sg rounds to 1 at s >= 17)
    q = (zc * zc - 1) / sd
    Eq = (2 * zc.abs() * Ezc + U * (zc * zc + (zc * zc - 1).abs())) / sd + q.abs() * (U + Esd / sd)
    inner = -ag[:, None] * q - eta32 / sd
    E_in = agc * Eq + U * (ag[:, None] * q).abs() + eta32 / sd * (U + Esd / sd) + U * inner.abs()
    P = sg * (1 - sg)
    E_P = (1 - sg) * Esg + sg * (Esg + U * (1 - sg)) + U * P
    bound("dout s", dout[:, A:], gr[:, A:], c * (E_in * P + inner.abs() * E_P) + 6 * U * gr[:, A:].abs())
    # per row: log_prob terms -0.5 zc^2 - log sd - log sqrt(2 pi): |zc| Ezc, logf 1 ulp + Esd / sd, a rounding of each term,
    # and A roundings of the running sum; the entropy the same without zc
    lsd = sd.log()
    Elsd = Esd / sd + 2 * U * lsd.abs()
    lpn = -0.5 * zc * zc - lsd - 0.5 * math.log(2 * math.pi)
    lp_terms = (zc.abs() * Ezc + Elsd + 4 * U * (0.5 * zc * zc + lsd.abs() + 1)).sum(-1) + A * U * lpn.abs().sum(-1)
    ent = pi.entropy().detach()
    Eent = (Elsd + 3 * U * (lsd.abs() + 1.5)).sum(-1) + A * U * ent.abs()
    Erow = w * (ag.abs() * lp_terms + eta32 * Eent) + 3 * U * per.detach().abs()
    # the double sums: exact row values, float64 additions over <= 37 500 rows
    bound("sums[0]", sums[0], pre[0] + per.detach().sum(), Erow.sum() + 1e-12 * (per.detach().abs().sum() + 1))
    bound("sums[1]", sums[1], pre[1] + ent.sum(), Eent.sum() + 1e-12 * (ent.abs().sum() + 1))


@gpu
def test_zero_weights_and_zero_agae_leave_only_the_entropy_gradient(ops):
    """w = 0 rows get zero gradient and add nothing to the loss; agae = 0 leaves -c eta / sd * sg (1 - sg) on s and 0 on m."""
    rows, A = 45, 3
    out, a, ag, w, eta32 = loss_case(rows, A, 1e-3, seed=5)
    w[::2] = 0.0
    ag[1::4] = 0.0
    dout, sums = run_loss(ops, out, a, ag, w, eta32, pre=(0.0, 0.0))
    sync()
    assert (dout[::2] == 0).all()
    assert (dout[1::4, :A] == 0).all()
    mu, sg, sd, *_ = nt_terms(out, A)
    want = -(w / rows)[:, None] * eta32 / sd * sg * (1 - sg)
    got = dout[1::4, A:].double()
    # 1 - sg is absolute to a few U: where sg rounds to 1 (s >= 17) the gradient is 0 against the float64 1e-14
    assert torch.allclose(got, want[1::4], rtol=1e-5, atol=1e-9)


@gpu
@pytest.mark.parametrize("rows", [333, 37_500])
def test_sums_and_gradients_are_bit_identical_across_launches(ops, rows):
    A = 12
    out, a, ag, w, eta32 = loss_case(rows, A, 1e-3, seed=rows)
    d1, s1 = run_loss(ops, out, a, ag, w, eta32)
    d2, s2 = run_loss(ops, out, a, ag, w, eta32)
    sync()
    assert torch.equal(s1, s2) and torch.equal(d1, d2)


@gpu
def test_tanh_normal_entry_points_are_unchanged_by_the_shared_kernels(ops):
    """The tanh_normal pair still computes its own policy (functions.py:69-78), not normal_tanh's."""
    rows, A = 45, 3
    out = nt_inputs(rows, A, seed=9)
    eps = fp32(Gen(3).normal(rows, A))
    act = torch.empty(rows, A, device=DEV)
    ops.tanh_normal_sample(f32(out), f32(eps), act)
    sync()
    mu = 5 * torch.tanh(out[:, :A] / 5)
    sd = torch.nn.functional.softplus(out[:, A:]) + 0.1
    assert torch.allclose(act.double(), torch.tanh(mu + sd * eps), rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------------------------------- host-side checks
def z(*shape):
    return torch.zeros(*shape, device=DEV)


def strided(rows, n, ld):
    """A (rows, n) view whose rows are ld apart (ld < n: overlapping rows, a row pitch the kernels refuse)."""
    return torch.as_strided(z(rows * max(ld, n) + n), (rows, n), (ld, 1))


def loss_call(rows=4, A=3, ldo=None, lda=None, lddo=None):
    ldo, lda, lddo = ldo or 2 * A, lda or A, lddo or 2 * A
    return lambda o: o.actor_loss_normal_tanh(1e-3, strided(rows, 2 * A, ldo), strided(rows, A, lda), z(rows), z(rows) + 1,
                                              strided(rows, 2 * A, lddo), torch.zeros(2, dtype=f64, device=DEV))


def sample_call(rows=4, A=3, ldo=None, lda=None):
    ldo, lda = ldo or 2 * A, lda or A
    return lambda o: o.normal_tanh_sample(strided(rows, 2 * A, ldo), z(rows, A), strided(rows, A, lda))


# name: (a call just inside the boundary, the same call just outside it); rows >= 0 has its own test below
CASES = {
    "loss_A_ge_1": (loss_call(A=1), loss_call(A=0, ldo=2, lda=1, lddo=2)),
    "loss_ldo_ge_2A": (loss_call(ldo=6), loss_call(ldo=5)),
    "loss_lda_ge_A": (loss_call(lda=3), loss_call(lda=2)),
    "loss_lddo_ge_2A": (loss_call(lddo=6), loss_call(lddo=5)),
    "sample_A_ge_1": (sample_call(A=1), sample_call(A=0, ldo=2, lda=1)),
    "sample_ldo_ge_2A": (sample_call(ldo=6), sample_call(ldo=5)),
    "sample_lda_ge_A": (sample_call(lda=3), sample_call(lda=2)),
}


@pytest.mark.gpu
@pytest.mark.skipif(CPU, reason="native host-side checks")
@pytest.mark.parametrize("what", list(CASES))
def test_reference_table_accepts_and_refuses_what_the_native_table_does(native_ops, what):
    from tests.test_gemm_conv_f64_gpu import refused
    inside, outside = CASES[what]
    ref = NtRefOps(DEV)
    inside(native_ops)
    inside(ref)
    torch.cuda.synchronize()
    refused(native_ops, lambda: outside(native_ops))
    with pytest.raises(RuntimeError, match="unsupported"):
        outside(ref)


@pytest.mark.gpu
@pytest.mark.skipif(CPU, reason="native host-side checks")
def test_zero_rows_launch_nothing_and_negative_rows_are_refused(native_ops):
    """rows = 0 is accepted by both tables and launches nothing; rows < 0 (reachable only through the C ABI) is refused
    before any launch."""
    from tests.test_gemm_conv_f64_gpu import refused
    A = 3
    ref = NtRefOps(DEV)
    for o in (native_ops, ref):
        sums = torch.tensor([0.5, 1.5], dtype=f64, device=DEV)
        n0 = native_ops.launch_count()
        o.actor_loss_normal_tanh(1e-3, z(0, 2 * A), z(0, A), z(0), z(0), z(0, 2 * A), sums)
        o.normal_tanh_sample(z(0, 2 * A), z(0, A), z(0, A))
        torch.cuda.synchronize()
        assert native_ops.launch_count() == n0
        assert sums.tolist() == [0.5, 1.5]
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    out, a, v, sums = z(4, 2 * A), z(4, A), z(4), torch.zeros(2, dtype=f64, device=DEV)
    lib, h, ck = native_ops.lib, native_ops.h, native_ops._ck
    refused(native_ops, lambda: ck(lib.pd_actor_loss_normal_tanh(h, -1, A, 1e-3, p(out), 2 * A, p(a), A, p(v), p(v), p(out),
                                                                  2 * A, p(sums), None), "pd_actor_loss_normal_tanh"))
    refused(native_ops, lambda: ck(lib.pd_normal_tanh_sample(h, -1, A, p(out), 2 * A, p(a), p(a), A, None),
                                   "pd_normal_tanh_sample"))

"""Shared helpers: rebuild the seeded inputs of a committed golden case (no reference checkout needed), and the fixtures,
seeded generators and float64 comparison helpers of the kernel-level tests (test_*_f64_gpu.py, test_rssm_persistent_gpu.py)."""
import json
import os

import pytest
import torch

from oracle import dreamer_oracle as O
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.replay import synthetic_batch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("tiny_onehot", "tiny_iwae3", "tiny_dmc", "tiny_klbal05")


def load_fixture(name):
    with open(os.path.join(GOLDEN_DIR, name + ".json")) as f:
        return json.load(f)


def build_case(name, device="cpu", fx=None):
    """-> (fixture, conf, obs, in_state, noise).  `fx` (instead of the committed fixture `name`): a dict with the
    fixture's `preset`, `overrides` and `seeds` keys, for a case that has no reference outputs."""
    fx = fx or load_fixture(name)
    conf = make_conf(fx["preset"], device=str(device), **fx["overrides"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    obs = synthetic_batch(conf, seed=fx["seeds"]["data"])
    g = torch.Generator().manual_seed(fx["seeds"]["state"])
    D, Z = conf.deter_dim, conf.stoch_dim * conf.stoch_discrete
    state = (torch.tanh(torch.randn((B * I, D), generator=g)), torch.zeros(B * I, Z))
    torch.manual_seed(fx["seeds"]["noise"])
    noise = O.draw_noise(conf, T, B)
    mv = lambda d: {k: v.to(device) for k, v in d.items()}
    return fx, conf, mv(obs), tuple(s.to(device) for s in state), mv(noise)


def seeded_weights(model_state_dict, fx):
    return seeded_state_dict(model_state_dict, fx["seeds"]["weights"])


def rel_err(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


# ----------------------------------------------------------------------------------------------------- kernel-level tests
# PD_TEST_DEV=cpu runs a kernel test file with the float32 torch twins of oracle/ref_ops.py in place of the kernels: a dry
# run of its references and bounds without a GPU.
DEV = os.environ.get("PD_TEST_DEV", "cuda:0")
CPU = DEV == "cpu"
f64 = torch.float64


@pytest.fixture(scope="module")
def ops(request):
    """NativeOps on cuda:0 (the float32 RefOps twin under PD_TEST_DEV=cpu); puts the handle back to its defaults after."""
    if CPU:
        from oracle.ref_ops import RefOps

        yield RefOps("cpu")
        return
    o = request.getfixturevalue("native_ops")
    yield o
    o.set_round_operands(True)
    o.set_gemm_impl(0)


@pytest.fixture(params=[0, 1], ids=lambda v: f"round_out{v}")
def round_out(request, ops):
    """Runs a test with operand rounding (set_round_operands) off and on."""
    ops.set_round_operands(bool(request.param))
    yield request.param
    ops.set_round_operands(True)


class Gen:
    """Seeded float64 draws (CPU generator: the same values on every machine), returned on `dev`."""

    def __init__(self, seed, dev=None):
        self.g = torch.Generator().manual_seed(seed)
        self.dev = DEV if dev is None else dev

    def uniform(self, *shape, bound=1.0):
        return ((torch.rand(*shape, generator=self.g, dtype=f64) * 2 - 1) * bound).to(self.dev)

    def normal(self, *shape, scale=1.0):
        return (torch.randn(*shape, generator=self.g, dtype=f64) * scale).to(self.dev)

    def rand(self, *shape):
        return torch.rand(*shape, generator=self.g, dtype=f64).to(self.dev)


def fp32(x):                                    # float64 copy of the fp32 value the kernel reads
    return x.float().double()


def fp16(x):
    return x.to(torch.float16).to(f64)


def ulp(x, min_exp, mant):
    """ulp of a binary float with `mant` explicit mantissa bits and minimum normal exponent min_exp at |x| (float64)."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** min_exp))
    return torch.ldexp(torch.ones_like(x), e - 1 - mant)


def tf32_rna(x):
    """cvt.rna.tf32.f32 of x (float64 -> fp32 -> tf32, ties away from zero), as float64."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32).double()


def bound(name, got, ref, lim):
    """|got - ref| <= lim elementwise (lim: float64 tensor of the propagated error); equal infinities pass.  Returns
    max(|got - ref| / lim), the share of the bound used."""
    got = got.double()
    ref = torch.as_tensor(ref, dtype=f64, device=got.device).expand_as(got)
    lim = torch.as_tensor(lim, dtype=f64, device=got.device).expand_as(got)
    assert not torch.isnan(got).any(), f"{name}: {int(torch.isnan(got).sum())} elements not written or NaN"
    same = got == ref
    err = torch.where(same, torch.zeros_like(got), (got - ref).abs())
    bad = err > lim
    ratio = torch.where(same, torch.zeros_like(err), err / lim.clamp_min(1e-300))
    if bad.any():
        i = int(torch.argmax(torch.where(bad, ratio, torch.zeros_like(err)).reshape(-1)))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements out of bound; worst flat index {i}: "
                             f"got {got.reshape(-1)[i].item():.9g} ref {ref.reshape(-1)[i].item():.9g} "
                             f"bound {lim.reshape(-1)[i].item():.3g}")
    return float(ratio.max()) if ratio.numel() else 0.0


def rounded(name, got, ref, err, kind, stats):
    """A value the kernel rounds to fp16 / tf32 (rna): equal to the rounded reference unless the reference lies within its
    fp32 error `err` of a rounding boundary (then the kernel's fp32 value may sit on the other side); never more than one
    ulp (+ err) away."""
    rnd, u = (fp16, lambda v: ulp(v, -14, 10)) if kind == "fp16" else (tf32_rna, lambda v: ulp(v, -126, 10))
    got64 = got.double()
    bound(name, got64, ref, u(torch.maximum(ref.abs(), got64.abs())) + err)
    straddle = rnd(ref - err) != rnd(ref + err)
    bad = (got64 != rnd(ref)) & ~straddle
    assert not bad.any(), (f"{name}: {int(bad.sum())} elements differ from the {kind}-rounded reference away from a "
                           f"rounding boundary")
    stats[name] = stats.get(name, 0) + int(straddle.sum())

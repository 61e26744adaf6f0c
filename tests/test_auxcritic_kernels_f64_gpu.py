"""Kernel-level tests of what the auxiliary critic adds: pd_gae_critic_obs against a float64 reference computed from the
kernel's own fp32 inputs, its host-side refusals, and the GEMM route each aux-critic GEMM of the `atari_auxcritic` and
`tiny_auxcritic_iwae3` shapes takes (the latter reads and writes the sample-0 rows of the features as a strided view).
Conventions of tests/test_catreward_kernels_f64_gpu.py: per-element bounds in U = 2^-24, outputs pre-filled with NaN
inside sentinel guard bands.

PD_TEST_DEV=cpu runs the file with the float32 torch twin of oracle/auxcritic_ops.py in place of the kernels."""
import ctypes

import pytest
import torch

import tests.test_vecobs_kernels_f64_gpu as V
from tests.test_gemm_conv_f64_gpu import refused
from tests.test_rowwise_misc_f64_gpu import Bufs
from tests.util import CPU, DEV, Gen, bound, f64, fp32, round_out  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def ops(request):
    """NativeOps on cuda:0 (the float32 AuxRefOps twin under PD_TEST_DEV=cpu); puts the handle back to its defaults after."""
    if CPU:
        from oracle.auxcritic_ops import AuxRefOps

        yield AuxRefOps("cpu")
        return
    o = request.getfixturevalue("native_ops")
    yield o
    o.set_round_operands(True)
    o.set_gemm_impl(0)


def gae_case(T, B, seed):
    """Values, rewards and 0/1 terminals of T rows x B columns: column 0 ends at row 0, column 1 mid-sequence, column 2 at
    the last row, column 3 twice; the other columns have none."""
    g = Gen(seed)
    vt, v = fp32(g.normal(T, B)), fp32(g.normal(T, B))
    rew = fp32(torch.tanh(g.normal(T, B)))
    term = torch.zeros(T, B, dtype=f64, device=DEV)
    for col, rows in ((0, (0,)), (1, (T // 2,)), (2, (T - 1,)), (3, (1, T - 1))):
        if col < B:
            term[list(rows), col] = 1.0
    return vt, v, rew, term


def reference(T, B, gamma, lam, vt, v, rew, term, scale):
    """float64 results and the magnitude each fp32 target accumulates (for the error bound)."""
    H = T - 1
    a = -vt[:-1] + rew[1:] + gamma * (1 - term[1:]) * vt[1:]
    mag_a = vt[:-1].abs() + rew[1:].abs() + gamma * vt[1:].abs()
    ag, mag = torch.zeros_like(a), torch.zeros_like(a)
    for j in reversed(range(H)):
        c = lam * gamma * (1 - term[j + 1])
        ag[j] = a[j] + (c * ag[j + 1] if j < H - 1 else 0)
        mag[j] = mag_a[j] + (c * mag[j + 1] if j < H - 1 else 0)
    w = torch.cumprod(1 - term[:-1], 0)                   # exp(cumsum(log(1 - t))) for 0/1 terminals
    d = ag + vt[:-1] - v[:-1]
    coef = scale / (H * B)
    return dict(dv=-d * w * coef, loss=(0.5 * d * d * w).sum(), vsum=v[:-1].sum(), w=w, d=d,
                err_d=8 * U * (mag + vt[:-1].abs() + v[:-1].abs()) * (H + 2), coef=coef)


def run(ops, T, B, gamma, lam, vt, v, rew, term, scale, bufs):
    dv = bufs.out("dv", (T - 1, B))
    sums = torch.full((8,), 123.0, dtype=f64, device=DEV)
    sums[:2] = 0
    f = lambda x: x.float().contiguous()
    ops.gae_critic_obs(T, B, gamma, lam, f(vt), f(v), f(rew), f(term), scale, dv, sums)
    bufs.check()
    assert (sums[2:] == 123.0).all(), "sums past the two outputs were written"
    return dv, sums


@gpu
@pytest.mark.parametrize("gam,lam,scale", [(0.99, 0.95, 1.0), (1.0, 1.0, 0.3), (0.99, 0.0, 2.0)])
@pytest.mark.parametrize("B", [1, 3, 50])
@pytest.mark.parametrize("T", [2, 50, 128])
def test_gae_critic_obs_against_float64(ops, T, B, gam, lam, scale):
    vt, v, rew, term = gae_case(T, B, T * 1000 + B)
    bufs = Bufs()
    dv, sums = run(ops, T, B, gam, lam, vt, v, rew, term, scale, bufs)
    r = reference(T, B, gam, lam, vt, v, rew, term, scale)
    dv_err = r["coef"] * r["w"] * r["err_d"] + U * r["dv"].abs()
    bound("dv", dv, r["dv"], dv_err)
    assert (dv[r["w"] == 0] == 0).all(), "rows at and after a terminal carry a gradient"
    sum_err = (U if CPU else 1e-13) * T * B            # the kernel adds in double; its float32 twin in float32
    loss_err = (r["w"] * (r["d"].abs() * r["err_d"] + r["err_d"] ** 2)).sum() + sum_err * (0.5 * r["d"] ** 2 * r["w"]).sum()
    bound("loss sum", sums[0:1], r["loss"].reshape(1), loss_err.reshape(1))
    bound("value sum", sums[1:2], r["vsum"].reshape(1), (sum_err * v[:-1].abs().sum()).reshape(1))


@gpu
def test_terminal_columns_get_zero_weight_and_no_nan(ops):
    """A terminal of 1 gives log 0 = -inf in the reference's reality weight: weight 0 at its row and after, never NaN, in
    the gradient and the loss sum alike."""
    T, B = 6, 4
    vt, v, rew, term = gae_case(T, B, 3)
    dv, sums = run(ops, T, B, 0.99, 0.95, vt, v, rew, term, 1.0, Bufs())
    assert torch.isfinite(dv).all() and torch.isfinite(sums[:2]).all()
    assert (dv[:, 0] == 0).all()                                   # terminal at row 0: nothing of the column is real
    assert (dv[T // 2:, 1] == 0).all() and (dv[:T // 2, 1] != 0).all()
    assert (dv[:, 2] != 0).all()                                   # a terminal at the last row weights no row of H


@gpu
def test_gae_critic_obs_is_bit_identical_run_to_run(ops):
    T, B = 50, 3000
    vt, v, rew, term = gae_case(T, B, 9)
    outs = [run(ops, T, B, 0.99, 0.95, vt, v, rew, term, 1.0, Bufs()) for _ in range(3)]
    for dv, sums in outs[1:]:
        assert torch.equal(dv, outs[0][0]) and torch.equal(sums, outs[0][1])


@gpu
@pytest.mark.parametrize("what", ["T1", "T129", "B0", "null_term"])
def test_gae_critic_obs_refusals_launch_nothing(ops, what):
    buf = torch.zeros(130 * 4, device=DEV)
    sums = torch.zeros(2, dtype=f64, device=DEV)
    p, ps = ctypes.c_void_p(buf.data_ptr()), ctypes.c_void_p(sums.data_ptr())

    def raw(T, B, term=True):
        ops._ck(ops.lib.pd_gae_critic_obs(ops.h, T, B, 0.99, 0.95, p, p, p, p if term else None, 1.0, p, ps, ops._s()),
                "pd_gae_critic_obs")

    calls = dict(T1=lambda: raw(1, 2), T129=lambda: raw(129, 2), B0=lambda: raw(4, 0), null_term=lambda: raw(4, 2, False))
    refused(ops, calls[what])


# ----------------------------------------------------------------------------------------------------- GEMM routes
R, F = 2500, 3072                                # atari_auxcritic: T*B sample-0 rows of 2048 + 32*32 features
RB = R - 50                                      # the first T - 1 steps carry the critic loss
FI, RI, RIB = 96, 12, 9                          # tiny_auxcritic_iwae3: F = 64 + 4*8, T*B = 12, (T-1)*B = 9, rows I*F apart
ROUTES = [
    V.gcase("atari_fwd_l0", R, 400, F, F, F, 400, "wgmma", bias=True),
    V.gcase("atari_out", R, 1, 400, 400, 400, 1, "gemv", bias=True),
    V.gcase("atari_wgrad_l0", 400, F, RB, 400, F, F, "mma", a_mn=1, b_mn=1, acc=True),
    V.gcase("atari_wgrad_out", 1, 400, RB, 1, 400, 400, "wcolsum", a_mn=1, b_mn=1, acc=True),
    V.gcase("atari_dx_l0_into_dfeat", RB, F, 400, 400, F, F, "mma", b_mn=1, res="inplace"),
    V.gcase("iwae3_fwd_l0_strided_rows", RI, 400, FI, 3 * FI, FI, 400, "wgmma", bias=True),
    V.gcase("iwae3_wgrad_l0_strided_rows", 400, FI, RIB, 400, 3 * FI, FI, "mma", a_mn=1, b_mn=1, acc=True),
    V.gcase("iwae3_dx_l0_into_strided_dfeat", RIB, FI, 400, 400, FI, 3 * FI, "mma", b_mn=1, res="inplace"),
]


@gpu
@pytest.mark.parametrize("c", ROUTES)
def test_aux_critic_gemm_routes_match_float64_reference(ops, round_out, c):
    V.test_vecobs_gemm_shapes_match_float64_reference(ops, round_out, c)

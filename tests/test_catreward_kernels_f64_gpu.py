"""Kernel-level tests of what the categorical reward head adds: pd_support_head against a float64 reference computed from
the kernel's own fp32 inputs, its host-side refusals, and the GEMM route each reward-head GEMM of the `atari_catreward`
shape takes (S = 3 outputs at a row pitch of 4, and S = 33 at a pitch of 36).  Conventions of
tests/test_vecobs_kernels_f64_gpu.py: per-element bounds in U = 2^-24, outputs pre-filled with NaN inside sentinel guard
bands, operand gap columns holding NaN (so a padding column that leaked into a product would show).

PD_TEST_DEV=cpu runs the file with the float32 torch twin of oracle/catreward_ops.py in place of the kernels."""
import ctypes
import math

import pytest
import torch

import tests.test_vecobs_kernels_f64_gpu as V
from pydreamer_b200.ops import SUPPORT_MAX
from tests.test_gemm_conv_f64_gpu import refused
from tests.test_rowwise_misc_f64_gpu import Bufs
from tests.util import CPU, DEV, Gen, bound, f64, fp32, round_out  # noqa: F401

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def ops(request):
    """NativeOps on cuda:0 (the float32 CatRefOps twin under PD_TEST_DEV=cpu); puts the handle back to its defaults after."""
    if CPU:
        from oracle.catreward_ops import CatRefOps

        yield CatRefOps("cpu")
        return
    o = request.getfixturevalue("native_ops")
    yield o
    o.set_round_operands(True)
    o.set_gemm_impl(0)


def support_case(S, div, seed):
    """Logits (M rows, some of them at +-80), an unsorted support on the 1/8 grid with a duplicated value, and targets:
    uniform draws, support values and exact midpoints between two support values (a tie the first index wins)."""
    M = (37 if S >= 255 else 501) * div
    g = Gen(seed)
    y = fp32(g.normal(M, S, scale=3.0))
    y[0] = 80.0
    y[0, S // 2] = -80.0
    y[1, ::2] = -80.0
    y[1, 1::2] = 80.0
    grid = torch.randperm(max(S, 16), generator=g.g)[:S].to(f64) / 8 - 1
    if S >= 3:
        grid[-1] = grid[0]
    sup = grid.to(DEV)
    R = M // div
    t = fp32(g.uniform(R, bound=1.5))
    pick = torch.randint(0, S, (R, 2), generator=g.g).to(DEV)
    t[0::3] = sup[pick[0::3, 0]]
    t[1::3] = (sup[pick[1::3, 0]] + sup[pick[1::3, 1]]) / 2          # exact on the 1/8 grid
    return M, y, sup, t


def reference(y, sup, t, div):
    """float64 results; the bucket is torch's argmin of the fp32 squared distances, as the reference computes it."""
    M, S = y.shape
    k = torch.square(t.float()[:, None] - sup.float()).argmin(-1).cpu().to(DEV)
    k = k.repeat_interleave(div, 0)
    p = torch.softmax(y, -1)
    rec = p @ sup
    loss = torch.logsumexp(y, -1) - y.gather(-1, k[:, None])[:, 0]
    dy = p - torch.nn.functional.one_hot(k, S).to(f64)
    return k, p, rec, loss, dy


@gpu
@pytest.mark.parametrize("mode", ["target", "expectation"])
@pytest.mark.parametrize("gap", [0, 5])
@pytest.mark.parametrize("div", [1, 3])
@pytest.mark.parametrize("S", [2, 3, 4, 5, 31, 32, 33, 255, SUPPORT_MAX])
def test_support_head_against_float64(ops, S, div, gap, mode):
    M, y, sup, t = support_case(S, div, S * 10 + div + gap)
    k, p, rec_r, loss_r, dy_r = reference(y, sup, t, div)
    B = Bufs()
    rec = B.out("rec", (M,))
    yd = y.float()
    if gap:                                     # a padded row pitch: the gap columns hold NaN
        yv = torch.full((M, S + gap), float("nan"), device=DEV)
        yv[:, :S] = yd
        yd = yv[:, :S]
    if mode == "target":
        loss, dy, idx = (B.out("loss", (M,)), B.out("dy", (M, S), gap=gap),
                          B.out("idx", (M, 1), dtype=torch.int32, fill=-7))
        ops.support_head(yd, sup.float(), t.float(), div, rec, loss, dy, idx.view(-1))
    else:
        ops.support_head(yd, sup.float(), None, div, rec)
    B.check()
    chain = math.ceil(S / 32) + 5               # a lane's chain of additions, then the 5 levels of the xor tree
    mx = y.amax(-1)
    # exp(y - max) carries 2 U plus U |y - max| from rounding its argument; the sums chain U; the division 1 U
    ep = (chain + 6 + (y - mx[:, None]).abs()) * U * p
    bound("rec", rec, rec_r, ep @ sup.abs() + (chain + 6) * U * (p @ sup.abs()) + 2.0 ** -126)
    if mode != "target":
        return
    assert torch.equal(idx.view(-1).long(), k), "bucket indices differ from torch's argmin"
    yk = y.gather(-1, k[:, None])[:, 0]
    bound("loss", loss, loss_r, (chain + 6) * U + 2 * U * (mx.abs() + yk.abs() + loss_r.abs()))
    bound("dy", dy, dy_r, 2 * ep + U * dy_r.abs() + 2.0 ** -126)


@gpu
def test_support_head_is_bit_identical_run_to_run(ops):
    M, y, sup, t = support_case(33, 1, 5)
    y, sup, t = y.float(), sup.float(), t.float()
    outs = []
    for _ in range(3):
        o = [torch.empty(M, device=DEV), torch.empty(M, device=DEV), torch.empty(M, 33, device=DEV),
             torch.empty(M, dtype=torch.int32, device=DEV)]
        ops.support_head(y, sup, t, 1, *o)
        outs.append(o)
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))


@gpu
@pytest.mark.parametrize("what", ["S1", "S_above_max", "ldy_below_S", "tgt_div0", "no_target_no_rec", "target_no_dy"])
def test_support_head_refusals_launch_nothing(ops, what):
    z = lambda *s: torch.zeros(*s, device=DEV)

    def raw(S, ldy, target=True, rec=True, dy=True, div=1):    # the C entry point: ops.support_head derives ld from views
        buf = z(64 * (SUPPORT_MAX + 1))
        p = ctypes.c_void_p(buf.data_ptr())
        ops._ck(ops.lib.pd_support_head(ops.h, 8, S, p, ldy, p, p if target else None, div, p if rec else None, p,
                                        p if dy else None, max(S, 1), None, ops._s()), "pd_support_head")

    calls = {
        "S1": lambda: ops.support_head(z(8, 1), z(1), z(8), 1, z(8), z(8), z(8, 1)),
        "S_above_max": lambda: raw(SUPPORT_MAX + 1, SUPPORT_MAX + 1),
        "ldy_below_S": lambda: raw(3, 2),
        "tgt_div0": lambda: raw(3, 4, div=0),
        "no_target_no_rec": lambda: raw(3, 4, target=False, rec=False),
        "target_no_dy": lambda: raw(3, 4, dy=False),
    }
    refused(ops, calls[what])


# ----------------------------------------------------------------------------------------------------- GEMM routes
R, RJ = 2500, 16 * 2500                          # atari_catreward: T*B world-model rows, (H+1)*T*B dreamed rows
ROUTES = [
    # S = 3 at pitch 4: the output layer (N = 3 <= 4, K-major, storing) runs gemv_rows on both row counts; its weight
    # gradient (A = the logit gradient [rows][3] at lda = 4) is TMA-addressable and runs on the tensor cores; its input
    # gradient (K = 3 < 8) runs the generic CUDA-core kernel
    V.gcase("s3_out", R, 3, 400, 400, 400, 4, "gemv", bias=True),
    V.gcase("s3_out_dream_rows", RJ, 3, 400, 400, 400, 4, "gemv", bias=True),
    V.gcase("s3_wgrad_lda4", 3, 400, R, 4, 400, 400, "mma", a_mn=1, b_mn=1, acc=True),
    V.gcase("s3_dx_k3_lda4", R, 400, 3, 4, 400, 400, "simt", b_mn=1),
    # S = 33 at pitch 36: every reward-head GEMM on the tensor cores, with partial k-blocks and column tiles
    V.gcase("s33_wgrad_lda36", 33, 400, R, 36, 400, 400, "mma", a_mn=1, b_mn=1, acc=True),
    V.gcase("s33_dx_k33_lda36", R, 400, 33, 36, 400, 400, "mma", b_mn=1),
]


@gpu
@pytest.mark.parametrize("c", ROUTES)
def test_reward_head_gemm_routes_match_float64_reference(ops, round_out, c):
    V.test_vecobs_gemm_shapes_match_float64_reference(ops, round_out, c)


@gpu
@pytest.mark.parametrize("rows,ld", [(R, 36), (RJ, 36), (R, 40)])
def test_s33_output_layer_store_at_a_padded_pitch(ops, rows, ld):
    """The S = 33 output layer on the tensor cores stores its rows through a TMA map 33 columns wide at a row pitch of 36
    (or 40).  The store fills each row up to its next 16-byte boundary: columns 33-35 receive zeros, which nothing reads.
    Columns past that boundary and rows past the last stay untouched, and every real column is exact."""
    N, Nb = 33, 36
    c = dict(M=rows, N=N, K=400, bias=True)
    assert V.dispatch(c, 400, 400, ld) == "wgmma"
    g = Gen(rows + ld)
    A, Bm = V.tf32_rna(g.normal(rows, 400)), V.tf32_rna(g.normal(N, 400, scale=0.05))
    bias = fp32(g.normal(N, scale=0.5))
    flat = torch.full(((rows + 8) * ld,), float("nan"), device=DEV)
    full = flat[:rows * ld].view(rows, ld)
    C = full[:, :N]
    ops.gemm(A.float(), Bm.float(), C, bias=bias.float())
    if not CPU:
        torch.cuda.synchronize()
    assert torch.isnan(flat[rows * ld:]).all(), "rows past the last one were written"
    assert torch.isnan(full[:, Nb:]).all(), "columns past the row's 16-byte boundary were written"
    if not CPU:                                 # (the float32 twin writes the real columns only)
        assert (full[:, N:Nb] == 0).all(), "the padding columns up to the 16-byte boundary hold something other than 0"
    ref, err, _ = V.gemm_ref(dict(c, res=None), A, Bm, bias, None, None, CPU)
    V.check_out("C", C, ref, err, False, {})

"""Kernel-level tests of the categorical grid-image front end: pd_cat_image_loss, pd_grid_enc_input and
pd_image_ids_onehot against float64 references computed from the kernel's own fp32 inputs, and the GEMM route each new
layer takes at the `minigrid` shapes.

PD_TEST_DEV=cpu runs the file with the float32 torch twins of oracle/grid_ops.py in place of the kernels."""
import pytest
import torch

from oracle.grid_ops import cat_image_terms
from tests.test_gemm_conv_f64_gpu import refused
from tests.util import CPU, DEV, Gen, bound, f64

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def ops(request):
    """NativeOps on cuda:0 (the float32 GridRefOps twin under PD_TEST_DEV=cpu)."""
    if CPU:
        from oracle.grid_ops import GridRefOps

        yield GridRefOps("cpu")
        return
    o = request.getfixturevalue("native_ops")
    yield o
    o.set_round_operands(True)
    o.set_gemm_impl(0)


def onehot_target(g, G, C, P, ties=False, zeros=False):
    k = (g.rand(G, P) * C).long().clamp_max(C - 1)
    t = torch.nn.functional.one_hot(k, C).movedim(-1, 1).to(f64)
    if ties:                                    # a second maximum after the first in some pixels
        t[:, -1, ::3] = 1.0
    if zeros:
        t[:, :, 1::4] = 0.0
    return t.reshape(G, C * P).float()


# ----------------------------------------------------------------------------------------------------- pd_cat_image_loss
@gpu
@pytest.mark.parametrize("min_prob", [0.0, 0.1])
@pytest.mark.parametrize("div", [1, 3])
@pytest.mark.parametrize("C,P", [(2, 1), (4, 49), (33, 25), (64, 49), (4, 4096), (2, 4096)])
def test_cat_image_loss_against_float64(ops, C, P, div, min_prob):
    g = Gen(C * 131 + P + div)
    G = 5 if P < 4096 else 2
    M = G * div
    y = (g.normal(M, C * P) * 3).float()
    y[0, :C] = 80.0 * torch.sign(y[0, :C])      # large logits
    t = onehot_target(g, G, C, P, ties=True, zeros=True).to(y.device)
    loss, dy = torch.full((M,), float("nan"), device=y.device), torch.full((M, C * P), float("nan"), device=y.device)
    rec = torch.full((G, C * P), float("nan"), device=y.device)
    ops.cat_image_loss(y, C, t, div, min_prob, loss, dy, rec)
    l_ref, dy_ref, rec_ref = cat_image_terms(y.double(), C, t.double(), div, min_prob)
    # the target class is torch.argmax's: first maximum, all-zero pixels give class 0
    El = (2 * C + 20) * U * (l_ref.abs() + P * (y.abs().amax(1).double() + 1.0)) + 1e-30
    bound("loss", loss, l_ref, El)
    bound("dy", dy, dy_ref, (4 * C + 40) * U * (1.0 + y.abs().amax(1, keepdim=True).double()))
    bound("rec", rec, rec_ref, (8 * C + 80) * U * (1.0 + rec_ref.abs() + y.abs().amax().double()))


@gpu
def test_cat_image_loss_is_bit_identical_run_to_run(ops):
    g = Gen(9)
    C, P, div, G = 33, 49, 3, 300
    y = g.normal(G * div, C * P).float()
    t = onehot_target(g, G, C, P).to(y.device)
    outs = []
    for _ in range(3):
        o = (torch.empty(G * div, device=y.device), torch.empty(G * div, C * P, device=y.device),
             torch.empty(G, C * P, device=y.device))
        ops.cat_image_loss(y, C, t, div, 0.1, *o)
        outs.append(o)
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))


@gpu
@pytest.mark.parametrize("what", ["C1", "C65", "P4097", "div_not_dividing", "min_prob1"])
def test_cat_image_loss_refusals_launch_nothing(ops, what):
    z = lambda *s: torch.zeros(*s, device=DEV)
    calls = {
        "C1": lambda: ops.cat_image_loss(z(4, 49), 1, z(4, 49), 1, 0.0, z(4), z(4, 49)),
        "C65": lambda: ops.cat_image_loss(z(4, 65 * 4), 65, z(4, 65 * 4), 1, 0.0, z(4), z(4, 65 * 4)),
        "P4097": lambda: ops.cat_image_loss(z(2, 2 * 4097), 2, z(2, 2 * 4097), 1, 0.0, z(2), z(2, 2 * 4097)),
        "div_not_dividing": lambda: ops.cat_image_loss(z(4, 8), 2, z(2, 8), 3, 0.0, z(4), z(4, 8)),
        "min_prob1": lambda: ops.cat_image_loss(z(4, 8), 2, z(4, 8), 1, 1.0, z(4), z(4, 8)),
    }
    refused(ops, calls[what])


# ----------------------------------------------------------------------------------------------------- encoder input
@gpu
@pytest.mark.parametrize("C,H", [(4, 7), (3, 5)])
def test_grid_enc_input_is_the_exact_concatenation(ops, C, H):
    g = Gen(C + H)
    NB = 37
    img = g.normal(NB, C, H, H).float()
    rew, term = g.normal(NB).float(), (g.rand(NB) < 0.5).float()
    out = torch.full((NB, (C + 2) * H * H), float("nan"), device=img.device)
    ops.grid_enc_input(img, rew, term, out)
    want = torch.cat([img, rew.view(NB, 1, 1, 1).expand(NB, 1, H, H), term.view(NB, 1, 1, 1).expand(NB, 1, H, H)], 1)
    assert torch.equal(out, want.reshape(NB, -1))


# ----------------------------------------------------------------------------------------------------- one-hot ids
@gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int32, torch.int64])
def test_image_ids_onehot_and_out_of_range_ids(ops, dtype):
    g = Gen(3)
    T, B, H, W, C = 3, 4, 7, 7, 4
    ids = (g.rand(T, B, H, W) * C).long().clamp_max(C - 1)
    ids[0, 0, 0, 0] = C                             # out of range: NaN channels
    if dtype != torch.uint8:
        ids[1, 1, 1, 1] = -1
    guard = torch.full((T * B * C * H * W + 64,), -7.0, device=DEV)
    out = guard[:T * B * C * H * W].view(T, B, C, H, W)
    ops.image_ids_onehot(ids.to(dtype).to(DEV), out)
    bad = (ids < 0) | (ids >= C)
    want = torch.nn.functional.one_hot(ids.clamp(0, C - 1), C).movedim(-1, 2).float().to(DEV)
    ok = ~bad.to(DEV).unsqueeze(2).expand_as(out)
    assert torch.equal(out[ok], want[ok])
    assert torch.isnan(out[~ok]).all() and int((~ok).sum()) == C * int(bad.sum())
    assert (guard[T * B * C * H * W:] == -7.0).all(), "written past the output"


# ----------------------------------------------------------------------------------------------------- GEMM routes
@gpu
@pytest.mark.parametrize("K", [294, 75])
def test_first_encoder_layer_and_its_weight_gradient_match_float64(ops, K):
    """The first dense-encoder layer reads rows of K = (C+2) H W floats (294 at `minigrid`, 75 at 5x5x3): not 16-byte rows,
    so the forward GEMM and the weight gradient take the generic CUDA-core route; both against float64."""
    g = Gen(K)
    M, N = 480, 400
    x = g.normal(M, K).float()
    w = (g.normal(N, K) / K ** 0.5).float()
    out = torch.empty(M, N, device=x.device)
    ops.gemm(x, w, out)
    ref = x.double() @ w.double().T
    bound("fwd", out, ref, (K + 4) * 2 ** -10 * (x.double().abs() @ w.double().abs().T))
    dx = g.normal(M, N).float()
    gw = torch.zeros(N, K, device=x.device)
    ops.gemm(dx, x, gw, a_mn=True, b_mn=True, accumulate=True)
    ref = dx.double().T @ x.double()
    bound("wgrad", gw, ref, (M + 4) * 2 ** -10 * (dx.double().abs().T @ x.double().abs()))

"""The imagination rollout (Dreamer._dream) and the actor-critic update (Dreamer._actor_critic) of a real training step,
checked STAGE BY STAGE against a float64 reference computed on the device.

Harness.  `Dreamer(conf)` with seeded weights runs `training_step` on a synthetic batch with explicit sampling noise (an
eager step; the product settings otherwise: fp16 forward GEMMs, the default `overlap`, the persistent RSSM kernels).  The
step's workspace is then read back (`ws`: the key must already exist, so a renamed buffer fails loudly) and every stage
is recomputed in float64 from the step's OWN inputs to that stage (teacher forcing), so an error never compounds and each
comparison owns one piece of wiring:
  1. actor forward of every imagination step (pre-norm x, LayerNorm statistics and y of each hidden layer in the saved
     rows [i N, (i+1) N), then the logits from the saved last y);
  2. the action sample (one-hot: argmax(p / q); tanh_normal: the float64 formula on the kernel's logits and noise);
  3. the RSSM cell and GRU of every step: aa, x, za and its statistics, gi, gh and h';
  4. the prior head and the latent sample of every step (yp, pp and its statistics, the logits, the sample), and
     feats16 == fp16(feats) bit for bit;
  5. the reward / terminal / target-critic / critic heads on the (H+1) N dreamed rows (the critic layer by layer);
  6. `gae_critic` from the kernel's rew / v / vt / terminal logits;
  7. the actor loss and the seven returned metrics;
  8. every actor and critic parameter gradient and each layer's input gradient, from the kernel's dv / dlogits and the
     saved activations (critic_target gets none);
  9. the logging dream (do_dream_tensors: B rows, T - 1 steps, stages 1-7) and the dream tensors the step returns;
 10. all of it again after grad_clip and an optimizer step (target_interval 1 and 2), so a stale tf32 / fp16 shadow, a
     stale a_mlp^T or a stale critic_target fails.

References.  Weights are the fp32 masters (`_raw`) rounded the way the kernel reads them: fp16 for the fp16 GEMMs,
tf32 (rna) for `ops.gemm`, raw fp32 for biases and LayerNorm affine.  Operands are the exact values the kernel read (the
fp16 feature copy, the fp16 copy of a saved y, the fp32 features where the kernel reads fp32).  The op twins of
oracle/ref_ops.py are never the reference.

Bounds reuse the machinery of tests/test_gemm_conv_f64_gpu.py and tests/test_rowwise_misc_f64_gpu.py: a contraction is
held to C_ACC * depth * U * sum_k |a_k b_k| with the depth of the route the GEMM dispatcher takes (tc_depth for the
tensor-core and skinny routes, simt_depth for the CUDA-core one), + TF32_OP * sum_k |a_k b_k| for an fp32 operand that is
not tf32-exact on the tensor-core route (the actual difference of its truncated or rounded copy where the other operand
is exact), + the epilogue's additions; LayerNorm, GRU, softmax, GAE and actor-loss bounds are those files' own.  The step
keeps some intermediates in scratch only or for its last imagination step only (the hidden layers of the reward, terminal
and target-critic heads, the cell and prior head of each step, the layer gradients of the backward).  Those are replayed
on the step's own inputs into test-owned buffers: the replay must reproduce what the step kept bit for bit (h' and the
fp16 h' of every step, the last step's buffers, the heads' outputs, the parameter gradients; every sum of the step is
added in a fixed order), and is then checked stage by stage like the rest.  Every element has its own bound; max(err /
bound) per stage is printed (run with -s), values stored tf32-rounded apart, and so is the share of the value the bound
takes (the median over elements), which must stay small (VACUOUS).

Sampled classes must be argmax(p / q) of the float64 softmax, except near-ties: the top two log(p / q) within their
propagated error.  Near-ties are counted, printed and bounded.

The exact arm (`exact`) runs the CUDA-core GEMM (set_gemm_impl(1)) with operand rounding off and fp16_forward off: every
bound is then an fp32 one.

PD_TEST_DEV=cpu runs the tiny cases on the CPU with the float32 torch twins installed as the op table: a dry run of the
references and bounds without a GPU (the twins do not round, so there every rounding is the identity)."""
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import dreamer_oracle as O
from oracle.grid_oracle import seeded_state_dict as grid_seeded_state_dict
from oracle.weights import seeded_state_dict
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_gemm_conv_f64_gpu import C_ACC, TF32_OP, U, cdiv, simt_depth, tc_depth
from tests.test_rowwise_misc_f64_gpu import KS, TINY, colsum_depth, gae_ref, ln_col_depth, ln_fwd_ref, softmax_err
from tests.test_rssm_persistent_gpu import ln_bwd_ref
from tests.util import CPU, DEV, bound, f64, fp16, rounded, tf32_rna, ulp

gpu = pytest.mark.gpu if not CPU else (lambda f: f)
# The bound of a value may take at most this share of it (median over elements).  The widest are the weight gradients: sums
# of H * N = 37 500 rows that cancel, whose worst-case fp32 chain on the CUDA-core route (K + 16 roundings) reaches ~10 %.
VACUOUS = 0.125
SEED_W, SEED_DATA, SEED_NOISE = 11, 100, 7

# name: (preset, overrides)
TINY_CASES = {
    "tiny": ("tiny", {}),
    "tiny_dmc": ("tiny_dmc", {}),
    "tiny_catreward_wide": ("tiny_catreward_wide", {}),
    "tiny_hd42": ("tiny", dict(hidden_dim=42)),                # Hd % 4 != 0: the a_mlp GEMM branch, fp16 path off
    "tiny_grid_h1": ("tiny_grid", dict(imag_horizon=1)),       # H = 1
    "tiny_iwae3": ("tiny", dict(iwae_samples=3)),
}
FULL_CASES = {
    "atari": ("atari", {}),                                    # one-hot actor, gather branch, fp16 path
    "dmc": ("dmc", {}),                                        # tanh_normal actor
    "atari_iwae_b16": ("atari_iwae", dict(batch_size=16)),     # N = 50 * 16 * 4 = 3200
    "atari_catreward": ("atari_catreward", {}),
}
CASES = dict(TINY_CASES, **({} if CPU else FULL_CASES))


# ----------------------------------------------------------------------------------------------------------- harness
@pytest.fixture(scope="module", autouse=True)
def op_table():
    """The dry run installs the float32 twins (the grid table carries every op a tiny case uses) as the op table."""
    if CPU:
        from oracle.grid_ops import GridRefOps

        pd_ops.set_ops_for_testing(GridRefOps("cpu"))
    yield
    if CPU:
        pd_ops.set_ops_for_testing(None)


def ws(m, name, *shape, dtype=torch.float32):
    """A workspace buffer the step already wrote (never a fresh one: _buf would allocate a missing key)."""
    assert (name, shape, dtype) in m._ws, f"no workspace buffer {name} {shape} {dtype}"
    return m._buf(name, *shape, dtype=dtype)


def make_model(case, exact=False, **extra):
    preset, over = CASES[case]
    conf = make_conf(preset, device=DEV, **dict(over, **extra))
    m = Dreamer(conf).to(DEV)
    seeded = grid_seeded_state_dict if conf.image_decoder == "dense" else seeded_state_dict
    m.load_state_dict(seeded(m.state_dict(), SEED_W))
    if exact:
        m._ensure_arena()                        # (a new arena comes with a new op table)
        m.fp16_forward = False
        m.ops.set_gemm_impl(1)
        m.ops.set_round_operands(False)
    return conf, m


def run_step(m, conf, seed):
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    obs = synthetic_batch(conf, seed=seed, device=DEV)
    torch.manual_seed(seed + SEED_NOISE)
    noise = {k: v.to(DEV) for k, v in O.draw_noise(conf, T, B, dream_log=True).items()}
    out = m.training_step(obs, m.init_state(B * I), noise=noise, do_dream_tensors=True)
    if not CPU:
        torch.cuda.synchronize()
    return obs, noise, out


class Ctx:
    """What the stage checks share: the model, the rounding the kernels apply, and the per-stage record of
    max(err / bound), of bound / value scale, and of the near-ties."""

    def __init__(self, m, exact):
        self.m, self.d, self.conf = m, m.d, m.conf
        self.exact = exact
        self.round = not CPU and not exact          # producers round to tf32, tensor-core GEMMs read tf32
        self.f16 = m._fp16_forward_ok()
        self.ratio, self.scale, self.ties, self.straddle = {}, {}, {}, {}
        self.ratio_rnd, self.err_ulp, self.worst = {}, {}, {}
        self.stage, self.prefix = "?", ""

    def at(self, stage):
        self.stage = self.prefix + stage

    # weights as the kernel reads them
    def raw(self, p):
        return self.m._raw(p).double()

    def wtc(self, p):
        return self.rtf(self.raw(p))

    def w16(self, p):
        return fp16(self.raw(p))

    def rtf(self, v):
        return tf32_rna(v) if self.round else v

    # recording
    def note(self, lim, ref):
        """The share of the value the bound takes: the median over elements of bound / |value|, over the elements whose
        |value| is at least 1 % of the tensor's rms (a value that cancels to ~0 has no scale of its own)."""
        lim, ref = lim.double().expand_as(ref).reshape(-1), ref.double().reshape(-1)
        a = ref.abs()
        keep = a >= 0.01 * a.pow(2).mean().sqrt()
        sc = float((lim[keep] / a[keep]).median()) if bool(keep.any()) else 0.0
        if sc >= self.scale.get(self.stage, 0.0):
            self.scale[self.stage], self.worst[self.stage] = sc, self.name

    def check(self, name, got, ref, err):
        """An fp32 value the kernel does not round."""
        self.name = name
        r = bound(f"{self.stage}: {name}", got, ref, err)
        self.ratio[self.stage] = max(self.ratio.get(self.stage, 0.0), r)
        self.note(err, ref)

    def check_rnd(self, name, got, ref, err):
        """An fp32 value the kernel stores tf32-rounded (rna) when operand rounding is on.  Then its fp32 error is not
        observable below the rounding: `rounded` requires got == tf32(ref) away from a boundary, the slack against
        err + 1 ulp is recorded apart, and so is the size of the fp32 error term in ulps.  With rounding off (the exact
        arm) the value is held to err alone like any other."""
        if not self.round:
            return self.check(name, got, ref, err)
        assert ((got.float().contiguous().view(torch.int32) & 0x1FFF) == 0).all(), f"{self.stage}: {name} not tf32-rounded"
        self.name = name
        rounded(f"{self.stage}: {name}", got, ref, err, "tf32", self.straddle)
        u = ulp(torch.maximum(ref.abs(), got.double().abs()), -126, 10)
        r = bound(f"{self.stage}: {name}", got, ref, err + u)
        self.ratio_rnd[self.stage] = max(self.ratio_rnd.get(self.stage, 0.0), r)
        self.err_ulp[self.stage] = max(self.err_ulp.get(self.stage, 0.0), float((err / u).max()))
        self.note(err + u, ref)

    def report(self, label):
        print(f"\n[{label}] f16 path {self.f16}, exact arm {self.exact}")
        for s in self.scale:
            line = f"  {s:<32} bound/value {self.scale[s]:.2e} ({self.worst[s]})"
            if s in self.ratio:
                line += f"   max err/bound {self.ratio[s]:.3g}"
            if s in self.ratio_rnd:
                line += f"   tf32-stored: max err/(bound + ulp) {self.ratio_rnd[s]:.3g}, fp32 bound <= {self.err_ulp[s]:.2g} ulp"
            print(line)
        print(f"  near-ties {self.ties}; tf32 values within error of a rounding boundary {sum(self.straddle.values())}")
        for s, v in self.scale.items():
            assert v < VACUOUS, f"{label} {s} {self.worst[s]}: the bound takes {v:.3g} of the value (median over elements)"


def vals(t):
    return t.double()


# ---------------------------------------------------------------------------------------------- reference pieces
def mm(c, A, W, bias=None, res=None, *, f16=False, lda=None, ldb=None, acc=False, exact_ops=False):
    """float64 A @ W^T (+ bias + res) and the error bound of the route pd_gemm / pd_gemm_f16 take for this launch:
    fp16 operands and tf32 launches with 16-byte rows and N, K >= 8 on tensor cores (tc_depth), the rest (and the
    exact arm) on the CUDA-core kernel (simt_depth).  exact_ops: the kernel's operands are known tf32 values."""
    M, K = A.shape
    N = W.shape[0]
    lda = K if lda is None else lda
    ldb = K if ldb is None else ldb
    simt = not f16 and (c.exact or not (lda % 4 == 0 and ldb % 4 == 0 and N >= 8 and K >= 8))
    depth = simt_depth(K) if simt else tc_depth(M, N, cdiv(K, 64 if f16 else 32), acc)[0]
    ref = A @ W.t()
    S = A.abs() @ W.abs().t()
    err = C_ACC * depth * U * S
    if c.round and not simt and not f16 and not exact_ops:
        err = err + operand_err(A, W, S)
    extra = torch.zeros_like(ref)
    if bias is not None:
        ref, extra = ref + bias, extra + bias.abs()
    if res is not None:
        ref, extra = ref + res, extra + res.abs()
    err = err + 2 * U * (S + extra)
    return ref, err


def tf32_trunc(x):
    """The low 13 bits of the fp32 x dropped (float64)."""
    return (x.float().contiguous().view(torch.int32) & -0x2000).view(torch.float32).double()


def operand_err(A, W, S):
    """The error of reading raw fp32 operands as tf32 on the tensor cores, which truncate or round the low 13 bits.  With
    one operand tf32-exact it is the larger of the two actual differences |(t(A) - A) . W^T| (t = truncation or rna
    rounding), plus one tf32 ulp of the elements that sit exactly on a tie (where rn and rna part); otherwise
    TF32_OP * sum |a b| (test_gemm_conv_f64_gpu.py)."""
    a_raw, w_raw = bool((tf32_rna(A) != A).any()), bool((tf32_rna(W) != W).any())
    if a_raw and w_raw:
        return TF32_OP * S
    if not (a_raw or w_raw):
        return torch.zeros_like(S)
    X, Y = (A, W) if a_raw else (W, A)
    ties = ((X.float().contiguous().view(torch.int32) & 0x1FFF) == 0x1000).double() * ulp(X, -126, 10)
    e = torch.maximum(((tf32_trunc(X) - X) @ Y.t()).abs(), ((tf32_rna(X) - X) @ Y.t()).abs()) + ties @ Y.abs().t()
    return e if a_raw else e.t()


def gru_ref(gi, gh, hp):
    """The nn.GRUCell equations in float64 and the bound of pd_gru_fwd's fp32 evaluation on the kernel's gi / gh
    (test_gru_fwd_against_float64)."""
    D = hp.shape[1]
    s = lambda v, j: v[:, j * D:(j + 1) * D]
    r = torch.sigmoid(s(gi, 0) + s(gh, 0))
    u = torch.sigmoid(s(gi, 1) + s(gh, 1))
    ghn = s(gh, 2)
    arg = s(gi, 2) + r * ghn
    n = torch.tanh(arg)
    h = (1 - u) * n + u * hp
    E_r = 4 * U * r + U * (s(gi, 0) + s(gh, 0)).abs() * r * (1 - r)
    E_u = 4 * U * u + U * (s(gi, 1) + s(gh, 1)).abs() * u * (1 - u)
    E_n = (1 - n * n) * (ghn.abs() * E_r + U * ((r * ghn).abs() + arg.abs())) + 3 * U * n.abs()
    E_h = (n - hp).abs() * E_u + (1 - u + E_u) * E_n + 4 * U * (((1 - u) * n).abs() + (u * hp).abs()) + U * u * n.abs()
    return h, E_h


def check_sample(c, name, z, logits, e_logit, noise, G, C):
    """z (one-hot rows of G groups of C) against argmax(p / q) of the float64 softmax of `logits`.  log(p / q) carries
    e_c + max e (the logit bound through the log-softmax) and the kernel's own fp32 softmax and division error
    (softmax_err); a group whose top two scores are within the sum of theirs is a near-tie."""
    M = logits.shape[0]
    z = vals(z).reshape(M, G, C)
    k = z.argmax(-1)
    assert torch.equal(z, F.one_hot(k, C).to(f64)), f"{c.stage}: {name} is not one-hot"
    lp, _, Elp, _ = softmax_err(logits, G, C)
    score = lp - torch.log(noise.double().reshape(M, G, C))
    el = e_logit.reshape(M, G, C)
    es = el + el.amax(-1, keepdim=True) + 2 * Elp + 14 * U
    want = score.argmax(-1)
    near = torch.zeros(M, G, dtype=torch.bool, device=z.device)
    if C > 1:
        top = score.topk(2, -1)
        i0, i1 = top.indices[..., :1], top.indices[..., 1:2]
        near = (top.values[..., 0] - top.values[..., 1]) <= (es.gather(-1, i0) + es.gather(-1, i1))[..., 0]
    wrong = (k != want) & ~near
    assert not wrong.any(), f"{c.stage}: {name}: {int(wrong.sum())} samples differ from argmax(p/q) away from a near-tie"
    n = int(near.sum())
    c.ties[c.stage] = c.ties.get(c.stage, 0) + n
    assert n <= max(2, 0.01 * M * G), f"{c.stage}: {name}: {n} near-ties of {M * G} samples"
    return k


def replay_fwd(c, mp, X32, X16, out_k, name):
    """The step keeps the hidden activations of the reward / terminal / target-critic heads in scratch only: replay the
    head's forward (Dreamer._mlp_fwd on the step's own inputs) into saved buffers; it must reproduce the step's output bit
    for bit, and its activations are then checked layer by layer."""
    m = c.m
    rows = X32.shape[0]
    saved = m._mlp_saved(mp, "replay." + name, rows)
    out = torch.empty_like(out_k)
    m._mlp_fwd(mp, X32, out, saved, x16=X16)
    if not CPU:
        torch.cuda.synchronize()
    assert torch.equal(out, out_k), f"{name}: the replayed head differs from the step's output"
    return saved


def mlp_ref(c, mp, X16, X32, saved, rows, out, out_name):
    """Forward of an MLP of the step (Dreamer._mlp_fwd) in float64, each layer from the kernel's own input to it: X16 /
    X32 the fp16 / fp32 input the kernel read (X16 None off the fp16 path), then the saved activations `saved` (rows
    `rows`); x, y, the LayerNorm statistics of every hidden layer and the output `out` are checked."""
    f16 = X16 is not None
    A, lda, yk = (X16 if f16 else X32), X32.shape[1], None
    for l in range(mp.L):
        W = c.w16(mp.lin[l].weight) if f16 else c.wtc(mp.lin[l].weight)
        gamma, beta = c.raw(mp.ln[l].weight), c.raw(mp.ln[l].bias)
        xs = vals(saved.x[l][rows])
        c.check(f"{out_name} x{l}", xs, *mm(c, A, W, c.raw(mp.lin[l].bias), f16=f16, lda=lda))
        y, mu, r, e_y, e_mu, e_r = ln_fwd_ref(xs, gamma, beta)
        c.check_rnd(f"{out_name} y{l}", saved.y[l][rows], y, e_y)
        c.check(f"{out_name} mean{l}", saved.m[l][rows], mu, e_mu)
        c.check(f"{out_name} rstd{l}", saved.r[l][rows], r, e_r)
        yk = vals(saved.y[l][rows])
        A, lda = (fp16(yk) if f16 else yk), mp.hid
    # the narrow output layer reads the fp32 y (or, without hidden layers, the fp32 input)
    c.check(out_name, out, *mm(c, yk if mp.L else X32, c.wtc(mp.out.weight), c.raw(mp.out.bias), lda=lda))


def replay_cell(c, f_k, f16_k, act_k, aidx, N):
    """One imagination step of the RSSM cell and GRU (the body of Dreamer._dream's loop) restated with the op table on the
    kernel's own inputs of the step (feats[i], its fp16 copy, the sampled action) and the weights as this file reads them:
    a_mlp^T rows (one-hot action, Hd % 4 == 0) or the a_mlp GEMM, z_mlp on the latent columns, LayerNorm+ELU, W_ih and
    W_hh, the GRU gates.  It must reproduce the step's h' bit for bit, which ties the step's wiring to this restatement;
    its intermediates are then each checked in float64."""
    m, d, D = c.m, c.d, c.d.D
    ops = m.ops
    cell = m.wm.core.cell
    gru = cell.gru.layers[0]
    dev = m._arena.device
    e = lambda *shape, dtype=torch.float32: torch.full(shape, float("nan"), dtype=dtype, device=dev)
    f32 = lambda t: t.float().contiguous()
    w = lambda p: c.w16(p).half().contiguous() if c.f16 else f32(c.wtc(p))
    mm_ = lambda a, p, out, **kw: (ops.gemm_f16 if c.f16 else ops.gemm)(a, w(p), out, **kw)
    r = SimpleNamespace(aa=e(N, d.Hd), x=e(N, d.Hd), za=e(N, d.Hd), m=e(N), r=e(N), gi=e(N, 3 * D), gh=e(N, 3 * D),
                        h=e(N, D), za16=e(N, d.Hd, dtype=torch.float16) if c.f16 else None,
                        h16=e(N, D, dtype=torch.float16) if c.f16 else None)
    WaT = f32(c.wtc(cell.a_mlp.weight).t())
    if aidx is not None:
        ops.gather_rows(aidx.to(torch.int32).contiguous(), WaT, r.aa)
    else:
        ops.gemm(act_k, f32(c.wtc(cell.a_mlp.weight)), r.aa)
    x_in = f16_k if c.f16 else f_k
    mm_(x_in[:, D:], cell.z_mlp.weight, r.x, bias=f32(c.raw(cell.z_mlp.bias)), res=r.aa)
    ops.ln_elu_fwd(r.x, f32(c.raw(cell.in_norm.weight)), f32(c.raw(cell.in_norm.bias)), 1e-3, r.za, r.m, r.r, r.za16)
    mm_(r.za16 if c.f16 else r.za, gru.weight_ih, r.gi, bias=f32(c.raw(gru.bias_ih)))
    mm_(x_in[:, :D], gru.weight_hh, r.gh, bias=f32(c.raw(gru.bias_hh)))
    ops.gru_fwd(r.gi, r.gh, f_k[:, :D], r.h, h16=r.h16)
    if not CPU:
        torch.cuda.synchronize()
    return r


def cell_check(c, fx_i, f_i, act, aidx, rc, h_next):
    """aa, x, za (and its LayerNorm statistics), gi, gh and h' of one step, each from the kernel's own input to it."""
    m, d, D = c.m, c.d, c.d.D
    cell = m.wm.core.cell
    gru = cell.gru.layers[0]
    Wa = c.wtc(cell.a_mlp.weight)
    if aidx is not None:
        assert torch.equal(vals(rc.aa), Wa.t()[aidx]), "aa != the a_mlp^T row of the sampled action"
    else:
        c.check("aa", rc.aa, *mm(c, act, Wa, lda=d.A, ldb=d.A))
    Wz = c.w16(cell.z_mlp.weight) if c.f16 else c.wtc(cell.z_mlp.weight)
    c.check("x", rc.x, *mm(c, fx_i[:, D:], Wz, c.raw(cell.z_mlp.bias), vals(rc.aa), f16=c.f16, lda=d.F))
    za, mu, r, e_za, e_mu, e_r = ln_fwd_ref(vals(rc.x), c.raw(cell.in_norm.weight), c.raw(cell.in_norm.bias))
    c.check_rnd("za", rc.za, za, e_za)
    c.check("mean", rc.m, mu, e_mu)
    c.check("rstd", rc.r, r, e_r)
    if c.f16:
        assert torch.equal(vals(rc.za16), fp16(vals(rc.za))), "za16 != fp16(za)"
    za_op = vals(rc.za16) if c.f16 else vals(rc.za)
    Wih = c.w16(gru.weight_ih) if c.f16 else c.wtc(gru.weight_ih)
    Whh = c.w16(gru.weight_hh) if c.f16 else c.wtc(gru.weight_hh)
    c.check("gi", rc.gi, *mm(c, za_op, Wih, c.raw(gru.bias_ih), f16=c.f16))
    c.check("gh", rc.gh, *mm(c, fx_i[:, :D], Whh, c.raw(gru.bias_hh), f16=c.f16, lda=d.F))
    c.check_rnd("h'", h_next, *gru_ref(vals(rc.gi), vals(rc.gh), f_i[:, :D]))


def replay_prior(c, h_k, N):
    """The step keeps the prior head's activations of the last imagination step only: replay the head
    (Dreamer._head_fwd on the kernel's h' of the step, as the step reads it) into test-owned buffers.  At the last step the
    replay must reproduce the step's buffers bit for bit."""
    m, d = c.m, c.d
    dev = m._arena.device
    e = lambda *shape, dtype=torch.float32: torch.full(shape, float("nan"), dtype=dtype, device=dev)
    r = SimpleNamespace(yp=e(N, d.Hd), pp=e(N, d.Hd), m=e(N), r=e(N), prior=e(N, d.Z),
                        pp16=e(N, d.Hd, dtype=torch.float16) if c.f16 else None)
    m._head_fwd(m._rssm_head(prior=True), h_k, r.yp, r.pp, r.m, r.r, r.prior, c.f16, r.pp16)
    if not CPU:
        torch.cuda.synchronize()
    return r


def prior_head_check(c, h, rp):
    """yp, pp, its LayerNorm statistics and the prior logits of one step, each from the kernel's own input to it."""
    d = c.d
    ph, pn, pm = c.m._rssm_head(prior=True)
    Wph = c.w16(ph.weight) if c.f16 else c.wtc(ph.weight)
    Wpm = c.w16(pm.weight) if c.f16 else c.wtc(pm.weight)
    yp_k = vals(rp.yp)
    c.check("yp", yp_k, *mm(c, h, Wph, c.raw(ph.bias), f16=c.f16, lda=d.F))
    pp, mu, r, e_pp, e_mu, e_r = ln_fwd_ref(yp_k, c.raw(pn.weight), c.raw(pn.bias))
    c.check_rnd("pp", rp.pp, pp, e_pp)
    c.check("mean", rp.m, mu, e_mu)
    c.check("rstd", rp.r, r, e_r)
    if c.f16:
        assert torch.equal(vals(rp.pp16), fp16(vals(rp.pp))), "pp16 != fp16(pp)"
    prior_k = vals(rp.prior)
    c.check("prior", prior_k, *mm(c, vals(rp.pp16) if c.f16 else vals(rp.pp), Wpm, c.raw(pm.bias), f16=c.f16))
    return prior_k


# ---------------------------------------------------------------------------------------------- stages 1-4: the dream
def dream_stages(c, tag, N, H, noise_actor, noise_prior):
    m, d, conf = c.m, c.d, c.conf
    cell = m.wm.core.cell
    gru = cell.gru.layers[0]
    ap = m._mlp_params(m.ac.actor)
    D, Z, A = d.D, d.Z, d.A
    feats = vals(ws(m, tag + "feats", H + 1, N, d.F))
    feats_k = ws(m, tag + "feats", H + 1, N, d.F)
    f16buf = ws(m, tag + "feats16", H + 1, N, d.F, dtype=torch.float16) if c.f16 else None
    fx = vals(f16buf) if c.f16 else feats                       # the GEMM operand copy of the features
    alog = ws(m, tag + "dream.alog", H, N, d.Ap)[..., :d.Aout]
    actions = ws(m, tag + "dream.actions", H, N, A)
    for l in range(ap.L):
        for k in ("x", "y"):
            ws(m, f"{tag}actor.{k}{l}", H * N, ap.hid)
        for k in ("m", "r"):
            ws(m, f"{tag}actor.{k}{l}", H * N)
    saved = m._mlp_saved(ap, tag + "actor", H * N)
    onehot = conf.actor_dist == "onehot"
    gather = onehot and d.Hd % 4 == 0
    kact = None

    for i in range(H):
        rows = slice(i * N, (i + 1) * N)
        # 1: actor forward from the saved rows of step i
        c.at("1 actor forward")
        mlp_ref(c, ap, fx[i] if c.f16 else None, feats[i], saved, rows, alog[i], "alog")
        # 2: action sample from the kernel's logits and noise
        c.at("2 action sample")
        al = vals(alog[i])
        if onehot:
            kact = check_sample(c, f"actions[{i}]", actions[i], al, torch.zeros_like(al), noise_actor[i], 1, A)
        else:
            eps = noise_actor[i].double()
            th = torch.tanh(al[:, :A] / 5)
            mu, sd = 5 * th, F.softplus(al[:, A:]) + 0.1
            arg = mu + sd * eps
            a = torch.tanh(arg)
            Emu = 5 * (3 * U * th.abs() + (1 - th * th) * U * (al[:, :A] / 5).abs()) + U * mu.abs()
            c.check(f"actions[{i}]", actions[i], a, (1 - a * a) * (Emu + eps.abs() * 4 * U * sd +
                                                                    2 * U * ((sd * eps).abs() + arg.abs())) + 3 * U * a.abs())
        # 3: cell and GRU, composed from feats[i], the kernel's action and the weights
        c.at("3 cell+GRU every step")
        rc = replay_cell(c, feats_k[i], f16buf[i] if c.f16 else None, actions[i], kact[:, 0] if gather else None, N)
        assert torch.equal(rc.h, feats_k[i + 1][:, :D]), f"h'[{i + 1}]: the replayed cell differs from the step"
        if c.f16:
            assert torch.equal(rc.h16, f16buf[i + 1][:, :D]), f"fp16 h'[{i + 1}]: the replayed cell differs from the step"
        if i == H - 1:
            for n_, t_ in (("aa", rc.aa), ("x", rc.x), ("za", rc.za), ("gi", rc.gi), ("gh", rc.gh)):
                assert torch.equal(t_, ws(m, tag + "dream." + n_, *t_.shape)), f"dream.{n_}: the replayed cell differs"
            if c.f16:
                assert torch.equal(rc.za16, ws(m, tag + "dream.za16", N, d.Hd, dtype=torch.float16)), \
                    "dream.za16: the replayed cell differs"
        cell_check(c, fx[i], feats[i], vals(actions[i]), kact[:, 0] if gather else None, rc, feats[i + 1][:, :D])
        # 4: prior head on the kernel's h' and the latent sample
        c.at("4 prior head every step")
        rp = replay_prior(c, (f16buf if c.f16 else feats_k)[i + 1][:, :D], N)
        if i == H - 1:
            for n_, t_ in (("yp", rp.yp), ("pp", rp.pp), ("m", rp.m), ("r", rp.r), ("prior", rp.prior)):
                shape = t_.shape
                assert torch.equal(t_, ws(m, tag + "dream." + n_, *shape)), f"dream.{n_}: the replayed prior head differs"
            if c.f16:
                assert torch.equal(rp.pp16, ws(m, tag + "dream.pp16", N, d.Hd, dtype=torch.float16)), \
                    "dream.pp16: the replayed prior head differs"
        prior_k = prior_head_check(c, fx[i + 1][:, :D], rp)
        c.at("4 latent sample every step")
        check_sample(c, f"z[{i + 1}]", feats[i + 1][:, D:], prior_k, torch.zeros_like(prior_k), noise_prior[i], d.G, d.C)

    # 4 (every step): feats16 is the fp16 copy of feats, bit for bit
    if c.f16:
        c.at("4 feats16")
        assert torch.equal(vals(f16buf), fp16(feats)), f"{tag}feats16 != fp16(feats)"

    # 3 / 4 (last step): every intermediate the cell and the prior head kept, one by one
    i = H - 1
    return feats, fx, alog, actions, saved


# ---------------------------------------------------------------------------------- stages 5-7: the actor-critic
def ac_stages(c, tag, N, H, feats, fx, alog, actions, metrics=None):
    m, d, conf = c.m, c.d, c.conf
    J = H + 1
    fall, fall16 = feats.view(J * N, d.F), (fx.view(J * N, d.F) if c.f16 else None)
    rp, tp = m._mlp_params(m.wm.decoder.reward.model), m._mlp_params(m.wm.decoder.terminal.model)
    cp, ctp = m._mlp_params(m.ac.critic), m._mlp_params(m.ac.critic_target)
    b = lambda name, *s, **kw: ws(m, tag + name, *s, **kw)
    rew, tlog, vt, v = (b(n, J * N, 1) for n in ("ac.rew", "ac.tlog", "ac.vt", "ac.v"))
    for l in range(cp.L):
        for k in ("x", "y"):
            b(f"critic.{k}{l}", J * N, cp.hid)
        for k in ("m", "r"):
            b(f"critic.{k}{l}", J * N)
    critic = m._mlp_saved(cp, tag + "critic", J * N)
    feats_k = ws(m, tag + "feats", J, N, d.F)
    fx16_k = ws(m, tag + "feats16", J, N, d.F, dtype=torch.float16) if c.f16 else None
    rlog_k = b("ac.rlog", J * N, d.Sp)[:, :d.S] if m._catreward else None

    c.at("5 heads")
    allr = slice(0, J * N)
    f16k, f32k = (fx16_k.view(J * N, d.F) if c.f16 else None), feats_k.view(J * N, d.F)
    heads = {n: replay_fwd(c, mp, f32k, f16k, t, n) for n, mp, t in
             ((("rlog", rp, rlog_k) if m._catreward else ("rew", rp, rew)), ("tlog", tp, tlog), ("vt", ctp, vt))}
    if m._catreward:
        rlog = b("ac.rlog", J * N, d.Sp)[:, :d.S]
        mlp_ref(c, rp, fall16, fall, heads["rlog"], allr, rlog, "rlog")
        y = vals(rlog)
        sup = c.raw(m.wm.decoder.reward._support)
        _, p, _, Ep = softmax_err(y, 1, d.S)
        p, Ep = p[:, 0], Ep[:, 0]
        ref = (p * sup).sum(-1, keepdim=True)
        c.check("expected reward", rew, ref, (Ep * sup.abs()).sum(-1, keepdim=True) +
                (d.S + 2) * U * (p * sup.abs()).sum(-1, keepdim=True))
    else:
        mlp_ref(c, rp, fall16, fall, heads["rew"], allr, rew, "rew")
    mlp_ref(c, tp, fall16, fall, heads["tlog"], allr, tlog, "tlog")
    # the target critic reads the critic_target weights (synced from the critic at the start of a step with gradients)
    mlp_ref(c, ctp, fall16, fall, heads["vt"], allr, vt, "vt")
    mlp_ref(c, cp, fall16, fall, critic, slice(0, J * N), v, "v")

    c.at("6 gae_critic")
    term = b("ac.term", J, N)
    tl = vals(tlog).view(J, N)
    tr = torch.sigmoid(tl)
    c.check("term", term, tr, 4 * U * tr + TINY)
    ref, s_ref, Es = gae_ref(H, N, conf.gamma, conf.lambda_gae, vals(vt), vals(v), vals(rew), vals(term))
    outs = dict(adv=b("ac.adv", H, N), agae=b("ac.agae", H, N), target=b("ac.target", H, N),
                weight=b("ac.weight", H, N), dv=b("ac.dv", H * N, 1).view(H, N))
    for n, (r_, e_) in ref.items():
        c.check(n, outs[n], r_, e_)
    sums = b("ac.sums", 8, dtype=torch.float64)
    vv, rr = vals(v).view(J, N), vals(rew).view(J, N)
    mag = torch.stack([s_ref[0].abs(), vv[0].abs().sum(), vv[:-1].abs().sum(), rr[1:].abs().sum(), (rr[1:] ** 2).sum()]) + 1
    if CPU:
        mag = mag * (H * N * U * 1e12)          # the float32 twin sums in fp32, the kernel in double
    c.check("sums[0:5]", sums[:5], s_ref, Es + 1e-12 * mag)
    agae = vals(outs["agae"])
    kappa = float(vv.abs().max() / agae.pow(2).mean().sqrt().clamp_min(1e-30))

    c.at("7 actor loss")
    rows = H * N
    al = vals(alog).reshape(rows, d.Aout)
    acts = vals(actions).reshape(rows, d.A)
    ag, w = agae.reshape(rows), vals(outs["weight"]).reshape(rows)
    dal = b("ac.dalog", rows, d.Ap)[:, :d.Aout]
    eta = float(torch.tensor(conf.entropy, dtype=torch.float32))
    if conf.actor_dist == "onehot":
        dl_ref, E, per, ent, Erow, Eent = actor_onehot_ref(al, acts, ag, w, eta, rows)
    else:
        dl_ref, E, per, ent, Erow, Eent = actor_tanh_ref(al, acts, ag, w, eta, rows, d.A)
    c.check("dlogits", dal, dl_ref, E)
    c.check("sums[5]", sums[5], per.sum(), Erow.sum() + 1e-12 * (per.abs().sum() + 1) * (rows * U * 1e12 if CPU else 1))
    c.check("sums[6]", sums[6], ent.sum(), Eent.sum() + 1e-12 * (ent.abs().sum() + 1) * (rows * U * 1e12 if CPU else 1))
    if metrics is not None:
        # the returned metrics: float64 of the stage sums, rounded once to fp32 (the std: + its sqrt)
        s, hm = sums.double(), float(rows)
        r_var = torch.clamp((s[4] - s[3] * s[3] / hm) / (hm - 1.0), min=0.0)
        want = dict(loss_critic=s[0] / hm, loss_actor=s[5] / hm, policy_entropy=s[6] / hm, policy_value=s[1] / N,
                    policy_value_im=s[2] / hm, policy_reward=s[3] / hm, policy_reward_std=r_var.sqrt())
        for k_, v_ in want.items():
            c.check(f"metric {k_}", metrics[k_].reshape(()), v_, 2 * U * v_.abs() + TINY)
    return critic, kappa


def actor_onehot_ref(l, acts, ag, w, eta, rows):
    """d loss_actor / d logits of the one-hot actor by autograd, and the bounds of test_actor_loss_onehot."""
    lg = l.clone().requires_grad_(True)
    pi = torch.distributions.OneHotCategorical(logits=lg)
    ent_t = pi.entropy()
    per = (-pi.log_prob(acts) * ag - eta * ent_t) * w
    per.mean().backward()
    A = l.shape[1]
    lp, p, Elp, Ep = (v[:, 0] for v in softmax_err(l, 1, A))
    Eent = (Ep * lp.abs() + p * Elp).sum(-1) + 7 * U * (p * lp.abs()).sum(-1)
    en = ent_t.detach()
    c_ = (w / rows)[:, None]
    E = c_ * (ag.abs()[:, None] * (Ep + U * (acts + p)) + eta * (Ep * (lp + en[:, None]).abs() + p * (Elp + Eent[:, None]))
              + 4 * U * (ag.abs()[:, None] * (acts + p) + eta * p * (lp.abs() + en.abs()[:, None]))) + 2 * U * lg.grad.abs()
    lpa = (lp * acts).sum(-1)
    Erow = w * (ag.abs() * Elp[:, 0] + eta * Eent + 3 * U * ((lpa * ag).abs() + eta * en.abs()))
    return lg.grad, E, per.detach(), en, Erow, Eent


def actor_tanh_ref(out, a, ag, w, eta, rows, A):
    """The tanh_normal actor's gradient by autograd, and the bounds of test_actor_loss_tanh_normal (actions clamped to
    +-(1 - 2^-23) as the kernel does)."""
    ac = a.clamp(-1 + 2.0 ** -23, 1 - 2.0 ** -23)
    og = out.clone().requires_grad_(True)
    mg, sg = og[:, :A], og[:, A:]
    normal = torch.distributions.Independent(torch.distributions.Normal(5 * torch.tanh(mg / 5), F.softplus(sg) + 0.1), 1)
    pi = torch.distributions.TransformedDistribution(normal, [torch.distributions.TanhTransform()])
    per = (-pi.log_prob(ac) * ag - eta * normal.entropy()) * w
    per.mean().backward()
    th = torch.tanh(out[:, :A] / 5)
    mu, sd = 5 * th, F.softplus(out[:, A:]) + 0.1
    x = torch.atanh(ac)
    zc = (x - mu) / sd
    Emu = 5 * (3 * U * th.abs() + (1 - th * th) * U * (out[:, :A] / 5).abs()) + U * mu.abs()
    Esd = 4 * U * sd
    Ezc = (3 * U * x.abs() + Emu + U * (x - mu).abs()) / sd + zc.abs() * (Esd / sd + U)
    c_ = (w / rows)[:, None]
    E_m = c_ * ag.abs()[:, None] * ((Ezc / sd + zc.abs() * Esd / sd ** 2) * (1 - th * th)
                                    + zc.abs() / sd * (5 * U + 2 * U * (out[:, :A] / 5).abs()) + 4 * U * (zc / sd).abs() * (1 - th * th))
    sig = torch.sigmoid(out[:, A:])
    gr = og.grad
    E_s = c_ * sig * (ag.abs()[:, None] * ((2 * zc.abs() * Ezc + (zc * zc + 1) * Esd / sd) / sd + 4 * U * (zc * zc + 1) / sd)
                      + eta * (Esd / sd ** 2 + 2 * U / sd)) + 4 * U * gr[:, A:].abs()
    E = torch.cat([E_m + 2 * U * gr[:, :A].abs(), E_s], 1)
    lpn = -0.5 * zc * zc - sd.log() - 0.5 * math.log(2 * math.pi)
    ladj = 2 * (math.log(2) - x - F.softplus(-2 * x))
    lp_terms = ((zc.abs() * Ezc + Esd / sd + 6 * U * (0.5 * zc * zc + sd.log().abs() + 1 + x.abs()) + 12 * U * x.abs()).sum(-1)
                + A * U * (lpn.abs() + ladj.abs()).sum(-1))
    ent = normal.entropy().detach()
    Eent = (Esd / sd + 3 * U * (sd.log().abs() + 1.5)).sum(-1) + A * U * ent.abs()
    Erow = w * (ag.abs() * lp_terms + eta * Eent) + 3 * U * per.detach().abs()
    return gr, E, per.detach(), ent, Erow, Eent


# --------------------------------------------------------------------------------------------- stage 8: backward
class _Recorder:
    """The op table of a model, recording the gradient each LayerNorm+ELU backward reads (dy) and writes (dx)."""

    def __init__(self, ops):
        self._ops, self.calls = ops, []

    def __getattr__(self, k):
        return getattr(self._ops, k)

    def ln_elu_bwd(self, dy, x, y, gamma, mean, rstd, dx, *rest):
        before = dy.clone()
        self._ops.ln_elu_bwd(dy, x, y, gamma, mean, rstd, dx, *rest)
        self.calls.append((before, dx.clone()))


def mlp_bwd_check(c, mp, X, X_k, dout_k, saved, name):
    """Every parameter gradient of an MLP (Dreamer._mlp_bwd) in float64 from the kernel's output gradient `dout_k` through
    its saved activations (rows [0, rows)).  The step keeps the layer gradients dy / dx in scratch only, so the backward is
    replayed on the step's own buffers with the op table recording them; the replay must reproduce the step's parameter
    gradients bit for bit (every sum of the step is added in a fixed order), and each layer is then checked from the
    recorded gradient it read."""
    m = c.m
    rows, hid = X.shape[0], mp.hid
    params = [mp.out.weight, mp.out.bias] + [q for l in range(mp.L) for q in (mp.lin[l].weight, mp.lin[l].bias,
                                                                   mp.ln[l].weight, mp.ln[l].bias)]
    step = {id(p): m._g(p).clone() for p in params}
    for p in params:
        m._g(p).zero_()
    rec, keep = _Recorder(m.ops), m._ops
    m._ops = rec
    try:
        m._mlp_bwd(mp, X_k, dout_k, saved)
    finally:
        m._ops = keep
    if not CPU:
        torch.cuda.synchronize()
    for p in params:
        assert torch.equal(m._g(p), step[id(p)]), f"{name}: the replayed backward differs from the step's"
    g = lambda p: m._g(p).double()
    sv = lambda s, l: vals(s[l][:rows])
    dout, ld_out = vals(dout_k), dout_k.stride(0)
    inp = sv(saved.y, mp.L - 1) if mp.L else X
    # output layer: dW = dout^T y (accumulated into the zeroed arena), db = column sums of dout
    ref, err = mm(c, dout.t().contiguous(), inp.t().contiguous(), lda=ld_out, ldb=inp.shape[1], acc=True)
    c.check(f"{name} out.weight", g(mp.out.weight), ref, err + U * ref.abs())
    ref = dout.sum(0)
    c.check(f"{name} out.bias", g(mp.out.bias), ref, colsum_depth(rows, mp.out_dim) * U * dout.abs().sum(0) + U * ref.abs())
    W, lda = c.wtc(mp.out.weight), ld_out
    src = dout
    depth_col = ln_col_depth(rows, hid) + 2
    assert len(rec.calls) == mp.L
    for l in reversed(range(mp.L)):
        dy_k, dx_k = (vals(t) for t in rec.calls[mp.L - 1 - l])
        # dy = (gradient below) . W, W read as stored (b_mn)
        c.check(f"{name} dy{l}", dy_k, *mm(c, src, W.t().contiguous(), lda=lda, ldb=hid, exact_ops=l < mp.L - 1))
        gamma = c.raw(mp.ln[l].weight)
        dx, e_dx, g_, xh, terms = ln_bwd_ref(dy_k, torch.zeros_like(dy_k), sv(saved.x, l), sv(saved.y, l), gamma,
                                             sv(saved.m, l), sv(saved.r, l))
        # the row means c1 = mean(dxh), c2 = mean(dxh x^) are fp32 sums of `hid` terms (KS roundings each, as in
        # test_ln_elu_fwd_bwd_against_float64_autograd): an absolute error, which 1e-5 |c| misses where they cancel
        dxh = (g_ * gamma).abs()
        e_dx = e_dx + sv(saved.r, l)[:, None] * KS * U * (dxh.mean(-1, keepdim=True) +
                                                           xh.abs() * (dxh * xh.abs()).mean(-1, keepdim=True))
        c.check_rnd(f"{name} dx{l}", dx_k, dx, e_dx)
        terms["x"] = (dx, e_dx)             # the bias gradient sums dx before it is rounded for storage
        for key, p, pname in (("g", mp.ln[l].weight, f"ln{l}.weight"), ("b", mp.ln[l].bias, f"ln{l}.bias"),
                              ("x", mp.lin[l].bias, f"lin{l}.bias")):
            v_, e_ = terms[key]
            ref = v_.sum(0)
            c.check(f"{name} {pname}", g(p), ref, e_.sum(0) + depth_col * U * v_.abs().sum(0) + U * ref.abs())
        a_in = X if l == 0 else sv(saved.y, l - 1)
        ref, err = mm(c, dx_k.t().contiguous(), a_in.t().contiguous(), lda=hid, ldb=X_k.stride(0) if l == 0 else hid,
                      acc=True)
        c.check(f"{name} lin{l}.weight", g(mp.lin[l].weight), ref, err + U * ref.abs())
        src, W, lda = dx_k, c.wtc(mp.lin[l].weight), hid


def backward_stage(c, N, H, feats, critic):
    m = c.m
    c.at("8 backward")
    fH = feats.view(-1, c.d.F)[:H * N]
    cp, ap = m._mlp_params(m.ac.critic), m._mlp_params(m.ac.actor)
    fH_k = ws(m, "feats", H + 1, N, c.d.F).view(-1, c.d.F)[:H * N]
    mlp_bwd_check(c, cp, fH, fH_k, ws(m, "ac.dv", H * N, 1), critic, "critic")
    actor = m._mlp_saved(ap, "actor", H * N)
    mlp_bwd_check(c, ap, fH, fH_k, ws(m, "ac.dalog", H * N, c.d.Ap)[:, :c.d.Aout], actor, "actor")
    for p in m.ac.critic_target.parameters():
        assert p.grad is None, "critic_target has a gradient"


# ------------------------------------------------------------------------------------------------------- driver
def check_step(c, conf, obs, noise, out, label):
    """Stages 1-9 of one step."""
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    metrics, dream = out[2], out[4]
    feats, fx, alog, actions, _ = dream_stages(c, "", N, H, noise["actor"], noise["prior"])
    critic, kappa = ac_stages(c, "", N, H, feats, fx, alog, actions, metrics)
    backward_stage(c, N, H, feats, critic)
    c.report(label)
    print(f"  kappa = max|V| / rms(agae) = {kappa:.3g}")
    # 9: the logging dream from the first posterior state of each sequence (B rows, T - 1 steps)
    Hl = T - 1
    fl0 = ws(c.m, "dl.feats", Hl + 1, B, c.d.F)[0]
    assert torch.equal(fl0, ws(c.m, "feats", H + 1, N, c.d.F)[0][0:B * I:I]), "dl.feats[0] != the first posterior states"
    c.ratio, c.scale, c.ties, c.ratio_rnd, c.err_ulp, c.worst, c.prefix = {}, {}, {}, {}, {}, {}, "9 dl "
    flf, flx, fla, flac, _ = dream_stages(c, "dl.", B, Hl, noise["dream_log_actor"], noise["dream_log_prior"])
    ac_stages(c, "dl.", B, Hl, flf, flx, fla, flac)
    c.at("dream tensors")
    J = Hl + 1
    b = lambda name, *s: ws(c.m, "dl." + name, *s)
    for k_, buf in (("value", b("ac.v", J * B, 1).view(J, B)), ("reward_pred", b("ac.rew", J * B, 1).view(J, B)),
                    ("terminal_pred", b("ac.term", J, B)), ("value_target", b("ac.target", Hl, B)),
                    ("value_advantage", b("ac.adv", Hl, B)), ("value_advantage_gae", b("ac.agae", Hl, B)),
                    ("value_weight", b("ac.weight", Hl, B))):
        assert torch.equal(dream[k_], buf), f"dream tensor {k_} is not the logging dream's buffer"
    assert torch.equal(dream["action_pred"][1:], b("dream.actions", Hl, B, c.d.A)), "action_pred[1:] != dl.dream.actions"
    assert torch.equal(dream["action_pred"][:1], obs["action"][:1]), "action_pred[0] != the first observed action"
    c.report(label + ", logging dream")
    return kappa


@gpu
@pytest.mark.parametrize("case", list(CASES))
def test_imagination_stages(case):
    conf, m = make_model(case)
    obs, noise, out = run_step(m, conf, SEED_DATA)
    c = Ctx(m, exact=False)
    # the branches the case exists for
    if case == "tiny_hd42":
        assert not c.f16 and m.d.Hd % 4 != 0
    if case in ("tiny", "atari"):
        assert c.f16 and m.d.Hd % 4 == 0 and conf.actor_dist == "onehot"
    check_step(c, conf, obs, noise, out, case)


@gpu
@pytest.mark.parametrize("case", ["tiny"] + ([] if CPU else ["atari"]))
def test_imagination_stages_exact_arm(case):
    """CUDA-core fp32 GEMMs, no operand rounding, fp16 forward off: the same stages held to fp32-only bounds."""
    conf, m = make_model(case, exact=True)
    try:
        obs, noise, out = run_step(m, conf, SEED_DATA)
        check_step(Ctx(m, exact=True), conf, obs, noise, out, case + " exact")
    finally:
        m.ops.set_gemm_impl(0)
        m.ops.set_round_operands(True)


@gpu
@pytest.mark.parametrize("interval", [1, 2], ids=lambda v: f"target_interval{v}")
@pytest.mark.parametrize("case", ["tiny", "tiny_dmc"] + ([] if CPU else ["atari"]))
def test_imagination_stages_after_optimizer_step(case, interval):
    """grad_clip and the four optimizer steps, then a second step: every stage again against the updated master weights,
    so a shadow arena, a_mlp^T or critic_target left stale by the update fails.  target_interval = 1 syncs the target
    critic to the updated critic at the second step; 2 keeps the first step's copy, so there the target critic and the
    critic differ and a head reading the wrong one fails."""
    conf, m = make_model(case, target_interval=interval)
    opts = m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    run_step(m, conf, SEED_DATA)
    before = m._arena.clone()
    m.grad_clip(conf.grad_clip, conf.grad_clip_ac)
    for o in opts:
        o.step()
    for gid in ("wm", "actor", "critic"):
        a, b_ = m._group_range[gid]
        assert not torch.equal(m._arena[a:b_], before[a:b_]), f"the {gid} optimizer step changed nothing"
    obs, noise, out = run_step(m, conf, SEED_DATA + 1)
    tg, cr = m._group_slice("target", m._arena), m._group_slice("critic", m._arena)
    if interval == 1:
        assert torch.equal(tg, cr), "critic_target was not synced to the updated critic"
    else:
        assert torch.equal(tg, m._group_slice("critic", before)) and not torch.equal(tg, cr), \
            "critic_target is not the copy of the first step"
    check_step(Ctx(m, exact=False), conf, obs, noise, out, f"{case} after an optimizer step, target_interval {interval}")

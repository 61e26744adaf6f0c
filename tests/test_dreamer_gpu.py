"""GPU parity of the full drop-in module (CUDA kernels through the C ABI) against the committed reference
goldens and the oracle.

  * exact arm  (SIMT fp32 GEMM, operand rounding off): must reproduce the reference's losses / metrics / gradient
    norms within 2e-4 and the sampled categorical indices bit-exactly;
  * product arm (tensor-core TF32 GEMM, rna operand rounding): compared with the oracle TEACHER-FORCED on the indices /
    actions the GPU run sampled (SURVEY.md §7 'bit-exact categorical indices'): 1e-3 relative on losses, 3e-3 on
    per-tensor gradient norms (north_star tolerance 1e-3 on outputs; gradients of tiny tensors are noisier);
    the number of free-running index flips is reported."""
import pytest
import torch

from oracle import dreamer_oracle as O
from pydreamer_b200.dreamer import Dreamer
from tests.util import CASES, build_case, seeded_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_gpu(case, impl, rounding, persistent=False):
    fx, conf, obs, state, noise = build_case(case, DEV)
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    model.persistent_rssm = persistent        # posterior unroll as one cooperative kernel (pd_rssm_unroll_fwd)
    model.persistent_bptt = persistent        # ... and its BPTT as one cooperative kernel (pd_rssm_unroll_bwd)
    model.fp16_forward = (impl == 0)          # the exact arm keeps every GEMM in fp32
    model.implicit_conv = (impl == 0)         # ... and uses the explicit im2col + SIMT GEMM path
    model._ensure_arena()
    model.ops.set_gemm_impl(impl)
    model.ops.set_round_operands(rounding)
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    n0 = model.ops.launch_count()
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    assert model.ops.launch_count() - n0 > 100          # the native kernels really ran
    return fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors


@pytest.mark.parametrize("case", CASES)
def test_exact_arm_matches_reference_golden(case):
    fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors = run_gpu(case, impl=1, rounding=False)
    check_exact_arm(fx, conf, model, losses, metrics, tensors)


def check_exact_arm(fx, conf, model, losses, metrics, tensors):
    """The exact arm's step (SIMT fp32 GEMM, no operand rounding) against the reference's committed outputs."""
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-5 * max(1.0, abs(want)), (got, want)
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= 2e-4 * max(1.0, abs(want)), k
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        assert abs(got - want) <= 1e-3 * max(want, 1e-6) + 1e-9, (k, got, want)
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    idx = model._buf("rssm.idx", T, B * I, conf.stoch_dim, dtype=torch.int32)
    assert idx[0].reshape(-1).tolist() == fx["post_sample_indices_t0"]        # bit-exact sampled indices
    assert int(idx.sum()) == fx["post_sample_index_sum"]
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= 3e-4 * max(want, 1e-6), (k, got, want)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
@pytest.mark.parametrize("case", CASES)
def test_product_arm_tcgen05_teacher_forced_against_oracle(case, persistent):
    fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors = run_gpu(case, impl=0, rounding=True,
                                                                                      persistent=persistent)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples) == persistent
    assert model._persistent_bptt_ok(conf.batch_size * conf.iwae_samples) == persistent
    check_teacher_forced_against_oracle(case, conf, obs, state, noise, model, losses, metrics, tensors)


def check_teacher_forced_against_oracle(case, conf, obs, state, noise, model, losses, metrics, tensors, target_synced=True,
                                        tol=1.0):
    """The step's losses, metrics, every parameter gradient, the reconstructed image and the posterior logits (read from
    `model` after the four backward calls) against the oracle on the same weights, inputs and noise, teacher-forced on the
    posterior / prior indices and the actions the GPU sampled.  target_synced: the step copied the critic to its target
    first (a2c.py:76-79).  tol scales every tolerance (1: those of the TF32 product arm)."""
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    N, G, C, D = T * B * I, conf.stoch_dim, conf.stoch_discrete, conf.deter_dim
    post_idx = model._buf("rssm.idx", T, B * I, G, dtype=torch.int32).long().cpu()
    feats = model._buf("feats", H + 1, N, D + G * C).cpu()
    prior_idx = feats[1:, :, D:].reshape(H, N, G, C).argmax(-1)
    actions = model._buf("dream.actions", H, N, conf.action_dim).cpu()
    sd = {k: v.detach().cpu().clone().requires_grad_(not k.startswith("ac.critic_target"))
          for k, v in model.state_dict().items()}
    cpu = lambda d: {k: v.cpu() for k, v in d.items()}
    free = O.training_step({k: v.detach() for k, v in sd.items()}, conf, cpu(obs), tuple(s.cpu() for s in state), cpu(noise))
    flips = int((free["inter"]["post_idx"] != post_idx).sum())
    print(f"[{case}] free-running posterior index flips under TF32: {flips} / {post_idx.numel()}")
    res = O.training_step(sd, conf, cpu(obs), tuple(s.cpu() for s in state), cpu(noise),
                          force=dict(post_idx=post_idx, actor=actions, prior_idx=prior_idx), target_synced=target_synced)
    for l in res["losses"]:
        l.backward()
    for i, (got, want) in enumerate(zip(losses, res["losses"])):
        g, w = float(got.detach().reshape(-1)[0]), float(want.detach().reshape(-1)[0])
        assert abs(g - w) <= tol * 1e-3 * max(1.0, abs(w)), (i, g, w)
    for k, want in res["metrics"].items():
        assert abs(float(metrics[k]) - float(want)) <= tol * 2e-3 * max(1.0, abs(float(want))), k
    named = dict(model.named_parameters())
    worst = ("", 0.0)
    for k, v in sd.items():
        if v.grad is None:
            continue
        w, g = float(v.grad.double().norm()), float(named[k].grad.double().norm())
        err = abs(g - w) / max(w, 1e-6)
        worst = max(worst, (k, err), key=lambda t: t[1])
        dot = float((named[k].grad.double().cpu() * v.grad.double()).sum()) / max(w * max(g, 1e-12), 1e-12)
        assert err <= tol * (3e-3 + 1e-7 / max(w, 1e-12)), (k, g, w)
        if w > 1e-6:
            assert dot > 0.999, (k, dot)       # direction of every gradient tensor
    print(f"[{case}] worst grad-norm rel err {worst[1]:.2e} ({worst[0]})")
    rel = lambda a, b: ((a.double().cpu() - b.double()).abs().max() / (b.double().abs().max() + 1e-12)).item()
    assert rel(tensors["image_rec"], res["tensors"]["image_rec"]) < tol * 2e-3
    assert rel(model._buf("rssm.post", T, B * I, G * C), res["inter"]["posts"]) < tol * 2e-3


def test_optimizer_step_and_second_step_on_gpu():
    fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors = run_gpu("tiny_onehot", 0, True)
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    before = model.wm.core.cell.z_mlp.weight.detach().clone()
    norms = model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
    for o in opts:
        o.step()
    assert float(norms["grad_norm"]) > 0 and not torch.equal(before, model.wm.core.cell.z_mlp.weight.detach())
    losses2, out_state2, *_ = model.training_step(obs, out_state)           # internally drawn noise
    for l in losses2:
        l.backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(l).all() for l in losses2)


@pytest.mark.parametrize("case", ("tiny_onehot_log", "tiny_dmc_log", "tiny_iwae3_log"))
def test_logging_eval_and_inference_branches_on_gpu(case):
    """do_image_pred + do_dream_tensors, open-loop evaluation and inference() through the native kernels (tensor-core TF32
    product arm) against the reference's committed outputs.  Tolerance 2e-3 (TF32 operands; sums over tensors)."""
    from tests.test_dreamer_cpu import check_log_case, run_log_case
    fx, conf, out = run_log_case(case, DEV)
    check_log_case(fx, conf, out, 2e-3)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
def test_full_atari_shape_subbatch_parity_with_oracle(persistent):
    """BASELINE.json configs[1] at FULL size (T=B=50, deter 2048, stoch 32x32, H=15) on the product arm.  Sequences of a
    batch are independent (every loss is a batch mean), so the oracle re-runs just the first 2 sequences on the CPU with the
    same weights, the matching noise slices and the GPU's sampled indices (teacher forcing) and must reproduce the
    per-(t,b) tensors of those sequences: 2e-3 relative (TF32 / fp16-forward operands through a 50-step recurrence)."""
    from pydreamer_b200.config import make_conf
    from pydreamer_b200.replay import synthetic_batch
    from oracle.weights import seeded_state_dict

    conf = make_conf("atari", device=DEV)
    T, B, I, H = conf.batch_length, conf.batch_size, 1, conf.imag_horizon
    D, G, C, A = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete, conf.action_dim
    Z, N = G * C, T * B
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
    model.persistent_rssm = persistent
    obs = synthetic_batch(conf, seed=77, device=DEV)
    state = (torch.tanh(torch.randn(B, D, device=DEV)), torch.zeros(B, Z, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(5)
    noise = dict(post=torch.empty(T, B, Z, device=DEV).exponential_(generator=g),
                 actor=torch.empty(H, N, A, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(l).all() for l in losses)
    assert float(metrics["loss_kl"]) >= 0 and 0 < float(metrics["entropy_post"]) <= G * torch.log(torch.tensor(float(C))) + 1e-3
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.requires_grad)
    # ---- oracle on the first S sequences
    S = 2
    sub = lambda x: x[:, :S].contiguous().cpu()
    obs_s = {k: sub(v) for k, v in obs.items()}
    rows = lambda x: x.view(H, T, B, -1)[:, :, :S].reshape(H, T * S, -1).cpu()
    noise_s = dict(post=sub(noise["post"]), actor=rows(noise["actor"]), prior=rows(noise["prior"]))
    post_idx = model._buf("rssm.idx", T, B, G, dtype=torch.int32)[:, :S].long().cpu()
    feats = model._buf("feats", H + 1, N, D + Z)
    prior_idx = feats[1:, :, D:].reshape(H, T, B, G, C)[:, :, :S].argmax(-1).reshape(H, T * S, G).cpu()
    actions = rows(model._buf("dream.actions", H, N, A))
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    res = O.training_step(sd, conf, obs_s, (state[0][:S].cpu(), state[1][:S].cpu()), noise_s,
                          force=dict(post_idx=post_idx, actor=actions, prior_idx=prior_idx))
    rel = lambda a, b: ((a.double().cpu() - b.double()).abs().max() / (b.double().abs().max() + 1e-12)).item()
    worst = {}
    for k in ("loss_image", "loss_kl", "reward_rec", "terminal_rec", "entropy_prior", "entropy_post", "policy_value", "image_rec"):
        worst[k] = rel(tensors[k][:, :S], res["tensors"][k])
    worst["posts"] = rel(model._buf("rssm.post", T, B, Z)[:, :S], res["inter"]["posts"])
    worst["dream_features_h"] = rel(feats.view(H + 1, T, B, D + Z)[:, :, :S, :D].reshape(H + 1, T * S, D), res["inter"]["dream_features"][..., :D])
    print("full-size sub-batch parity, max rel err per tensor:", {k: f"{v:.1e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v < 2e-3, (k, v)


@pytest.mark.parametrize("preset", ("atari", "atari_iwae"), ids=("atari", "atari_iwae4_BI200"))
def test_persistent_rssm_kernel_matches_the_per_step_chain_at_full_size(preset):
    """pd_rssm_unroll_fwd (one cooperative kernel, fp16 mma.sync) against the chain of per-timestep launches (TF32
    tensor-core GEMMs) on the Atari shape, same weights / batch / noise: both round operands to 10 mantissa bits, so logits agree to
    accumulation order and the sampled indices are the same except at numerical near-ties.  `atari_iwae` (B=50 x 4 samples
    = 200 batch rows) exercises the kernel's batch-row blocks (4 blocks of 64) and strided row owners (200 rows > 132 CTAs)."""
    from pydreamer_b200.config import make_conf
    from pydreamer_b200.replay import synthetic_batch
    from oracle.weights import seeded_state_dict

    conf = make_conf(preset, device=DEV)
    T, B, H, I = conf.batch_length, conf.batch_size * conf.iwae_samples, conf.imag_horizon, conf.iwae_samples
    D, G, C, A = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete, conf.action_dim
    Z, N, Hd = G * C, T * B, conf.hidden_dim
    obs = synthetic_batch(conf, seed=3, device=DEV)
    state = (torch.tanh(torch.randn(B, D, device=DEV)), torch.zeros(B, Z, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(9)
    noise = dict(post=torch.empty(T, B, Z, device=DEV).exponential_(generator=g),
                 actor=torch.empty(H, N, A, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    got = {}
    for mode in (False, True):
        model = Dreamer(conf).to(DEV)
        model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
        model.persistent_rssm = mode
        with torch.no_grad():
            model.training_step(obs, state, noise=noise)
        torch.cuda.synchronize()
        assert model._persistent_rssm_ok(B) == mode
        names = dict(post=("rssm.post", (T, B, Z)), x1=("rssm.x1", (T, B, Hd)), za=("rssm.za", (T, B, Hd)),
                     y2=("rssm.y2", (T, B, Hd)), pin=("rssm.pin", (T, B, Hd)), gates=("rssm.gates", (T, B, 4 * D)),
                     hin=("rssm.hin", (T, B, D)), zin=("rssm.zin", (T, B, Z)), m1=("rssm.m1", (T, B)), r2=("rssm.r2", (T, B)))
        got[mode] = {k: model._buf(n, *shp).clone() for k, (n, shp) in names.items()}
        got[mode]["idx"] = model._buf("rssm.idx", T, B, G, dtype=torch.int32).clone()
        got[mode]["feat"] = model._buf("feats", H + 1, N, D + Z)[0].view(T, B, D + Z).clone()
        del model
    a, b = got[False], got[True]
    same = (a["idx"] == b["idx"]).all(-1)                      # (T, B): all 32 groups agree
    alive = torch.cumprod(same.long(), 0).bool()               # sequences still on the same trajectory at step t
    frac = float(alive.float().mean())
    print(f"persistent vs chain: identical-trajectory fraction {frac:.4f}; first step all-equal: {bool(same[0].all())}")
    assert bool(same[0].all()) and frac > 0.9
    # wherever the two runs are still on the same trajectory, every saved activation agrees
    prev_alive = torch.cat([torch.ones_like(alive[:1]), alive[:-1]], 0)
    for k in ("x1", "za", "gates", "hin", "zin", "y2", "pin", "post", "feat", "m1", "r2"):
        x, y = a[k][prev_alive].double(), b[k][prev_alive].double()
        if k == "feat":
            x, y = x[..., :D], y[..., :D]
        err = float((x - y).abs().max() / (x.abs().max() + 1e-12))
        assert err < 2e-3, (k, err)


@pytest.mark.parametrize("preset,over", (("atari", {}), ("dmc", {}), ("atari_iwae", dict(batch_size=16))),
                         ids=("atari", "dmc", "atari_iwae4_b16"))
def test_persistent_bptt_kernel_matches_the_per_step_chain_at_full_size(preset, over):
    """pd_rssm_unroll_bwd (one cooperative kernel: TMA-staged fp16 weight tiles, tf32 mma.sync) against the chain of
    per-timestep launches (TF32 tensor-core GEMMs + row-wise kernels) on the SAME forward pass: both contract 10-bit operands,
    so every tensor the kernel writes agrees with the chain's to accumulation order and weight rounding (fp16 vs tf32
    rounding of the same master weight)."""
    from pydreamer_b200.config import make_conf
    from pydreamer_b200.replay import synthetic_batch
    from oracle.weights import seeded_state_dict

    conf = make_conf(preset, device=DEV, **over)
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    D, G, C, A = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete, conf.action_dim
    Z, BI, N, Hd = G * C, B * I, T * B * I, conf.hidden_dim
    obs = synthetic_batch(conf, seed=3, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(9)
    state = (torch.tanh(torch.randn(BI, D, device=DEV, generator=g)), torch.zeros(BI, Z, device=DEV))
    noise = dict(post=torch.empty(T, BI, Z, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    noise["actor"] = (torch.empty(H, N, A, device=DEV).exponential_(generator=g) if conf.actor_dist == "onehot"
                      else torch.empty(H, N, A, device=DEV).normal_(generator=g))
    got = {}
    for mode in (False, True):
        model = Dreamer(conf).to(DEV)
        model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
        model.persistent_bptt = mode                           # opt-in switch (PD_B200_PERSISTENT_BPTT)
        losses, *_ = model.training_step(obs, state, noise=noise)
        for l in losses:
            l.backward()
        torch.cuda.synchronize()
        assert model._persistent_bptt_ok(BI) == mode
        names = dict(dpost=("bwd.dpost", (T, BI, Z)), dy2=("bwd.dy2", (T, BI, Hd)), dgi=("bwd.dgi", (T, BI, 3 * D)),
                     dgh=("bwd.dgh", (T, BI, 3 * D)), dx1=("bwd.dx1", (T, BI, Hd)))
        got[mode] = {k: model._buf(n, *shp).clone() for k, (n, shp) in names.items()}
        got[mode]["idx"] = model._buf("rssm.idx", T, BI, G, dtype=torch.int32).clone()
        cell = model.wm.core.cell
        got[mode]["grads"] = {k: p.grad.detach().clone() for k, p in model.named_parameters()
                              if k.startswith("wm.core.") or k.startswith("wm.encoder.")}
        del model
    a, b = got[False], got[True]
    assert torch.equal(a["idx"], b["idx"])                     # same forward pass, same samples
    worst = {}
    for k in ("dpost", "dy2", "dgi", "dgh", "dx1"):
        x, y = a[k].double(), b[k].double()
        worst[k] = (float((x - y).norm() / (x.norm() + 1e-30)), float((x - y).abs().max() / (x.abs().max() + 1e-30)))
    gw = {}
    for k in a["grads"]:
        x, y = a["grads"][k].double(), b["grads"][k].double()
        gw[k] = float((x - y).norm() / (x.norm() + 1e-30))
    kworst = max(gw, key=gw.get)
    print(f"[{preset}] persistent BPTT vs chain (l2-relative, worst-element/max):", {k: f"{v[0]:.1e}/{v[1]:.1e}" for k, v in worst.items()},
          f"; worst parameter gradient {kworst} {gw[kworst]:.1e}")
    for k, (l2, mx) in worst.items():
        assert l2 < 1e-3 and mx < 3e-3, (k, l2, mx)
    for k, v in gw.items():
        assert v < 1.5e-3, (k, v)

"""Host-side composition + hand-written backward of pydreamer_b200.Dreamer, checked on CPU.

The module is run on the reference op table (oracle/ref_ops.py, plain torch) instead of the CUDA kernels, so
this isolates the schedule written in pydreamer_b200/dreamer.py (what feeds what, the manual BPTT, gradient
routing to the four optimizers) from the kernels themselves (tests/test_kernels_gpu.py).  Expected values are
the committed outputs of the unmodified reference (tests/golden).  Tolerance: 2e-4 relative."""
import pytest
import torch

from oracle.ref_ops import RefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.dreamer import Dreamer
from tests.util import CASES, build_case, seeded_weights


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(RefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def run_model(case, fp16_forward=False, persistent_rssm=False, persistent_bptt=False):
    fx, conf, obs, state, noise = build_case(case)
    model = Dreamer(conf)
    model.fp16_forward = fp16_forward
    model.persistent_rssm = persistent_rssm
    model.persistent_bptt = persistent_bptt
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    losses, out_state, metrics, tensors, dream = model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    for l in losses:
        l.backward()
    return fx, conf, model, opts, losses, out_state, metrics, tensors


@pytest.mark.parametrize("case", CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case)
    check_golden(fx, model, losses, out_state, metrics, tensors)


def check_golden(fx, model, losses, out_state, metrics, tensors):
    """A step run on the reference op table (fp32 throughout) against the reference's committed outputs: 2e-4 relative."""
    assert [tuple(l.shape) for l in losses] == [(), (1,), (), ()]          # SURVEY.md App. E
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 2e-5 * max(1.0, abs(want))
    assert set(metrics) == set(fx["metrics"])
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= 2e-4 * max(1.0, abs(want)), k
    assert set(tensors) == set(fx["tensor_sums"])
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= 2e-4 * max(want, 1e-6), (k, got, want)
    named = dict(model.named_parameters())
    assert {k for k, p in named.items() if p.requires_grad} == set(fx["grad_norms"])
    worst = ("", 0.0)
    for k, want in fx["grad_norms"].items():
        g = named[k].grad
        assert g is not None, k
        got = float(g.double().norm())
        err = abs(got - want) / max(want, 1e-6)
        if err > worst[1]:
            worst = (k, err)
        assert abs(got - want) <= 2e-4 * max(want, 1e-6) + 1e-9, (k, got, want)
        assert abs(float(g.double().sum()) - fx["grad_sums"][k]) <= 5e-4 * max(want, 1e-6) * g.numel() ** 0.5 + 1e-8, k
    assert not out_state[0].requires_grad and abs(float(out_state[0].double().sum()) - fx["out_state_h_sum"]) < 1e-3
    assert all(p.grad is None for p in model.ac.critic_target.parameters())


def test_fp16_forward_plumbing_stays_within_tolerance(ref_ops):
    """Imagination rollout / dreamed-feature heads with fp16 GEMM operands (forward-only layers): same schedule, fp16
    copies of activations and weights; the posterior samples are untouched, actor/critic losses move by < 2e-3."""
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model("tiny_onehot", fp16_forward=True)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= (5e-5 if i < 2 else 5e-3) * max(1.0, abs(want)), (i, got, want)
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        if k.startswith("wm."):                       # world-model gradients do not depend on the dream
            assert abs(float(named[k].grad.double().norm()) - want) <= 2e-4 * max(want, 1e-6) + 1e-9, k


@pytest.mark.parametrize("case", CASES)
def test_persistent_rssm_branch_of_the_schedule(ref_ops, case):
    """The host branch that hands the whole posterior unroll to ONE call (pd_rssm_unroll_fwd on the GPU, its torch twin
    here): same goldens; fp16-rounded operands in the recurrence move losses by < 2e-3 and may flip a near-tie sample."""
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case, fp16_forward=True, persistent_rssm=True)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples)
    T, BI = conf.batch_length, conf.batch_size * conf.iwae_samples
    assert ("rssm.gi", (T, BI, 3 * conf.deter_dim), torch.float32) not in model._ws      # the per-step chain did not run
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-3 * max(1.0, abs(want)), (i, got, want)
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        if k.startswith("wm.") and want > 1e-6:
            assert abs(float(named[k].grad.double().norm()) - want) <= 2e-2 * want + 1e-7, k


@pytest.mark.parametrize("case", CASES)
def test_persistent_bptt_branch_of_the_schedule(ref_ops, case):
    """The host branch that hands BPTT through the posterior unroll to ONE call (pd_rssm_unroll_bwd on the GPU, its torch
    twin here): same goldens; the recurrent weights enter as transposed fp16 copies (10 mantissa bits, like the TF32 chain
    on the GPU), which moves world-model gradients by < 2e-3."""
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case, persistent_bptt=True)
    T, BI = conf.batch_length, conf.batch_size * conf.iwae_samples
    assert model._persistent_bptt_ok(BI)
    assert ("bwd.dhin", (T, BI, conf.deter_dim), torch.float32) in model._ws                 # allocated ...
    assert float(model._buf("bwd.dpost", T, BI, conf.stoch_dim * conf.stoch_discrete).abs().sum()) > 0
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 2e-5 * max(1.0, abs(want)), (i, got, want)
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        tol = 2e-3 if k.startswith("wm.") else 2e-4
        assert abs(got - want) <= tol * max(want, 1e-6) + 1e-8, (k, got, want)


def test_state_dict_roundtrip_and_grad_clip_and_optimizer(ref_ops):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model("tiny_onehot")
    sd = model.state_dict()
    assert "wm.core.cell.gru.layers.0.weight_hh" in sd and "ac.critic_target.model.12.bias" in sd
    assert "probe_model.dummy" in sd and "wm.decoder.image.model.8.weight" in sd
    # torch reference for clip + AdamW on a copy of params/grads
    named = dict(model.named_parameters())
    groups = dict(wm=list(model.wm.parameters()), actor=list(model.ac.actor.parameters()),
                  critic=list(model.ac.critic.parameters()))
    clones = {g: [torch.nn.Parameter(p.detach().clone()) for p in ps] for g, ps in groups.items()}
    for g, ps in groups.items():
        for c, p in zip(clones[g], ps):
            c.grad = p.grad.detach().clone()
    norms = model.grad_clip(0.5, 0.01)           # tiny thresholds so that clipping is active
    assert set(norms) == {"grad_norm", "grad_norm_probe", "grad_norm_actor", "grad_norm_critic"}
    tn = {g: torch.nn.utils.clip_grad_norm_(clones[g], 0.5 if g == "wm" else 0.01) for g in clones}
    assert abs(float(norms["grad_norm"]) - float(tn["wm"])) <= 1e-4 * float(tn["wm"])
    assert abs(float(norms["grad_norm_actor"]) - float(tn["actor"])) <= 1e-4 * float(tn["actor"])
    topts = dict(wm=torch.optim.AdamW(clones["wm"], lr=conf.adam_lr, eps=conf.adam_eps),
                 actor=torch.optim.AdamW(clones["actor"], lr=conf.adam_lr_actor, eps=conf.adam_eps),
                 critic=torch.optim.AdamW(clones["critic"], lr=conf.adam_lr_critic, eps=conf.adam_eps))
    for o in opts:
        o.step()
    for o in topts.values():
        o.step()
    for g, ps in groups.items():
        for c, p in zip(clones[g], ps):
            assert torch.allclose(c.detach(), p.detach(), rtol=1e-5, atol=1e-7), g
    # second step reuses the workspace, carries state, target critic no longer synced
    fx2, conf2, obs, state, noise = build_case("tiny_onehot")
    losses2, out_state2, *_ = model.training_step(obs, out_state, noise=noise)
    assert all(torch.isfinite(l).all() for l in losses2)
    assert model.ac.train_steps == 2


def test_no_grad_mode_skips_backward_and_unsupported_configs_raise(ref_ops):
    fx, conf, obs, state, noise = build_case("tiny_onehot")
    model = Dreamer(conf)
    with torch.no_grad():
        losses, *_ = model.training_step(obs, state, noise=noise)
    assert not losses[0].requires_grad and model.ac.train_steps == 0
    from pydreamer_b200.config import make_conf
    for bad in (dict(gru_type="gru_layernorm"), dict(image_encoder="dense"), dict(actor_grad="dynamics"),
                dict(probe_model="map"), dict(stoch_discrete=0)):
        with pytest.raises(NotImplementedError):
            Dreamer(make_conf("tiny", **bad))
    with pytest.raises(NotImplementedError):
        model.training_step(obs, state, do_open_loop=True)          # evaluation branch: only under no_grad


LOG_CASES = ("tiny_onehot_log", "tiny_dmc_log", "tiny_iwae3_log")


def check_sums(got, want, rtol=3e-4, what=""):
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    for k, (sm, ab, shape) in want.items():
        g = got[k].double()
        assert list(g.shape) == shape, (what, k, list(g.shape), shape)
        assert abs(float(g.abs().nansum()) - ab) <= rtol * max(ab, 1e-6) + 1e-5, (what, k, float(g.abs().nansum()), ab)
        assert abs(float(g.nansum()) - sm) <= rtol * max(ab, 1e-6) + 1e-5, (what, k)


def run_log_case(case, device="cpu"):
    """Shared by the CPU (reference op table) and GPU (native kernels) tests."""
    import torch
    from oracle import dreamer_oracle as O
    from tests.util import load_fixture
    from pydreamer_b200.config import make_conf
    from pydreamer_b200.replay import synthetic_batch
    fx = load_fixture(case)
    conf = make_conf(fx["preset"], device=str(device), **fx["overrides"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    mv = lambda d_: {k: v.to(device) for k, v in d_.items()}
    obs = mv(synthetic_batch(conf, seed=fx["seeds"]["data"]))
    g = torch.Generator().manual_seed(fx["seeds"]["state"])
    state = (torch.tanh(torch.randn((B * I, conf.deter_dim), generator=g)).to(device),
             torch.zeros(B * I, conf.stoch_dim * conf.stoch_discrete, device=device))
    model = Dreamer(conf).to(device)
    model.fp16_forward = str(device) != "cpu"
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    out = {}

    def snap(x):      # returned metrics / tensors are views of the step workspace (valid until the next call): copy
        if isinstance(x, torch.Tensor):
            return x.detach().clone()
        if isinstance(x, dict):
            return {k: snap(v) for k, v in x.items()}
        if isinstance(x, (tuple, list)):
            return type(x)(snap(v) for v in x)
        return x

    torch.manual_seed(fx["seeds"]["noise"])
    noise = mv(O.draw_noise(conf, T, B, image_pred=True, dream_log=True))
    out["train_log"] = snap(model.training_step(obs, state, do_image_pred=True, do_dream_tensors=True, noise=noise))
    with torch.no_grad():
        torch.manual_seed(fx["seeds"]["noise"])
        noise = mv(O.draw_noise(conf, T, B, image_pred=True))
        out["open_loop"] = snap(model.training_step(obs, state, do_open_loop=True, do_image_pred=True, noise=noise))
        torch.manual_seed(fx["seeds"]["noise"])
        model._test_inference_noise = torch.empty(B * conf.stoch_dim, conf.stoch_discrete).exponential_().reshape(1, B, -1).to(device)
        out["inference"] = model.inference({k: v[:1] for k, v in obs.items()}, (state[0][:B], state[1][:B]))
    return fx, conf, out


def _close(a, b, tol):
    import math
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= tol * max(1.0, abs(b))


def check_log_case(fx, conf, out, rtol):
    losses, out_state, metrics, tensors, dream = out["train_log"]
    w = fx["train_log"]
    for a, b in zip(losses, w["losses"]):
        assert abs(float(a.detach().reshape(-1)[0]) - b) <= rtol * max(1.0, abs(b))
    assert set(metrics) == set(w["metrics"])
    for k, v in w["metrics"].items():
        assert _close(float(metrics[k]), v, 2 * rtol), k
    check_sums(tensors, w["tensors"], rtol, "tensors")
    check_sums(dream, w["dream"], rtol, "dream_tensors")
    losses, out_state, metrics, tensors, _ = out["open_loop"]
    w = fx["open_loop"]
    for a, b in zip(losses, w["losses"]):
        assert abs(float(a.detach().reshape(-1)[0]) - b) <= rtol * max(1.0, abs(b))
    for k, v in w["metrics"].items():
        assert _close(float(metrics[k]), v, 2 * rtol), k
    check_sums(tensors, w["tensors"], rtol, "open-loop tensors")
    atol_h = 1e-3 if rtol < 1e-3 else 2e-2          # sum over B*D recurrent-state elements (TF32 arm: ~3e-4 each)
    assert abs(float(out_state[0].double().sum()) - w["out_state_h_sum"]) <= atol_h
    dist, os3, m3 = out["inference"]
    w = fx["inference"]
    import torch
    lg = dist.logits if conf.actor_dist == "onehot" else torch.cat([dist.base_dist.base_dist.loc, dist.base_dist.base_dist.scale], -1)
    assert abs(float(lg.double().abs().sum()) - w["dist_param_abs"]) <= rtol * w["dist_param_abs"]
    assert abs(float(os3[0].double().sum()) - w["out_state_h_sum"]) <= atol_h
    assert abs(float(os3[1].double().sum()) - w["out_state_z_sum"]) <= 1e-6      # same sampled latent
    assert abs(float(m3["policy_value"]) - w["policy_value"]) <= 2 * rtol * max(1.0, abs(w["policy_value"]))
    a = dist.sample()
    assert a.shape == (1, conf.batch_size, conf.action_dim) and torch.isfinite(dist.log_prob(a)).all()


@pytest.mark.parametrize("case", LOG_CASES)
def test_logging_eval_and_inference_branches_match_reference(ref_ops, case):
    fx, conf, out = run_log_case(case)
    check_log_case(fx, conf, out, 3e-4)


def test_dream_tensors_start_from_the_same_calls_posterior(ref_ops):
    """do_dream_tensors dreams from the posterior features of its own call, also when that call's imag_horizon differs from
    an earlier call's: a model that already ran a step on other observations returns the dream tensors of a fresh one."""
    fx, conf, obs_b, state, _ = build_case("tiny_onehot")
    obs_a = {k: v.flip(0) if v.is_floating_point() else v for k, v in obs_b.items()}
    H = conf.imag_horizon

    def model():
        m = Dreamer(conf)
        m.load_state_dict(seeded_weights(m.state_dict(), fx))
        return m

    def dream(m, obs, seed, **kw):
        torch.manual_seed(seed)
        return m.training_step(obs, state, **kw)[4]

    a, b = model(), model()
    with torch.no_grad():
        dream(a, obs_a, 1)
        got = dream(a, obs_b, 2, imag_horizon=H - 1, do_dream_tensors=True)
        want = dream(b, obs_b, 2, imag_horizon=H - 1, do_dream_tensors=True)
    assert set(got) == set(want) and "value_target" in got
    for k in want:
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))

"""The normal_tanh actor (`actor_dist: normal_tanh`), checked on CPU.

The module runs on the reference op table (oracle/normaltanh_ops.py over oracle/ref_ops.py and its extensions) as in tests/test_dreamer_cpu.py, against
fixtures written from the unmodified reference by tests/golden/make_golden_normaltanh.py: the DMC shape, the DMC shape with
three importance samples, and a model without an image.  The policy is Independent(Normal(tanh(m), sigmoid(s) + 0.01), 1)
with no transform on the action (functions.py:59-66), so the dreamed actions are not bounded to (-1, 1).  The auxiliary
critic and a two-layer GRU, which have no fixtures with this actor, are held to oracle/normaltanh_oracle.py."""
import json
import math
import os
from types import SimpleNamespace

import pytest
import torch
import torch.distributions as D

import tests.test_dreamer_cpu as TD
from oracle import dreamer_oracle as DO
from oracle import normaltanh_oracle
from oracle.normaltanh_ops import NtGruRefOps, NtRefOps
from oracle.weights import seeded_state_dict
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.util import GOLDEN_DIR, build_case, seeded_weights

CASES = ("tiny_dmc_normaltanh", "tiny_dmc_normaltanh_iwae3", "tiny_vector_normaltanh")
PRESETS = CASES + ("dmc_normaltanh",)


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(NtRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def run_model(case, **attrs):
    """tests/test_dreamer_cpu.run_model: fp32 forward and the per-timestep chains unless `attrs` say otherwise."""
    fx, conf, obs, state, noise = build_case(case)
    model = Dreamer(conf)
    for k, v in dict(dict(fp16_forward=False, persistent_rssm=False, persistent_bptt=False), **attrs).items():
        setattr(model, k, v)
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    for l in losses:
        l.backward()
    return fx, conf, model, opts, losses, out_state, metrics, tensors


@pytest.mark.parametrize("case", CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case)
    TD.check_golden(fx, model, losses, out_state, metrics, tensors)


def test_dreamed_actions_are_the_unbounded_normal_sample(ref_ops):
    """a = tanh(m) + (sigmoid(s) + 0.01) eps on the actor's outputs, with no squashing: with the fixture's noise some
    actions leave (-1, 1), and their sum is the reference's."""
    fx, conf, model, *_ = run_model("tiny_dmc_normaltanh")
    H, N, A = conf.imag_horizon, conf.batch_length * conf.batch_size, conf.action_dim
    acts = model._buf("dream.actions", H, N, A)
    alog = model._buf("dream.alog", H, N, model.d.Ap)[..., :2 * A]
    _, _, _, _, noise = build_case("tiny_dmc_normaltanh")
    want = torch.tanh(alog[..., :A]) + (torch.sigmoid(alog[..., A:]) + 0.01) * noise["actor"]
    assert torch.allclose(acts, want, rtol=1e-6, atol=1e-6)
    assert float(acts.abs().max()) > 1.0
    assert abs(float(acts.double().sum()) - fx["dream_action_sum"]) <= 1e-4 * max(1.0, abs(fx["dream_action_sum"]))


def test_fp16_forward_and_persistent_branches(ref_ops):
    fx, conf, model, opts, losses, *_ = run_model("tiny_dmc_normaltanh", fp16_forward=True, persistent_rssm=True,
                                                  persistent_bptt=True)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):      # fp16 operands: the actor-critic losses move most
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= (5e-3 if i < 2 else 2e-2) * max(1.0, abs(want)), (i, got, want)


def test_logging_eval_and_inference_branches_match_reference(ref_ops):
    fx, conf, out = TD.run_log_case("tiny_dmc_normaltanh_log")
    dist, os3, m3 = out["inference"]
    # check_log_case reads the Normal's parameters two levels down (tanh_normal's TransformedDistribution of an
    # Independent): hand it the Independent as the outer level's base
    shim = SimpleNamespace(base_dist=dist, sample=dist.sample, log_prob=dist.log_prob)
    TD.check_log_case(fx, conf, dict(out, inference=(shim, os3, m3)), 3e-4)


def test_inference_returns_the_reference_distribution(ref_ops):
    """inference() returns Independent(Normal(tanh(m), sigmoid(s) + 0.01), 1) over (1, B, A), as functions.py:59-66
    builds it: .mean is tanh(m), .sample() is unbounded, entropy and log_prob are the Normal's own."""
    fx, conf, out = TD.run_log_case("tiny_dmc_normaltanh_log")
    dist = out["inference"][0]
    B, A = conf.batch_size, conf.action_dim
    assert type(dist) is D.Independent and type(dist.base_dist) is D.Normal and dist.reinterpreted_batch_ndims == 1
    assert dist.batch_shape == (1, B) and dist.event_shape == (A,)
    loc, scale = dist.base_dist.loc, dist.base_dist.scale
    assert float(loc.abs().max()) < 1.0 and float(scale.min()) > 0.01 and float(scale.max()) < 1.01
    lg = torch.cat([loc, scale], -1)
    w = fx["inference"]
    assert abs(float(lg.double().sum()) - w["dist_param_sum"]) <= 3e-4 * max(1.0, abs(w["dist_param_sum"]))
    assert torch.equal(dist.mean, loc)
    ent = (0.5 + 0.5 * math.log(2 * math.pi) + scale.log()).sum(-1)
    assert torch.allclose(dist.entropy(), ent, rtol=1e-6, atol=1e-6)
    a = loc + 3.0 * scale
    lp = (-0.5 * ((a - loc) / scale) ** 2 - scale.log() - 0.5 * math.log(2 * math.pi)).sum(-1)
    assert torch.allclose(dist.log_prob(a), lp, rtol=1e-5, atol=1e-5)


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "normaltanh_state_dict.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("preset", PRESETS)
def test_state_dict_keys_shapes_and_parameter_order_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g


def test_checkpoint_round_trips_with_torch_adamw(ref_ops):
    """The actor optimizer's state_dict is torch.optim.AdamW's over the same parameter list (the reference's checkpoint,
    tools.py:171-172, 195-196), and a fresh model loads the module and every optimizer state back."""
    fx, conf, model, opts, losses, *_ = run_model("tiny_dmc_normaltanh")
    actor = list(model.ac.actor.parameters())
    clones = [torch.nn.Parameter(p.detach().clone()) for p in actor]
    for c, p in zip(clones, actor):
        c.grad = p.grad.detach().clone()
    topt = torch.optim.AdamW(clones, lr=conf.adam_lr_actor, eps=conf.adam_eps)
    for o in opts:
        o.step()
    topt.step()
    ours, theirs = opts[2].state_dict(), topt.state_dict()
    assert ours["param_groups"][0]["params"] == theirs["param_groups"][0]["params"]
    for i, st in theirs["state"].items():
        assert torch.allclose(st["exp_avg"], ours["state"][i]["exp_avg"], rtol=1e-5, atol=1e-9), i
        assert torch.allclose(st["exp_avg_sq"], ours["state"][i]["exp_avg_sq"], rtol=1e-5, atol=1e-12), i
    for c, p in zip(clones, actor):
        assert torch.allclose(c.detach(), p.detach(), rtol=1e-6, atol=1e-7)
    fresh = Dreamer(conf)
    fresh.load_state_dict(model.state_dict(), strict=True)
    fopts = fresh.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    for fo, o in zip(fopts, opts):
        fo.load_state_dict(o.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(fresh.state_dict().values(), model.state_dict().values()))
    for fo, o in zip(fopts, opts):
        for i, st in o.state_dict()["state"].items():
            got = fo.state_dict()["state"][i]
            assert all(torch.equal(got[k], v) for k, v in st.items() if isinstance(v, torch.Tensor)), i


def _against_oracle(oracle, conf, seed=77):
    """A step of the module on a batch, weights and noise other than the fixtures' against oracle.training_step: losses,
    metrics and every gradient."""
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    obs = synthetic_batch(conf, seed=seed)
    g = torch.Generator().manual_seed(8)
    state = (torch.tanh(torch.randn(B * I, conf.deter_dim, generator=g)), torch.zeros(B * I, conf.stoch_dim * conf.stoch_discrete))
    torch.manual_seed(5)
    noise = DO.draw_noise(conf, T, B)
    model = Dreamer(conf)
    model.fp16_forward = model.persistent_rssm = model.persistent_bptt = False
    sd = seeded_state_dict(model.state_dict(), 11)
    model.load_state_dict(sd)
    model.init_optimizers(conf.adam_lr)
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    sdo = {k: v.clone().requires_grad_(v.is_floating_point() and "critic_target" not in k) for k, v in sd.items()}
    res = oracle.training_step(sdo, conf, obs, state, noise)
    for l in res["losses"]:
        l.backward()
    for a, b in zip(losses, res["losses"]):
        a, b = float(a.detach().reshape(-1)[0]), float(b.detach().reshape(-1)[0])
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (a, b)
    for k, v in res["metrics"].items():
        assert abs(float(metrics[k]) - float(v)) <= 2e-4 * max(1.0, abs(float(v))), k
    acts = model._buf("dream.actions", conf.imag_horizon, T * B * I, conf.action_dim)
    assert torch.allclose(acts, res["inter"]["dream_actions"], rtol=1e-5, atol=1e-5)
    for n, p in model.named_parameters():
        want = sdo[n].grad
        if want is None:
            assert p.grad is None or not p.grad.any(), n
            continue
        assert torch.allclose(p.grad, want, rtol=1e-4, atol=1e-4 * float(want.abs().max()) + 1e-12), n


@pytest.mark.parametrize("preset,over,table", [
    ("tiny_dmc_normaltanh", {}, NtRefOps),
    ("tiny_dmc_normaltanh", dict(aux_critic=True), NtRefOps),
    ("tiny_vector_normaltanh", dict(aux_critic=True), NtRefOps),
    ("tiny_dmc_normaltanh", dict(gru_layers=2), NtGruRefOps),
    ("tiny_dmc_normaltanh_iwae3", dict(gru_layers=2), NtGruRefOps),
], ids=["dmc", "dmc_aux", "vector_aux", "dmc_gru2", "dmc_iwae3_gru2"])
def test_matches_oracle_with_aux_critic_and_stacked_gru(preset, over, table):
    pd_ops.set_ops_for_testing(table("cpu"))
    try:
        _against_oracle(normaltanh_oracle, make_conf(preset, device="cpu", **over))
    finally:
        pd_ops.set_ops_for_testing(None)


def test_aux_critic_actor_has_two_outputs_per_action():
    model = Dreamer(make_conf("tiny_dmc_normaltanh", aux_critic=True))
    A = model.conf.action_dim
    assert model.wm.ac_aux.actor.model[-1].weight.shape[0] == 2 * A
    assert model.ac.actor.model[-1].weight.shape[0] == 2 * A


def test_other_actor_settings_stay_refused():
    with pytest.raises(NotImplementedError, match="actor_grad"):
        Dreamer(make_conf("tiny_dmc_normaltanh", actor_grad="dynamics"))
    with pytest.raises(NotImplementedError, match="actor_dist"):
        Dreamer(make_conf("tiny_dmc_normaltanh", actor_dist="normal"))


def test_twin_samples_and_loss_follow_the_formulas():
    """The float32 twins on the reference op table against float64 restatements of functions.py:59-66 and a2c.py:119-130
    (autograd for the gradient)."""
    ops = NtRefOps("cpu")
    g = torch.Generator().manual_seed(3)
    rows, A, eta = 45, 3, 3e-3
    out = torch.randn(rows, 2 * A, generator=g) * 3
    eps = torch.randn(rows, A, generator=g)
    act = torch.empty(rows, A)
    ops.normal_tanh_sample(out, eps, act)
    o64 = out.double().requires_grad_()
    mu, sd = torch.tanh(o64[:, :A]), torch.sigmoid(o64[:, A:]) + 0.01
    assert torch.allclose(act.double(), mu + sd * eps.double(), rtol=1e-6, atol=1e-6)
    ag, w = torch.randn(rows, generator=g), torch.rand(rows, generator=g)
    dout, sums = torch.zeros(rows, 2 * A), torch.zeros(2, dtype=torch.float64)
    ops.actor_loss_normal_tanh(eta, out, act, ag, w, dout, sums)
    dist = D.Independent(D.Normal(mu, sd), 1)
    lp, ent = dist.log_prob(act.double()), dist.entropy()
    loss = ((-lp * ag.double() - eta * ent) * w.double()).mean()
    loss.backward()
    assert torch.allclose(sums, torch.stack([loss.detach() * rows, ent.sum().detach()]), rtol=1e-5, atol=1e-5)
    assert torch.allclose(dout.double(), o64.grad, rtol=1e-4, atol=1e-7)

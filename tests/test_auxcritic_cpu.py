"""The world model's auxiliary critic (`aux_critic`), checked on CPU.

The module runs on the reference op table with the aux-critic scan twin (oracle/auxcritic_ops.py) as in
tests/test_dreamer_cpu.py, against fixtures written from the unmodified reference by tests/golden/make_golden_auxcritic.py:
the Atari shape, three importance samples, the tanh_normal actor and a model without images.  Every batch carries the
terminal pattern of `force_terminals`.  Also: the aux critic's place in the state dict, the optimizer and the arena (its
actor and target never receive a gradient), the target copies, and the configurations the module refuses."""
import json
import os

import pytest
import torch

import tests.test_dreamer_cpu as TD
from oracle import auxcritic_oracle as O
from oracle.auxcritic_ops import AuxRefOps
from oracle.ref_ops import RefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200 import replay
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from tests.test_dreamer_cpu import check_log_case
from tests.util import GOLDEN_DIR, build_case, load_fixture

CASES = ("tiny_auxcritic", "tiny_auxcritic_iwae3", "tiny_dmc_auxcritic", "tiny_vector_auxcritic")
NEVER_GRAD = ("wm.ac_aux.actor.", "wm.ac_aux.critic_target.")


def force_terminals(obs):
    """The terminal pattern of every auxiliary-critic fixture: a terminal at t = 0 in column 0, at t = T // 2 in column 1
    and none in the other columns (synthetic Bernoulli(0.01) terminals almost never occur in a tiny batch)."""
    term = torch.zeros_like(obs["terminal"])
    term[0, 0] = 1.0
    term[term.shape[0] // 2, 1] = 1.0
    return dict(obs, terminal=term)


def build_aux_case(name, device="cpu", fx=None):
    fx, conf, obs, state, noise = build_case(name, device, fx)
    return fx, conf, force_terminals(obs), state, noise


@pytest.fixture()
def ref_ops(monkeypatch):
    monkeypatch.setattr(TD, "build_case", build_aux_case)
    pd_ops.set_ops_for_testing(AuxRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "auxcritic_state_dict.json")) as f:
        return json.load(f)


def check_aux_golden(fx, model, losses, out_state, metrics, tensors, rtol=2e-4):
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 0.1 * rtol * max(1.0, abs(want))
    assert set(metrics) == set(fx["metrics"]) and {"loss_critic_aux", "policy_value_aux"} <= set(metrics)
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= rtol * max(1.0, abs(want)), k
    assert set(tensors) == set(fx["tensor_sums"])
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= rtol * max(want, 1e-6), (k, got, want)
    assert torch.allclose(tensors["policy_value_aux"].double(), torch.tensor(fx["policy_value_aux"], dtype=torch.float64),
                          rtol=rtol, atol=rtol)
    named = dict(model.named_parameters())
    assert {k for k, p in named.items() if p.grad is not None} == set(fx["grad_norms"])
    for k, want in fx["grad_norms"].items():
        g = named[k].grad
        got = float(g.double().norm())
        assert abs(got - want) <= rtol * max(want, 1e-6) + 1e-9, (k, got, want)
        assert abs(float(g.double().sum()) - fx["grad_sums"][k]) <= 2.5 * rtol * max(want, 1e-6) * g.numel() ** 0.5 + 1e-8, k
    assert abs(float(out_state[0].double().sum()) - fx["out_state_h_sum"]) < 1e-3
    assert all(p.grad is None for n, p in named.items() if n.startswith(NEVER_GRAD))


@pytest.mark.parametrize("case", CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = TD.run_model(case)
    assert fx["terminals"] == force_terminals(build_case(case)[2])["terminal"].tolist()
    check_aux_golden(fx, model, losses, out_state, metrics, tensors)


@pytest.mark.parametrize("case", CASES)
def test_fp16_forward_and_persistent_branches(ref_ops, case):
    fx, conf, model, opts, losses, *_ = TD.run_model(case, fp16_forward=True, persistent_rssm=True, persistent_bptt=True)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-3 * max(1.0, abs(want)), (i, got, want)


def test_logging_eval_and_inference_branches_match_reference(ref_ops, monkeypatch):
    batch = replay.synthetic_batch
    monkeypatch.setattr(replay, "synthetic_batch", lambda *a, **k: force_terminals(batch(*a, **k)))
    fx, conf, out = TD.run_log_case("tiny_auxcritic_log")
    check_log_case(fx, conf, out, 3e-4)
    for key in ("train_log", "open_loop"):
        metrics, tensors = out[key][2], out[key][3]
        assert {"loss_critic_aux", "policy_value_aux"} <= set(metrics) and tensors["policy_value_aux"].shape == (4, 3)


def test_matches_oracle_with_a_stale_target_and_another_weight(ref_ops):
    """Call 1 of a model whose aux target was synced at call 0 and whose critic then changed: the target critic is the
    stale copy (target_interval_aux > 1); aux_critic_weight 0.3 scales both the loss term and its gradients."""
    fx, conf, obs, state, noise = build_aux_case("tiny_auxcritic")
    conf.aux_critic_weight = 0.3
    model = Dreamer(conf)
    sd = TD.seeded_weights(model.state_dict(), fx)
    model.load_state_dict(sd)
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    aux = model.wm.ac_aux
    with torch.no_grad():
        for p in aux.critic.parameters():
            p.mul_(0.9)
    model._weights_dirty = True
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    losses, _, metrics, _, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    assert aux.train_steps == 2
    sdo = {k: v.clone().requires_grad_(k.startswith("wm.") and not k.startswith(("wm.ac_aux.actor", "wm.ac_aux.critic_target")))
           for k, v in sd.items()}
    res = O.training_step(sdo, conf, obs, state, noise, target_synced=False, aux_target_synced=False)
    res["losses"][0].backward()
    assert abs(float(losses[0].detach()) - float(res["losses"][0])) <= 2e-5 * max(1.0, abs(float(res["losses"][0])))
    for k in ("loss_critic_aux", "policy_value_aux", "loss_model"):
        assert abs(float(metrics[k]) - float(res["metrics"][k])) <= 2e-4 * max(1.0, abs(float(res["metrics"][k]))), k
    for n, p in model.named_parameters():
        if n.startswith("wm.") and sdo[n].grad is not None:
            g, want = p.grad.double(), sdo[n].grad.double()
            assert (g - want).abs().max() <= 1e-3 * want.abs().max() + 1e-9, n        # fp32 both sides, other sum orders


def test_target_copies_at_every_target_interval(ref_ops):
    fx, conf, obs, state, noise = build_aux_case("tiny_auxcritic")
    conf.target_interval_aux = 3
    model = Dreamer(conf)
    model.load_state_dict(TD.seeded_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    aux = model.wm.ac_aux
    flat = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()])
    synced = []
    for call in range(7):
        before = flat(aux.critic_target).clone()
        losses = model.training_step(obs, state, noise=noise)[0]
        synced.append(torch.equal(flat(aux.critic_target), flat(aux.critic)) and not torch.equal(before, flat(aux.critic)))
        if call in (0, 3, 6):
            assert torch.equal(flat(aux.critic_target), flat(aux.critic)), call
        else:
            assert torch.equal(flat(aux.critic_target), before), call
        for o in opts:
            o.zero_grad()
        for l in losses:
            l.backward()
        for o in opts:
            o.step()
    with torch.no_grad():                                  # an evaluation call neither copies nor counts
        model.training_step(obs, state, noise=noise)
    assert aux.train_steps == 7


def test_never_trained_parameters_stay_outside_the_trained_arena_and_unchanged(ref_ops):
    fx, conf, model, opts, *_ = TD.run_model("tiny_auxcritic")
    aux = model.wm.ac_aux
    never = list(aux.actor.parameters()) + list(aux.critic_target.parameters())
    for p in never:
        off = model._offsets[id(p)]
        assert off >= model._group_range["target"][1] and off >= model._train_numel and p.grad is None
    for p in aux.critic.parameters():
        a, b = model._group_range["wm"]
        assert a <= model._offsets[id(p)] < b and p.grad is not None
    actor = [p.detach().clone() for p in aux.actor.parameters()]
    target = [p.detach().clone() for p in aux.critic_target.parameters()]
    model.grad_clip(0.5, 0.01)
    for o in opts:
        o.step()
    assert all(torch.equal(p, q) for p, q in zip(aux.actor.parameters(), actor))
    assert all(torch.equal(p, q) for p, q in zip(aux.critic_target.parameters(), target))
    assert all(p.grad is None for p in never)


@pytest.mark.parametrize("preset", ("tiny_auxcritic", "tiny_dmc_auxcritic", "atari_auxcritic"))
def test_state_dict_keys_shapes_and_parameter_order_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g


@pytest.mark.parametrize("preset", ("tiny_auxcritic", "tiny_dmc_auxcritic"))
def test_optimizer_state_matches_torch_adamw_and_round_trips(ref_ops, preset):
    """torch.optim.AdamW over the reference's world-model parameters keeps no state for the aux actor and target (their
    grad is None): _FusedAdamW keeps state for the reference's indices, equals torch's state there and loads it back."""
    fx = build_aux_case("tiny_auxcritic")[0]
    fx = dict(fx, preset=preset, overrides={})
    _, conf, obs, state, noise = build_aux_case(preset, fx=fx)
    model = Dreamer(conf)
    model.load_state_dict(TD.seeded_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    for l in model.training_step(obs, state, noise=noise)[0]:
        l.backward()
    wm = list(model.wm.parameters())
    clones = [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in wm]
    for c, p in zip(clones, wm):
        c.grad = None if p.grad is None else p.grad.detach().clone()
    topt = torch.optim.AdamW(clones, lr=conf.adam_lr, eps=conf.adam_eps)
    opts[0].step()
    topt.step()
    ours, theirs = opts[0].state_dict(), topt.state_dict()
    assert sorted(ours["state"]) == sorted(theirs["state"]) == _state_dict_fixture()[preset]["wm_adamw_state"]
    for i, st in theirs["state"].items():
        assert torch.allclose(st["exp_avg"], ours["state"][i]["exp_avg"], rtol=1e-5, atol=1e-9), i
        assert torch.allclose(st["exp_avg_sq"], ours["state"][i]["exp_avg_sq"], rtol=1e-5, atol=1e-12), i
    for c, p in zip(clones, wm):
        assert torch.allclose(c.detach(), p.detach(), rtol=1e-5, atol=1e-7)
    opts[0].load_state_dict(theirs)                     # torch -> fused
    back = opts[0].state_dict()
    t2 = torch.optim.AdamW([torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in wm],
                           lr=conf.adam_lr, eps=conf.adam_eps)
    t2.load_state_dict(back)                            # fused -> torch
    for i, st in theirs["state"].items():
        assert torch.equal(t2.state_dict()["state"][i]["exp_avg"], st["exp_avg"]), i


def test_state_dict_loads_strictly_both_ways():
    conf = make_conf("tiny_auxcritic", device="cpu")
    a, b = Dreamer(conf), Dreamer(conf)
    fx = _state_dict_fixture()["tiny_auxcritic"]["state_dict"]
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(shape, generator=g) for k, shape in fx}
    a.load_state_dict(sd, strict=True)
    a._ensure_arena()
    out = a.state_dict()
    assert list(out) == [k for k, _ in fx] and all(torch.equal(out[k], sd[k]) for k in sd)
    b.load_state_dict(out, strict=True)
    assert all(torch.equal(b.state_dict()[k], sd[k]) for k in sd)


def test_refused_configurations(ref_ops):
    for T in (1, 129):
        with pytest.raises(NotImplementedError):
            Dreamer(make_conf("tiny_auxcritic", batch_length=T))
        Dreamer(make_conf("tiny", batch_length=T))                  # without the aux critic the length is not limited
    Dreamer(make_conf("tiny_auxcritic", batch_length=2))
    Dreamer(make_conf("tiny_auxcritic", batch_length=128))
    fx, conf, obs, state, noise = build_aux_case("tiny_auxcritic")
    model = Dreamer(conf)
    with pytest.raises(NotImplementedError):
        model.training_step({k: v[:1] for k, v in obs.items()}, state)
    ops = AuxRefOps("cpu")
    z = lambda *s: torch.zeros(*s)
    for T in (1, 129):
        with pytest.raises(RuntimeError):
            ops.gae_critic_obs(T, 2, 0.99, 0.95, z(T * 2), z(T * 2), z(T * 2), z(T * 2), 1.0, z(max(T - 1, 1) * 2),
                               torch.zeros(2, dtype=torch.float64))


def test_aux_off_layout_parameters_and_metrics_are_unchanged(monkeypatch):
    """Without aux_critic the arena, the parameter lists and the metric keys are those of the parent's schedule."""
    pd_ops.set_ops_for_testing(RefOps("cpu"))
    try:
        base, aux = Dreamer(make_conf("tiny", device="cpu")), Dreamer(make_conf("tiny_auxcritic", device="cpu"))
        assert base.wm.ac_aux is None and not base._frozen
        assert base._arena_numel == base._group_range["target"][1] == base._train_numel + (
            base._group_range["target"][1] - base._group_range["target"][0])
        n = len(list(base.wm.parameters()))
        assert [p.shape for p in base.wm.parameters()] == [p.shape for p in aux.wm.parameters()][:n]
        assert list(base.state_dict()) == [k for k in aux.state_dict() if not k.startswith("wm.ac_aux.")]
        for g in ("probe", "actor", "critic", "target"):
            assert [p.shape for p in base._group_params[g]] == [p.shape for p in aux._group_params[g]]
        fx, conf, obs, state, noise = build_case("tiny_onehot")
        metrics = TD.run_model("tiny_onehot")[6]
        assert "loss_critic_aux" not in metrics and "policy_value_aux" not in metrics
        assert set(metrics) == set(load_fixture("tiny_onehot")["metrics"])
    finally:
        pd_ops.set_ops_for_testing(None)

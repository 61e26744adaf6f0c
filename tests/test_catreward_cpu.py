"""The categorical reward head (`reward_decoder_categorical`), checked on CPU.

The module runs on the reference op table with the support-head twin (oracle/catreward_ops.py) as in
tests/test_dreamer_cpu.py, against fixtures written from the unmodified reference by tests/golden/make_golden_catreward.py:
[-1, 0, 1] through tanh clipping (also with three importance samples), [0, 1] unclipped under the tanh_normal actor, and
33 unsorted, duplicated support values.  Also: the support's place in the state dict, the optimizer and the arena (it is a
parameter that is never trained), and the configurations the module refuses."""
import json
import os

import numpy as np
import pytest
import torch

import tests.test_dreamer_cpu as TD
from oracle import catreward_oracle as O
from oracle.catreward_ops import CatRefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from tests.test_dreamer_cpu import check_log_case
from tests.util import GOLDEN_DIR, build_case, load_fixture

CASES = ("tiny_catreward", "tiny_catreward_iwae3", "tiny_dmc_catreward", "tiny_catreward_wide")
SUPPORT = O.SUPPORT


@pytest.fixture()
def ref_ops(monkeypatch):
    # the runners of tests/test_dreamer_cpu.py load seeded weights; the fixtures keep the configured support
    monkeypatch.setattr(TD, "seeded_weights", lambda template, fx: O.seeded_weights(template, fx["seeds"]["weights"]))
    pd_ops.set_ops_for_testing(CatRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "catreward_state_dict.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = TD.run_model(case)
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
    for k, want in fx["grad_norms"].items():
        g = named[k].grad
        assert g is not None, k
        assert abs(float(g.double().norm()) - want) <= 2e-4 * max(want, 1e-6) + 1e-9, (k, float(g.double().norm()), want)
        assert abs(float(g.double().sum()) - fx["grad_sums"][k]) <= 5e-4 * max(want, 1e-6) * g.numel() ** 0.5 + 1e-8, k
    assert abs(float(out_state[0].double().sum()) - fx["out_state_h_sum"]) < 1e-3
    assert named[SUPPORT].grad is None
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    kr = model._buf("head.kr", T * B * I, dtype=torch.int32).view(T, B, I)
    assert (kr == kr[:, :, :1]).all() and kr[:, :, 0].reshape(-1).tolist() == fx["reward_buckets"]


def test_wide_support_resolves_ties_to_the_first_index():
    fx = load_fixture("tiny_catreward_wide")
    sup = torch.tensor(make_conf("tiny_catreward_wide").reward_decoder_categorical).float()
    firsts = {float(v): int((sup == v).nonzero()[0]) for v in sup}
    dup = [k for k in fx["reward_buckets"] if int((sup == sup[k]).sum()) > 1]
    assert len(dup) >= len(fx["reward_buckets"]) // 2                  # the case exercises ties
    assert all(firsts[float(sup[k])] == k for k in fx["reward_buckets"])


@pytest.mark.parametrize("case", CASES)
def test_persistent_rssm_and_bptt_branches(ref_ops, case):
    fx, conf, model, opts, losses, *_ = TD.run_model(case, fp16_forward=True, persistent_rssm=True, persistent_bptt=True)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-3 * max(1.0, abs(want)), (i, got, want)


@pytest.mark.parametrize("case", [c + "_log" for c in CASES])
def test_logging_eval_and_inference_branches_match_reference(ref_ops, case):
    fx, conf, out = TD.run_log_case(case)
    check_log_case(fx, conf, out, 3e-4)
    metrics, tensors, dream = out["train_log"][2], out["train_log"][3], out["train_log"][4]
    S = len(conf.reward_decoder_categorical)
    assert {f"logprob_reward{i}" for i in range(S)} <= set(metrics) and "logprob_reward-1" not in metrics
    assert "reward_pred" in tensors and dream["reward_pred"].shape == (conf.batch_length, conf.batch_size)


@pytest.mark.parametrize("preset", ("tiny_catreward", "tiny_dmc_catreward", "tiny_catreward_wide", "atari_catreward"))
def test_state_dict_keys_shapes_parameter_order_and_support_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g
    sup = model.wm.decoder.reward._support
    assert sup.dtype == torch.float32 and not sup.requires_grad and sup.tolist() == fx["support"]


def test_state_dict_loads_strictly_both_ways(ref_ops):
    conf = make_conf("tiny_catreward", device="cpu")
    a, b = Dreamer(conf), Dreamer(conf)
    fx = _state_dict_fixture()["tiny_catreward"]["state_dict"]
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(shape, generator=g) if shape else torch.randn((), generator=g) for k, shape in fx}
    a.load_state_dict(sd, strict=True)
    a._ensure_arena()                                   # the support moves into the arena with its loaded values
    out = a.state_dict()
    assert list(out) == [k for k, _ in fx] and all(torch.equal(out[k], sd[k]) for k in sd)
    b.load_state_dict(out, strict=True)
    assert all(torch.equal(b.state_dict()[k], sd[k]) for k in sd)


def _grad_clones(model):
    groups = dict(wm=list(model.wm.parameters()), actor=list(model.ac.actor.parameters()),
                  critic=list(model.ac.critic.parameters()))
    clones = {g: [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in ps]
              for g, ps in groups.items()}
    for g, ps in groups.items():
        for c, p in zip(clones[g], ps):
            c.grad = None if p.grad is None else p.grad.detach().clone()
    return groups, clones


def test_support_survives_clip_and_adamw_steps_and_grad_clip_matches_torch(ref_ops):
    fx, conf, model, opts, *_ = TD.run_model("tiny_catreward")
    sup = model.wm.decoder.reward._support
    before = sup.detach().clone()
    for step in range(3):
        if step:
            _, _, obs, state, noise = build_case("tiny_catreward")
            losses = model.training_step(obs, state, noise=noise)[0]
            for o in opts:
                o.zero_grad()
            for l in losses:
                l.backward()
        groups, clones = _grad_clones(model)
        norms = model.grad_clip(0.5, 0.01)
        for g, key, mx in (("wm", "grad_norm", 0.5), ("actor", "grad_norm_actor", 0.01), ("critic", "grad_norm_critic", 0.01)):
            want = float(torch.nn.utils.clip_grad_norm_(clones[g], mx))
            assert abs(float(norms[key]) - want) <= 1e-4 * want, (step, g)
        for o in opts:
            o.step()
        assert sup.grad is None and torch.equal(sup.detach(), before), step
    assert torch.equal(model.state_dict()[SUPPORT], before)


def test_optimizer_state_dict_round_trips_with_torch_adamw(ref_ops):
    """torch.optim.AdamW over the reference's parameter list keeps no state for the support (its grad is None):
    _FusedAdamW writes none at its index, equals torch's state elsewhere, and loads torch's state back (both ways)."""
    fx, conf, model, opts, *_ = TD.run_model("tiny_catreward")
    wm = list(model.wm.parameters())
    i_sup = next(i for i, p in enumerate(wm) if p is model.wm.decoder.reward._support)
    assert i_sup == 18
    groups, clones = _grad_clones(model)
    topt = torch.optim.AdamW(clones["wm"], lr=conf.adam_lr, eps=conf.adam_eps)
    opts[0].step()
    topt.step()
    ours, theirs = opts[0].state_dict(), topt.state_dict()
    assert ours["param_groups"][0]["params"] == theirs["param_groups"][0]["params"] == list(range(len(wm)))
    assert set(ours["state"]) == set(theirs["state"]) and i_sup not in ours["state"]
    for i, st in theirs["state"].items():
        assert torch.allclose(st["exp_avg"], ours["state"][i]["exp_avg"], rtol=1e-5, atol=1e-9), i
        assert torch.allclose(st["exp_avg_sq"], ours["state"][i]["exp_avg_sq"], rtol=1e-5, atol=1e-12), i
    for c, p in zip(clones["wm"], wm):
        assert torch.allclose(c.detach(), p.detach(), rtol=1e-5, atol=1e-7)
    opts[0].load_state_dict(theirs)                     # torch -> fused
    assert int(opts[0].step_t.item()) == 1
    back = opts[0].state_dict()
    t2 = torch.optim.AdamW([torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in wm],
                           lr=conf.adam_lr, eps=conf.adam_eps)
    t2.load_state_dict(back)                            # fused -> torch
    assert set(t2.state_dict()["state"]) == set(theirs["state"])
    for i, st in theirs["state"].items():
        assert torch.equal(t2.state_dict()["state"][i]["exp_avg"], st["exp_avg"]), i


def test_support_is_stored_outside_the_trained_arena(ref_ops):
    model = Dreamer(make_conf("tiny_catreward", device="cpu"))
    model._ensure_arena()
    sup = model.wm.decoder.reward._support
    off = model._offsets[id(sup)]
    assert off >= model._group_range["target"][1] and off >= model._train_numel
    assert sup.grad is None and sup.data_ptr() == model._arena[off:].data_ptr()
    normal = Dreamer(make_conf("tiny", device="cpu"))                  # the Normal head: the arena layout is unchanged
    assert not normal._frozen and normal._arena_numel == normal._group_range["target"][1]


def test_refused_configurations():
    for sup in ([1.0], list(np.linspace(-1, 1, 1025))):                  # S = 1 (the reference cannot run it), S > 1024
        with pytest.raises(NotImplementedError):
            Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=sup))
    with pytest.raises(ValueError):                                       # log1p(-1) = -inf
        Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=[-1.0, 0.0, 1.0], clip_rewards="log1p"))
    with pytest.raises(ValueError):
        Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=[0.0, float("nan")], clip_rewards=None))
    with pytest.raises(AssertionError):                                   # decoders.py:329
        Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=(0.0, 1.0), clip_rewards=None))
    Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=(0.0, 1.0)))       # tanh turns the tuple into an array
    Dreamer(make_conf("tiny_catreward", reward_decoder_categorical=list(np.linspace(-1, 1, 1024))))

"""Boundary semantics of the drop-in module that the reference's callers rely on (train.py:143-198, tools.py:164-197),
checked on CPU with the reference op table: optimizer state in torch.optim.AdamW's layout, weight reloads, non-unit
grad_output (GradScaler / scaled losses), metric lifetime."""
import json
import os
import warnings

import pytest
import torch

from oracle.ref_ops import RefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from tests.util import GOLDEN_DIR, build_case, seeded_weights



@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(RefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def _stepped_model(case="tiny_onehot"):
    fx, conf, obs, state, noise = build_case(case)
    model = Dreamer(conf)
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    for l in losses:
        l.backward()
    return fx, conf, obs, state, noise, model, opts, losses, metrics


@pytest.mark.parametrize("preset", ("tiny", "tiny_dmc"))
def test_parameter_order_per_optimizer_equals_the_reference(preset):
    """torch optimizers key their state by parameter index: same enumeration order as the reference module
    (fixture written from the unmodified reference by tests/golden/make_param_order.py)."""
    with open(os.path.join(GOLDEN_DIR, "param_order.json")) as f:
        want = json.load(f)[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    names = {id(p): n for n, p in model.named_parameters()}
    for g in ("wm", "probe", "actor", "critic"):
        got = [[names[id(p)], list(p.shape)] for p in model._group_params[g]]
        assert got == want[g], g


def test_optimizer_state_dict_is_torch_adamw_layout_both_ways(ref_ops):
    fx, conf, obs, state, noise, model, opts, losses, metrics = _stepped_model()
    assert opts[0].state_dict()["state"] == {}                       # like torch: no per-parameter state before step 1
    groups = dict(wm=0, actor=2, critic=3)
    clones = {g: [torch.nn.Parameter(p.detach().clone()) for p in model._group_params[g]] for g in groups}
    for g in groups:
        for c, p in zip(clones[g], model._group_params[g]):
            c.grad = p.grad.detach().clone()
    lrs = dict(wm=conf.adam_lr, actor=conf.adam_lr_actor, critic=conf.adam_lr_critic)
    topts = {g: torch.optim.AdamW(clones[g], lr=lrs[g], eps=conf.adam_eps) for g in groups}
    for o in opts:
        o.step()
    for o in topts.values():
        o.step()
    for g, i in groups.items():
        ours, theirs = opts[i].state_dict(), topts[g].state_dict()
        assert set(ours) == {"state", "param_groups"} and sorted(ours["state"]) == sorted(theirs["state"])
        assert ours["param_groups"][0]["params"] == theirs["param_groups"][0]["params"]
        for k in theirs["state"]:
            assert set(ours["state"][k]) == {"step", "exp_avg", "exp_avg_sq"}
            assert float(ours["state"][k]["step"]) == float(theirs["state"][k]["step"]) == 1.0
            for n in ("exp_avg", "exp_avg_sq"):
                assert ours["state"][k][n].shape == theirs["state"][k][n].shape
                assert torch.allclose(ours["state"][k][n], theirs["state"][k][n], rtol=1e-5, atol=1e-10), (g, k, n)
        # ours -> a fresh torch.optim.AdamW (what tools.py:195-196 does with a reference-side optimizer)
        fresh = torch.optim.AdamW([torch.nn.Parameter(c.detach().clone()) for c in clones[g]], lr=1.0)
        fresh.load_state_dict(ours)
        assert fresh.param_groups[0]["lr"] == lrs[g] and float(fresh.state[fresh.param_groups[0]["params"][3]]["step"]) == 1.0
    # torch's state -> a fresh fused optimizer of a second model, then one more identical step on both sides
    model2 = Dreamer(conf)
    model2.load_state_dict(model.state_dict())
    opts2 = model2.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    for g, i in groups.items():
        opts2[i].load_state_dict(topts[g].state_dict())
        assert int(opts2[i].step_t) == 1
    model2._ensure_arena()
    for g, i in groups.items():
        for p2, c in zip(model2._group_params[g], clones[g]):
            model2._g(p2).copy_(c.grad)
        opts2[i].step()
        topts[g].step()
        for p2, c in zip(model2._group_params[g], clones[g]):
            assert torch.allclose(p2.detach(), c.detach(), rtol=1e-5, atol=1e-7), g
    with pytest.raises(ValueError):
        opts2[0].load_state_dict(topts["actor"].state_dict())       # wrong group: parameter count differs


def test_load_state_dict_refreshes_the_operand_shadows(ref_ops):
    """inference() -> reload weights -> inference() must act with the NEW weights (generator.py:105-116 reloads
    latest.pt into a live model): nn.Module.load_state_dict writes the arena in place, the hook marks the tf32 / fp16
    shadows and re-laid conv weights stale."""
    fx, conf, obs, state, noise = build_case("tiny_onehot")
    model = Dreamer(conf)
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    B = conf.batch_size
    o1 = {k: v[:1] for k, v in obs.items()}
    model._test_inference_noise = torch.empty(1, B, conf.stoch_dim * conf.stoch_discrete).exponential_()
    d1, s1, m1 = model.inference(o1, (state[0][:B], state[1][:B]))
    assert model._weights_dirty is False
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    for k in sd:
        if k.startswith("wm.encoder") or k.startswith("ac.actor"):
            sd[k] = sd[k] * 1.5 + 0.01
    model.load_state_dict(sd)
    assert model._weights_dirty is True
    d2, s2, m2 = model.inference(o1, (state[0][:B], state[1][:B]))
    assert not torch.allclose(d1.logits, d2.logits)
    fresh = Dreamer(conf)
    fresh.load_state_dict(sd)
    fresh._test_inference_noise = model._test_inference_noise
    d3, s3, m3 = fresh.inference(o1, (state[0][:B], state[1][:B]))
    assert torch.allclose(d2.logits, d3.logits, atol=1e-6) and torch.equal(s2[1], s3[1])


def test_non_unit_grad_output_scales_the_delivered_gradients(ref_ops):
    """(k * loss).backward() — what a GradScaler does under amp=True (train.py:143,184-187) — must scale that group's
    gradients by k; groups backwarded with the default grad_output stay untouched."""
    fx, conf, obs, state, noise, model, opts, losses, metrics = _stepped_model()
    base = {g: model._group_slice(g, model._garena).clone() for g in ("wm", "actor", "critic")}
    losses2, *_ = model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    (losses2[0] * 1024.0).backward()
    losses2[1].backward()
    losses2[2].backward(torch.tensor(0.5))
    losses2[3].backward()
    assert torch.allclose(model._group_slice("wm", model._garena), base["wm"] * 1024.0, rtol=1e-6)
    assert torch.allclose(model._group_slice("actor", model._garena), base["actor"] * 0.5, rtol=1e-6)
    assert torch.equal(model._group_slice("critic", model._garena), base["critic"])
    scaler_unscaled = model.wm.core.cell.z_mlp.weight.grad / 1024.0
    assert torch.allclose(scaler_unscaled, base["wm"][model._offsets[id(model.wm.core.cell.z_mlp.weight)]:][:scaler_unscaled.numel()].view_as(scaler_unscaled), rtol=1e-6)


def test_metrics_are_private_copies_and_accumulation_warns(ref_ops):
    fx, conf, obs, state, noise, model, opts, losses, metrics = _stepped_model()
    norms = model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
    kept = {k: float(v) for k, v in metrics.items()}
    kept_n = {k: float(v) for k, v in norms.items()}
    for o in opts:
        o.step()
    obs2 = {k: v.clone() for k, v in obs.items()}
    obs2["image"] = obs2["image"] * 0.5
    with warnings.catch_warnings():
        warnings.simplefilter("error")                     # step / zero_grad consumed the gradients: no warning
        losses2, _, metrics2, _, _ = model.training_step(obs2, state, noise=noise)
    for l in losses2:
        l.backward()
    model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
    assert abs(float(metrics2["loss_image"]) - kept["loss_image"]) > 1e-6
    for k, v in kept.items():
        assert float(metrics[k]) == v, k                   # the first step's metrics did not change under the caller
    for k, v in kept_n.items():
        assert float(norms[k]) == v, k
    with pytest.warns(UserWarning, match="gradient accumulation"):
        model.training_step(obs2, state, noise=noise)      # second backward pass without step / zero_grad in between

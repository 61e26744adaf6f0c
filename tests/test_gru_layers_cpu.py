"""A stacked GRU in the RSSM (`gru_layers` > 1), checked on CPU.

The module runs on the reference op table (oracle/ref_ops.py with the twins of oracle/vecobs_ops.py and
oracle/gru_ops.py) as in
tests/test_dreamer_cpu.py, against fixtures written from the unmodified reference by tests/golden/make_golden_gru.py: two and
four layers (the latter with three importance samples), the tanh_normal actor, a model without an image, and deter 66 in
three 22-unit layers."""
import json
import os

import pytest
import torch

import tests.test_dreamer_cpu as TD
from oracle import dreamer_oracle as DO
from oracle import gru_oracle as GO
from oracle.gru_ops import GruRefOps
from oracle.weights import seeded_state_dict
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.util import GOLDEN_DIR, build_case, seeded_weights

GRU_CASES = ("tiny_gru2", "tiny_gru4_iwae3", "tiny_dmc_gru2", "tiny_vector_gru2", "tiny_gru3_odd")
GRU_PRESETS = GRU_CASES + ("atari_gru2",)


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(GruRefOps("cpu"))
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


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "gru_state_dict.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", GRU_CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case)
    TD.check_golden(fx, model, losses, out_state, metrics, tensors)


@pytest.mark.parametrize("case", GRU_CASES)
def test_fp16_forward_and_persistent_unroll_branch(ref_ops, case):
    """With the fp16 forward and both persistent kernels switched on, a stacked model runs the persistent posterior unroll
    (its float32 twin) where D / L allows it, and the BPTT chain (the persistent BPTT runs one GRU cell)."""
    fx, conf, model, opts, losses, *_ = run_model(case, fp16_forward=True, persistent_rssm=True, persistent_bptt=True)
    BI = conf.batch_size * conf.iwae_samples
    assert model._persistent_rssm_ok(BI) == (case != "tiny_gru3_odd") and not model._persistent_bptt_ok(BI)
    assert model._fp16_forward_ok() == (case != "tiny_gru3_odd")
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):      # fp16 operands: the actor-critic losses move most
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= (5e-3 if i < 2 else 2e-2) * max(1.0, abs(want)), (i, got, want)


@pytest.mark.parametrize("case", ("tiny_gru2_log", "tiny_gru4_iwae3_log"))
def test_logging_eval_and_inference_branches_match_reference(ref_ops, case):
    fx, conf, out = TD.run_log_case(case)
    TD.check_log_case(fx, conf, out, 3e-4)


@pytest.mark.parametrize("preset", GRU_PRESETS)
def test_state_dict_keys_shapes_and_parameter_order_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g


def test_layer_shapes_follow_the_reference_stack():
    conf = make_conf("tiny_gru4_iwae3", device="cpu")
    sd = Dreamer(conf).state_dict()
    D, Hd, L = conf.deter_dim, conf.hidden_dim, conf.gru_layers
    for l in range(L):
        p = f"wm.core.cell.gru.layers.{l}."
        assert tuple(sd[p + "weight_ih"].shape) == (3 * D // L, Hd if l == 0 else D // L)
        assert tuple(sd[p + "weight_hh"].shape) == (3 * D // L, D // L)
        assert tuple(sd[p + "bias_ih"].shape) == tuple(sd[p + "bias_hh"].shape) == (3 * D // L,)
    assert f"wm.core.cell.gru.layers.{L}.weight_ih" not in sd


def test_checkpoint_round_trips_with_torch_adamw_over_the_reference_module(ref_ops):
    """The world-model optimizer's state_dict is torch.optim.AdamW's over the same parameter list (the reference's
    checkpoint, tools.py:171-172, 195-196), and loads back."""
    fx, conf, model, opts, losses, *_ = run_model("tiny_gru2")
    wm = list(model.wm.parameters())
    clones = [torch.nn.Parameter(p.detach().clone()) for p in wm]
    for c, p in zip(clones, wm):
        c.grad = p.grad.detach().clone()
    topt = torch.optim.AdamW(clones, lr=conf.adam_lr, eps=conf.adam_eps)
    opts[0].step()
    topt.step()
    ours, theirs = opts[0].state_dict(), topt.state_dict()
    assert ours["param_groups"][0]["params"] == theirs["param_groups"][0]["params"]
    assert set(ours["state"]) == set(theirs["state"])
    for i, st in theirs["state"].items():
        assert torch.allclose(st["exp_avg"], ours["state"][i]["exp_avg"], rtol=1e-5, atol=1e-9), i
        assert torch.allclose(st["exp_avg_sq"], ours["state"][i]["exp_avg_sq"], rtol=1e-5, atol=1e-12), i
    for c, p in zip(clones, wm):                                     # the stepped parameters too
        assert torch.allclose(c.detach(), p.detach(), rtol=1e-6, atol=1e-7)
    fresh = Dreamer(conf)
    fresh.load_state_dict(model.state_dict(), strict=True)
    fopts = fresh.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    fopts[0].load_state_dict(theirs)
    assert int(fopts[0].step_t.item()) == 1
    assert all(torch.equal(a, b) for a, b in zip(fresh.state_dict().values(), model.state_dict().values()))


def test_indivisible_deter_dim_and_other_cells_stay_refused():
    with pytest.raises(AssertionError, match="Must be divisible"):
        Dreamer(make_conf("tiny_gru2", gru_layers=3))                 # 64 % 3 != 0
    for cell in ("gru_layernorm", "gru_layernorm_dv2"):
        with pytest.raises(NotImplementedError, match="gru_type"):
            Dreamer(make_conf("tiny_gru2", gru_type=cell))
    with pytest.raises(NotImplementedError, match="gru_layers"):
        Dreamer(make_conf("tiny", gru_layers=0))


def test_single_layer_models_build_the_same_module():
    """gru_layers = 1 keeps its state_dict and the persistent routes."""
    a = Dreamer(make_conf("tiny"))
    assert [k for k in a.state_dict() if ".gru." in k] == [f"wm.core.cell.gru.layers.0.{n}" for n in
                                                         ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    assert a.d.L == 1 and a.d.Dl == a.d.D


def test_oracle_reproduces_the_module_on_a_fresh_batch(ref_ops):
    """The stacked-cell oracle and the module agree on a batch, weights and noise other than the fixtures'."""
    conf = make_conf("tiny_gru4_iwae3", device="cpu")
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    obs = synthetic_batch(conf, seed=77)
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
    sdo = {k: v.clone().requires_grad_(not k.startswith("ac.critic_target")) for k, v in sd.items()}
    res = GO.training_step(sdo, conf, obs, state, noise)
    for l in res["losses"]:
        l.backward()
    for a, b in zip(losses, res["losses"]):
        a, b = float(a.detach().reshape(-1)[0]), float(b.detach().reshape(-1)[0])
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b))
    assert torch.allclose(out_state[0], res["out_state"][0], rtol=1e-5, atol=1e-5)
    for n, p in model.named_parameters():
        if ".gru." in n:
            want = sdo[n].grad
            assert torch.allclose(p.grad, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), n

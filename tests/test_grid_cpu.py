"""Categorical grid images (`image_encoder: dense`, `image_decoder: dense`, `image_categorical`, `reward_input`), checked on
CPU.

The module runs on the reference op table (oracle/ref_ops.py with the twins of oracle/grid_ops.py) as in
tests/test_dreamer_cpu.py, against fixtures written from the unmodified reference by tests/golden/make_golden_grid.py: a
7x7x4 grid with reward and terminal planes (`tiny_grid`, also with three importance samples, with image_decoder_min_prob
and with MLPs without hidden layers), a 5x5x3 grid without planes and a grid plus a 27-float vector."""
import json
import os

import numpy as np
import pytest
import torch

import tests.test_dreamer_cpu as TD
from oracle import dreamer_oracle as DO
from oracle.grid_ops import GridRefOps
from oracle.grid_oracle import seeded_state_dict
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.util import GOLDEN_DIR, build_case

GRID_CASES = ("tiny_grid", "tiny_grid_iwae3", "tiny_grid_minprob", "tiny_grid_layers0", "tiny_grid_plain",
              "tiny_grid_vecobs")
GRID_PRESETS = GRID_CASES + ("minigrid",)


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(GridRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def grid_weights(model_state_dict, fx):
    return seeded_state_dict(model_state_dict, fx["seeds"]["weights"])


def run_model(case, device="cpu", **attrs):
    """tests/test_dreamer_cpu.run_model for the grid cases: fp32 forward and the per-timestep chains unless `attrs` (module
    attributes such as fp16_forward) say otherwise."""
    fx, conf, obs, state, noise = build_case(case, device)
    model = Dreamer(conf).to(device)
    attrs = dict(dict(fp16_forward=False, persistent_rssm=False, persistent_bptt=False), **attrs)
    for k, v in attrs.items():
        setattr(model, k, v)
    model.load_state_dict(grid_weights(model.state_dict(), fx))
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for o in opts:
        o.zero_grad()
    for l in losses:
        l.backward()
    return fx, conf, model, opts, losses, out_state, metrics, tensors


def run_log_case(case, monkeypatch, device="cpu"):
    monkeypatch.setattr(TD, "seeded_weights", grid_weights)
    return TD.run_log_case(case, device)


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "grid_state_dict.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", GRID_CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case)
    TD.check_golden(fx, model, losses, out_state, metrics, tensors)
    s = conf.image_size
    assert tensors["image_rec"].shape == (conf.batch_length, conf.batch_size, conf.image_channels, s, s)


@pytest.mark.parametrize("case", GRID_CASES)
def test_persistent_rssm_and_bptt_branches(ref_ops, case):
    fx, conf, model, opts, losses, *_ = run_model(case, fp16_forward=True, persistent_rssm=True, persistent_bptt=True)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):      # fp16 operands: the actor-critic losses move most
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= (5e-3 if i < 2 else 2e-2) * max(1.0, abs(want)), (i, got, want)


@pytest.mark.parametrize("case", ("tiny_grid_log", "tiny_grid_iwae3_log"))
def test_logging_eval_and_inference_branches_match_reference(ref_ops, monkeypatch, case):
    fx, conf, out = run_log_case(case, monkeypatch)
    TD.check_log_case(fx, conf, out, 3e-4)
    tensors, dream = out["train_log"][3], out["train_log"][4]
    s = conf.image_size
    shape = (conf.batch_length, conf.batch_size, conf.image_channels, s, s)
    assert tensors["image_pred"].shape == shape and dream["image_pred"].shape == shape
    assert "logprob_image" in out["train_log"][2]


@pytest.mark.parametrize("preset", GRID_PRESETS)
def test_state_dict_keys_shapes_and_parameter_order_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g


def test_state_dict_loads_strictly_both_ways(ref_ops):
    conf = make_conf("tiny_grid", device="cpu")
    a, b = Dreamer(conf), Dreamer(conf)
    fx = _state_dict_fixture()["tiny_grid"]["state_dict"]
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(shape, generator=g) if shape else torch.randn((), generator=g) for k, shape in fx}
    a.load_state_dict(sd, strict=True)
    out = a.state_dict()
    assert list(out) == [k for k, _ in fx] and all(torch.equal(out[k], sd[k]) for k in sd)
    b.load_state_dict(out, strict=True)
    assert all(torch.equal(b.state_dict()[k], sd[k]) for k in sd)


def test_optimizer_state_dict_matches_torch_adamw(ref_ops):
    fx, conf, model, opts, losses, *_ = run_model("tiny_grid")
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
    opts[0].load_state_dict(theirs)
    assert int(opts[0].step_t.item()) == 1


def test_new_limits_refuse_just_past_each_bound():
    for over, kernel in ((dict(image_channels=65), "pd_cat_image_loss"), (dict(image_channels=1), "pd_cat_image_loss"),
                         (dict(image_size=65), "pd_cat_image_loss")):
        with pytest.raises(NotImplementedError, match=kernel):
            Dreamer(make_conf("tiny_grid", **over))
    Dreamer(make_conf("tiny_grid", image_channels=64, image_size=64, image_encoder_layers=0, image_decoder_layers=0))
    Dreamer(make_conf("tiny_grid", image_channels=2))
    # the conv path keeps its own channel limit
    with pytest.raises(NotImplementedError, match="pd_col2im_imgloss"):
        Dreamer(make_conf("tiny", image_channels=17))


def test_combinations_that_stay_refused():
    with pytest.raises(NotImplementedError):
        Dreamer(make_conf("tiny_grid", probe_model="map"))
    with pytest.raises(NotImplementedError):
        Dreamer(make_conf("minigrid", probe_model="map"))
    for bad in (dict(image_decoder="cnn"), dict(image_encoder="cnn"), dict(image_decoder=None), dict(layer_norm=False),
                dict(stoch_discrete=0)):
        with pytest.raises(NotImplementedError):
            Dreamer(make_conf("tiny_grid", **bad))
    with pytest.raises(NotImplementedError, match="categorical"):
        Dreamer(make_conf("tiny_grid", image_categorical=False))
    with pytest.raises(NotImplementedError, match="reward_input"):
        Dreamer(make_conf("tiny", reward_input=True))


def test_conv_and_image_less_models_build_no_grid_buffers(ref_ops):
    for case in ("tiny_onehot",):
        fx, conf, obs, state, noise = build_case(case)
        model = Dreamer(conf)
        model.training_step(obs, state, noise=noise)
        assert not any(k[0].startswith(("enc.gin", "gdec.", "denc.")) for k in model._ws)
    fx, conf, obs, state, noise = build_case("tiny_grid")
    model = Dreamer(conf)
    model.training_step(obs, state, noise=noise)
    names = {k[0] for k in model._ws}
    assert "enc.gin" in names and "gdec.y" in names and not any(n.startswith(("enc.a", "dec.", "encw", "decw")) for n in names)


def test_synthetic_batches_are_one_hot_and_leave_other_batches_unchanged():
    conf = make_conf("tiny_grid")
    obs = synthetic_batch(conf, seed=5)
    img = obs["image"]
    assert img.shape == (4, 3, 4, 7, 7) and torch.equal(img.sum(2), torch.ones(4, 3, 7, 7))
    plain = synthetic_batch(make_conf("tiny_grid", image_categorical=False), seed=5)
    assert torch.equal(img, torch.nn.functional.one_hot(plain["image"].argmax(2), 4).movedim(-1, 2).float())
    assert all(torch.equal(obs[k], plain[k]) for k in obs if k != "image")


@pytest.mark.parametrize("dtype", (torch.uint8, torch.int32, torch.int64, torch.int16))
def test_preprocessor_one_hot_matches_reference_preprocessor(ref_ops, dtype):
    from pydreamer_b200.preprocess import GpuPreprocessor

    conf = make_conf("tiny_grid", device="cpu")
    T, B, C = 4, 3, conf.image_channels
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, C, (T, B, 7, 7), generator=g)
    raw = dict(image=ids.to(dtype), action=torch.randint(0, 7, (T, B)), reward=torch.randn(T, B), terminal=torch.zeros(T, B),
               reset=torch.zeros(T, B, dtype=torch.bool))
    out = GpuPreprocessor(conf, "cpu").apply(raw)
    # preprocessing.py:10-19 (img_to_onehot)
    want = np.eye(C, dtype=np.float32)[ids.numpy()].transpose(0, 1, 4, 2, 3)
    assert out["image"].dtype == torch.float32 and torch.equal(out["image"], torch.from_numpy(want))


def test_out_of_range_ids_give_nan_channels_and_nan_losses(ref_ops):
    from pydreamer_b200.preprocess import GpuPreprocessor

    conf = make_conf("tiny_grid", device="cpu")
    T, B, C = conf.batch_length, conf.batch_size, conf.image_channels
    ids = torch.randint(0, C, (T, B, 7, 7), generator=torch.Generator().manual_seed(4)).to(torch.uint8)
    ids[1, 2, 3, 4] = C
    raw = dict(image=ids, action=torch.randint(0, 7, (T, B)), reward=torch.randn(T, B), terminal=torch.zeros(T, B),
               reset=torch.zeros(T, B, dtype=torch.bool))
    obs = GpuPreprocessor(conf, "cpu").apply(raw)
    img = obs["image"]
    assert torch.isnan(img[1, 2, :, 3, 4]).all() and int(torch.isnan(img).sum()) == C
    model = Dreamer(conf)
    losses, *_ = model.training_step(obs, model.init_state(B))
    assert torch.isnan(losses[0])


def test_oracle_reproduces_the_module_with_teacher_forced_samples(ref_ops):
    """The grid oracle and the module agree on a fresh synthetic batch (seed other than the fixtures')."""
    from oracle import grid_oracle as GO

    conf = make_conf("tiny_grid_iwae3", device="cpu")
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    obs = synthetic_batch(conf, seed=77)
    state = (torch.zeros(B * I, conf.deter_dim), torch.zeros(B * I, conf.stoch_dim * conf.stoch_discrete))
    torch.manual_seed(5)
    noise = DO.draw_noise(conf, T, B)
    model = Dreamer(conf)
    model.fp16_forward = model.persistent_rssm = model.persistent_bptt = False
    sd = seeded_state_dict(model.state_dict(), 11)
    model.load_state_dict(sd)
    losses, _, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    res = GO.training_step(sd, conf, obs, state, noise)
    for a, b in zip(losses, res["losses"]):
        assert abs(float(a.detach().reshape(-1)[0]) - float(b.reshape(-1)[0])) <= 2e-5 * max(1.0, abs(float(b.reshape(-1)[0])))
    assert torch.allclose(tensors["image_rec"], res["tensors"]["image_rec"], rtol=1e-5, atol=1e-5)
    assert torch.allclose(tensors["loss_image"], res["tensors"]["loss_image"], rtol=1e-5, atol=1e-4)

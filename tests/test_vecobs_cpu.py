"""Vector observations (`vecobs_size`) with and without the image encoder / decoder, checked on CPU.

The module runs on the reference op table (oracle/ref_ops.py, with the vecobs twins of oracle/vecobs_ops.py) as in
tests/test_dreamer_cpu.py, against fixtures written from the unmodified reference by tests/golden/make_golden_vecobs.py:
a 64x64 image plus a 27-float vector (`tiny_vecobs`, also with three importance samples) and a 4-float vector without any
image (`tiny_vector`)."""
import json
import os

import pytest
import torch

from oracle.vecobs_ops import VecRefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_dreamer_cpu import check_log_case, run_log_case, run_model
from tests.util import GOLDEN_DIR, build_case

VEC_CASES = ("tiny_vecobs", "tiny_vecobs_iwae3", "tiny_vector")


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(VecRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def _state_dict_fixture():
    with open(os.path.join(GOLDEN_DIR, "vecobs_state_dict.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", VEC_CASES)
def test_training_step_matches_reference_golden(ref_ops, case):
    fx, conf, model, opts, losses, out_state, metrics, tensors = run_model(case)
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 2e-5 * max(1.0, abs(want))
    assert set(metrics) == set(fx["metrics"]) and "loss_vecobs" in metrics
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= 2e-4 * max(1.0, abs(want)), k
    assert set(tensors) == set(fx["tensor_sums"])
    assert tensors["vecobs_rec"].shape == (conf.batch_length, conf.batch_size, conf.vecobs_size)
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


@pytest.mark.parametrize("case", VEC_CASES)
def test_persistent_rssm_and_bptt_branches(ref_ops, case):
    """The single-call posterior unroll and BPTT branches read only the hoisted embedding product: same goldens within
    the fp16-operand tolerances of tests/test_dreamer_cpu.py."""
    fx, conf, model, opts, losses, *_ = run_model(case, fp16_forward=True, persistent_rssm=True, persistent_bptt=True)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples)
    for i, (got, want) in enumerate(zip(losses, fx["losses"])):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-3 * max(1.0, abs(want)), (i, got, want)


@pytest.mark.parametrize("case", [c + "_log" for c in VEC_CASES])
def test_logging_eval_and_inference_branches_match_reference(ref_ops, case):
    fx, conf, out = run_log_case(case)
    check_log_case(fx, conf, out, 3e-4)
    tensors, dream = out["train_log"][3], out["train_log"][4]
    assert "vecobs_pred" in tensors and "logprob_vecobs" in out["train_log"][2]
    if not conf.image_decoder:
        assert dream == {} and not any("image" in k for k in tensors)


@pytest.mark.parametrize("preset", ("tiny_vecobs", "tiny_vector", "vectorenv", "minecraft"))
def test_state_dict_keys_shapes_and_parameter_order_match_reference(preset):
    fx = _state_dict_fixture()[preset]
    model = Dreamer(make_conf(preset, device="cpu"))
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == fx["state_dict"]
    groups = dict(wm=model.wm, probe=model.probe_model, actor=model.ac.actor, critic=model.ac.critic)
    names = {id(p): n for n, p in model.named_parameters()}
    for g, mod in groups.items():
        assert [[names[id(p)], list(p.shape)] for p in mod.parameters()] == fx["params"][g], g


def test_state_dict_loads_strictly_both_ways(ref_ops):
    """A reference-layout state dict (keys, shapes, values) loads strictly, and what the module saves carries the same
    keys and values back."""
    conf = make_conf("tiny_vecobs", device="cpu")
    a, b = Dreamer(conf), Dreamer(conf)
    fx = _state_dict_fixture()["tiny_vecobs"]["state_dict"]
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(shape, generator=g) if shape else torch.randn((), generator=g) for k, shape in fx}
    a.load_state_dict(sd, strict=True)
    out = a.state_dict()
    assert list(out) == [k for k, _ in fx] and all(torch.equal(out[k], sd[k]) for k in sd)
    b.load_state_dict(out, strict=True)
    assert all(torch.equal(b.state_dict()[k], sd[k]) for k in sd)


def test_optimizer_state_dict_matches_torch_adamw(ref_ops):
    """_FusedAdamW indexes parameters by position: with the vecobs MLPs registered in the reference's module order its
    state_dict equals that of torch.optim.AdamW over the same parameters, and loads back."""
    fx, conf, model, opts, losses, *_ = run_model("tiny_vecobs")
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
        assert st["exp_avg"].shape == ours["state"][i]["exp_avg"].shape
        assert torch.allclose(st["exp_avg"], ours["state"][i]["exp_avg"], rtol=1e-5, atol=1e-9), i
        assert torch.allclose(st["exp_avg_sq"], ours["state"][i]["exp_avg_sq"], rtol=1e-5, atol=1e-12), i
    opts[0].load_state_dict(theirs)
    assert int(opts[0].step_t.item()) == 1


def test_refused_combinations():
    for bad in (dict(image_encoder="cnn", image_decoder=None), dict(image_encoder=None, image_decoder="cnn"),
                dict(image_encoder="dense", image_decoder="dense"), dict(reward_input=True),
                dict(probe_model="map")):
        with pytest.raises(NotImplementedError):
            Dreamer(make_conf("tiny_vecobs", **bad))
    with pytest.raises(AssertionError):
        Dreamer(make_conf("tiny_vector", vecobs_size=0))                   # encoders.py:38
    Dreamer(make_conf("tiny_vector", image_size=32))                        # no image: image_size is not read


def test_image_less_model_allocates_no_image_buffers_and_synthetic_batches(ref_ops):
    fx, conf, obs, state, noise = build_case("tiny_vector")
    assert "image" not in obs and obs["vecobs"].shape == (conf.batch_length, conf.batch_size, 4)
    model = Dreamer(conf)
    model.training_step(obs, state, noise=noise)
    names = {k[0] for k in model._ws}
    assert not any(n.startswith(("enc.a", "enc.col", "dec.", "bwd.dd", "bwd.gdec", "bwd.genc", "bwd.da", "encw", "decw"))
                   for n in names), sorted(names)
    assert "enc.vembed" in names and "head.yv" in names
    # batches of the image-only configurations do not change when the vector draw is added after them
    c = make_conf("tiny")
    a = synthetic_batch(c, seed=5)
    b = synthetic_batch(make_conf("tiny", vecobs_size=3), seed=5)
    assert set(b) == set(a) | {"vecobs"} and all(torch.equal(a[k], b[k]) for k in a)


def test_preprocessor_passes_vecobs_through_without_an_image(ref_ops):
    from pydreamer_b200.preprocess import GpuPreprocessor

    conf = make_conf("tiny_vector", device="cpu")
    pre = GpuPreprocessor(conf, "cpu")
    T, B = 4, 3
    raw = dict(vecobs=torch.randn(T, B, 4, dtype=torch.float64), action=torch.randint(0, 3, (T, B)),
               reward=torch.randn(T, B), terminal=torch.zeros(T, B), reset=torch.zeros(T, B, dtype=torch.bool))
    out = pre.apply(raw)
    assert "image" not in out and out["vecobs"].dtype == torch.float32
    assert torch.equal(out["vecobs"], raw["vecobs"].float()) and out["action"].shape == (T, B, 3)

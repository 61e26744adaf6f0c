"""Learner step + checkpoint format (SURVEY.md §8f N1) on CPU with the reference op table; the checkpoint carries every
key of the UNMODIFIED reference Dreamer's state_dict, and only those, with their shapes (tests/golden/state_dict_keys.json)."""
import json
import os

import pytest
import torch

from oracle.ref_ops import RefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.learner import Learner
from pydreamer_b200.replay import synthetic_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(RefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def test_learner_steps_carry_state_and_checkpoint_roundtrip(ref_ops, tmp_path):
    conf = make_conf("tiny", device="cpu")
    lr = Learner(conf, "cpu")
    m0 = {k: v.clone() for k, v in lr.model.state_dict().items()}
    b1, b2 = synthetic_batch(conf, seed=1), synthetic_batch(conf, seed=2, first=False)
    met1, tensors, _ = lr.step(b1)
    assert {"loss_model", "loss_kl", "grad_norm", "grad_norm_actor", "grad_norm_critic", "grad_norm_probe"} <= set(met1)
    assert 0 in lr.states and lr.states[0][0].shape == (conf.batch_size, conf.deter_dim)
    met2, _, _ = lr.step(b2, do_image_pred=True)
    assert "logprob_image" in met2 and lr.steps == 2
    changed = sum(not torch.equal(m0[k], v) for k, v in lr.model.state_dict().items())
    assert changed > 100                                      # parameters moved
    path = str(tmp_path / "latest.pt")
    lr.save_checkpoint(path)
    ck = torch.load(path)
    assert set(ck) == {"epoch", "model_state_dict", "optimizer_0_state_dict", "optimizer_1_state_dict",
                       "optimizer_2_state_dict", "optimizer_3_state_dict"}                       # tools.py:164-174
    lr2 = Learner(conf, "cpu")
    assert lr2.load_checkpoint(path) == 2
    for (k, a), (_, b_) in zip(lr.model.state_dict().items(), lr2.model.state_dict().items()):
        assert torch.equal(a, b_), k
    # the reference module loads the checkpoint strictly (generator.py:109): exactly its state_dict keys, with its shapes
    # (tests/golden/state_dict_keys.json, written from the reference by tests/golden/make_param_order.py)
    with open(os.path.join(ROOT, "tests", "golden", "state_dict_keys.json")) as f:
        want = {k: shape for k, shape in json.load(f)["tiny"]}
    assert set(ck["model_state_dict"]) == set(want)
    for name, shape in want.items():
        assert list(ck["model_state_dict"][name].shape) == shape, name


def test_learner_trains_from_raw_replay_batches(ref_ops):
    """Raw replay batches (uint8 HWC images, integer actions: what the reference's DataSequential yields) -> device-side
    preprocessing -> gradient steps, state carried across consecutive windows."""
    import numpy as np

    conf = make_conf("tiny", device="cpu", reset_interval=0)
    rng = np.random.default_rng(0)
    T, B = conf.batch_length, conf.batch_size

    def batches():
        first = True
        while True:
            reset = np.zeros((T, B), bool)
            reset[0] = first
            first = False
            yield dict(image=rng.integers(0, 256, (T, B, 64, 64, 3), dtype=np.uint8),
                       action=rng.integers(0, conf.action_dim, (T, B)), reward=rng.normal(size=(T, B)).astype(np.float32),
                       terminal=np.zeros((T, B), bool), reset=reset)

    lr = Learner(conf, "cpu")
    metrics = lr.train_on_batches(batches(), 3)
    assert lr.steps == 3 and torch.isfinite(metrics["loss_model"]) and float(metrics["grad_norm"]) > 0
    assert lr.states[0][0].shape == (conf.batch_size, conf.deter_dim)          # state carried across the windows

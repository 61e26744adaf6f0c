"""A stacked GRU in the RSSM (`gru_layers` > 1) through the native kernels: the module against the reference goldens (exact
arm) and against the teacher-forced stacked-cell oracle (TF32 product arm, the posterior unroll as a chain and as one
persistent kernel), the logging / evaluation / inference branches, graph replay and the concurrent branches bit for bit
against one-stream eager launches, and the full-size `atari_gru2` step with the persistent unroll against the chain."""
import pytest
import torch

import tests.test_vecobs_gpu as TV
from oracle import gru_oracle
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_step_schedule_gpu import train_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRU_CASES = ("tiny_gru2", "tiny_gru4_iwae3", "tiny_dmc_gru2", "tiny_vector_gru2", "tiny_gru3_odd")


@pytest.fixture()
def gru_oracle_checks(monkeypatch):
    """tests/test_vecobs_gpu.check_against_oracle with the stacked-cell oracle."""
    monkeypatch.setattr(TV, "O", gru_oracle)
    return TV.check_against_oracle


@pytest.mark.parametrize("case", GRU_CASES)
def test_exact_arm_matches_reference_golden(case):
    TV.test_exact_arm_matches_reference_golden(case)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
@pytest.mark.parametrize("case", GRU_CASES)
def test_product_arm_teacher_forced_against_oracle(gru_oracle_checks, case, persistent):
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = TV.run_gpu(case, impl=0, rounding=True,
                                                                                   persistent=persistent)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples) == (persistent and case != "tiny_gru3_odd")
    gru_oracle_checks(conf, obs, state, noise, model, losses, metrics, tensors)


@pytest.mark.parametrize("case,rtol", [("tiny_gru2_log", 2e-3), ("tiny_gru4_iwae3_log", 6e-3)])
def test_logging_eval_and_inference_branches_on_gpu(case, rtol):
    """As tests/test_vecobs_gpu.py: the TF32 product arm against the reference's outputs; 6e-3 with importance samples."""
    from tests.test_dreamer_cpu import check_log_case, run_log_case
    fx, conf, out = run_log_case(case, DEV)
    check_log_case(fx, conf, out, rtol)


@pytest.mark.parametrize("preset", ("tiny_gru2", "tiny_dmc_gru2", "tiny_gru3_odd"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    """(Presets without importance samples: the shared helper carries a state of batch_size rows.)"""
    TV.test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset)


@pytest.mark.parametrize("preset", ("tiny_gru2", "atari_gru2"))
def test_three_eager_steps_are_identical(preset):
    TV.test_three_eager_steps_are_identical(preset)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
def test_full_size_atari_gru2_step_teacher_forced_against_oracle(gru_oracle_checks, persistent):
    """The Atari benchmark shape with two 1024-unit layers (T=B=50, deter 2048) on the product arm, the posterior unroll as
    the chain and as the persistent kernel; the oracle re-runs the first 2 sequences teacher-forced on the GPU's samples:
    2e-3 relative on the per-(t,b) tensors, as at the Atari shape."""
    conf = make_conf("atari_gru2", device=DEV)
    T, B, H = conf.batch_length, conf.batch_size, conf.imag_horizon
    Z, N = conf.stoch_dim * conf.stoch_discrete, T * B
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
    model.persistent_rssm = persistent
    obs = synthetic_batch(conf, seed=77, device=DEV)
    state = (torch.tanh(torch.randn(B, conf.deter_dim, device=DEV)), torch.zeros(B, Z, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(5)
    noise = dict(post=torch.empty(T, B, Z, device=DEV).exponential_(generator=g),
                 actor=torch.empty(H, N, conf.action_dim, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    losses, _, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    assert model._persistent_rssm_ok(B) == persistent and model._fp16_forward_ok()
    assert all(torch.isfinite(l).all() for l in losses)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.requires_grad)
    gru_oracle_checks(conf, obs, state, noise, model, losses, metrics, tensors, S=2)


def test_single_layer_and_stacked_models_differ_only_in_the_recurrent_launches():
    """Same shape, L = 1 against L = 2 on the chain: the stack adds (L - 1) x 3 forward launches per posterior and dream
    step (the extra layer's W_ih and W_hh products and its gate kernel), and (L - 1) x 3 per BPTT step plus 4 weight /
    bias gradient launches."""
    counts = {}
    for L in (1, 2):
        conf = make_conf("tiny", device=DEV, gru_layers=L)
        m = Dreamer(conf).to(DEV)
        m.persistent_rssm = m.persistent_bptt = False
        m.use_cuda_graph = False
        opts = m.init_optimizers(conf.adam_lr)
        obs = synthetic_batch(conf, seed=7, device=DEV)
        state = m.init_state(conf.batch_size)
        train_step(m, opts, conf, obs, state)                      # loads the kernels, allocates the workspace
        counts[L] = train_step(m, opts, conf, obs, state)[2]       # the library launches of training_step
    T, H = conf.batch_length, conf.imag_horizon
    assert counts[2] - counts[1] == 3 * T + 3 * H + 3 * T + 4, counts

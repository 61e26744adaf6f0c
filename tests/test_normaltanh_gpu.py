"""The normal_tanh actor (`actor_dist: normal_tanh`) through the native kernels: the module against the reference goldens
(exact arm) and against the teacher-forced oracle (TF32 product arm, the posterior unroll as a chain and as one persistent
kernel), the logging / evaluation / inference branches, graph replay and the concurrent branches bit for bit against
one-stream eager launches, identical seeded runs, and the full-size `dmc_normaltanh` shape: one step against the oracle and
a few optimizer steps through the learner."""
from types import SimpleNamespace

import pytest
import torch

import tests.test_vecobs_gpu as TV
from oracle import normaltanh_oracle
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_step_schedule_gpu import graph_state

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = ("tiny_dmc_normaltanh", "tiny_dmc_normaltanh_iwae3", "tiny_vector_normaltanh")


@pytest.fixture(autouse=True)
def normaltanh_oracle_checks(monkeypatch):
    """tests/test_vecobs_gpu.check_against_oracle with the normal_tanh oracle."""
    monkeypatch.setattr(TV, "O", normaltanh_oracle)


@pytest.mark.parametrize("case", CASES)
def test_exact_arm_matches_reference_golden(case):
    TV.test_exact_arm_matches_reference_golden(case)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
@pytest.mark.parametrize("case", CASES)
def test_product_arm_teacher_forced_against_oracle(case, persistent):
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = TV.run_gpu(case, impl=0, rounding=True,
                                                                                   persistent=persistent)
    H, N, A = conf.imag_horizon, conf.batch_length * conf.batch_size * conf.iwae_samples, conf.action_dim
    acts, alog = model._buf("dream.actions", H, N, A), model._buf("dream.alog", H, N, model.d.Ap)[..., :2 * A]
    want = torch.tanh(alog[..., :A].double()) + (torch.sigmoid(alog[..., A:].double()) + 0.01) * noise["actor"].double()
    assert torch.allclose(acts.double(), want, rtol=1e-6, atol=1e-6)        # the unbounded sample on the GPU's logits
    TV.check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors)


@pytest.mark.parametrize("over", [dict(aux_critic=True), dict(gru_layers=2)], ids=("aux_critic", "gru2"))
@pytest.mark.parametrize("case", ("tiny_dmc_normaltanh", "tiny_vector_normaltanh"))
def test_aux_critic_and_stacked_gru_teacher_forced_against_oracle(monkeypatch, case, over):
    """The same step with the auxiliary critic or a two-layer GRU (no reference fixtures: the preset's seeds, held to the
    oracle) on the exact arm: with TF32 products the unbounded actions carry the rounding of the dream into the critic's
    output-bias gradient, a signed sum over the H*N dreamed rows, past the product arm's bounds."""
    from tests.util import load_fixture
    fx = dict(load_fixture(case), overrides=over)
    monkeypatch.setattr("tests.util.load_fixture", lambda name: fx)
    _, conf, obs, state, noise, model, losses, metrics, tensors, _ = TV.run_gpu(case, impl=1, rounding=False)
    assert all(getattr(conf, k) == v for k, v in over.items())
    TV.check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors)


def test_logging_eval_and_inference_branches_on_gpu():
    """The TF32 product arm against the reference's logging, open-loop and inference outputs; inference returns the
    reference's Independent(Normal) (tests/test_normaltanh_cpu.py explains the shim).  6e-3, as with importance samples
    in tests/test_vecobs_gpu.py: the logged dream's signed advantage sum moves by 2e-3 of its absolute sum under TF32."""
    from tests.test_dreamer_cpu import check_log_case, run_log_case
    fx, conf, out = run_log_case("tiny_dmc_normaltanh_log", DEV)
    dist, os3, m3 = out["inference"]
    assert type(dist) is torch.distributions.Independent and type(dist.base_dist) is torch.distributions.Normal
    shim = SimpleNamespace(base_dist=dist, sample=dist.sample, log_prob=dist.log_prob)
    check_log_case(fx, conf, dict(out, inference=(shim, os3, m3)), 6e-3)


@pytest.mark.parametrize("preset", ("tiny_dmc_normaltanh", "tiny_vector_normaltanh"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    TV.test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset)


@pytest.mark.parametrize("preset", ("tiny_dmc_normaltanh", "dmc_normaltanh"))
def test_three_eager_steps_are_identical(preset):
    TV.test_three_eager_steps_are_identical(preset)


def test_full_size_dmc_normaltanh_step_teacher_forced_against_oracle():
    """The DMC benchmark shape (T=B=50, deter 1024, A=12) on the product arm; the oracle re-runs the first 2 sequences
    teacher-forced on the GPU's samples: 2e-3 relative on the per-(t,b) tensors."""
    conf = make_conf("dmc_normaltanh", device=DEV)
    T, B, H = conf.batch_length, conf.batch_size, conf.imag_horizon
    Z, N = conf.stoch_dim * conf.stoch_discrete, T * B
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
    obs = synthetic_batch(conf, seed=77, device=DEV)
    state = (torch.tanh(torch.randn(B, conf.deter_dim, device=DEV)), torch.zeros(B, Z, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(5)
    noise = dict(post=torch.empty(T, B, Z, device=DEV).exponential_(generator=g),
                 actor=torch.empty(H, N, conf.action_dim, device=DEV).normal_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    losses, _, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(l).all() for l in losses)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.requires_grad)
    assert float(model._buf("dream.actions", H, N, conf.action_dim).abs().max()) > 1.0      # not squashed
    TV.check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, S=2)


def test_dmc_normaltanh_trains_through_the_learner_with_graph_replay():
    """A few optimizer steps at the benchmark shape: finite losses, metrics and gradient norms, and the step captured."""
    from pydreamer_b200.learner import Learner
    conf = make_conf("dmc_normaltanh", device=DEV)
    lr = Learner(conf, DEV)
    for i in range(4):
        metrics, tensors, _ = lr.step(synthetic_batch(conf, seed=i, first=(i == 0), device=DEV))
    torch.cuda.synchronize()
    st = graph_state(lr.model)
    assert st["graph"] is not None and not st.get("failed")
    assert all(torch.isfinite(v).all() for v in metrics.values()), metrics
    for k in ("loss_actor", "policy_entropy", "grad_norm", "grad_norm_actor", "grad_norm_critic"):
        assert k in metrics, k
    assert all(p.isfinite().all() for p in lr.model.parameters())

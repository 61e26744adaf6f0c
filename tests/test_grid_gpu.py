"""Categorical grid images through the native kernels: the module against the reference goldens (exact arm), against the
teacher-forced grid oracle (TF32 product arm), graph replay and the concurrent branches bit for bit against one-stream
eager launches, the shipped `minigrid` shape through the learner from raw uint8 category ids, and the full-size `minigrid`
step and the B = 10, T = 10 shape against the fp32 oracle."""
import weakref

import pytest
import torch

import tests.test_dreamer_cpu as TD
import tests.test_vecobs_gpu as VG
from oracle import grid_oracle as GO
from oracle.grid_oracle import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_grid_cpu import GRID_CASES, grid_weights, run_log_case
from tests.test_step_schedule_gpu import assert_identical, graph_state, released, train_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture()
def grid_oracle(monkeypatch):
    """tests/test_vecobs_gpu.check_against_oracle and its weight seeding with the grid restatement."""
    monkeypatch.setattr(VG, "O", GO)
    monkeypatch.setattr(VG, "seeded_weights", grid_weights)
    monkeypatch.setattr(VG, "seeded_state_dict", seeded_state_dict)


@pytest.mark.parametrize("case", GRID_CASES)
def test_exact_arm_matches_reference_golden(grid_oracle, case):
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = VG.run_gpu(case, impl=1, rounding=False)
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-5 * max(1.0, abs(want)), (got, want)
    assert set(metrics) == set(fx["metrics"])
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= 2e-4 * max(1.0, abs(want)), k
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        assert abs(got - want) <= 1e-3 * max(want, 1e-6) + 1e-9, (k, got, want)
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= 3e-4 * max(want, 1e-6), (k, got, want)


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
@pytest.mark.parametrize("case", GRID_CASES)
def test_product_arm_teacher_forced_against_oracle(grid_oracle, case, persistent):
    """tests/test_vecobs_gpu.py's criteria at 2.5x: the bias gradients of the reward head are signed sums over every row,
    which at the 5x5x3 shape cancel to ~6e-3 of their terms under TF32 operands."""
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = VG.run_gpu(case, impl=0, rounding=True,
                                                                                   persistent=persistent)
    VG.check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, tol=2.5)


@pytest.mark.parametrize("case,rtol", [("tiny_grid_log", 2e-2), ("tiny_grid_iwae3_log", 6e-3)])
def test_logging_eval_and_inference_branches_on_gpu(monkeypatch, case, rtol):
    """The logging / evaluation branches through the product arm (fp16 operands in the dream) against the reference's
    outputs.  At `tiny_grid` (B = 3, H = 3) the actor loss, a sum of advantage-weighted terms that largely cancel, moves by
    ~1e-2 of its magnitude: 2e-2 there."""
    fx, conf, out = run_log_case(case, monkeypatch, DEV)
    TD.check_log_case(fx, conf, out, rtol)


def make_model(preset, graphs, overlap):
    conf = make_conf(preset, device=DEV, target_interval=2)
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    m = Dreamer(conf).to(DEV)
    m.load_state_dict(seeded_state_dict(m.state_dict(), 11))
    m.use_cuda_graph, m.overlap, m.persistent_rssm, m.persistent_bptt = graphs, overlap, True, False
    return conf, m, m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)


@pytest.mark.parametrize("preset", ("tiny_grid", "tiny_grid_iwae3"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    STEPS = 5
    conf, m, opts = make_model(preset, graphs=True, overlap=Dreamer.overlap)
    obs = [synthetic_batch(conf, seed=100 + i, first=(i == 0), device=DEV) for i in range(STEPS)]
    state = m.init_state(conf.batch_size * conf.iwae_samples)
    arms, noises = {"graph": []}, []
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state)
        assert not warned, warned
        noises.append(VG.drawn_noise(m, conf, obs[i]))
        arms["graph"].append(rec)
    st = graph_state(m)
    assert st["graph"] is not None and not st.get("failed")
    ref = weakref.ref(m)
    del m, opts
    released(ref)
    for mask in range(1, 8):
        conf, m, opts = make_model(preset, graphs=False, overlap=mask)
        state = m.init_state(conf.batch_size * conf.iwae_samples)
        arms[f"overlap{mask}"] = []
        for i in range(2):
            rec, state, n, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i])
            arms[f"overlap{mask}"].append(rec)
        del m, opts
    conf, m, opts = make_model(preset, graphs=False, overlap=0)
    state = m.init_state(conf.batch_size * conf.iwae_samples)
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i])
        for name, recs in arms.items():
            if i < len(recs):
                assert_identical(f"[{preset}] {name} step {i + 1}", rec, recs[i])
        if i == 2:
            assert st["kernels"] == n


def test_minigrid_trains_through_the_learner_from_uint8_ids_with_graph_replay():
    from pydreamer_b200.learner import Learner
    conf = make_conf("minigrid", device=DEV)
    lr = Learner(conf, DEV)
    T, B = conf.batch_length, conf.batch_size

    def raw(i):
        g = torch.Generator().manual_seed(i)
        r = dict(image=torch.randint(0, conf.image_channels, (T, B, 7, 7), generator=g).to(torch.uint8),
                 action=torch.randint(0, conf.action_dim, (T, B), generator=g), reward=torch.rand(T, B, generator=g),
                 terminal=(torch.rand(T, B, generator=g) < 0.02).float(), reset=torch.zeros(T, B, dtype=torch.bool))
        r["reset"][0] = i == 0
        return r

    metrics = lr.train_on_batches((raw(i) for i in range(4)), 4)
    torch.cuda.synchronize()
    st = graph_state(lr.model)
    assert st["graph"] is not None and not st.get("failed")
    assert all(torch.isfinite(v).all() for v in metrics.values()), metrics
    assert "loss_image" in metrics


def _full_step(preset, S, **over):
    conf = make_conf(preset, device=DEV, **over)
    T, B, H = conf.batch_length, conf.batch_size, conf.imag_horizon
    Z, N = conf.stoch_dim * conf.stoch_discrete, T * B
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 11))
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
    assert all(torch.isfinite(l).all() for l in losses)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.requires_grad)
    VG.check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, S=S)


def test_full_size_minigrid_step_teacher_forced_against_oracle(grid_oracle):
    """The shipped `minigrid` shape (T = 48, B = 32, deter 2048, H = 1); the oracle re-runs the first 2 sequences."""
    _full_step("minigrid", S=2)


def test_baseline_minigrid_shape_teacher_forced_against_oracle(grid_oracle):
    """B = 10, T = 10 (the `--configs defaults minigrid` benchmark shape): every loss, metric, per-(t,b) tensor and
    parameter gradient of the whole batch against the oracle."""
    _full_step("minigrid", S=None, batch_size=10, batch_length=10)

"""Vector observations through the native kernels: the module against the reference goldens (exact arm), against the
teacher-forced oracle (TF32 product arm, posterior unroll as a chain and as one persistent kernel), graph replay and the
concurrent branches bit for bit against one-stream eager launches, and one full-size `minecraft` step."""
import weakref

import pytest
import torch

from oracle import vecobs_oracle as O
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_step_schedule_gpu import assert_identical, graph_state, released, train_step, ws
from tests.util import build_case, seeded_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VEC_CASES = ("tiny_vecobs", "tiny_vecobs_iwae3", "tiny_vector")


def run_gpu(case, impl, rounding, persistent=False):
    fx, conf, obs, state, noise = build_case(case, DEV)
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_weights(model.state_dict(), fx))
    model.persistent_rssm = model.persistent_bptt = persistent
    model.fp16_forward = model.implicit_conv = (impl == 0)
    model._ensure_arena()
    model.ops.set_gemm_impl(impl)
    model.ops.set_round_operands(rounding)
    n0 = model.ops.launch_count()
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    launches = model.ops.launch_count() - n0
    model.ops.set_gemm_impl(0)
    model.ops.set_round_operands(True)
    return fx, conf, obs, state, noise, model, losses, metrics, tensors, launches


@pytest.mark.parametrize("case", VEC_CASES)
def test_exact_arm_matches_reference_golden(case):
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = run_gpu(case, impl=1, rounding=False)
    for got, want in zip(losses, fx["losses"]):
        assert abs(float(got.detach().reshape(-1)[0]) - want) <= 5e-5 * max(1.0, abs(want)), (got, want)
    assert set(metrics) == set(fx["metrics"])
    for k, want in fx["metrics"].items():
        assert abs(float(metrics[k]) - want) <= 2e-4 * max(1.0, abs(want)), k
    named = dict(model.named_parameters())
    for k, want in fx["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        assert abs(got - want) <= 1e-3 * max(want, 1e-6) + 1e-9, (k, got, want)
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    idx = model._buf("rssm.idx", T, B * I, conf.stoch_dim, dtype=torch.int32)
    assert idx[0].reshape(-1).tolist() == fx["post_sample_indices_t0"]        # bit-exact sampled indices
    assert int(idx.sum()) == fx["post_sample_index_sum"]
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= 3e-4 * max(want, 1e-6), (k, got, want)


def check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, S=None, tol=1.0):
    """Losses, metrics, parameter gradients (full batch) or per-(t,b) tensors (first S sequences) against the oracle on the
    same weights, teacher-forced on the posterior / prior indices and actions the GPU sampled."""
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    G, C, D, A = conf.stoch_dim, conf.stoch_discrete, conf.deter_dim, conf.action_dim
    Z, N = G * C, T * B * I
    S = S or B
    sub = lambda x: x[:, :S].contiguous().cpu()
    rows = lambda x: x.reshape(H, T, B * I, -1)[:, :, :S * I].reshape(H, T * S * I, -1).cpu()
    post_idx = model._buf("rssm.idx", T, B * I, G, dtype=torch.int32)[:, :S * I].long().cpu()
    feats = model._buf("feats", H + 1, N, D + Z)
    prior_idx = rows(feats[1:, :, D:].reshape(H, N, G, C).argmax(-1))
    sd = {k: v.detach().cpu().clone().requires_grad_(S == B and not k.startswith("ac.critic_target"))
          for k, v in model.state_dict().items()}
    noise_s = dict(post=noise["post"][:, :S * I].contiguous().cpu(), actor=rows(noise["actor"]), prior=rows(noise["prior"]))
    res = O.training_step(sd, conf, {k: sub(v) for k, v in obs.items()}, (state[0][:S * I].cpu(), state[1][:S * I].cpu()),
                          noise_s, force=dict(post_idx=post_idx, actor=rows(model._buf("dream.actions", H, N, A)),
                                              prior_idx=prior_idx))
    rel = lambda a, b: ((a.double().cpu() - b.double()).abs().max() / (b.double().abs().max() + 1e-12)).item()
    for k in res["tensors"]:
        assert rel(tensors[k][:, :S], res["tensors"][k]) < tol * 2e-3, k
    assert rel(model._buf("rssm.post", T, B * I, Z)[:, :S * I], res["inter"]["posts"]) < tol * 2e-3
    if S < B:
        return
    for l in res["losses"]:
        l.backward()
    for i, (got, want) in enumerate(zip(losses, res["losses"])):
        g, w = float(got.detach().reshape(-1)[0]), float(want.detach().reshape(-1)[0])
        assert abs(g - w) <= tol * 1e-3 * max(1.0, abs(w)), (i, g, w)
    for k, want in res["metrics"].items():
        assert abs(float(metrics[k]) - float(want)) <= tol * 2e-3 * max(1.0, abs(float(want))), k
    named = dict(model.named_parameters())
    for k, v in sd.items():
        if v.grad is None:
            continue
        w, g = float(v.grad.double().norm()), float(named[k].grad.double().norm())
        # actor-critic gradients come from fp16-operand dreams, and an output bias's gradient is a signed sum over all H*N
        # dreamed rows: with the 4-float vector model's small critic errors that sum cancels to ~1e-2 of its terms
        rtol = 3e-3 if k.startswith("wm.") else 3e-2
        assert abs(g - w) / max(w, 1e-6) <= tol * (rtol + 1e-7 / max(w, 1e-12)), (k, g, w)
        if w > 1e-6:
            dot = float((named[k].grad.double().cpu() * v.grad.double()).sum()) / max(w * max(g, 1e-12), 1e-12)
            assert dot > 0.999, (k, dot)       # direction of every gradient tensor


@pytest.mark.parametrize("persistent", (False, True), ids=("chain", "persistent_rssm"))
@pytest.mark.parametrize("case", VEC_CASES)
def test_product_arm_teacher_forced_against_oracle(case, persistent):
    fx, conf, obs, state, noise, model, losses, metrics, tensors, _ = run_gpu(case, impl=0, rounding=True,
                                                                                persistent=persistent)
    assert model._persistent_rssm_ok(conf.batch_size * conf.iwae_samples) == persistent
    check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors)


@pytest.mark.parametrize("case,rtol", [("tiny_vecobs_log", 2e-3), ("tiny_vecobs_iwae3_log", 6e-3), ("tiny_vector_log", 2e-3)])
def test_logging_eval_and_inference_branches_on_gpu(case, rtol):
    """The logging / evaluation branches through the TF32 product arm against the reference's outputs.  With three
    importance samples the open-loop prior unroll carries TF32 error through every step into masked reward sums over a
    handful of elements: 6e-3 there."""
    from tests.test_dreamer_cpu import check_log_case, run_log_case
    fx, conf, out = run_log_case(case, DEV)
    check_log_case(fx, conf, out, rtol)


def test_image_less_model_launches_no_image_kernels():
    *_, vec_model, _, _, _, n_vec = run_gpu("tiny_vecobs", impl=0, rounding=True)
    *_, model, _, _, _, n = run_gpu("tiny_vector", impl=0, rounding=True)
    names = {k[0] for k in model._ws}
    assert not any(s.startswith(("enc.a", "enc.col", "dec.", "bwd.dd", "bwd.gdec", "bwd.genc", "bwd.da", "encw", "decw"))
                   for s in names), sorted(names)
    assert 100 < n < n_vec, (n, n_vec)


# ------------------------------------------------------------------------ graph replay / concurrency / run to run
def make_model(preset, graphs, overlap):
    conf = make_conf(preset, device=DEV, target_interval=2)
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    m = Dreamer(conf).to(DEV)
    m.load_state_dict(seeded_state_dict(m.state_dict(), 11))
    m.use_cuda_graph, m.overlap, m.persistent_rssm, m.persistent_bptt = graphs, overlap, True, False
    return conf, m, m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)


def drawn_noise(m, conf, obs):
    d, (T, B) = m.d, obs["action"].shape[:2]
    I, H = conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    return {k: v.clone() for k, v in dict(post=ws(m, "noise.post", T, B * I, d.Z), actor=ws(m, "noise.actor", H, N, d.A),
                                          prior=ws(m, "noise.prior", H, N, d.Z)).items()}


@pytest.mark.parametrize("preset", ("tiny_vecobs", "tiny_vector"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    """Calls 1-2 eager, 3 captures, 4-5 replay (default overlap); then every overlap mask launched eagerly; each against
    one-stream eager launches fed the noise the tested arm drew."""
    STEPS = 5
    conf, m, opts = make_model(preset, graphs=True, overlap=Dreamer.overlap)
    obs = [synthetic_batch(conf, seed=100 + i, first=(i == 0), device=DEV) for i in range(STEPS)]
    state = m.init_state(conf.batch_size)
    arms, noises = {"graph": []}, []
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state)
        assert not warned, warned
        noises.append(drawn_noise(m, conf, obs[i]))
        arms["graph"].append(rec)
    st = graph_state(m)
    assert st["graph"] is not None and not st.get("failed")
    ref = weakref.ref(m)
    del m, opts
    released(ref)
    for mask in range(1, 8):
        conf, m, opts = make_model(preset, graphs=False, overlap=mask)
        state = m.init_state(conf.batch_size)
        arms[f"overlap{mask}"] = []
        for i in range(2):
            rec, state, n, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i])
            arms[f"overlap{mask}"].append(rec)
        del m, opts
    conf, m, opts = make_model(preset, graphs=False, overlap=0)
    state = m.init_state(conf.batch_size)
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i])
        for name, recs in arms.items():
            if i < len(recs):
                assert_identical(f"[{preset}] {name} step {i + 1}", rec, recs[i])
        if i == 2:
            assert st["kernels"] == n


@pytest.mark.parametrize("preset", ("tiny_vecobs", "tiny_vector"))
def test_three_eager_steps_are_identical(preset):
    recs = []
    for _ in range(3):
        conf, m, opts = make_model(preset, graphs=False, overlap=Dreamer.overlap)
        obs = synthetic_batch(conf, seed=7, device=DEV)
        torch.manual_seed(3)
        recs.append(train_step(m, opts, conf, obs, m.init_state(conf.batch_size))[0])
        del m, opts
    assert_identical(f"[{preset}] run 2", recs[0], recs[1])
    assert_identical(f"[{preset}] run 3", recs[0], recs[2])


@pytest.mark.parametrize("preset", ("vectorenv", "minecraft"))
def test_shipped_configs_train_through_the_learner_with_graph_replay(preset):
    from pydreamer_b200.learner import Learner
    conf = make_conf(preset, device=DEV)
    lr = Learner(conf, DEV)
    for i in range(4):
        metrics, tensors, _ = lr.step(synthetic_batch(conf, seed=i, first=(i == 0), device=DEV))
    torch.cuda.synchronize()
    st = graph_state(lr.model)
    assert st["graph"] is not None and not st.get("failed")
    assert all(torch.isfinite(v).all() for v in metrics.values()), metrics
    assert "loss_vecobs" in metrics and ("loss_image" in metrics) == (preset == "minecraft")


def test_full_size_minecraft_step_teacher_forced_against_oracle():
    """The shipped `minecraft` shape (T=48, B=32, deter 2048, 64x64x3 image + 27-float vector) on the product arm; the
    oracle re-runs the first 2 sequences (sequences of a batch are independent) teacher-forced on the GPU's samples:
    2e-3 relative on the per-(t,b) tensors, as tests/test_dreamer_gpu.py at the Atari shape."""
    conf = make_conf("minecraft", device=DEV)
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
    check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, S=2)

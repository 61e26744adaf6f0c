"""The categorical reward head through the native kernels: the module against the reference goldens (exact arm) and their
logging branches (product arm), graph replay and every overlap mask bit for bit against one-stream eager launches, and
one full-size `atari_catreward` step against the oracle restatement."""
import weakref

import pytest
import torch

from oracle import catreward_oracle as O
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_step_schedule_gpu import assert_identical, graph_state, released, train_step, ws
from tests.util import build_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = ("tiny_catreward", "tiny_catreward_iwae3", "tiny_dmc_catreward", "tiny_catreward_wide")


def run_gpu(case, impl, rounding):
    fx, conf, obs, state, noise = build_case(case, DEV)
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(O.seeded_weights(model.state_dict(), fx["seeds"]["weights"]))
    model.persistent_rssm = model.persistent_bptt = False
    model.fp16_forward = model.implicit_conv = (impl == 0)
    model._ensure_arena()
    model.ops.set_gemm_impl(impl)
    model.ops.set_round_operands(rounding)
    losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
    for l in losses:
        l.backward()
    torch.cuda.synchronize()
    model.ops.set_gemm_impl(0)
    model.ops.set_round_operands(True)
    return fx, conf, model, losses, metrics, tensors


@pytest.mark.parametrize("case", CASES)
def test_exact_arm_matches_reference_golden(case):
    fx, conf, model, losses, metrics, tensors = run_gpu(case, impl=1, rounding=False)
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
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    kr = model._buf("head.kr", T * B * I, dtype=torch.int32).view(T, B, I)[:, :, 0]
    assert kr.reshape(-1).tolist() == fx["reward_buckets"]                   # bit-exact target buckets
    assert model.wm.decoder.reward._support.grad is None


@pytest.mark.parametrize("case,rtol", [("tiny_catreward_log", 2e-3), ("tiny_catreward_iwae3_log", 6e-3),
                                       ("tiny_dmc_catreward_log", 2e-3), ("tiny_catreward_wide_log", 2e-3)])
def test_logging_eval_and_inference_branches_on_gpu(case, rtol, monkeypatch):
    import tests.test_dreamer_cpu as TD
    monkeypatch.setattr(TD, "seeded_weights", lambda template, fx: O.seeded_weights(template, fx["seeds"]["weights"]))
    fx, conf, out = TD.run_log_case(case, DEV)
    TD.check_log_case(fx, conf, out, rtol)


# ------------------------------------------------------------------------ graph replay / concurrency / run to run
def make_model(preset, graphs, overlap):
    conf = make_conf(preset, device=DEV, target_interval=2)
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    m = Dreamer(conf).to(DEV)
    m.load_state_dict(O.seeded_weights(m.state_dict(), 11))
    m.use_cuda_graph, m.overlap, m.persistent_rssm, m.persistent_bptt = graphs, overlap, True, False
    return conf, m, m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)


def drawn_noise(m, conf, obs):
    d, (T, B) = m.d, obs["action"].shape[:2]
    I, H = conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    return {k: v.clone() for k, v in dict(post=ws(m, "noise.post", T, B * I, d.Z), actor=ws(m, "noise.actor", H, N, d.A),
                                          prior=ws(m, "noise.prior", H, N, d.Z)).items()}


@pytest.mark.parametrize("preset", ("tiny_catreward", "tiny_catreward_wide"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    """Calls 1-2 eager, 3 captures, 4-5 replay (default overlap); then every overlap mask launched eagerly; each against
    one-stream eager launches fed the noise the tested arm drew.  The support stays bit-identical through the steps."""
    STEPS = 5
    conf, m, opts = make_model(preset, graphs=True, overlap=Dreamer.overlap)
    sup0 = m.wm.decoder.reward._support.detach().clone()
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
    assert torch.equal(m.wm.decoder.reward._support.detach(), sup0) and m.wm.decoder.reward._support.grad is None
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


@pytest.fixture()
def parity(monkeypatch):
    """tests/test_parity_full_gpu.py's runner and checks with the categorical-head oracle and seeded weights that keep the
    configured support.  The oracle result of its check is kept for the imagined-reward comparison."""
    import tests.test_parity_full_gpu as P
    monkeypatch.setattr(P, "O", O)
    monkeypatch.setattr(P, "seeded_state_dict", O.seeded_weights)
    last, oracle = {}, P._oracle

    def kept(*a, **k):
        last["sd"], last["res"] = oracle(*a, **k)
        return last["sd"], last["res"]

    monkeypatch.setattr(P, "_oracle", kept)
    return P, last


def run_and_check(parity, case):
    """One product-arm step teacher-forced against the oracle with tests/test_parity_full_gpu.py's criteria (every loss
    and metric, the per-(t,b) tensors, every gradient tensor element-wise), and the expected rewards of the imagination
    rollout (fp16 hidden layers, pd_support_head without a target) at the same 2-norm and worst-element tolerances."""
    P, last = parity
    conf = make_conf(case, device=DEV)
    model, obs, state, noise, losses, metrics, tensors = P._run_gpu(conf, 11, 77, 5)
    P._check(case, conf=conf, model=model, obs=obs, state=state, noise=noise, losses=losses, metrics=metrics,
             tensors=tensors)
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    l2, mx = P._err(model._buf("ac.rew", (H + 1) * N, 1).view(H + 1, N), last["res"]["inter"]["rewards"].reshape(H + 1, N))
    print(f"[{case}] imagined rewards: l2-relative {l2:.1e}, worst-element/max {mx:.1e}")
    assert l2 <= P.L2_TOL and mx <= P.MAX_TOL, (case, "imagined rewards", l2, mx)
    assert model.wm.decoder.reward._support.grad is None


@pytest.mark.parametrize("case", CASES)
def test_product_arm_step_at_tiny_size(parity, case):
    """The product arm (tensor-core and fp16-forward GEMMs, persistent RSSM) at the tiny shapes, teacher-forced against the
    oracle.  S = 3 takes the gemv, tensor-core and CUDA-core routes of `atari_catreward`; `tiny_catreward_wide` (S = 33,
    pitch 36) runs the reward head's output layer, weight gradient and input gradient on the tensor cores.
    Losses, metrics, the per-(t,b) tensors, the imagined rewards and every gradient of the reward head (the logit-gradient
    seed through rowscale, colsum and both GEMMs) are held to tests/test_parity_full_gpu.py's tolerances.  Every other
    gradient is held as tests/test_vecobs_gpu.py holds its tiny models (3e-3 on the norm of world-model gradients, 3e-2 on
    actor / critic ones, direction within 0.999).  Measured on an H100: at this size the conv-encoder bias gradients, the
    far end of the chain from every loss seed, differ from the oracle by up to 4.9e-3 (2-norm) with the categorical head
    and 1.7e-3 with the Normal head; every other gradient stays within the full-size element-wise bounds, and the
    full-size `atari_catreward` step below meets them for every gradient."""
    P, last = parity
    conf = make_conf(case, device=DEV)
    model, obs, state, noise, losses, metrics, tensors = P._run_gpu(conf, 11, 77, 5)
    sd, res = P._oracle(model, conf, obs, state, noise)
    for i, (got, want) in enumerate(zip(losses, res["losses"])):
        g, w = float(got.detach().reshape(-1)[0]), float(want.detach().reshape(-1)[0])
        assert abs(g - w) <= P.SCALAR_TOL * max(1.0, abs(w)), ("loss", i, g, w)
    for k, want in res["metrics"].items():
        assert abs(float(metrics[k]) - float(want)) <= P.SCALAR_TOL * max(1.0, abs(float(want))), ("metric", k)
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    fwd = {k: (tensors[k], res["tensors"][k]) for k in res["tensors"]}
    fwd["imagined rewards"] = (model._buf("ac.rew", (H + 1) * N, 1).view(H + 1, N), res["inter"]["rewards"].reshape(H + 1, N))
    named = dict(model.named_parameters())
    head = [k for k, v in sd.items() if k.startswith("wm.decoder.reward.") and v.grad is not None]
    assert len(head) == 4 * conf.reward_decoder_layers + 2                   # Linear + LayerNorm per hidden layer, output
    for k in head:
        fwd["grad " + k] = (named[k].grad, sd[k].grad)
    for k, (got, want) in fwd.items():
        l2, mx = P._err(got, want)
        assert l2 <= P.L2_TOL and mx <= P.MAX_TOL, (case, k, l2, mx)
    for k, v in sd.items():
        if v.grad is None or k in head:
            continue
        w, g = float(v.grad.double().norm()), float(named[k].grad.double().norm())
        rtol = 3e-3 if k.startswith("wm.") else 3e-2
        assert abs(g - w) <= rtol * w + 1e-7, (case, k, g, w)
        if w > 1e-6:
            dot = float((named[k].grad.double().cpu() * v.grad.double()).sum()) / (w * max(g, 1e-12))
            assert dot > 0.999, (case, k, dot)
    assert named[O.SUPPORT].grad is None


def test_full_atari_catreward_every_gradient_elementwise(parity):
    """`atari_catreward` (T = B = 50, deter 2048, S = 3) over the whole batch at the tolerances of
    tests/test_parity_full_gpu.py: losses and metrics 1e-3, per-(t,b) tensors and every gradient tensor 2e-3 in the 2-norm
    and 3e-3 worst element (actor / critic gradients with the measured advantage error on top)."""
    run_and_check(parity, "atari_catreward")

"""The auxiliary critic through the native kernels: the module against the reference goldens (exact arm) and its logging
branches (product arm), graph replay and every overlap mask bit for bit against one-stream eager launches, and one
full-size `atari_auxcritic` step against the oracle restatement."""
import weakref

import pytest
import torch

from oracle import auxcritic_oracle as O
from oracle.weights import seeded_state_dict
from pydreamer_b200 import replay
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from tests.test_auxcritic_cpu import CASES, NEVER_GRAD, build_aux_case, force_terminals
from tests.test_step_schedule_gpu import assert_identical, graph_state, released, train_step, ws

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_gpu(case, impl, rounding):
    fx, conf, obs, state, noise = build_aux_case(case, DEV)
    model = Dreamer(conf).to(DEV)
    model.load_state_dict(seeded_state_dict(model.state_dict(), fx["seeds"]["weights"]))
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
    assert {k for k, p in named.items() if p.grad is not None} == set(fx["grad_norms"])
    for k, want in fx["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        assert abs(got - want) <= 1e-3 * max(want, 1e-6) + 1e-9, (k, got, want)
    for k, want in fx["tensor_abs_sums"].items():
        got = float(tensors[k].double().abs().sum())
        assert abs(got - want) <= 3e-4 * max(want, 1e-6), (k, got, want)
    assert torch.allclose(tensors["policy_value_aux"].double().cpu(), torch.tensor(fx["policy_value_aux"], dtype=torch.float64),
                          rtol=2e-4, atol=2e-4)
    assert all(p.grad is None for n, p in named.items() if n.startswith(NEVER_GRAD))


def test_logging_eval_and_inference_branches_on_gpu(monkeypatch):
    import tests.test_dreamer_cpu as TD
    batch = replay.synthetic_batch
    monkeypatch.setattr(replay, "synthetic_batch", lambda *a, **k: force_terminals(batch(*a, **k)))
    fx, conf, out = TD.run_log_case("tiny_auxcritic_log", DEV)
    TD.check_log_case(fx, conf, out, 2e-3)


# ------------------------------------------------------------------------ graph replay / concurrency / run to run
def make_model(preset, graphs, overlap):
    conf = make_conf(preset, device=DEV, target_interval=2, target_interval_aux=2)
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


@pytest.mark.parametrize("preset", ("tiny_auxcritic", "tiny_auxcritic_iwae3"))
def test_graph_replay_and_every_overlap_mask_equal_the_one_stream_eager_step(preset):
    """Calls 1-2 eager, 3 captures, 4-5 replay (default overlap); then every overlap mask launched eagerly; each against
    one-stream eager launches fed the noise the tested arm drew.  target_interval_aux = 2: the aux target is copied on the
    host before calls 1, 3 and 5, outside the graph, and every replay reads the copied weights."""
    STEPS = 5
    conf, m, opts = make_model(preset, graphs=True, overlap=Dreamer.overlap)
    obs = [force_terminals(replay.synthetic_batch(conf, seed=100 + i, first=(i == 0), device=DEV)) for i in range(STEPS)]
    state = m.init_state(conf.batch_size * conf.iwae_samples)
    arms, noises = {"graph": []}, []
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state)
        assert not warned, warned
        noises.append(drawn_noise(m, conf, obs[i]))
        arms["graph"].append(rec)
    st = graph_state(m)
    assert st["graph"] is not None and not st.get("failed")
    assert m.wm.ac_aux.train_steps == STEPS
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


def test_full_atari_auxcritic_every_gradient_elementwise(monkeypatch):
    """`atari_auxcritic` (T = B = 50, deter 2048) over the whole batch at the tolerances of tests/test_parity_full_gpu.py:
    losses and metrics 1e-3, per-(t,b) tensors (policy_value_aux among them) and every gradient tensor 2e-3 in the 2-norm
    and 3e-3 worst element."""
    import tests.test_parity_full_gpu as P
    monkeypatch.setattr(P, "O", O)
    conf = make_conf("atari_auxcritic", device=DEV)
    model, obs, state, noise, losses, metrics, tensors = P._run_gpu(conf, 11, 77, 5)
    errs = P._check("atari_auxcritic", conf=conf, model=model, obs=obs, state=state, noise=noise, losses=losses,
                    metrics=metrics, tensors=tensors)
    assert sum(k.startswith("wm.ac_aux.critic.") for k in errs) == 18              # 4 x (Linear + LayerNorm) + output
    assert all(p.grad is None for n, p in model.named_parameters() if n.startswith(NEVER_GRAD))

"""Generates tests/golden/*.json from the UNMODIFIED reference (jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  For each case it (1) builds the reference Dreamer, loads seeded weights, (2) seeds the global RNG and runs
training_step + the four backward passes exactly as train.py:171-187 does, (3) re-draws the same RNG stream as
explicit noise (SURVEY.md App. D) and checks oracle/dreamer_oracle.py reproduces losses, metrics and gradients,
(4) stores the REFERENCE's numbers as the fixture.  Fixtures hold seeds + expected outputs only."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.abspath(sys.argv[1]))  # a checkout of the reference

from pydreamer.models import Dreamer as RefDreamer  # noqa: E402  (the reference)

from oracle import dreamer_oracle as O  # noqa: E402
from oracle.weights import seeded_state_dict  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402
from pydreamer_b200.replay import synthetic_batch  # noqa: E402

CASES = {
    "tiny_onehot": dict(preset="tiny", over={}),
    "tiny_iwae3": dict(preset="tiny", over=dict(iwae_samples=3)),
    "tiny_dmc": dict(preset="tiny_dmc", over={}),
    "tiny_klbal05": dict(preset="tiny", over=dict(kl_balance=0.5, kl_weight=1.0)),
    # shapes off the multiples of 8 / 4 the tensor-core paths need, and heads without hidden layers
    "tiny_heads0": dict(preset="tiny", over=dict(reward_decoder_layers=0, terminal_decoder_layers=0)),
    "tiny_odd_dims": dict(preset="tiny", over=dict(hidden_dim=42, deter_dim=70, stoch_dim=5, stoch_discrete=7, cnn_depth=6,
                                                   image_channels=1)),
    "tiny_z2": dict(preset="tiny", over=dict(stoch_dim=1, stoch_discrete=2, batch_length=1, imag_horizon=1)),
}
NOISE_SEED, DATA_SEED, WEIGHT_SEED = 4321, 1234, 7


def run_case(name, spec):
    torch.distributions.Distribution.set_default_validate_args(False)   # train.py:30
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    torch.manual_seed(0)
    ref = RefDreamer(conf)
    sd = seeded_state_dict(ref.state_dict(), WEIGHT_SEED)
    ref.load_state_dict(sd)
    obs = synthetic_batch(conf, seed=DATA_SEED)
    state = ref.init_state(B * I)
    # a non-trivial carried state exercises the reset masking
    g = torch.Generator().manual_seed(99)
    state = (torch.tanh(torch.randn(state[0].shape, generator=g)), torch.zeros_like(state[1]))
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, _ = ref.training_step(obs, state)
    for l in losses:
        l.backward()
    ref_grads = {n: p.grad.clone() for n, p in ref.named_parameters() if p.grad is not None}

    # the restatement, fed the same RNG stream as explicit noise
    torch.manual_seed(NOISE_SEED)
    noise = O.draw_noise(conf, T, B)
    sdo = {k: v.clone().requires_grad_(not k.startswith("ac.critic_target")) for k, v in sd.items()}
    res = O.training_step(sdo, conf, obs, state, noise)
    for l in res["losses"]:
        l.backward()
    for i, (a, b) in enumerate(zip(losses, res["losses"])):
        assert torch.allclose(a.detach().reshape(-1), b.detach().reshape(-1), rtol=2e-5, atol=1e-6), (name, i, a, b)
    for k, v in metrics.items():
        assert torch.allclose(v, res["metrics"][k], rtol=2e-4, atol=1e-6), (name, k, v, res["metrics"][k])
    worst = 0.0
    for n, gr in ref_grads.items():
        go = sdo[n].grad
        assert go is not None, n
        err = (gr - go).abs().max().item() / (gr.abs().max().item() + 1e-12)
        worst = max(worst, err)
        assert err < 2e-4, (name, n, err)
    for k in ("image_rec", "reward_rec", "loss_kl", "policy_value"):
        assert torch.allclose(tensors[k], res["tensors"][k], rtol=1e-4, atol=1e-5), (name, k)
    assert torch.equal(out_state[1].round(), res["out_state"][1].round())   # same samples => noise stream aligned

    fix = dict(
        case=name, preset=spec["preset"], overrides=spec["over"],
        seeds=dict(noise=NOISE_SEED, data=DATA_SEED, weights=WEIGHT_SEED, state=99),
        reference="jurgisp/pydreamer (Dreamer.training_step + 4x backward, CPU fp32, torch %s)" % torch.__version__,
        losses=[float(l.detach().reshape(-1)[0]) for l in losses],
        metrics={k: float(v) for k, v in metrics.items()},
        grad_norms={n: float(g_.double().norm()) for n, g_ in ref_grads.items()},
        grad_sums={n: float(g_.double().sum()) for n, g_ in ref_grads.items()},
        tensor_sums={k: float(v.double().sum()) for k, v in tensors.items()},
        tensor_abs_sums={k: float(v.double().abs().sum()) for k, v in tensors.items()},
        out_state_h_sum=float(out_state[0].double().sum()),
        post_sample_index_sum=int(res["inter"]["post_idx"].sum()),
        post_sample_indices_t0=res["inter"]["post_idx"][0].reshape(-1).tolist(),
        dream_action_sum=float(res["inter"]["dream_actions"].double().sum()),
        oracle_vs_reference_worst_grad_rel_err=worst,
    )
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: losses {fix['losses']}  oracle-vs-reference worst grad rel err {worst:.2e} -> {path}")


def run_log_case(name, spec):
    """Logging / evaluation branches of the reference (do_image_pred + do_dream_tensors, open-loop eval, inference):
    the REFERENCE's outputs are the fixture; the module is checked against them in tests/test_dreamer_cpu.py and
    tests/test_dreamer_gpu.py (there is no oracle restatement of these logging branches)."""
    torch.distributions.Distribution.set_default_validate_args(False)
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    torch.manual_seed(0)
    ref = RefDreamer(conf)
    ref.load_state_dict(seeded_state_dict(ref.state_dict(), WEIGHT_SEED))
    obs = synthetic_batch(conf, seed=DATA_SEED)
    g = torch.Generator().manual_seed(99)
    state = (torch.tanh(torch.randn((B * I, conf.deter_dim), generator=g)), torch.zeros(B * I, conf.stoch_dim * conf.stoch_discrete))
    sums = lambda d: {k: [float(v.double().nansum()), float(v.double().abs().nansum()), list(v.shape)] for k, v in d.items()}
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, dream = ref.training_step(obs, state, do_image_pred=True, do_dream_tensors=True)
    fix = dict(case=name, preset=spec["preset"], overrides=spec["over"],
               seeds=dict(noise=NOISE_SEED, data=DATA_SEED, weights=WEIGHT_SEED, state=99),
               train_log=dict(losses=[float(l.detach().reshape(-1)[0]) for l in losses],
                              metrics={k: float(v) for k, v in metrics.items()}, tensors=sums(tensors), dream=sums(dream)))
    with torch.no_grad():
        torch.manual_seed(NOISE_SEED)
        l2, os2, m2, t2, _ = ref.training_step(obs, state, do_open_loop=True, do_image_pred=True)
    fix["open_loop"] = dict(losses=[float(l.detach().reshape(-1)[0]) for l in l2], metrics={k: float(v) for k, v in m2.items()},
                            tensors=sums(t2), out_state_h_sum=float(os2[0].double().sum()))
    with torch.no_grad():
        torch.manual_seed(NOISE_SEED)
        o1 = {k: v[:1] for k, v in obs.items()}
        dist, os3, m3 = ref.inference(o1, (state[0][:B], state[1][:B]))      # the actor path has no IWAE dimension
    lg = dist.logits if conf.actor_dist == "onehot" else torch.cat([dist.base_dist.base_dist.loc, dist.base_dist.base_dist.scale], -1)
    fix["inference"] = dict(dist_param_sum=float(lg.double().sum()), dist_param_abs=float(lg.double().abs().sum()),
                            out_state_h_sum=float(os3[0].double().sum()), out_state_z_sum=float(os3[1].double().sum()),
                            policy_value=float(m3["policy_value"]))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: log/eval/inference fixture -> {path}")


if __name__ == "__main__":
    wanted = sys.argv[2:]
    for n, sp in (("tiny_onehot_log", CASES["tiny_onehot"]), ("tiny_dmc_log", CASES["tiny_dmc"]),
                  ("tiny_iwae3_log", CASES["tiny_iwae3"])):
        if not wanted or n in wanted:
            run_log_case(n, sp)
    for n, s in CASES.items():
        if not wanted or n in wanted:
            run_case(n, s)

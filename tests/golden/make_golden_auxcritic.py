"""Generates the auxiliary-critic fixtures under tests/golden/ from the UNMODIFIED reference (jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden_auxcritic.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  Same procedure and seeds as tests/golden/make_golden_catreward.py: per
case (1) the reference Dreamer with seeded weights runs training_step + the four backward passes, (2)
oracle/auxcritic_oracle.py, fed the same RNG stream as explicit noise, must reproduce its losses, metrics and gradients,
(3) the REFERENCE's numbers are stored.  Synthetic terminals are Bernoulli(0.01), so every batch gets the terminal pattern
of tests/test_auxcritic_cpu.force_terminals (a terminal at t = 0 in column 0, at t = T // 2 in column 1, none in the
others).  The `_log` fixture holds the logging / evaluation branches (do_image_pred + do_dream_tensors, open loop,
inference) as tests/golden/make_golden.py writes them.  `auxcritic_state_dict` holds, per preset, the reference's
state_dict keys and shapes, the parameter order of each optimizer and, for the tiny presets, the indices of the
world-model parameters torch.optim.AdamW keeps state for after one step."""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402,F401  (puts the repository and the reference checkout of argv[1] on sys.path)
from make_golden import DATA_SEED, NOISE_SEED, WEIGHT_SEED, RefDreamer  # noqa: E402

from oracle import auxcritic_oracle as O  # noqa: E402
from oracle.weights import seeded_state_dict  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402
from pydreamer_b200.replay import synthetic_batch  # noqa: E402
from tests.test_auxcritic_cpu import force_terminals  # noqa: E402

CASES = {
    "tiny_auxcritic": dict(preset="tiny_auxcritic", over={}),
    "tiny_auxcritic_iwae3": dict(preset="tiny_auxcritic_iwae3", over={}),         # sample-0 rows t*B*I + b*I
    "tiny_dmc_auxcritic": dict(preset="tiny_dmc_auxcritic", over={}),             # tanh_normal: the aux actor is 2A wide
    "tiny_vector_auxcritic": dict(preset="tiny_vector_auxcritic", over={}),       # no image: the reward head writes dfeat first
}
LOG_CASES = {"tiny_auxcritic_log": dict(preset="tiny_auxcritic", over={})}
STATE_DICT_PRESETS = ("tiny_auxcritic", "tiny_dmc_auxcritic", "atari_auxcritic")


def reference_model(conf):
    torch.manual_seed(0)
    ref = RefDreamer(conf)
    sd = seeded_state_dict(ref.state_dict(), WEIGHT_SEED)
    ref.load_state_dict(sd)
    return ref, sd


def inputs(conf):
    B, I = conf.batch_size, conf.iwae_samples
    obs = force_terminals(synthetic_batch(conf, seed=DATA_SEED))
    g = torch.Generator().manual_seed(99)                       # a non-trivial carried state exercises the reset masking
    state = (torch.tanh(torch.randn((B * I, conf.deter_dim), generator=g)), torch.zeros(B * I, conf.stoch_dim * conf.stoch_discrete))
    return obs, state


def run_case(name, spec):
    torch.distributions.Distribution.set_default_validate_args(False)   # train.py:30
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B = conf.batch_length, conf.batch_size
    ref, sd = reference_model(conf)
    obs, state = inputs(conf)
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, _ = ref.training_step(obs, state)
    for l in losses:
        l.backward()
    ref_grads = {n: p.grad.clone() for n, p in ref.named_parameters() if p.grad is not None}
    assert not any(n.startswith(("wm.ac_aux.actor", "wm.ac_aux.critic_target")) for n in ref_grads)
    assert any(n.startswith("wm.ac_aux.critic.") for n in ref_grads)

    torch.manual_seed(NOISE_SEED)
    noise = O.draw_noise(conf, T, B)
    frozen = ("ac.critic_target", "wm.ac_aux.critic_target", "wm.ac_aux.actor")
    sdo = {k: v.clone().requires_grad_(not k.startswith(frozen)) for k, v in sd.items()}
    res = O.training_step(sdo, conf, obs, state, noise)
    for l in res["losses"]:
        l.backward()
    for i, (a, b) in enumerate(zip(losses, res["losses"])):
        assert torch.allclose(a.detach().reshape(-1), b.detach().reshape(-1), rtol=2e-5, atol=1e-6), (name, i, a, b)
    assert set(metrics) == set(res["metrics"]), (name, sorted(set(metrics) ^ set(res["metrics"])))
    for k, v in metrics.items():
        assert torch.allclose(v, res["metrics"][k], rtol=2e-4, atol=1e-6), (name, k, v, res["metrics"][k])
    worst = 0.0
    for n, gr in ref_grads.items():
        go = sdo[n].grad
        assert go is not None, n
        err = (gr - go).abs().max().item() / (gr.abs().max().item() + 1e-12)
        worst = max(worst, err)
        assert err < 2e-4, (name, n, err)
    assert not any(sdo[k].grad is not None for k in sdo if k.startswith(frozen))
    for k in ("reward_rec", "loss_reward", "loss_kl", "policy_value", "policy_value_aux"):
        assert torch.allclose(tensors[k], res["tensors"][k], rtol=1e-4, atol=1e-5), (name, k)
    assert torch.equal(out_state[1].round(), res["out_state"][1].round())   # same samples => noise stream aligned

    fix = dict(
        case=name, preset=spec["preset"], overrides=spec["over"], terminals=obs["terminal"].tolist(),
        seeds=dict(noise=NOISE_SEED, data=DATA_SEED, weights=WEIGHT_SEED, state=99),
        reference="jurgisp/pydreamer (Dreamer.training_step + 4x backward, CPU fp32, torch %s)" % torch.__version__,
        losses=[float(l.detach().reshape(-1)[0]) for l in losses],
        metrics={k: float(v) for k, v in metrics.items()},
        grad_norms={n: float(g_.double().norm()) for n, g_ in ref_grads.items()},
        grad_sums={n: float(g_.double().sum()) for n, g_ in ref_grads.items()},
        tensor_sums={k: float(v.double().sum()) for k, v in tensors.items()},
        tensor_abs_sums={k: float(v.double().abs().sum()) for k, v in tensors.items()},
        policy_value_aux=tensors["policy_value_aux"].tolist(),
        out_state_h_sum=float(out_state[0].double().sum()),
        oracle_vs_reference_worst_grad_rel_err=worst,
    )
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: losses {fix['losses']}  oracle-vs-reference worst grad rel err {worst:.2e} -> {path}")


def run_log_case(name, spec):
    """The logging / evaluation branches of the reference, as make_golden.run_log_case records them."""
    torch.distributions.Distribution.set_default_validate_args(False)
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    B = conf.batch_size
    ref, _ = reference_model(conf)
    obs, state = inputs(conf)
    sums = lambda d: {k: [float(v.double().nansum()), float(v.double().abs().nansum()), list(v.shape)] for k, v in d.items()}
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, dream = ref.training_step(obs, state, do_image_pred=True, do_dream_tensors=True)
    fix = dict(case=name, preset=spec["preset"], overrides=spec["over"], terminals=obs["terminal"].tolist(),
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
        dist, os3, m3 = ref.inference(o1, (state[0][:B], state[1][:B]))
    lg = dist.logits if conf.actor_dist == "onehot" else torch.cat([dist.base_dist.base_dist.loc, dist.base_dist.base_dist.scale], -1)
    fix["inference"] = dict(dist_param_sum=float(lg.double().sum()), dist_param_abs=float(lg.double().abs().sum()),
                            out_state_h_sum=float(os3[0].double().sum()), out_state_z_sum=float(os3[1].double().sum()),
                            policy_value=float(m3["policy_value"]))
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: log/eval/inference fixture -> {path}")


def adamw_state_indices(preset):
    """Indices of the world-model parameters torch.optim.AdamW keeps state for after one reference step."""
    torch.distributions.Distribution.set_default_validate_args(False)
    conf = make_conf(preset, device="cpu")
    ref, _ = reference_model(conf)
    opt = torch.optim.AdamW(ref.wm.parameters(), lr=conf.adam_lr, eps=conf.adam_eps)
    obs, state = inputs(conf)
    torch.manual_seed(NOISE_SEED)
    losses = ref.training_step(obs, state)[0]
    for l in losses:
        l.backward()
    opt.step()
    return sorted(opt.state_dict()["state"])


def write_state_dict_fixture(name):
    out = {}
    for preset in STATE_DICT_PRESETS:
        ref = RefDreamer(make_conf(preset, device="cpu"))
        names = {id(p): n for n, p in ref.named_parameters()}
        groups = dict(wm=ref.wm.parameters(), probe=ref.probe_model.parameters(), actor=ref.ac.actor.parameters(),
                      critic=ref.ac.critic.parameters())
        out[preset] = dict(state_dict=[[k, list(v.shape)] for k, v in ref.state_dict().items()],
                           params={g: [[names[id(p)], list(p.shape)] for p in ps] for g, ps in groups.items()})
        if preset.startswith("tiny"):
            out[preset]["wm_adamw_state"] = adamw_state_indices(preset)
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print(f"{name}: {len(out)} presets -> {path}")


if __name__ == "__main__":
    wanted = sys.argv[2:]
    for n, spec in LOG_CASES.items():
        if not wanted or n in wanted:
            run_log_case(n, spec)
    for n, spec in CASES.items():
        if not wanted or n in wanted:
            run_case(n, spec)
    if not wanted or "auxcritic_state_dict" in wanted:
        write_state_dict_fixture("auxcritic_state_dict")

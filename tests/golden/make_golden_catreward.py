"""Generates the categorical-reward-head fixtures under tests/golden/ from the UNMODIFIED reference (jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden_catreward.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  Same procedure and seeds as tests/golden/make_golden_vecobs.py: per case
(1) the reference Dreamer with seeded weights runs training_step + the four backward passes, (2)
oracle/catreward_oracle.py, fed the same RNG stream as explicit noise, must reproduce its losses, metrics and gradients,
(3) the REFERENCE's numbers are stored.  The seeded weights keep the configured support (catreward_oracle.seeded_weights).
The `_log` fixtures hold the logging / evaluation branches (do_image_pred + do_dream_tensors, open loop, inference) as
tests/golden/make_golden.py writes them.  `catreward_state_dict` holds, per preset, the reference's state_dict keys and
shapes, the parameter order of each optimizer and the support values."""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (puts the repository and the reference checkout of argv[1] on sys.path)
from make_golden import DATA_SEED, NOISE_SEED, WEIGHT_SEED, RefDreamer  # noqa: E402

from oracle import catreward_oracle as O  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402
from pydreamer_b200.replay import synthetic_batch  # noqa: E402

CASES = {
    "tiny_catreward": dict(preset="tiny_catreward", over={}),              # [-1, 0, 1] through tanh: S = 3
    "tiny_catreward_iwae3": dict(preset="tiny_catreward_iwae3", over={}),
    "tiny_dmc_catreward": dict(preset="tiny_dmc_catreward", over={}),      # tanh_normal actor, [0, 1] unclipped
    "tiny_catreward_wide": dict(preset="tiny_catreward_wide", over={}),    # 33 unsorted values, duplicated: ties
}
STATE_DICT_PRESETS = ("tiny_catreward", "tiny_dmc_catreward", "tiny_catreward_wide", "atari_catreward")


def reference_model(conf):
    torch.manual_seed(0)
    ref = RefDreamer(conf)
    sd = O.seeded_weights(ref.state_dict(), WEIGHT_SEED)
    ref.load_state_dict(sd)
    return ref, sd


def run_case(name, spec):
    torch.distributions.Distribution.set_default_validate_args(False)   # train.py:30
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    ref, sd = reference_model(conf)
    obs = synthetic_batch(conf, seed=DATA_SEED)
    g = torch.Generator().manual_seed(99)                       # a non-trivial carried state exercises the reset masking
    state = ref.init_state(B * I)
    state = (torch.tanh(torch.randn(state[0].shape, generator=g)), torch.zeros_like(state[1]))
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, _ = ref.training_step(obs, state)
    for l in losses:
        l.backward()
    ref_grads = {n: p.grad.clone() for n, p in ref.named_parameters() if p.grad is not None}
    assert "wm.decoder.reward._support" not in ref_grads

    torch.manual_seed(NOISE_SEED)
    noise = O.draw_noise(conf, T, B)
    sdo = {k: v.clone().requires_grad_(not k.startswith("ac.critic_target") and k != O.SUPPORT) for k, v in sd.items()}
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
    for k in ("image_rec", "reward_rec", "loss_reward", "loss_kl", "policy_value"):
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
        reward_buckets=ref.wm.decoder.reward.to_categorical(obs["reward"]).reshape(-1).tolist(),
        oracle_vs_reference_worst_grad_rel_err=worst,
    )
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: losses {fix['losses']}  oracle-vs-reference worst grad rel err {worst:.2e} -> {path}")


def run_log_case(name, spec):
    """The logging / evaluation branches of the reference, as make_golden.run_log_case records them, with the seeded
    weights keeping the configured support."""
    torch.distributions.Distribution.set_default_validate_args(False)
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    ref, _ = reference_model(conf)
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
        dist, os3, m3 = ref.inference(o1, (state[0][:B], state[1][:B]))
    lg = dist.logits if conf.actor_dist == "onehot" else torch.cat([dist.base_dist.base_dist.loc, dist.base_dist.base_dist.scale], -1)
    fix["inference"] = dict(dist_param_sum=float(lg.double().sum()), dist_param_abs=float(lg.double().abs().sum()),
                            out_state_h_sum=float(os3[0].double().sum()), out_state_z_sum=float(os3[1].double().sum()),
                            policy_value=float(m3["policy_value"]))
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: log/eval/inference fixture -> {path}")


def write_state_dict_fixture(name):
    out = {}
    for preset in STATE_DICT_PRESETS:
        ref = RefDreamer(make_conf(preset, device="cpu"))
        names = {id(p): n for n, p in ref.named_parameters()}
        groups = dict(wm=ref.wm.parameters(), probe=ref.probe_model.parameters(), actor=ref.ac.actor.parameters(),
                      critic=ref.ac.critic.parameters())
        out[preset] = dict(state_dict=[[k, list(v.shape)] for k, v in ref.state_dict().items()],
                           params={g: [[names[id(p)], list(p.shape)] for p in ps] for g, ps in groups.items()},
                           support=ref.wm.decoder.reward._support.tolist())
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print(f"{name}: {len(out)} presets -> {path}")


if __name__ == "__main__":
    wanted = sys.argv[2:]
    for n, spec in CASES.items():
        if not wanted or n + "_log" in wanted:
            run_log_case(n + "_log", spec)
    for n, spec in CASES.items():
        if not wanted or n in wanted:
            run_case(n, spec)
    if not wanted or "catreward_state_dict" in wanted:
        write_state_dict_fixture("catreward_state_dict")

"""Generates the normal_tanh actor fixtures (`actor_dist: normal_tanh`) under tests/golden/ from the UNMODIFIED reference
(jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden_normaltanh.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  Same procedure and seeds as tests/golden/make_golden_vecobs.py, whose case
runner it uses with oracle/normaltanh_oracle.py in place of the vector-observation oracle: per case (1) the reference
Dreamer with seeded weights runs training_step + the four backward passes, (2) the oracle, fed the same RNG stream as
explicit noise, must reproduce its losses, metrics and gradients, (3) the REFERENCE's numbers are stored.  The reference
samples the action as Normal.sample(), i.e. torch.normal(mean, std), which draws N(0, 1) into the output and scales it:
the draws the oracle takes as its Gaussian noise.  The `_log` cases hold
the reference's logging, open-loop and inference outputs as tests/golden/make_golden.py writes them, except that the
inference policy is Independent(Normal(mean, std), 1) itself, so its parameters are `base_dist.loc` / `base_dist.scale`.
`normaltanh_state_dict` holds, per normal_tanh preset, the reference's state_dict keys and shapes and the parameter order of
each optimizer."""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (puts the repository and the reference checkout of argv[1] on sys.path)
import make_golden_vecobs as MV  # noqa: E402
from make_golden import DATA_SEED, NOISE_SEED, WEIGHT_SEED, RefDreamer  # noqa: E402

from oracle import normaltanh_oracle  # noqa: E402
from oracle.weights import seeded_state_dict  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402
from pydreamer_b200.replay import synthetic_batch  # noqa: E402

CASES = {n: dict(preset=n, over={}) for n in ("tiny_dmc_normaltanh", "tiny_dmc_normaltanh_iwae3", "tiny_vector_normaltanh")}
LOG_CASES = ("tiny_dmc_normaltanh",)
STATE_DICT_PRESETS = tuple(CASES) + ("dmc_normaltanh",)


def run_log_case(name, spec):
    """make_golden.run_log_case for the normal_tanh policy."""
    torch.distributions.Distribution.set_default_validate_args(False)
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    assert conf.actor_dist == "normal_tanh"
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
        dist, os3, m3 = ref.inference(o1, (state[0][:B], state[1][:B]))
    assert type(dist) is torch.distributions.Independent and type(dist.base_dist) is torch.distributions.Normal
    lg = torch.cat([dist.base_dist.loc, dist.base_dist.scale], -1)
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
                           params={g: [[names[id(p)], list(p.shape)] for p in ps] for g, ps in groups.items()})
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print(f"{name}: {len(out)} presets -> {path}")


if __name__ == "__main__":
    MV.O = normaltanh_oracle                          # the case runner checks the reference against the normal_tanh oracle
    wanted = sys.argv[2:]
    for n in LOG_CASES:
        if not wanted or n + "_log" in wanted:
            run_log_case(n + "_log", CASES[n])
    for n, spec in CASES.items():
        if not wanted or n in wanted:
            MV.run_case(n, spec)
    if not wanted or "normaltanh_state_dict" in wanted:
        write_state_dict_fixture("normaltanh_state_dict")

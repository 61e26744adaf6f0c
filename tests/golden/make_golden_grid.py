"""Generates the categorical grid-image fixtures under tests/golden/ from the UNMODIFIED reference (jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden_grid.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  Same procedure and seeds as tests/golden/make_golden_vecobs.py: per case
(1) the reference Dreamer with seeded weights runs training_step + the four backward passes, (2) oracle/grid_oracle.py,
fed the same RNG stream as explicit noise, must reproduce its losses, metrics, gradients and decoded image, (3) the
REFERENCE's numbers are stored.  The `_log` cases hold the reference's logging, open-loop and inference outputs.
`grid_state_dict` holds, per grid preset and `minigrid`, the reference's state_dict keys and shapes and the parameter
order of each optimizer."""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (puts the repository and the reference checkout of argv[1] on sys.path)
from make_golden import DATA_SEED, NOISE_SEED, WEIGHT_SEED, RefDreamer  # noqa: E402

from oracle import grid_oracle as O  # noqa: E402
from oracle.grid_oracle import seeded_state_dict  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402
from pydreamer_b200.replay import synthetic_batch  # noqa: E402

CASES = {n: dict(preset=n, over={}) for n in ("tiny_grid", "tiny_grid_iwae3", "tiny_grid_minprob", "tiny_grid_layers0",
                                               "tiny_grid_plain", "tiny_grid_vecobs")}
LOG_CASES = ("tiny_grid", "tiny_grid_iwae3")
GRID_PRESETS = tuple(CASES) + ("minigrid",)


def run_case(name, spec):
    torch.distributions.Distribution.set_default_validate_args(False)   # train.py:30
    conf = make_conf(spec["preset"], device="cpu", **spec["over"])
    T, B, I = conf.batch_length, conf.batch_size, conf.iwae_samples
    torch.manual_seed(0)
    ref = RefDreamer(conf)
    sd = seeded_state_dict(ref.state_dict(), WEIGHT_SEED)
    ref.load_state_dict(sd)
    obs = synthetic_batch(conf, seed=DATA_SEED)
    g = torch.Generator().manual_seed(99)                       # a non-trivial carried state exercises the reset masking
    state = ref.init_state(B * I)
    state = (torch.tanh(torch.randn(state[0].shape, generator=g)), torch.zeros_like(state[1]))
    torch.manual_seed(NOISE_SEED)
    losses, out_state, metrics, tensors, _ = ref.training_step(obs, state)
    for l in losses:
        l.backward()
    ref_grads = {n: p.grad.clone() for n, p in ref.named_parameters() if p.grad is not None}

    torch.manual_seed(NOISE_SEED)
    noise = O.draw_noise(conf, T, B)
    sdo = {k: v.clone().requires_grad_(not k.startswith("ac.critic_target")) for k, v in sd.items()}
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
    for k in ("image_rec", "loss_image", "vecobs_rec", "reward_rec", "loss_kl", "policy_value"):
        if k in tensors:
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
    path = os.path.join(HERE, name + ".json")
    with open(path, "w") as f:
        json.dump(fix, f, indent=1, sort_keys=True)
    print(f"{name}: losses {fix['losses']}  oracle-vs-reference worst grad rel err {worst:.2e} -> {path}")


def write_state_dict_fixture(name):
    out = {}
    for preset in GRID_PRESETS:
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
    MG.seeded_state_dict = seeded_state_dict           # the logging cases draw their weights with the grid-aware rule
    wanted = sys.argv[2:]
    for n in LOG_CASES:
        if not wanted or n + "_log" in wanted:
            MG.run_log_case(n + "_log", CASES[n])        # the logging branches: the reference's outputs, no oracle involved
    for n, spec in CASES.items():
        if not wanted or n in wanted:
            run_case(n, spec)
    if not wanted or "grid_state_dict" in wanted:
        write_state_dict_fixture("grid_state_dict")

"""Generates the stacked-GRU fixtures (`gru_layers` > 1) under tests/golden/ from the UNMODIFIED reference (jurgisp/pydreamer).

Run with a checkout of the reference:
    python tests/golden/make_golden_gru.py <reference checkout> [fixture name ...]
(without names every fixture below is written).  Same procedure and seeds as tests/golden/make_golden_vecobs.py, whose case
runner it uses with oracle/gru_oracle.py in place of the vector-observation oracle: per case (1) the reference Dreamer with
seeded weights runs training_step + the four backward passes, (2) the oracle, fed the same RNG stream as explicit noise,
must reproduce its losses, metrics and gradients, (3) the REFERENCE's numbers are stored.  The `_log` cases hold the
reference's logging, open-loop and inference outputs.  `gru_state_dict` holds, per stacked-GRU preset, the reference's
state_dict keys and shapes and the parameter order of each optimizer."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (puts the repository and the reference checkout of argv[1] on sys.path)
import make_golden_vecobs as MV  # noqa: E402
from make_golden import RefDreamer  # noqa: E402

from oracle import gru_oracle  # noqa: E402
from pydreamer_b200.config import make_conf  # noqa: E402

CASES = {n: dict(preset=n, over={}) for n in ("tiny_gru2", "tiny_gru4_iwae3", "tiny_dmc_gru2", "tiny_vector_gru2",
                                               "tiny_gru3_odd")}
LOG_CASES = ("tiny_gru2", "tiny_gru4_iwae3")
GRU_PRESETS = tuple(CASES) + ("atari_gru2",)


def write_state_dict_fixture(name):
    out = {}
    for preset in GRU_PRESETS:
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
    MV.O = gru_oracle                                 # the case runner checks the reference against the stacked-cell oracle
    wanted = sys.argv[2:]
    for n in LOG_CASES:
        if not wanted or n + "_log" in wanted:
            MG.run_log_case(n + "_log", CASES[n])    # the logging branches: the reference's outputs, no oracle involved
    for n, spec in CASES.items():
        if not wanted or n in wanted:
            MV.run_case(n, spec)
    if not wanted or "gru_state_dict" in wanted:
        write_state_dict_fixture("gru_state_dict")

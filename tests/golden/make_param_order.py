"""Writes tests/golden/param_order.json from the UNMODIFIED reference: for each optimizer `Dreamer.init_optimizers`
builds (pydreamer/models/dreamer.py:60-71) the parameter NAMES in `.parameters()` order; and state_dict_keys.json, every
key of the reference's state_dict with its shape (what a strict load_state_dict checks).  torch.optim state dicts key the
per-parameter state by that index, so a checkpoint's optimizer state only round-trips if the drop-in module enumerates
its parameters in the same order.  Run with a checkout of the reference:  python tests/golden/make_param_order.py <reference checkout>"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.abspath(sys.argv[1]))  # a checkout of the reference

from pydreamer.models import Dreamer as RefDreamer  # noqa: E402  (the reference)

from pydreamer_b200.config import make_conf  # noqa: E402

out, keys = {}, {}
for preset in ("tiny", "tiny_dmc"):
    ref = RefDreamer(make_conf(preset, device="cpu"))
    keys[preset] = [[k, list(v.shape)] for k, v in ref.state_dict().items()]   # parameters and buffers: strict-load key set
    names = {id(p): n for n, p in ref.named_parameters()}
    groups = dict(wm=ref.wm.parameters(), probe=ref.probe_model.parameters(), actor=ref.ac.actor.parameters(),
                  critic=ref.ac.critic.parameters())
    out[preset] = {g: [[names[id(p)], list(p.shape)] for p in ps] for g, ps in groups.items()}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "param_order.json"), "w") as f:
    json.dump(out, f, indent=0)
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "state_dict_keys.json"), "w") as f:
    json.dump(keys, f, indent=0)
print({k: {g: len(v) for g, v in d.items()} for k, d in out.items()})

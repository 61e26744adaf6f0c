"""Training-step throughput of the observation layouts side by side: `vectorenv` (a 4-float vector, no image), `minecraft`
(64x64x3 image + a 27-float vector) and `atari` (image only), as shipped in the reference's config/defaults.yaml.

Each preset gets its own model and seeded batch; every step is one iteration of the reference training loop
(training_step, four backward calls, grad_clip, four optimizer steps) with CUDA-graph replay on.  After a warm-up (which
captures each graph), the presets are timed in alternating rounds with CUDA events, so a drift of the shared machine
falls on all of them alike.  Prints one JSON line: per preset the median steps/s over the rounds, their spread and the
library kernels per step (nodes of the captured graph), plus the card's name and power limit.

    python tools/bench_obs.py [--steps 10] [--warmup 5] [--rounds 5] [--presets vectorenv,minecraft,atari] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["", ""])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "")
    return dict(name=name, power_limit=power)


class Arm:
    def __init__(self, preset, dev):
        from oracle.grid_oracle import seeded_state_dict      # the weights of oracle/weights.py, grid-aware
        from pydreamer_b200.config import make_conf
        from pydreamer_b200.dreamer import Dreamer
        from pydreamer_b200.replay import synthetic_batch

        self.conf = c = make_conf(preset, device=dev)
        self.model = Dreamer(c).to(dev)
        self.model.load_state_dict(seeded_state_dict(self.model.state_dict(), 11))
        self.opts = self.model.init_optimizers(c.adam_lr, c.adam_lr_actor, c.adam_lr_critic, c.adam_eps)
        self.obs = synthetic_batch(c, seed=1234, device=dev)
        self.state = self.model.init_state(c.batch_size * c.iwae_samples)

    def step(self):
        m, c = self.model, self.conf
        losses, self.state, metrics, _, _ = m.training_step(self.obs, self.state)
        for o in self.opts:
            o.zero_grad()
        for l in losses:
            l.backward()
        m.grad_clip(c.grad_clip, c.grad_clip_ac)
        for o in self.opts:
            o.step()
        return losses

    def kernels(self):
        (st,) = self.model._graphs.values()
        assert st["graph"] is not None and not st.get("failed"), "the step was not captured"
        return st["kernels"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--presets", default="vectorenv,minecraft,atari")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_obs.py measures on a CUDA device; there is none")
    dev = "cuda:0"
    torch.manual_seed(0)
    arms = {p: Arm(p, dev) for p in a.presets.split(",")}
    for arm in arms.values():
        for _ in range(max(a.warmup, 3)):                 # calls 1-2 eager, 3 captures the graph
            arm.step()
    torch.cuda.synchronize()
    rates = {p: [] for p in arms}
    for _ in range(a.rounds):
        for p, arm in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                losses = arm.step()
            e1.record()
            e1.synchronize()
            rates[p].append(a.steps / (e0.elapsed_time(e1) / 1e3))
            assert all(torch.isfinite(l).all() for l in losses), p
    res = dict(card=card(), steps=a.steps, warmup=a.warmup, rounds=a.rounds, graphs=True, results={
        p: dict(steps_per_s=round(statistics.median(r), 3), min=round(min(r), 3), max=round(max(r), 3),
                launches_per_step=arms[p].kernels(), batch=[arms[p].conf.batch_length, arms[p].conf.batch_size],
                vecobs_size=arms[p].conf.vecobs_size, image=bool(arms[p].conf.image_encoder)) for p, r in rates.items()})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

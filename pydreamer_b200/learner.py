"""Data-parallel learner step: the inner loop of the reference's train.py (146-303) around the drop-in Dreamer, without
mlflow.  SURVEY.md §8(f) row N1.

  * one process per GPU; each rank feeds its own replay shard (its own batch iterator: nothing here draws random
    numbers, so shards differ exactly as the caller's iterators do); gradients are all-reduced once per step (parallel.py)
  * truncated BPTT state carry per data stream (`states[wid]`, train.py:168-178, `keep_state`)
  * checkpoints in the reference's format (tools.py:164-174: {'epoch', 'model_state_dict', 'optimizer_{i}_state_dict'}), so the
    unmodified CPU generators (generator.py:105-116) keep loading `latest.pt` into the reference `Dreamer`.
"""
import torch

from .dreamer import Dreamer


class Learner:
    def __init__(self, conf, device="cuda:0", data_parallel=None):
        self.conf = conf
        self.device = torch.device(device)
        self.model = Dreamer(conf).to(self.device)
        self.model._ensure_arena()
        if data_parallel is not None:
            self.model._dp = data_parallel
            data_parallel.broadcast_params(self.model)
        self.optimizers = self.model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
        self.states = {}
        self.steps = 0

    def step(self, batch, wid=0, do_image_pred=False, do_dream_tensors=False):
        """One gradient step on `batch` (dict of (T,B,...) tensors, host or device).  Returns (metrics, tensors, dream)."""
        conf, model = self.conf, self.model
        obs = {k: v.to(self.device, non_blocking=True) for k, v in batch.items()}            # train.py:161
        B = obs["action"].shape[1]
        state = self.states.get(wid)
        if state is None:
            state = model.init_state(B * conf.iwae_samples)                                  # train.py:168-170
        losses, new_state, metrics, tensors, dream = model.training_step(
            obs, state, do_image_pred=do_image_pred, do_dream_tensors=do_dream_tensors)
        if conf.keep_state:
            self.states[wid] = tuple(s.clone() for s in new_state)                           # train.py:177-178
        for opt in self.optimizers:
            opt.zero_grad()
        for loss in losses:                                                                  # train.py:186-187
            loss.backward()
        grad_metrics = model.grad_clip(conf.grad_clip, conf.grad_clip_ac)                    # train.py:195
        for opt in self.optimizers:
            opt.step()                                                                       # train.py:196-197
        self.steps += 1
        metrics = dict(metrics)
        metrics.update(grad_metrics)
        return metrics, tensors, dream

    def train_on_batches(self, batches, num_steps):
        """Gradient steps from an iterator of RAW replay batches — what the reference's own `DataSequential`
        (pydreamer/data.py:127-305, which stays the caller's: the replay pipeline is outside this package) yields before
        its `Preprocessor`: uint8 HWC images, integer actions, (T,B,...) arrays.  They cross PCIe in that format and are
        converted on the device (preprocess.py; train.py:104-131,146-166 without the DataLoader workers).  In a
        data-parallel job every rank passes its OWN iterator (own replay shard / own numpy seed).  Returns the metrics of
        the last step."""
        from .preprocess import GpuPreprocessor

        pre = GpuPreprocessor(self.conf, self.device)
        keys = ("image", "vecobs", "action", "reward", "terminal", "reset")
        metrics = None
        for _, raw in zip(range(num_steps), batches):
            obs = pre.apply({k: raw[k] for k in keys if k in raw})
            metrics, _, _ = self.step(obs)
        return metrics

    # ---- tools.py:164-197
    def save_checkpoint(self, path):
        ck = {"epoch": self.steps, "model_state_dict": {k: v.detach().cpu() for k, v in self.model.state_dict().items()}}
        for i, opt in enumerate(self.optimizers):
            ck[f"optimizer_{i}_state_dict"] = opt.state_dict()
        torch.save(ck, path)

    def load_checkpoint(self, path, map_location=None):
        """tools.py:177-197.  The optimizer entries are torch.optim.AdamW state dicts (what the reference's loop writes and
        what `_FusedAdamW.state_dict` emits), so Adam moments and step counts resume whichever side wrote the file."""
        ck = torch.load(path, map_location=map_location or self.device)
        self.model.load_state_dict(ck["model_state_dict"])
        for i, opt in enumerate(self.optimizers):
            key = f"optimizer_{i}_state_dict"
            if key in ck:
                opt.load_state_dict(ck[key])
            else:
                import warnings
                warnings.warn(f"checkpoint {path} has no {key}: optimizer {i} restarts from zero moments")
        self.steps = ck["epoch"]
        return self.steps

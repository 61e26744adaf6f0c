"""Device-side restatement of the reference's batch Preprocessor (pydreamer/preprocessing.py:91-188) for the keys the hot
path reads.  The raw replay batch (uint8 HWC images, integer actions, raw rewards) crosses PCIe as is — 31 MB instead of
123 MB of fp32 per Atari batch — and is converted by three small kernels: SURVEY.md §8(f) row N3.

    image    uint8 (T,B,H,W,C)        -> fp32 (T,B,C,H,W) = x/255 - 0.5          preprocessing.py:21-29
             with image_categorical: category ids (T,B,H,W) of uint8 / int32 / int64 -> fp32 one-hot (T,B,C,H,W),
             C = image_channels (preprocessing.py:10-19, 105-110); an id outside [0, C) gives NaN channels
    action   int64 (T,B) | fp (T,B,A) -> fp32 one-hot (T,B,A) | as is             preprocessing.py:135-138
    reward   (T,B)                    -> fp32, tanh-clipped if clip_rewards=tanh  preprocessing.py:148-150, functions.py:153-160
    terminal (T,B) -> fp32 ; reset (T,B) bool stays                               preprocessing.py:148
    vecobs   (T,B,K)                  -> fp32                                     preprocessing.py:160-163
A batch without `image` (a model without an image encoder) passes without one.
"""
import torch

from . import ops as _ops


class GpuPreprocessor:
    def __init__(self, conf, device):
        self.conf, self.device = conf, torch.device(device)
        self._ops = None
        if conf.clip_rewards not in (None, "tanh"):
            raise NotImplementedError(f"clip_rewards={conf.clip_rewards}")       # log1p variant: not on the hot path

    @property
    def ops(self):
        if self._ops is None:
            self._ops = _ops.get_ops(self.device)
        return self._ops

    @torch.no_grad()
    def apply(self, batch):
        dev, conf = self.device, self.conf
        b = {k: (v if isinstance(v, torch.Tensor) else torch.as_tensor(v)).to(dev, non_blocking=True) for k, v in batch.items()}
        T, B = b["reward"].shape[:2]
        out = {}
        img = b.get("image")
        if img is None:
            pass
        elif conf.image_categorical:
            C = conf.image_channels
            H, W = img.shape[-2:]
            if img.dtype not in (torch.uint8, torch.int32, torch.int64):
                img = img.to(torch.int64)
            out["image"] = torch.empty(T, B, C, H, W, device=dev)
            self.ops.image_ids_onehot(img.contiguous(), out["image"])
        elif img.dtype == torch.uint8:
            H, W, C = img.shape[-3:]
            out["image"] = torch.empty(T, B, C, H, W, device=dev)
            self.ops.image_u8_to_f32(img.contiguous(), out["image"])
        else:
            out["image"] = img.to(torch.float32).movedim(-1, -3).contiguous()
        if "vecobs" in b:
            out["vecobs"] = b["vecobs"].to(torch.float32).contiguous()
        act = b["action"]
        if act.dim() == 2:
            out["action"] = torch.empty(T, B, conf.action_dim, device=dev)
            self.ops.onehot_i64(act.to(torch.int64).contiguous(), out["action"])
        else:
            out["action"] = act.to(torch.float32)
        rew = b["reward"].to(torch.float32).contiguous()
        if conf.clip_rewards == "tanh":
            out["reward"] = torch.empty_like(rew)
            self.ops.tanh(rew, out["reward"])
        else:
            out["reward"] = rew
        out["terminal"] = b.get("terminal", torch.zeros(T, B, device=dev)).to(torch.float32)
        out["reset"] = b["reset"].to(torch.bool)
        return out

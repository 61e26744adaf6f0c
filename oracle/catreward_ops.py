"""TEST INFRASTRUCTURE — plain-torch twin of the device op the categorical reward head adds, on top of
oracle/vecobs_ops.py.

`CatRefOps` is `VecRefOps` plus support_head: pd_support_head (decoders.py:322-362 DenseCategoricalSupportDecoder,
common.py:77-86 CategoricalSupport.mean), in float32.  For models with the Normal reward head it computes exactly what
VecRefOps computes.  Only tests/ may import it; the product path never does.
"""
import torch

from oracle.vecobs_ops import VecRefOps

SUPPORT_MAX = 1024                              # PD_SUPPORT_MAX of include/pd_b200.h


class CatRefOps(VecRefOps):
    def support_head(self, y, support, target, tgt_div, rec, loss=None, dy=None, idx=None):
        M, S = y.shape
        if not (2 <= S <= SUPPORT_MAX and tgt_div >= 1):
            raise RuntimeError(f"pd_support_head: S={S}, tgt_div={tgt_div} unsupported")
        p = torch.softmax(y, -1)
        if rec is not None:
            rec.view(-1).copy_((p * support).sum(-1))
        if target is None:
            return
        t = target.reshape(-1)[torch.arange(M, device=y.device) // tgt_div]
        k = torch.square(t[:, None] - support).argmin(-1)
        loss.view(-1).copy_(torch.logsumexp(y, -1) - y.gather(-1, k[:, None])[:, 0])
        dy.copy_(p - torch.nn.functional.one_hot(k, S).to(p.dtype))
        if idx is not None:
            idx.view(-1).copy_(k.to(torch.int32))

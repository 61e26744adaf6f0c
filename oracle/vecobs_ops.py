"""TEST INFRASTRUCTURE — plain-torch twins of the device ops the vector-observation path adds, on top of oracle/ref_ops.py.

`VecRefOps` is `RefOps` plus
  * vec_head_loss: pd_vec_head_loss (decoders.py:290-319, DenseNormalDecoder with out_dim = K);
  * wm_loss with the trailing `l_vec` / `w_vec` operands of pd_wm_loss and a NULL image loss (image-less models).
For image-only models it computes exactly what RefOps computes.  Only tests/ may import it; the product path never does.
"""
import torch
import torch.nn.functional as F

from oracle.ref_ops import RefOps

VEC_HEAD_MAX_K = 4096                           # PD_VEC_HEAD_MAX_K of include/pd_b200.h


class VecRefOps(RefOps):
    def vec_head_loss(self, y, target, tgt_div, loss, dy):
        M, K = y.shape
        if not (1 <= K <= VEC_HEAD_MAX_K and tgt_div >= 1):
            raise RuntimeError(f"pd_vec_head_loss: K={K}, tgt_div={tgt_div} unsupported")
        d = y - target[torch.arange(M, device=y.device) // tgt_div]
        dy.copy_(d)
        loss.view(-1).copy_(0.5 * (d * d).sum(-1))

    def wm_loss(self, TB, I, kl_weight, w_img, w_rew, w_term, l_img, l_rew, l_term, l_kl, kl_exact, ent_prior,
                ent_post, w, tb, l_vec=None, w_vec=0.0):
        img = l_img if l_img is not None else torch.zeros_like(l_rew)
        L = kl_weight * l_kl + w_img * img + w_rew * l_rew + w_term * l_term
        if l_vec is not None:
            L = L + w_vec * l_vec
        L = L.view(TB, I)
        tb[:, 0] = self._nlae(L)
        if I == 1:
            w.fill_(1.0 / TB)
        else:
            w.view(TB, I).copy_(F.softmax(-L, -1) / TB)
        for j, v in ((1, img), (2, l_rew), (3, l_term), (4, kl_exact)):
            tb[:, j] = self._nlae(v.view(TB, I))
        tb[:, 5] = ent_prior.view(TB, I).mean(-1)
        tb[:, 6] = ent_post.view(TB, I).mean(-1)
        tb[:, 7] = self._nlae(l_vec.view(TB, I)) if l_vec is not None else 0

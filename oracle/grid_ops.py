"""TEST INFRASTRUCTURE — plain-torch twins of the device ops the categorical grid-image front end adds, on top of
oracle/auxcritic_ops.py.

`GridRefOps` is `AuxRefOps` plus, in float32,
  * image_ids_onehot: pd_image_ids_onehot (preprocessing.py:10-19, 105-110; NaN channels for an id outside [0, C));
  * grid_enc_input:   pd_grid_enc_input (encoders.py:50-60: the one-hot image followed by reward and terminal planes);
  * cat_image_loss:   pd_cat_image_loss (decoders.py:212-254 CatImageDecoder.loss / training_step).
For models without grid images it computes exactly what AuxRefOps computes.  Only tests/ may import it; the product path
never does.
"""
import torch

from oracle.auxcritic_ops import AuxRefOps

CAT_IMAGE_MAX_C = 64                            # PD_CAT_IMAGE_MAX_C of include/pd_b200.h
CAT_IMAGE_MAX_P = 4096                          # PD_CAT_IMAGE_MAX_P


def first_argmax(t):
    """torch.argmax over dim 1 (the first maximum; NaN above everything)."""
    return t.argmax(1)


def cat_image_terms(y, C, target, tgt_div, min_prob):
    """-> (loss per row (M,), dy (M, C*P), rec (M / tgt_div, C*P)) of pd_cat_image_loss, in y's dtype."""
    M, CP = y.shape
    P = CP // C
    y3 = y.reshape(M, C, P)
    t3 = target.reshape(-1, C, P)[torch.arange(M, device=y.device) // tgt_div]
    k = first_argmax(t3)                                                # (M, P)
    lse = torch.logsumexp(y3, 1, keepdim=True)
    p = torch.exp(y3 - lse)
    onehot = torch.nn.functional.one_hot(k, C).movedim(-1, 1).to(y.dtype)
    yk = y3.gather(1, k[:, None])[:, 0]
    if min_prob == 0:
        loss = lse[:, 0] - yk
        dy = p - onehot
    else:
        pk = torch.softmax(y3, 1).gather(1, k[:, None])[:, 0]
        q = (1 - min_prob) * pk + min_prob / C
        loss = -torch.log(q)
        dy = ((1 - min_prob) * pk / q)[:, None] * (p - onehot)
    norm = y3 - lse
    r = torch.logsumexp(norm.reshape(M // tgt_div, tgt_div, C, P), 1)
    r = r - torch.logsumexp(r, 1, keepdim=True)
    return loss.sum(-1), dy.reshape(M, CP), r.reshape(M // tgt_div, CP)


class GridRefOps(AuxRefOps):
    def image_ids_onehot(self, ids, out):
        C = out.shape[-3]
        if ids.dtype not in (torch.uint8, torch.int32, torch.int64):
            raise TypeError(f"pd_image_ids_onehot: category ids of dtype {ids.dtype} (uint8, int32 or int64)")
        i = ids.long()
        bad = (i < 0) | (i >= C)
        x = torch.nn.functional.one_hot(i.clamp(0, C - 1), C).to(out.dtype).movedim(-1, -3)
        out.copy_(x.masked_fill(bad.unsqueeze(-3), float("nan")))

    def grid_enc_input(self, image, reward, terminal, out):
        NB, C, H, W = image.shape
        P = H * W
        out[:, :C * P] = image.reshape(NB, C * P)
        out[:, C * P:(C + 1) * P] = reward.reshape(NB, 1)
        out[:, (C + 1) * P:] = terminal.reshape(NB, 1)

    def cat_image_loss(self, y, C, target, tgt_div, min_prob, loss=None, dy=None, rec=None):
        M, CP = y.shape
        if not (2 <= C <= CAT_IMAGE_MAX_C and CP % C == 0 and 1 <= CP // C <= CAT_IMAGE_MAX_P and tgt_div >= 1
                and M % tgt_div == 0 and 0 <= min_prob < 1):
            raise RuntimeError(f"pd_cat_image_loss: M={M} C={C} P={CP // max(C, 1)} tgt_div={tgt_div} min_prob={min_prob} "
                               "unsupported")
        l_, d_, r_ = cat_image_terms(y, C, target, tgt_div, min_prob)
        if loss is not None:
            loss.view(-1).copy_(l_)
        if dy is not None:
            dy.copy_(d_)
        if rec is not None:
            rec.view(-1).copy_(r_.reshape(-1))

"""TEST INFRASTRUCTURE — plain-torch twin of the stacked-GRU form of pd_rssm_unroll_fwd, on top of oracle/vecobs_ops.py.

`GruRefOps` is `VecRefOps` whose rssm_unroll_fwd also takes `layers` = L in 2..4 (include/pd_b200.h, pd_rssm_fwd_args):
layer 0 reads za, layer l > 0 the fp16 h' of layer l - 1; `w_hh16` is the block-diagonal [3D, D] recurrent weight, `gates`
is laid out [L, T, BI, 4D/L].  For a single cell it is VecRefOps' statement.  It runs in the dtype of the tensors it is
given (float64 in tests/test_gru_layers_kernels_f64_gpu.py).  Only tests/ may import it; the product path never does.
"""
import torch
import torch.nn.functional as F

from oracle.ref_ops import SMS, _cdiv, _group_softmax, _require
from oracle.vecobs_ops import VecRefOps


class GruRefOps(VecRefOps):
    def rssm_unroll_fwd(self, dims, eps, **t):
        L = int(dims.get("layers", 0))
        w_ih_l, b_ih_l, b_hh_l = (t.pop(k, None) or [] for k in ("w_ih16_l", "b_ih_l", "b_hh_l"))
        if L <= 1:
            return super().rssm_unroll_fwd({k: v for k, v in dims.items() if k != "layers"}, eps, **t)
        T, BI, I, D, Hd, G, C = (int(dims[k]) for k in ("T", "BI", "I", "D", "Hd", "G", "C"))
        Dl = D // L
        RG = SMS // (4 if D % 256 == 0 else 1)
        _require(L <= 4 and D % L == 0 and Dl % 8 == 0 and len(w_ih_l) == L - 1 and T >= 1 and 1 <= BI <= 256 and I >= 1 and
                 BI % I == 0 and Hd <= 1024 and Hd % 8 == 0 and 1 <= C <= 32 and 1 <= G <= min(SMS, 256) and
                 _cdiv(Dl, SMS) <= 16 and _cdiv(D, RG) <= 64 and _cdiv(Hd, RG) <= 32, f"pd_rssm_unroll_fwd: shape {dict(dims)}")
        B = BI // I
        x1, za, m1, r1, gates, feat, hin, zin = (t[k] for k in ("x1", "za", "m1", "r1", "gates", "feat", "hin", "zin"))
        y2, pin, m2, r2, post, idx = (t[k] for k in ("y2", "pin", "m2", "r2", "post", "idx"))
        aa, ea, mask, noise = t["aa"], t.get("ea"), t["mask"], t["noise"]
        dt = x1.dtype
        Wz, Whh, Wph, Wpm = (t[k].to(dt) for k in ("w_z16", "w_hh16", "w_ph16", "w_pm16"))
        Wih = [t["w_ih16"].to(dt)] + [w.to(dt) for w in w_ih_l]
        bih, bhh = [t["b_ih"]] + list(b_ih_l), [t["b_hh"]] + list(b_hh_l)
        gl = gates.reshape(L, T, BI, 4 * Dl)
        h16 = lambda v: v.to(torch.float16).to(dt)
        rep = lambda v: v.repeat_interleave(I, 0) if I > 1 else v

        def ln(x, g, b):
            mu, var = x.mean(-1), x.var(-1, unbiased=False)
            r = 1.0 / torch.sqrt(var + eps)
            return h16(F.elu((x - mu[:, None]) * r[:, None] * g + b)), mu, r

        gh = h16(hin[0]) @ Whh.t()                                       # raw product, row gate * D + u; mask and bias at use
        for s in range(T):
            m = mask[s] if s > 0 else torch.ones_like(mask[0])
            if s > 0:
                zprev = feat[s - 1][:, D:]
                x1[s].copy_(m[:, None] * (zprev @ Wz.t()) + t["b_z"] + rep(aa[s * B:(s + 1) * B]))
                zin[s].copy_(zprev * m[:, None])
            x, mu, r = ln(x1[s], t["ln1_g"], t["ln1_b"])
            za[s].copy_(x); m1[s].copy_(mu); r1[s].copy_(r)
            ghm = m[:, None] * gh
            for l in range(L):
                cols = slice(l * Dl, (l + 1) * Dl)
                gi = x @ Wih[l].t() + bih[l]
                ghb = torch.cat([ghm[:, g * D + l * Dl:g * D + (l + 1) * Dl] for g in range(3)], 1) + bhh[l]
                rg = torch.sigmoid(gi[:, :Dl] + ghb[:, :Dl])
                ug = torch.sigmoid(gi[:, Dl:2 * Dl] + ghb[:, Dl:2 * Dl])
                ghn = ghb[:, 2 * Dl:]
                ng = torch.tanh(gi[:, 2 * Dl:] + rg * ghn)
                hn = h16((1 - ug) * ng + ug * hin[s][:, cols])
                feat[s][:, cols].copy_(hn)
                gl[l, s].view(BI, 4, Dl).copy_(torch.stack([rg, ug, ng, ghn], 1))
                if s + 1 < T:
                    hin[s + 1][:, cols].copy_(hn * mask[s + 1][:, None])
                x = hn
            hn = feat[s][:, :D]
            v = hn @ Wph.t() + t["b_ph"]
            if ea is not None:
                v = v + rep(ea[s * B:(s + 1) * B])
            y2[s].copy_(v)
            gh = hn @ Whh.t()
            y, mu, r = ln(y2[s], t["ln2_g"], t["ln2_b"])
            pin[s].copy_(y); m2[s].copy_(mu); r2[s].copy_(r)
            post[s].copy_(y @ Wpm.t() + t["b_pm"])
            _, p = _group_softmax(post[s], G, C)
            k = (p / noise[s].reshape(BI, G, C)).argmax(-1)
            idx[s].copy_(k.to(idx.dtype))
            feat[s][:, D:].copy_(F.one_hot(k, C).to(dt).reshape(BI, G * C))

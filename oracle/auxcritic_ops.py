"""TEST INFRASTRUCTURE — plain-torch twin of the device op the world model's auxiliary critic adds, on top of
oracle/catreward_ops.py.

`AuxRefOps` is `CatRefOps` plus gae_critic_obs: pd_gae_critic_obs (a2c.py:81-116 on the replayed sequence,
dreamer.py:347-365), in float32.  For models without `aux_critic` it computes exactly what CatRefOps computes.  Only
tests/ may import it; the product path never does.
"""
import torch

from oracle.catreward_ops import CatRefOps

AUX_T_MAX = 128                                 # the row bound of pd_gae_critic_obs (include/pd_b200.h)


class AuxRefOps(CatRefOps):
    def gae_critic_obs(self, T, B, gamma, lam, vt, v, rew, term, scale, dv, sums):
        if not (2 <= T <= AUX_T_MAX and B >= 1):
            raise RuntimeError(f"pd_gae_critic_obs: T={T}, B={B} unsupported")
        H = T - 1
        vt, v, rew, tm = vt.reshape(T, B), v.reshape(T, B), rew.reshape(T, B), term.reshape(T, B)
        r1, t0, t1 = rew[1:], tm[:-1], tm[1:]
        a = -vt[:-1] + r1 + gamma * (1.0 - t1) * vt[1:]
        ag = torch.zeros_like(a)
        last = None
        for j in reversed(range(H)):
            last = a[j] if last is None else a[j] + lam * gamma * (1.0 - t1[j]) * last
            ag[j] = last
        d = ag + vt[:-1] - v[:-1]
        wgt = (1 - t0).log().cumsum(0).exp()
        dv.view(H, B).copy_(-d * wgt * (scale / (H * B)))
        sums[:2] += torch.stack([(0.5 * d * d * wgt).sum(), v[:-1].sum()]).double()

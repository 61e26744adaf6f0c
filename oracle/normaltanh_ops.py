"""TEST INFRASTRUCTURE — plain-torch twins of the two device ops the normal_tanh actor adds, on top of the reference op
tables.

`NormalTanhTwins` holds pd_normal_tanh_sample and pd_actor_loss_normal_tanh (functions.py:59-66 with min_std 0.01, max_std 1;
a2c.py:119-130 reinforce) in float32, with the host-side argument checks (PD_REQUIRE) of the native entry points restated:
a call the twin refuses is one the native library refuses.  `NtRefOps` adds them to oracle/auxcritic_ops.py's table (image
and / or vector observations, the auxiliary critic), `NtGruRefOps` to oracle/gru_ops.py's (the stacked GRU).  Only tests/
may import it; the product path never does.
"""
import math

import torch

from oracle.auxcritic_ops import AuxRefOps
from oracle.gru_ops import GruRefOps
from oracle.ref_ops import _ld, _require


class NormalTanhTwins:
    def actor_loss_normal_tanh(self, eta, out, actions, agae, weight, dout, sums):
        rows, A = actions.shape
        _require(A >= 1 and _ld(out) >= 2 * A and _ld(dout) >= 2 * A and _ld(actions) >= A,
                 f"pd_actor_loss_normal_tanh: A={A} (>= 1), ldo={_ld(out)} / lddo={_ld(dout)} (>= 2A), "
                 f"lda={_ld(actions)} (>= A)")
        mu = torch.tanh(out[:, :A])
        sg = torch.sigmoid(out[:, A:2 * A])
        sd = sg + 0.01
        zc = (actions - mu) / sd
        lp = (-0.5 * zc * zc - sd.log() - 0.5 * math.log(2 * math.pi)).sum(-1)
        ent = (0.5 + 0.5 * math.log(2 * math.pi) + sd.log()).sum(-1)
        ag, w = agae.reshape(-1), weight.reshape(-1)
        c = (w / rows)[:, None]
        dout[:, :A] = c * (-ag[:, None] * (zc / sd)) * (1 - mu * mu)
        dout[:, A:2 * A] = c * (-ag[:, None] * ((zc * zc - 1) / sd) - eta / sd) * (sg * (1 - sg))
        sums[0] += ((-lp * ag - eta * ent) * w).sum().double()
        sums[1] += ent.sum().double()

    def normal_tanh_sample(self, out, eps, action):
        rows, A = action.shape
        _require(A >= 1 and _ld(out) >= 2 * A and _ld(action) >= A,
                 f"pd_normal_tanh_sample: A={A} (>= 1), ldo={_ld(out)} (>= 2A), lda={_ld(action)} (>= A)")
        sd = torch.sigmoid(out[:, A:2 * A]) + 0.01
        action.copy_(torch.tanh(out[:, :A]) + sd * eps.reshape(rows, A))


class NtRefOps(NormalTanhTwins, AuxRefOps):
    pass


class NtGruRefOps(NormalTanhTwins, GruRefOps):
    pass

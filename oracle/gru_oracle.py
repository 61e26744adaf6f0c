"""TEST INFRASTRUCTURE — CPU restatement of the reference's training step with a stacked GRU in the RSSM (`gru_layers` > 1,
rnn.py:40-67 GRUCellStack with cell_type gru, built at rssm.py:106-107).

The stack: L cells of D / L units; layer 0 reads the normalised input za, layer l > 0 the new state of layer l - 1 of the
same step; the state is the concatenation of the layers' states, layer l owning columns [l D / L, (l + 1) D / L).
Everything else is oracle/vecobs_oracle.py (conv image and / or vector observation), whose training step runs here with
its recurrent cell replaced by the stack.  Pinned against the real reference by tests/golden/make_golden_gru.py, which
asserts this restatement reproduces the reference's losses / metrics / gradients before storing the fixtures.
"""
import torch
import torch.nn.functional as F

from oracle import vecobs_oracle
from oracle.dreamer_oracle import draw_noise, gru_cell  # noqa: F401


def gru_stack(sd, c, x, h, L):
    """GRUCellStack.forward (rnn.py:60-67): x (..., Hd), h (..., D) -> the new state (..., D)."""
    out = []
    for l, hl in enumerate(h.chunk(L, -1)):
        x = gru_cell(sd, c + f"gru.layers.{l}", x, hl)
        out.append(x)
    return torch.cat(out, -1)


def cell_pre(sd, c, action, h, z, L):
    """RSSMCell up to the new state (rssm.py:133-141, 166-172): z_mlp + a_mlp -> in_norm -> ELU -> the GRU stack."""
    x = F.linear(z, sd[c + "z_mlp.weight"], sd[c + "z_mlp.bias"]) + F.linear(action, sd[c + "a_mlp.weight"])
    x = F.elu(F.layer_norm(x, x.shape[-1:], sd[c + "in_norm.weight"], sd[c + "in_norm.bias"], 1e-3))
    return gru_stack(sd, c, x, h, L)


def training_step(sd, conf, obs, in_state, noise, **kw):
    """oracle/vecobs_oracle.training_step (same arguments and result) with the stacked cell of conf.gru_layers layers."""
    single = vecobs_oracle.cell_pre
    vecobs_oracle.cell_pre = lambda sd_, c, action, h, z: cell_pre(sd_, c, action, h, z, conf.gru_layers)
    try:
        return vecobs_oracle.training_step(sd, conf, obs, in_state, noise, **kw)
    finally:
        vecobs_oracle.cell_pre = single

"""TEST INFRASTRUCTURE — CPU restatement of the reference's training step with the world model's auxiliary critic
(`aux_critic`).

oracle/vecobs_oracle.py's step (image and / or vector observations) plus dreamer.py:347-365 and a2c.py:61-116: the
critic `wm.ac_aux.critic` and its target on the posterior features of importance sample 0, GAE(lambda_gae_aux,
gamma_aux) over the OBSERVED rewards and terminals, the critic loss added to the world-model loss with weight
aux_critic_weight.  The gradient reaches the aux critic and, through the features, every world-model weight; the aux actor
and target receive none.  Pinned against the real reference by tests/golden/make_golden_auxcritic.py, which asserts this
restatement reproduces the reference's losses / metrics / gradients before storing the fixtures.
"""
import torch

from oracle import vecobs_oracle
from oracle.dreamer_oracle import draw_noise, mlp  # noqa: F401

AUX = "wm.ac_aux."


def aux_critic(sd, conf, obs, features, I, target_synced=True):
    """-> (loss_critic_aux, value (T,B)) of a2c.py:81-116 on the sample-0 rows of features (T, B*I, F)."""
    T, B = obs["reward"].shape
    f = features.reshape(T, B, I, -1)[:, :, 0]
    tgt = AUX + ("critic.model" if target_synced else "critic_target.model")
    value_t = mlp({k: v.detach() for k, v in sd.items()}, tgt, f.detach(), 4)
    rew, term = obs["reward"], obs["terminal"]
    reward1, terminal0, terminal1 = rew[1:], term[:-1], term[1:]
    g, lam = conf.gamma_aux, conf.lambda_gae_aux
    advantage = -value_t[:-1] + reward1 + g * (1.0 - terminal1) * value_t[1:]
    agae, out = None, []
    for adv, trm in zip(reversed(advantage.unbind()), reversed(terminal1.unbind())):
        agae = adv if agae is None else adv + lam * g * (1.0 - trm) * agae
        out.append(agae)
    out.reverse()
    value_target = torch.stack(out) + value_t[:-1]
    reality_weight = (1 - terminal0).log().cumsum(dim=0).exp()
    value = mlp(sd, AUX + "critic.model", f, 4)
    loss = (0.5 * torch.square(value_target.detach() - value[:-1]) * reality_weight).mean()
    return loss, value


def training_step(sd, conf, obs, in_state, noise, iwae_samples=None, imag_horizon=None, force=None, target_synced=True,
                  aux_target_synced=True):
    """vecobs_oracle.training_step with the auxiliary critic: the same dict(losses, metrics, tensors, inter), losses[0]
    including aux_critic_weight * loss_critic_aux, metrics loss_critic_aux / policy_value_aux, tensor policy_value_aux.
    aux_target_synced: wm.ac_aux.critic_target == wm.ac_aux.critic (its counter is 0 mod target_interval_aux)."""
    I = int(iwae_samples or conf.iwae_samples)
    res = vecobs_oracle.training_step(sd, conf, obs, in_state, noise, iwae_samples, imag_horizon, force, target_synced)
    loss, value = aux_critic(sd, conf, obs, res["inter"]["features"], I, aux_target_synced)
    l = res["losses"]
    res["losses"] = (l[0] + conf.aux_critic_weight * loss,) + tuple(l[1:])
    res["metrics"].update(loss_critic_aux=loss.detach(), policy_value_aux=value[:-1].mean().detach())
    res["tensors"].update(policy_value_aux=value.detach())
    return res

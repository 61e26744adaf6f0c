"""TEST INFRASTRUCTURE — CPU restatement of the reference's training step with the normal_tanh actor
(`actor_dist: normal_tanh`).

The policy (functions.py:59-66 with min_std 0.01, max_std 1) is Independent(Normal(tanh(m), sigmoid(s) + 0.01), 1) on the
actor's 2A outputs, with no transform on the action: the dream samples a = mean + std * eps (dreamer.py:196-200,
Normal.sample), unbounded, and the reinforce loss (a2c.py:119-130) takes the Normal's log-prob and its true entropy.

The world-model part is the step of oracle/vecobs_oracle.py (image and / or vector observations), of
oracle/auxcritic_oracle.py with `aux_critic`, or of oracle/gru_oracle.py with `gru_layers` > 1.  Its imagination and
actor-critic, which restate the other actor distributions, are replaced here by the dream and actor-critic of
dreamer.py:188-216 and a2c.py:61-149 with this policy, from the same posterior features.  Pinned against the real reference
by tests/golden/make_golden_normaltanh.py, which asserts this restatement reproduces the reference's losses / metrics /
gradients before storing the fixtures.
"""
import math

import torch

from oracle import auxcritic_oracle, gru_oracle, vecobs_oracle
from oracle.dreamer_oracle import cell_pre, draw_noise, mlp, prior_logits, st_sample  # noqa: F401


def policy(out, A):
    """functions.py:59-66: (mean, std) of the Normal from the actor's 2A outputs."""
    return torch.tanh(out[..., :A]), torch.sigmoid(out[..., A:2 * A]) + 0.01


def training_step(sd, conf, obs, in_state, noise, iwae_samples=None, imag_horizon=None, force=None, target_synced=True,
                  **kw):
    """The base oracle's training_step (same arguments and result) with the normal_tanh dream and actor-critic."""
    assert conf.actor_dist == "normal_tanh" and conf.actor_grad == "reinforce"
    base = auxcritic_oracle if conf.aux_critic else gru_oracle if conf.gru_layers > 1 else vecobs_oracle
    res = base.training_step(sd, conf, obs, in_state, noise, iwae_samples=iwae_samples, imag_horizon=imag_horizon,
                             force=force, target_synced=target_synced, **kw)
    H = int(imag_horizon or conf.imag_horizon)
    force = force or {}
    D, G, C, A = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete, conf.action_dim
    L = conf.gru_layers
    cell = (lambda s, c, a, h, z: gru_oracle.cell_pre(s, c, a, h, z, L)) if L > 1 else cell_pre
    c = "wm.core.cell."

    # ---- dream (dreamer.py:188-216): world model frozen, start from the detached posterior features
    sdd = {k: v.detach() if k.startswith("wm.") else v for k, v in sd.items()}
    features = res["inter"]["features"].detach()
    N = features.shape[0] * features.shape[1]
    h, z = features.reshape(N, -1).split([D, G * C], -1)
    feats, acts, prior_idx = [], [], []
    AL = 4
    for i in range(H):
        f = torch.cat((h, z), -1)
        if "actor" in force:
            a = force["actor"][i]
        else:
            mu, sd_ = policy(mlp(sdd, "ac.actor.model", f, AL), A)
            a = mu + sd_ * noise["actor"][i]
        a = a.detach()
        feats.append(f); acts.append(a)
        h = cell(sdd, c, a, h, z)
        z, k = st_sample(prior_logits(sdd, c, h), noise["prior"][i], G, C,
                         force["prior_idx"][i] if "prior_idx" in force else None)
        prior_idx.append(k)
    feats.append(torch.cat((h, z), -1))
    feats, acts = torch.stack(feats).detach(), torch.stack(acts).detach()      # (H+1,N,F), (H,N,A)
    rewards = mlp(sdd, "wm.decoder.reward.model.model", feats, conf.reward_decoder_layers).detach()
    terminals = torch.sigmoid(mlp(sdd, "wm.decoder.terminal.model.model", feats, conf.terminal_decoder_layers)).detach()

    # ---- actor critic (a2c.py:61-149)
    tgt_prefix = "ac.critic.model" if target_synced else "ac.critic_target.model"
    value_t = mlp({k: v.detach() for k, v in sd.items()}, tgt_prefix, feats, AL)
    reward1, terminal0, terminal1 = rewards[1:], terminals[:-1], terminals[1:]
    value0t, value1t = value_t[:-1], value_t[1:]
    advantage = -value0t + reward1 + conf.gamma * (1.0 - terminal1) * value1t
    agae, out_ = None, []
    for adv, trm in zip(reversed(advantage.unbind()), reversed(terminal1.unbind())):
        agae = adv if agae is None else adv + conf.lambda_gae * conf.gamma * (1.0 - trm) * agae
        out_.append(agae)
    out_.reverse()
    advantage_gae = torch.stack(out_)
    value_target = advantage_gae + value0t
    reality_weight = (1 - terminal0).log().cumsum(dim=0).exp()
    value = mlp(sd, "ac.critic.model", feats, AL)
    value0 = value[:-1]
    loss_critic = (0.5 * torch.square(value_target.detach() - value0) * reality_weight).mean()
    out = mlp(sd, "ac.actor.model", feats[:-1], AL)
    mu, sd_ = policy(out, A)
    lpn = -((acts - mu) ** 2) / (2 * sd_ ** 2) - sd_.log() - math.log(math.sqrt(2 * math.pi))   # Normal.log_prob
    action_logprob = lpn.sum(-1)
    policy_entropy = (0.5 + 0.5 * math.log(2 * math.pi) + sd_.log()).sum(-1)                     # Normal.entropy
    loss_policy = -action_logprob * advantage_gae.detach()
    loss_actor = ((loss_policy - conf.entropy * policy_entropy) * reality_weight).mean()
    with torch.no_grad():
        res["metrics"].update(loss_critic=loss_critic.detach(), loss_actor=loss_actor.detach(),
                              policy_entropy=policy_entropy.mean(), policy_value=value0[0].mean(),
                              policy_value_im=value0.mean(), policy_reward=reward1.mean(), policy_reward_std=reward1.std())
    res["losses"] = tuple(res["losses"][:2]) + (loss_actor, loss_critic)
    res["inter"].update(prior_idx=torch.stack(prior_idx) if prior_idx else None, dream_features=feats, dream_actions=acts,
                        rewards=rewards, terminals=terminals, value=value.detach(), value_target=value_target.detach(),
                        advantage_gae=advantage_gae.detach(), reality_weight=reality_weight.detach(),
                        actor_out=out.detach())
    return res

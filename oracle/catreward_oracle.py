"""TEST INFRASTRUCTURE — CPU restatement of the reference's hot path with the categorical reward head
(`reward_decoder_categorical`).

The restatement of oracle/vecobs_oracle.py (image and / or vector observations, helpers of oracle/dreamer_oracle.py) with
the reward head replaced by decoders.py:322-362 (DenseCategoricalSupportDecoder): S logits per row on the support
`wm.decoder.reward._support`, the loss -log softmax(y)[k*] of the target's nearest support value k*, the reconstruction
and the imagined rewards the actor-critic learns from as the expectation sum_k softmax(y)_k s_k (common.py:77-86).
Pinned against the real reference by tests/golden/make_golden_catreward.py, which asserts this restatement reproduces the
reference's losses / metrics / gradients before storing the fixtures.
"""
import math

import torch
import torch.nn.functional as F

from oracle.dreamer_oracle import (cat_probs, cell_pre, draw_noise, entropy_cat, kl_cat, logavgexp, mlp,  # noqa: F401
                                   prior_logits, st_sample)

SUPPORT = "wm.decoder.reward._support"


def to_categorical(target, support):
    """decoders.py:349-352: index of the nearest support value (fp32 squared distances, first index on ties)."""
    return torch.square(target.unsqueeze(-1) - support).argmin(-1)


def support_mean(logits, support):
    """common.py:84-86 (CategoricalSupport.mean)."""
    return torch.einsum("...i,i->...", torch.softmax(logits.float(), -1), support)


def training_step(sd, conf, obs, in_state, noise, iwae_samples=None, imag_horizon=None, force=None,
                  target_synced=True):
    """Returns dict(losses, metrics, tensors, inter).  `sd` tensors that require grad receive gradients when
    the caller backwards the losses.  force (optional): dict(post_idx (T,BI,G), actor (H,N,·), prior_idx (H,N,G))
    teacher-forces the sampled indices / actions.  target_synced: critic_target == critic (first call, a2c.py:76-79)."""
    I = int(iwae_samples or conf.iwae_samples)
    H = int(imag_horizon or conf.imag_horizon)
    T, B = obs["action"].shape[:2]
    D, G, C = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete
    Z = G * C
    BI, N = B * I, T * B * I
    force = force or {}

    # ---- encoder (encoders.py:42-96): image embedding, then the vector-observation MLP's, concatenated
    image = bool(conf.image_encoder)
    embeds = []
    if image:
        x = obs["image"].reshape((T * B,) + obs["image"].shape[2:])
        e = "wm.encoder.encoder_image.model."
        for i in (0, 2, 4, 6):
            x = F.elu(F.conv2d(x, sd[e + f"{i}.weight"], sd[e + f"{i}.bias"], stride=2))
        embeds.append(x.flatten(1).reshape(T, B, -1))
    if conf.vecobs_size:
        embeds.append(mlp(sd, "wm.encoder.encoder_vecobs.model", obs["vecobs"], 2))
    embed = torch.cat(embeds, -1)

    # ---- RSSM (rssm.py:21-78)
    def expand(v):
        return v.unsqueeze(2).expand(T, B, I, v.shape[-1]).reshape(T, BI, -1)
    embeds, actions = expand(embed), expand(obs["action"])
    masks = expand((~obs["reset"]).unsqueeze(2).to(embed.dtype))
    c = "wm.core.cell."
    h, z = in_state
    posts, hs, zs, post_idx = [], [], [], []
    for t in range(T):
        h, z = h * masks[t], z * masks[t]
        h = cell_pre(sd, c, actions[t], h, z)
        y = F.linear(h, sd[c + "post_mlp_h.weight"], sd[c + "post_mlp_h.bias"]) + F.linear(embeds[t], sd[c + "post_mlp_e.weight"])
        y = F.elu(F.layer_norm(y, y.shape[-1:], sd[c + "post_norm.weight"], sd[c + "post_norm.bias"], 1e-3))
        post = F.linear(y, sd[c + "post_mlp.weight"], sd[c + "post_mlp.bias"])
        z, k = st_sample(post, noise["post"][t], G, C, force["post_idx"][t] if "post_idx" in force else None)
        posts.append(post); hs.append(h); zs.append(z); post_idx.append(k)
    posts, hs, zs = torch.stack(posts), torch.stack(hs), torch.stack(zs)
    priors = prior_logits(sd, c, hs)
    features = torch.cat((hs, zs), -1)                              # (T,BI,F)
    out_state = (h.detach(), z.detach())
    feat4 = features.reshape(T, B, I, -1)

    # ---- decoders (decoders.py:50-108)
    std = 0.3989422804
    loss_reconstr = 0
    if image:
        dm = "wm.decoder.image.model."
        y = F.linear(feat4.reshape(N, -1), sd[dm + "0.weight"], sd[dm + "0.bias"]).reshape(N, -1, 1, 1)
        for i in (2, 4, 6):
            y = F.elu(F.conv_transpose2d(y, sd[dm + f"{i}.weight"], sd[dm + f"{i}.bias"], stride=2))
        y = F.conv_transpose2d(y, sd[dm + "8.weight"], sd[dm + "8.bias"], stride=2)
        decoded = y.reshape((T, B, I) + y.shape[1:])
        target = obs["image"].unsqueeze(2).expand_as(decoded)
        loss_image_tbi = 0.5 * torch.square(decoded - target).sum(dim=[-1, -2, -3])
        loss_reconstr = conf.image_weight * loss_image_tbi
    if conf.vecobs_size:                            # DenseNormalDecoder(out_dim=K): Independent Normal, loss * var
        vec = mlp(sd, "wm.decoder.vecobs.model.model", feat4, 4)
        vt = obs["vecobs"].unsqueeze(2).expand_as(vec)
        lp = -((vt - vec) ** 2) / (2 * std ** 2) - math.log(std) - math.log(math.sqrt(2 * math.pi))
        loss_vecobs_tbi = -lp.sum(-1) * std ** 2
        loss_reconstr = loss_reconstr + conf.vecobs_weight * loss_vecobs_tbi
    sup = sd[SUPPORT]
    rlog = mlp(sd, "wm.decoder.reward.model.model", feat4, conf.reward_decoder_layers)         # (T,B,I,S)
    rt = obs["reward"].unsqueeze(2).expand(T, B, I)
    lp_r = rlog - rlog.logsumexp(-1, keepdim=True)
    loss_reward_tbi = -lp_r.gather(-1, to_categorical(rt, sup).unsqueeze(-1)).squeeze(-1)
    rew = support_mean(rlog, sup)
    term = mlp(sd, "wm.decoder.terminal.model.model", feat4, conf.terminal_decoder_layers)
    tt = obs["terminal"].unsqueeze(2).expand(T, B, I)
    loss_terminal_tbi = F.binary_cross_entropy_with_logits(term, tt, reduction="none")
    loss_reconstr = loss_reconstr + conf.reward_weight * loss_reward_tbi + conf.terminal_weight * loss_terminal_tbi

    # ---- KL (dreamer.py:328-343)
    po, pr = posts.reshape(T, B, I, Z), priors.reshape(T, B, I, Z)
    kl_exact = kl_cat(po, pr, G, C)
    if I == 1:
        kb = None if conf.kl_balance == 0.5 else conf.kl_balance
        if not kb:
            loss_kl = kl_exact
        else:
            loss_kl = (1 - kb) * kl_cat(po, pr.detach(), G, C) + kb * kl_cat(po.detach(), pr, G, C)
    else:
        kidx = torch.stack(post_idx).reshape(T, B, I, G)
        lp, _ = cat_probs(po, G, C)
        lq, _ = cat_probs(pr, G, C)
        sel = lambda l: l.gather(-1, kidx.unsqueeze(-1)).squeeze(-1).sum(-1)
        loss_kl = sel(lp) - sel(lq)
    loss_model_tbi = conf.kl_weight * loss_kl + loss_reconstr
    loss_model_tb = -logavgexp(-loss_model_tbi, dim=2)
    loss_model = loss_model_tb.mean()

    with torch.no_grad():
        m_loss_kl = -logavgexp(-kl_exact, dim=2)
        ent_prior = entropy_cat(pr, G, C).mean(dim=2)
        ent_post = entropy_cat(po, G, C).mean(dim=2)
        loss_reward_tb = -logavgexp(-loss_reward_tbi, dim=2)
        loss_terminal_tb = -logavgexp(-loss_terminal_tbi, dim=2)
        tensors = dict(loss_reward=loss_reward_tb,
                       reward_rec=rew.mean(dim=2), loss_terminal=loss_terminal_tb,
                       terminal_rec=torch.sigmoid(term).mean(dim=2), loss_kl=m_loss_kl, entropy_prior=ent_prior,
                       entropy_post=ent_post)
        metrics = dict(loss_reward=loss_reward_tb.mean(),
                       loss_terminal=loss_terminal_tb.mean(), loss_model=loss_model_tb.mean().detach(),
                       loss_kl=m_loss_kl.mean(), entropy_prior=ent_prior.mean(), entropy_post=ent_post.mean())
        if image:
            loss_image_tb = -logavgexp(-loss_image_tbi, dim=2)
            tensors.update(loss_image=loss_image_tb, image_rec=decoded.mean(dim=2))
            metrics.update(loss_image=loss_image_tb.mean())
        if conf.vecobs_size:
            loss_vecobs_tb = -logavgexp(-loss_vecobs_tbi, dim=2)
            tensors.update(loss_vecobs=loss_vecobs_tb, vecobs_rec=vec.mean(dim=2))
            metrics.update(loss_vecobs=loss_vecobs_tb.mean())

    # ---- probe (probes.py:140-150)
    loss_probe = torch.square(sd["probe_model.dummy"])

    # ---- dream (dreamer.py:188-216): world model frozen, start from detached states
    sdd = {k: v.detach() if k.startswith("wm.") else v for k, v in sd.items()}
    h, z = hs.detach().reshape(N, D), zs.detach().reshape(N, Z)
    A = conf.action_dim
    feats, acts, prior_idx = [], [], []
    AL = 4
    for i in range(H):
        f = torch.cat((h, z), -1)
        out = mlp(sdd, "ac.actor.model", f, AL)
        if "actor" in force:
            a = force["actor"][i]
        elif conf.actor_dist == "onehot":
            _, p = cat_probs(out, 1, A)
            a = F.one_hot((p.squeeze(-2) / noise["actor"][i]).argmax(-1), A).to(out.dtype)
        else:
            mu = 5 * torch.tanh(out[:, :A] / 5)
            sd_ = F.softplus(out[:, A:]) + 0.1
            a = torch.tanh(mu + sd_ * noise["actor"][i])
        a = a.detach()
        feats.append(f); acts.append(a)
        h = cell_pre(sdd, c, a, h, z)
        z, k = st_sample(prior_logits(sdd, c, h), noise["prior"][i], G, C,
                         force["prior_idx"][i] if "prior_idx" in force else None)
        prior_idx.append(k)
    feats.append(torch.cat((h, z), -1))
    feats, acts = torch.stack(feats).detach(), torch.stack(acts).detach()      # (H+1,N,F), (H,N,A)
    rewards = support_mean(mlp(sdd, "wm.decoder.reward.model.model", feats, conf.reward_decoder_layers),
                           sdd[SUPPORT].detach()).detach()
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
    if conf.actor_dist == "onehot":
        lp = out - out.logsumexp(-1, keepdim=True)
        action_logprob = (lp * F.one_hot(acts.argmax(-1), A).to(lp.dtype)).sum(-1)
        policy_entropy = -(lp.exp() * lp).sum(-1)
    else:
        mu = 5 * torch.tanh(out[..., :A] / 5)
        sd_ = F.softplus(out[..., A:]) + 0.1
        eps = torch.finfo(torch.float32).eps
        xa = torch.atanh(acts.clamp(-1 + eps, 1 - eps))
        lpn = -((xa - mu) ** 2) / (2 * sd_ ** 2) - sd_.log() - math.log(math.sqrt(2 * math.pi))
        ladj = 2.0 * (math.log(2.0) - xa - F.softplus(-2.0 * xa))
        action_logprob = (lpn - ladj).sum(-1)
        policy_entropy = (0.5 + 0.5 * math.log(2 * math.pi) + sd_.log()).sum(-1)
    if conf.actor_grad != "reinforce":
        raise NotImplementedError("oracle restates actor_grad=reinforce (dynamics asserts upstream, a2c.py:131)")
    loss_policy = -action_logprob * advantage_gae.detach()
    loss_actor = ((loss_policy - conf.entropy * policy_entropy) * reality_weight).mean()
    with torch.no_grad():
        metrics.update(loss_critic=loss_critic.detach(), loss_actor=loss_actor.detach(),
                       policy_entropy=policy_entropy.mean(), policy_value=value0[0].mean(),
                       policy_value_im=value0.mean(), policy_reward=reward1.mean(), policy_reward_std=reward1.std())
        tensors.update(policy_value=value[0].reshape(T, B, I).mean(-1).detach())
    inter = dict(embed=embed, posts=posts, priors=priors, features=features, post_idx=torch.stack(post_idx),
                 prior_idx=torch.stack(prior_idx) if prior_idx else None, dream_features=feats, dream_actions=acts,
                 rewards=rewards, terminals=terminals, value=value.detach(), value_target=value_target.detach(),
                 advantage_gae=advantage_gae.detach(), reality_weight=reality_weight.detach(), actor_out=out.detach())
    return dict(losses=(loss_model, loss_probe, loss_actor, loss_critic), out_state=out_state, metrics=metrics,
                tensors=tensors, inter=inter)


def seeded_weights(template, seed):
    """oracle/weights.py's seeded state dict with the support left at the values in `template` (the configured support
    through clip_rewards), so that targets fall into the buckets the configuration names."""
    from oracle.weights import seeded_state_dict

    sd = seeded_state_dict(template, seed)
    sd[SUPPORT] = template[SUPPORT].detach().clone()
    return sd

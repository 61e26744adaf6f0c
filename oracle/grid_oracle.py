"""TEST INFRASTRUCTURE — CPU restatement of the reference's training step on categorical grid images: the dense image
encoder (encoders.py:10-69, 99-125, with reward_input the reward and terminal planes of encoders.py:50-60) and the
categorical image decoder (decoders.py:183-254 CatImageDecoder, with image_decoder_min_prob), optionally with a vector
observation.

The RSSM, reward / terminal / vecobs heads, KL, dream and actor-critic are those of oracle/vecobs_oracle.py, restated with
its helpers and those of oracle/dreamer_oracle.py.  Pinned against the real reference by tests/golden/make_golden_grid.py,
which asserts this restatement reproduces the reference's losses / metrics / gradients before storing the fixtures.
"""
import math

import torch
import torch.nn.functional as F

from oracle.dreamer_oracle import (cat_probs, cell_pre, draw_noise, entropy_cat, kl_cat, logavgexp, mlp,  # noqa: F401
                                   prior_logits, st_sample)


def seeded_state_dict(template, seed=0, dtype=torch.float32):
    """oracle/weights.seeded_state_dict for models with the categorical image decoder: the same draws in the same order,
    with the ConvTranspose2d fan-in rule applied to 4-D weights only (the decoder's Linear layers share the conv decoder's
    key names `wm.decoder.image.model.{2,4,6,8}.weight`).  For every other model it gives the same tensors."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name in sorted(template.keys()):
        shape = tuple(template[name].shape)
        r = torch.randn(shape, generator=g)
        if name.endswith("dummy"):
            v = torch.zeros(shape)
        elif len(shape) == 1:
            v = 1.0 + 0.1 * r if name.endswith(".weight") else 0.1 * r
        else:
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            if len(shape) == 4 and "decoder.image" in name and any(f"model.{i}.weight" in name for i in (2, 4, 6, 8)):
                fan_in = shape[0] * shape[2] * shape[3] // 4
            v = r * (1.0 / max(fan_in, 1)) ** 0.5
        out[name] = v.to(dtype)
    return out


def dense_encoder(sd, conf, obs):
    """encoders.py:42-60, 99-125 -> the image embedding (T, B, 256)."""
    image = obs["image"]
    T, B, C, H, W = image.shape
    if conf.reward_input:
        plane = lambda v: v.reshape(T, B, 1, 1, 1).expand(T, B, 1, H, W).to(image.dtype)
        image = torch.cat([image, plane(obs["reward"]), plane(obs["terminal"])], -3)
    x = image.reshape(T * B, -1)
    e = "wm.encoder.encoder_image.model."
    L = max(conf.image_encoder_layers, 1)
    for l in range(L):
        x = F.linear(x, sd[e + f"{1 + 3 * l}.weight"], sd[e + f"{1 + 3 * l}.bias"])
        x = F.elu(F.layer_norm(x, x.shape[-1:], sd[e + f"{2 + 3 * l}.weight"], sd[e + f"{2 + 3 * l}.bias"], 1e-3))
    x = F.elu(F.linear(x, sd[e + f"{1 + 3 * L}.weight"], sd[e + f"{1 + 3 * L}.bias"]))
    return x.reshape(T, B, -1)


def cat_decoder_logits(sd, conf, features):
    """CatImageDecoder.forward (decoders.py:212-216): features (..., F) -> logits (..., C, H, W)."""
    y = mlp(sd, "wm.decoder.image.model", features, conf.image_decoder_layers)
    return y.reshape(features.shape[:-1] + (conf.image_channels, conf.image_size, conf.image_size))


def cat_image_loss(conf, logits, target):
    """CatImageDecoder.loss (decoders.py:218-236): per-row loss summed over the pixels; target one-hot (..., C, H, W)."""
    k = target.argmax(-3)
    if conf.image_decoder_min_prob == 0:
        lp = F.log_softmax(logits, -3)
    else:
        m = conf.image_decoder_min_prob
        lp = ((1.0 - m) * F.softmax(logits, -3) + m / logits.shape[-3]).log()
    return -lp.gather(-3, k.unsqueeze(-3)).squeeze(-3).sum([-1, -2])


def cat_image_decoded(logits):
    """decoders.py:247-250: logits (T, B, I, C, H, W) -> the decoded image (T, B, C, H, W)."""
    x = logits - logits.logsumexp(-3, keepdim=True)
    x = torch.logsumexp(x, 2)
    return x - x.logsumexp(-3, keepdim=True)


def training_step(sd, conf, obs, in_state, noise, iwae_samples=None, imag_horizon=None, force=None,
                  target_synced=True):
    """Returns dict(losses, metrics, tensors, inter) as oracle/vecobs_oracle.training_step does."""
    I = int(iwae_samples or conf.iwae_samples)
    H = int(imag_horizon or conf.imag_horizon)
    T, B = obs["action"].shape[:2]
    D, G, C = conf.deter_dim, conf.stoch_dim, conf.stoch_discrete
    Z = G * C
    BI, N = B * I, T * B * I
    force = force or {}

    # ---- encoder (encoders.py:42-69): the dense image embedding, then the vector observation's, concatenated
    embeds = [dense_encoder(sd, conf, obs)]
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
    logits = cat_decoder_logits(sd, conf, feat4)                    # (T,B,I,C,H,W)
    target = obs["image"].unsqueeze(2).expand_as(logits)
    loss_image_tbi = cat_image_loss(conf, logits, target)
    loss_reconstr = conf.image_weight * loss_image_tbi
    if conf.vecobs_size:                            # DenseNormalDecoder(out_dim=K): Independent Normal, loss * var
        vec = mlp(sd, "wm.decoder.vecobs.model.model", feat4, 4)
        vt = obs["vecobs"].unsqueeze(2).expand_as(vec)
        lp = -((vt - vec) ** 2) / (2 * std ** 2) - math.log(std) - math.log(math.sqrt(2 * math.pi))
        loss_vecobs_tbi = -lp.sum(-1) * std ** 2
        loss_reconstr = loss_reconstr + conf.vecobs_weight * loss_vecobs_tbi
    rew = mlp(sd, "wm.decoder.reward.model.model", feat4, conf.reward_decoder_layers)
    rt = obs["reward"].unsqueeze(2).expand(T, B, I)
    loss_reward_tbi = -(-((rt - rew) ** 2) / (2 * std ** 2) - math.log(std) - math.log(math.sqrt(2 * math.pi))) * std ** 2
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
        loss_image_tb = -logavgexp(-loss_image_tbi, dim=2)
        tensors = dict(loss_image=loss_image_tb, image_rec=cat_image_decoded(logits), loss_reward=loss_reward_tb,
                       reward_rec=rew.mean(dim=2), loss_terminal=loss_terminal_tb,
                       terminal_rec=torch.sigmoid(term).mean(dim=2), loss_kl=m_loss_kl, entropy_prior=ent_prior,
                       entropy_post=ent_post)
        metrics = dict(loss_image=loss_image_tb.mean(), loss_reward=loss_reward_tb.mean(),
                       loss_terminal=loss_terminal_tb.mean(), loss_model=loss_model_tb.mean().detach(),
                       loss_kl=m_loss_kl.mean(), entropy_prior=ent_prior.mean(), entropy_post=ent_post.mean())
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
                 advantage_gae=advantage_gae.detach(), reality_weight=reality_weight.detach(), actor_out=out.detach(),
                 image_logits=logits.detach())
    return dict(losses=(loss_model, loss_probe, loss_actor, loss_critic), out_state=out_state, metrics=metrics,
                tensors=tensors, inter=inter)

"""Drop-in `Dreamer` module: the reference's API (pydreamer/models/dreamer.py:19-230) over hand-written
sm_90a kernels.

What is kept from the reference contract (SURVEY.md §8 b1):
  * ctor `Dreamer(conf)` with the reference's config keys; an nn.Module whose state_dict keys and
    shapes equal the reference's, so checkpoints round-trip with an unmodified reference Dreamer;
  * `init_state`, `training_step` (same arguments, same 5-tuple, same dict keys), `init_optimizers`
    (same tuple order), `grad_clip` (same dict keys); each returned loss is backwarded separately by
    the caller exactly as train.py:184-187 does.

What is different inside: the whole step — forward AND backward — is an explicit schedule of kernels
from libpd_b200.so (no autograd tape, no torch math).  `training_step` computes the gradients of the
four losses directly into a flat fp32 gradient arena; the returned loss tensors are connected to the
parameters through a tiny autograd.Function whose backward hands those precomputed gradients over,
so `loss.backward()` in the caller works unchanged.  Parameters live in one flat arena (views), which
is what the fused optimizer and the single-bucket data-parallel all-reduce operate on.
"""
import contextlib
import os
import warnings
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

from . import ops as _ops
from .ops import ACT_ELU, ACT_NONE, SUPPORT_MAX


def kl_balance_arg(kl_balance):
    """The `balance` argument of pd_kl for a configured kl_balance.  The reference (dreamer.py:241,334) maps 0.5 to None
    and takes the plain KL whenever `not self.kl_balance`, so 0 too means the plain KL (gradient weight 1 on both sides),
    which pd_kl spells as a negative balance."""
    return -1.0 if kl_balance in (0.0, 0.5) else float(kl_balance)


LN_MAX = 1024              # widest row pd_ln_elu_fwd / pd_ln_elu_bwd normalise
CAT_MAX = 32               # most classes per group pd_cat_sample / pd_cat_st_bwd / pd_kl / pd_actor_loss_onehot take
VEC_HEAD_MAX_K = 4096      # PD_VEC_HEAD_MAX_K: the widest vector observation pd_vec_head_loss takes
IMG_CHANNELS_MAX = 16      # image channels pd_col2im_imgloss takes
CAT_IMAGE_MAX_C = 64       # PD_CAT_IMAGE_MAX_C: the most categories per pixel pd_cat_image_loss takes (2 at least)
CAT_IMAGE_MAX_P = 4096     # PD_CAT_IMAGE_MAX_P: the most pixels per image pd_cat_image_loss takes
IMAG_HORIZON_MAX = 127     # pd_gae_critic keeps the H + 1 values of a row in registers, H + 1 <= 128
AUX_T_MAX = 128            # pd_gae_critic_obs scans the T rows of the replayed sequence with the same bound, 2 <= T


def _check_imag_horizon(H):
    if H > IMAG_HORIZON_MAX:
        raise NotImplementedError(f"imag_horizon={H}: the return / advantage kernel takes at most {IMAG_HORIZON_MAX} "
                                  "imagination steps (pd_gae_critic)")


def _check_aux_length(T):
    if not 2 <= T <= AUX_T_MAX:
        raise NotImplementedError(f"aux_critic with sequences of {T} steps: the auxiliary critic's return scan takes 2 to "
                                  f"{AUX_T_MAX} (pd_gae_critic_obs)")


def _fp16_path_ok(m):
    """Dreamer._fp16_forward_ok of module `m`: the fp16-forward path runs when it is switched on and its fp16 GEMMs
    (pd_gemm_f16) can take the shape.  They read 16-byte rows at 16-byte offsets, so the row lengths and column offsets
    D, Hd, Z = G * C and F = D + Z must be multiples of 8 halves, and they contract and produce at least 8 columns
    (Z % 8 == 0 implies Z >= 8)."""
    d = m.d
    return bool(m.fp16_forward) and d.D % 8 == 0 and d.Hd % 8 == 0 and (d.G * d.C) % 8 == 0


def _persistent_sms(m, enabled):
    """The shared preamble of Dreamer._persistent_rssm_ok / _persistent_bptt_ok: the SM count a persistent RSSM kernel of
    module `m` spreads over, or None when it cannot run (switched off, or neither a GPU nor the reference op table, whose
    stand-ins assume 148 SMs)."""
    on_gpu = m._arena.is_cuda
    if not (enabled and (on_gpu or m.ops.is_reference)):
        return None
    return torch.cuda.get_device_properties(m._arena.device).multi_processor_count if on_gpu else 148


# ======================================================================================
# parameter containers (names/shapes identical to the reference's module tree)
# ======================================================================================
def _mlp_seq(in_dim, out_dim, hidden_dim, hidden_layers, layer_norm):
    """common.py:37-65"""
    if not layer_norm:
        raise NotImplementedError("layer_norm=False is outside the accelerated path (SURVEY.md §8f N4)")
    layers, dim = [], in_dim
    for _ in range(hidden_layers):
        layers += [nn.Linear(dim, hidden_dim), nn.LayerNorm(hidden_dim, eps=1e-3), nn.ELU()]
        dim = hidden_dim
    layers += [nn.Linear(dim, out_dim)]
    if out_dim == 1:
        layers += [nn.Flatten(0)]
    return nn.Sequential(*layers)


class _MLP(nn.Module):
    def __init__(self, in_dim, out_dim, hidden_dim, hidden_layers, layer_norm):
        super().__init__()
        self.in_dim, self.out_dim, self.hidden_dim, self.hidden_layers = in_dim, out_dim, hidden_dim, hidden_layers
        self.model = _mlp_seq(in_dim, out_dim, hidden_dim, hidden_layers, layer_norm)


class _DenseHead(nn.Module):
    """decoders.py:257-319 (DenseBernoulliDecoder / DenseNormalDecoder): `.model` is an MLP"""

    def __init__(self, in_dim, hidden_layers, layer_norm, hidden_dim=400, out_dim=1):
        super().__init__()
        self.model = _MLP(in_dim, out_dim, hidden_dim, hidden_layers, layer_norm)


def _clip_rewards_np(x, type_):
    """functions.py:153-160"""
    if not type_:
        return x
    with np.errstate(all="ignore"):            # log1p(-1) = -inf: refused by _SupportHead with a clearer message
        if type_ == "tanh":
            return np.tanh(x)
        if type_ == "log1p":
            return np.log1p(x)
    raise AssertionError(type_)


class _SupportHead(nn.Module):
    """decoders.py:322-336 (DenseCategoricalSupportDecoder): `.model` is an MLP with one logit per support value;
    `_support` holds the support as a parameter that is never trained (its .grad stays None)."""

    def __init__(self, in_dim, support, hidden_layers, layer_norm):
        if not isinstance(support, (list, np.ndarray)):
            raise AssertionError()                                                     # decoders.py:329
        if not 2 <= len(support) <= SUPPORT_MAX:
            raise NotImplementedError(f"reward_decoder_categorical: {len(support)} support values; the categorical reward "
                                      f"head takes 2 to {SUPPORT_MAX}")
        super().__init__()
        self.model = _MLP(in_dim, len(support), 400, hidden_layers, layer_norm)
        self._support = nn.Parameter(torch.tensor(support).to(torch.float), requires_grad=False)
        if not torch.isfinite(self._support).all():
            raise ValueError(f"reward_decoder_categorical: the support after clip_rewards is not finite: "
                             f"{self._support.tolist()}")


class _ConvEncoder(nn.Module):
    """encoders.py:72-96"""

    def __init__(self, in_channels, d):
        super().__init__()
        self.out_dim = d * 32
        self.model = nn.Sequential(nn.Conv2d(in_channels, d, 4, 2), nn.ELU(), nn.Conv2d(d, d * 2, 4, 2), nn.ELU(),
                                   nn.Conv2d(d * 2, d * 4, 4, 2), nn.ELU(), nn.Conv2d(d * 4, d * 8, 4, 2), nn.ELU(),
                                   nn.Flatten())


def _image_modules(conf):
    """"cnn" for the conv image encoder + decoder pair, "dense" for the dense encoder + categorical decoder pair of grid
    images, None for a model without image observations."""
    if conf.image_encoder == "cnn" and conf.image_decoder == "cnn":
        return "cnn"
    if conf.image_encoder == "dense" and conf.image_decoder == "dense":
        if not conf.image_categorical:
            raise NotImplementedError("image_decoder=dense is a categorical image decoder (decoders.py:183-254): it takes "
                                      "the argmax over the channels of the target as the class, so a continuous image "
                                      "(image_categorical=False) would be trained on a meaningless target")
        return "dense"
    if not conf.image_encoder and not conf.image_decoder:
        return None
    raise NotImplementedError(f"accelerated path covers image_encoder / image_decoder both cnn, both dense or both empty, "
                              f"not {conf.image_encoder!r} / {conf.image_decoder!r} (SURVEY.md §2 rows 4-5)")


class _DenseEncoder(nn.Module):
    """encoders.py:99-125: Flatten, then max(hidden_layers, 1) x (Linear, LayerNorm, ELU) and Linear + ELU to 256.  The
    Linear / LayerNorm of hidden layer l sit at model[1 + 3 l] / model[2 + 3 l], the output Linear at model[1 + 3 L]."""

    def __init__(self, in_dim, hidden_layers, layer_norm, hidden_dim=400, out_dim=256):
        super().__init__()
        if not layer_norm:
            raise NotImplementedError("layer_norm=False is outside the accelerated path (SURVEY.md §8f N4)")
        self.in_dim, self.out_dim, self.hidden_dim = in_dim, out_dim, hidden_dim
        self.hidden_layers = max(hidden_layers, 1)          # the first hidden layer is always built
        layers, dim = [nn.Flatten()], in_dim
        for _ in range(self.hidden_layers):
            layers += [nn.Linear(dim, hidden_dim), nn.LayerNorm(hidden_dim, eps=1e-3), nn.ELU()]
            dim = hidden_dim
        layers += [nn.Linear(dim, out_dim), nn.ELU()]
        self.model = nn.Sequential(*layers)


class _CatImageDecoder(nn.Module):
    """decoders.py:183-210: hidden_layers x (Linear, LayerNorm, ELU), then Linear to C*H*W logits and Unflatten (one Linear
    without hidden layers): _mlp_seq's layer indices, with `.model` the Sequential itself."""

    def __init__(self, in_dim, out_shape, hidden_layers, layer_norm, hidden_dim=400):
        super().__init__()
        self.in_dim, self.out_dim, self.hidden_dim, self.hidden_layers = in_dim, int(np.prod(out_shape)), hidden_dim, hidden_layers
        seq = _mlp_seq(in_dim, self.out_dim, hidden_dim, hidden_layers, layer_norm)
        self.model = nn.Sequential(*seq, nn.Unflatten(-1, tuple(out_shape)))


class _MultiEncoder(nn.Module):
    """encoders.py:10-69: conv or dense embedding of the image and / or an MLP embedding of the vector observation,
    concatenated image part first.  With reward_input the dense encoder also reads reward and terminal planes."""

    def __init__(self, conf):
        super().__init__()
        image = _image_modules(conf)
        if conf.reward_input and image != "dense":
            raise NotImplementedError("accelerated path covers reward_input with the dense image encoder only "
                                      "(SURVEY.md §2 row 4)")
        if not image and not conf.vecobs_size:
            raise AssertionError("Either image_encoder or vecobs_size should be set")      # encoders.py:38
        if image == "dense":
            chans = conf.image_channels + (2 if conf.reward_input else 0)          # encoders.py:15-18
            self.encoder_image = _DenseEncoder(conf.image_size * conf.image_size * chans, conf.image_encoder_layers,
                                               conf.layer_norm)
        else:
            self.encoder_image = _ConvEncoder(conf.image_channels, conf.cnn_depth) if image else None
        self.encoder_vecobs = _MLP(conf.vecobs_size, 256, 400, 2, conf.layer_norm) if conf.vecobs_size else None
        self.out_dim = ((self.encoder_image.out_dim if image else 0) +
                        (self.encoder_vecobs.out_dim if conf.vecobs_size else 0))


class _ConvDecoder(nn.Module):
    """decoders.py:111-161"""

    def __init__(self, in_dim, out_channels, d):
        super().__init__()
        self.model = nn.Sequential(nn.Linear(in_dim, d * 32), nn.Unflatten(-1, (d * 32, 1, 1)),
                                   nn.ConvTranspose2d(d * 32, d * 4, 5, 2), nn.ELU(),
                                   nn.ConvTranspose2d(d * 4, d * 2, 5, 2), nn.ELU(),
                                   nn.ConvTranspose2d(d * 2, d, 6, 2), nn.ELU(),
                                   nn.ConvTranspose2d(d, out_channels, 6, 2))


class _MultiDecoder(nn.Module):
    def __init__(self, features_dim, conf):
        super().__init__()
        image = _image_modules(conf)
        if image == "cnn" and conf.image_size != 64:
            raise NotImplementedError("conv geometry is the reference's 64x64 one (encoders.py:77-90)")
        if image == "dense":
            self.image = _CatImageDecoder(features_dim, (conf.image_channels, conf.image_size, conf.image_size),
                                          conf.image_decoder_layers, conf.layer_norm)
        else:
            self.image = _ConvDecoder(features_dim, conf.image_channels, conf.cnn_depth) if image else None
        if conf.reward_decoder_categorical:         # decoders.py:34-40: the support values are clipped like rewards
            self.reward = _SupportHead(features_dim, _clip_rewards_np(conf.reward_decoder_categorical, conf.clip_rewards),
                                       conf.reward_decoder_layers, conf.layer_norm)
        else:
            self.reward = _DenseHead(features_dim, conf.reward_decoder_layers, conf.layer_norm)
        self.terminal = _DenseHead(features_dim, conf.terminal_decoder_layers, conf.layer_norm)
        # decoders.py:66-69: DenseNormalDecoder(out_dim=vecobs_size, hidden_layers=4)
        self.vecobs = _DenseHead(features_dim, 4, conf.layer_norm, out_dim=conf.vecobs_size) if conf.vecobs_size else None


class _GRUStack(nn.Module):
    """rnn.py:40-67 (GRUCellStack, cell_type gru): num_layers cells of hidden_size / num_layers units.  Layer 0 reads the
    input, layer l > 0 the new state of layer l - 1; the state is the concatenation of the layers' states."""

    def __init__(self, input_size, hidden_size, num_layers):
        super().__init__()
        self.num_layers = num_layers
        layer_size = hidden_size // num_layers
        if layer_size * num_layers != hidden_size:
            raise AssertionError("Must be divisible")                                        # rnn.py:45
        self.layers = nn.ModuleList([nn.GRUCell(input_size, layer_size)] +
                                    [nn.GRUCell(layer_size, layer_size) for _ in range(num_layers - 1)])


class _RSSMCell(nn.Module):
    """rssm.py:96-116"""

    def __init__(self, embed_dim, action_dim, deter_dim, stoch_dim, stoch_discrete, hidden_dim, gru_layers):
        super().__init__()
        z = stoch_dim * stoch_discrete
        self.z_mlp = nn.Linear(z, hidden_dim)
        self.a_mlp = nn.Linear(action_dim, hidden_dim, bias=False)
        self.in_norm = nn.LayerNorm(hidden_dim, eps=1e-3)
        self.gru = _GRUStack(hidden_dim, deter_dim, gru_layers)
        self.prior_mlp_h = nn.Linear(deter_dim, hidden_dim)
        self.prior_norm = nn.LayerNorm(hidden_dim, eps=1e-3)
        self.prior_mlp = nn.Linear(hidden_dim, z)
        self.post_mlp_h = nn.Linear(deter_dim, hidden_dim)
        self.post_mlp_e = nn.Linear(embed_dim, hidden_dim, bias=False)
        self.post_norm = nn.LayerNorm(hidden_dim, eps=1e-3)
        self.post_mlp = nn.Linear(hidden_dim, z)


class _RSSMCore(nn.Module):
    def __init__(self, *a):
        super().__init__()
        self.cell = _RSSMCell(*a)


def _init_weights_tf2(m):
    """functions.py:81-94"""
    if type(m) in (nn.Conv2d, nn.ConvTranspose2d, nn.Linear):
        nn.init.xavier_uniform_(m.weight.data)
        if m.bias is not None:
            nn.init.zeros_(m.bias.data)
    if type(m) == nn.GRUCell:
        nn.init.xavier_uniform_(m.weight_ih.data)
        nn.init.orthogonal_(m.weight_hh.data)
        nn.init.zeros_(m.bias_ih.data)
        nn.init.zeros_(m.bias_hh.data)


class _WorldModel(nn.Module):
    """dreamer.py:232-284"""

    def __init__(self, conf):
        super().__init__()
        if not conf.stoch_discrete:
            raise NotImplementedError("Gaussian latents (stoch_discrete=0) are outside the accelerated path (§8f N4)")
        if conf.gru_type != "gru" or conf.gru_layers < 1:
            raise NotImplementedError("accelerated path covers gru_type=gru with gru_layers >= 1 (SURVEY.md §2 row 3)")
        if conf.stoch_discrete > 32 or conf.stoch_dim > 32:
            raise NotImplementedError("categorical kernels handle <= 32 groups of <= 32 classes")
        self.encoder = _MultiEncoder(conf)
        features_dim = conf.deter_dim + conf.stoch_dim * conf.stoch_discrete
        self.decoder = _MultiDecoder(features_dim, conf)
        self.core = _RSSMCore(self.encoder.out_dim, conf.action_dim, conf.deter_dim, conf.stoch_dim,
                              conf.stoch_discrete, conf.hidden_dim, conf.gru_layers)
        # dreamer.py:267-279: the auxiliary critic learns the value of the observed rewards on the posterior features; its
        # actor is built (state_dict keys) but never trained
        self.ac_aux = _ActorCritic(features_dim, conf.action_dim, conf.layer_norm, conf.actor_dist) if conf.aux_critic else None
        for m in self.modules():
            _init_weights_tf2(m)


class _ActorCritic(nn.Module):
    """a2c.py:11-41"""

    def __init__(self, in_dim, out_actions, layer_norm, actor_dist, hidden_dim=400, hidden_layers=4):
        super().__init__()
        actor_out = out_actions if actor_dist == "onehot" else 2 * out_actions
        self.actor = _MLP(in_dim, actor_out, hidden_dim, hidden_layers, layer_norm)
        self.critic = _MLP(in_dim, 1, hidden_dim, hidden_layers, layer_norm)
        self.critic_target = _MLP(in_dim, 1, hidden_dim, hidden_layers, layer_norm)
        self.critic_target.requires_grad_(False)
        self.train_steps = 0


class _NoProbeHead(nn.Module):
    """probes.py:140-150"""

    def __init__(self):
        super().__init__()
        self.dummy = nn.Parameter(torch.zeros(1), requires_grad=True)


# ======================================================================================
# loss <-> precomputed-gradient bridge
# ======================================================================================
class _AttachGrads(torch.autograd.Function):
    """Returns `value` as a differentiable scalar whose backward delivers the gradients that the kernel
    schedule already wrote into the arena group `gid` (scaled by the incoming grad_output)."""

    @staticmethod
    def forward(ctx, value, owner, gid, *params):
        ctx.owner, ctx.gid = owner, gid
        return value.clone()

    @staticmethod
    def backward(ctx, grad_out):
        ctx.owner._deliver_grads(ctx.gid, grad_out)
        return (None, None, None) + tuple(None for _ in ctx.owner._group_params[ctx.gid])


class _FusedAdamW:
    """One optimizer of the tuple `init_optimizers` returns (dreamer.py:60-71): torch.optim.AdamW
    semantics (decoupled weight_decay=0.01, eps, no amsgrad) over one contiguous arena group.

    `state_dict()` / `load_state_dict()` speak torch.optim.AdamW's own layout (per-parameter `state` keyed by the
    parameter's index in the group, `param_groups[0]['params']` = those indices), so the reference's checkpoint code
    (tools.py:171-172 save, :195-196 load) round-trips both ways with a `torch.optim.AdamW` over the reference module."""

    def __init__(self, owner, gid, lr, eps, betas=(0.9, 0.999), weight_decay=0.01):
        self.owner, self.gid = owner, gid
        self.defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                             foreach=None, capturable=False, differentiable=False, fused=None)
        self.param_groups = [dict(params=list(owner._group_params[gid]), **self.defaults)]
        self._alloc()

    def _alloc(self):
        a = self.owner._group_slice(self.gid, self.owner._arena)
        self.exp_avg = torch.zeros_like(a)
        self.exp_avg_sq = torch.zeros_like(a)
        self.step_t = torch.zeros(1, dtype=torch.int32, device=a.device)

    def zero_grad(self, set_to_none=True):
        # every training_step overwrites the gradient arena, so there is nothing to clear; the call marks the previous
        # gradients as consumed (see Dreamer._note_new_grads: accumulation over several backward passes is not supported)
        self.owner._grads_pending.discard(self.gid)
        return None

    @torch.no_grad()
    def step(self, closure=None):
        o = self.owner
        o._ensure_arena()
        p = o._group_slice(self.gid, o._arena)
        g = o._group_slice(self.gid, o._garena)
        if self.exp_avg.device != p.device:
            self._alloc()
        pg = self.param_groups[0]
        o.ops.inc(self.step_t)
        o.ops.adamw(p, g, self.exp_avg, self.exp_avg_sq, pg["lr"], pg["betas"][0], pg["betas"][1], pg["eps"],
                    pg["weight_decay"], self.step_t)
        o._weights_dirty = True
        o._grads_pending.discard(self.gid)

    def _slices(self):
        """(index, offset in the group, numel, shape) of every trained parameter of the group, in torch's parameter order.
        A non-trainable one (never given a gradient) has no optimizer state, as in torch.optim.AdamW."""
        o = self.owner
        base = o._group_range[self.gid][0]
        return [(i, o._offsets[id(p)] - base, p.numel(), p.shape) for i, p in enumerate(o._group_params[self.gid])
                if id(p) not in o._frozen]

    def state_dict(self):
        step = int(self.step_t.item())
        state = {}
        if step > 0:                                          # torch creates the per-parameter state at the first step
            for i, off, n, shape in self._slices():
                state[i] = dict(step=torch.tensor(float(step)), exp_avg=self.exp_avg[off:off + n].view(shape).clone(),
                                exp_avg_sq=self.exp_avg_sq[off:off + n].view(shape).clone())
        pg = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        pg["params"] = list(range(len(self.owner._group_params[self.gid])))
        return dict(state=state, param_groups=[pg])

    def load_state_dict(self, sd):
        st = sd["state"]
        sl = self._slices()
        ids = list(sd["param_groups"][0]["params"]) if len(sd["param_groups"]) == 1 else []
        if len(sd["param_groups"]) != 1 or len(ids) != len(self.owner._group_params[self.gid]):
            raise ValueError("loaded state dict has a different number of parameter groups / parameters")
        with torch.no_grad():
            self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_t.zero_()
            steps = set()
            for i, off, n, shape in sl:
                e = st.get(ids[i])
                if e is None:
                    continue
                if tuple(e["exp_avg"].shape) != tuple(shape):
                    raise ValueError(f"optimizer state of parameter {i} has shape {tuple(e['exp_avg'].shape)}, expected {tuple(shape)}")
                self.exp_avg[off:off + n].copy_(e["exp_avg"].reshape(-1))
                self.exp_avg_sq[off:off + n].copy_(e["exp_avg_sq"].reshape(-1))
                steps.add(int(float(e["step"])))
            if len(steps) > 1:
                raise ValueError(f"parameters of one group carry different step counts {sorted(steps)}: the fused optimizer "
                                 "keeps one counter per group")
            if steps:
                self.step_t.fill_(steps.pop())
        for k, v in sd["param_groups"][0].items():
            if k != "params":
                self.param_groups[0][k] = v


# ======================================================================================
# the module
# ======================================================================================
GROUPS = ("wm", "probe", "actor", "critic")


class Dreamer(nn.Module):

    def __init__(self, conf):
        super().__init__()
        assert conf.action_dim > 0, "Need to set action_dim to match environment"   # dreamer.py:23
        if conf.probe_model != "none":
            raise NotImplementedError("probe heads are research probes outside the hot path (SURVEY.md §2 row 9)")
        if conf.probe_gradients:
            raise NotImplementedError("probe_gradients is for the baselines (SURVEY.md §2 row 10)")
        if conf.actor_dist not in ("onehot", "tanh_normal", "normal_tanh"):
            raise NotImplementedError(f"actor_dist={conf.actor_dist}")
        if conf.actor_grad != "reinforce":
            raise NotImplementedError("actor_grad=dynamics asserts upstream at a2c.py:131 (SURVEY.md §0.5); "
                                      "the accelerated path implements reinforce")
        # hard limits of the kernels (a config past one would otherwise fail partway through its first step)
        for over, what in ((conf.hidden_dim > LN_MAX, f"hidden_dim={conf.hidden_dim}: the LayerNorm kernels take rows of at most "
                                                      f"{LN_MAX} (pd_ln_elu_fwd / pd_ln_elu_bwd)"),
                           (conf.actor_dist == "onehot" and conf.action_dim > CAT_MAX,
                            f"action_dim={conf.action_dim}: the one-hot actor samples and differentiates at most {CAT_MAX} "
                            "classes (pd_cat_sample, pd_actor_loss_onehot)"),
                           (conf.vecobs_size > VEC_HEAD_MAX_K, f"vecobs_size={conf.vecobs_size}: the vector-observation loss "
                                                               f"takes at most {VEC_HEAD_MAX_K} values (pd_vec_head_loss)"),
                           (conf.image_encoder == "cnn" and conf.image_channels > IMG_CHANNELS_MAX,
                            f"image_channels={conf.image_channels}: the image loss takes at most {IMG_CHANNELS_MAX} channels "
                            "(pd_col2im_imgloss)"),
                           (conf.image_decoder == "dense" and not 2 <= conf.image_channels <= CAT_IMAGE_MAX_C,
                            f"image_channels={conf.image_channels}: the categorical image loss takes 2 to {CAT_IMAGE_MAX_C} "
                            "categories (pd_cat_image_loss)"),
                           (conf.image_decoder == "dense" and conf.image_size ** 2 > CAT_IMAGE_MAX_P,
                            f"image_size={conf.image_size}: the categorical image loss takes at most {CAT_IMAGE_MAX_P} "
                            "pixels (pd_cat_image_loss)")):
            if over:
                raise NotImplementedError(what)
        _check_imag_horizon(conf.imag_horizon)
        if conf.aux_critic:
            _check_aux_length(conf.batch_length)
        self.conf = conf
        self.iwae_samples = conf.iwae_samples
        self.imag_horizon = conf.imag_horizon
        self.probe_gradients = conf.probe_gradients
        features_dim = conf.deter_dim + conf.stoch_dim * conf.stoch_discrete
        self.wm = _WorldModel(conf)
        self.ac = _ActorCritic(features_dim, conf.action_dim, conf.layer_norm, conf.actor_dist)
        self.probe_model = _NoProbeHead()
        # static dims
        Aout = conf.action_dim if conf.actor_dist == "onehot" else 2 * conf.action_dim
        cd, IC = conf.cnn_depth, conf.image_channels
        enc = self.wm.encoder
        rew = self.wm.decoder.reward
        self._catreward = isinstance(rew, _SupportHead)
        S = rew._support.numel() if self._catreward else 1
        # embedding = cat(image part [Ei], vecobs part [Ev]); each part has its own buffer and meets W_pe's column slice
        self.d = SimpleNamespace(D=conf.deter_dim, L=conf.gru_layers, Dl=conf.deter_dim // conf.gru_layers,  # Dl: units per GRU layer
                                 G=conf.stoch_dim, C=conf.stoch_discrete,
                                 Z=conf.stoch_dim * conf.stoch_discrete, Hd=conf.hidden_dim, E=enc.out_dim,
                                 Ei=enc.encoder_image.out_dim if enc.encoder_image is not None else 0,
                                 Ev=enc.encoder_vecobs.out_dim if enc.encoder_vecobs is not None else 0,
                                 K=conf.vecobs_size, A=conf.action_dim, F=features_dim, cd=cd, IC=IC, Aout=Aout,
                                 Ap=(Aout + 3) // 4 * 4,   # row pitch of the actor outputs: 16-byte rows keep them TMA-addressable
                                 S=S, Sp=(S + 3) // 4 * 4 if self._catreward else 1)   # reward head outputs, their row pitch
        self._image = enc.encoder_image is not None
        self._dense = isinstance(enc.encoder_image, _DenseEncoder)     # categorical grid images (dense encoder / decoder)
        self._conv = self._image and not self._dense
        self._reward_input = bool(conf.reward_input) and self._dense
        d_ = self.d
        d_.P = conf.image_size * conf.image_size if self._dense else 0    # pixels of a grid image
        d_.CP = IC * d_.P                                                   # one-hot image floats (and decoder logits) per row
        # (input size, output size, in channels, out channels) of the four 4x4 stride-2 convolutions of the encoder
        self._enc_geo = ((64, 31, IC, cd), (31, 14, cd, 2 * cd), (14, 6, 2 * cd, 4 * cd), (6, 2, 4 * cd, 8 * cd))
        # (input size, output size, kernel, in channels, out channels) of the four stride-2 deconvolutions of the decoder
        self._dec_geo = ((1, 5, 5, 32 * cd, 4 * cd), (5, 13, 5, 4 * cd, 2 * cd), (13, 30, 6, 2 * cd, cd), (30, 64, 6, cd, IC))
        self._arena = None
        self._arena_device = None
        self._ws = {}
        self._graphs = {}
        self._ops = None
        self._weights_dirty = True
        self._dp = None           # optional data-parallel reducer (pydreamer_b200.parallel)
        self._grads_pending = set()
        # nn.Module.load_state_dict copies into the arena views in place: the tf32 / fp16 shadow arenas and the re-laid
        # conv weights must be rebuilt before the next kernel reads them
        self.register_load_state_dict_post_hook(lambda module, incompatible: setattr(module, "_weights_dirty", True))
        self._build_registry()

    # ------------------------------------------------------------------ arena
    def _build_registry(self):
        self._group_params = {
            "wm": list(self.wm.parameters()),
            "probe": list(self.probe_model.parameters()),
            "actor": list(self.ac.actor.parameters()),
            "critic": list(self.ac.critic.parameters()),
            "target": list(self.ac.critic_target.parameters()),
        }
        self._names = {id(p): n for n, p in self.named_parameters()}
        # members of a trained group that never receive a gradient (the categorical reward head's support, the auxiliary
        # critic's target and its actor, whose loss the reference discards) keep their place in the group's parameter list
        # but are stored after the target critic: outside every range the optimizer, grad clipping and the data-parallel
        # all-reduce walk, so their .grad stays None and torch.optim.AdamW would keep no state for them either
        self._frozen = {id(p) for g in GROUPS for p in self._group_params[g] if not p.requires_grad}
        if self.wm.ac_aux is not None:
            self._frozen |= {id(p) for p in self.wm.ac_aux.actor.parameters()}
        off = 0
        self._offsets, self._group_range = {}, {}

        def place(p):
            nonlocal off
            self._offsets[id(p)] = off
            off += (p.numel() + 7) // 8 * 8              # every tensor 16-byte aligned in the fp32 AND the fp16 arena (TMA)

        for gname in GROUPS + ("target",):
            start = off
            for p in self._group_params[gname]:
                if id(p) not in self._frozen:
                    place(p)
            self._group_range[gname] = (start, off)
        for g in GROUPS:
            for p in self._group_params[g]:
                if id(p) in self._frozen:
                    place(p)
        self._arena_numel = off
        self._train_numel = self._group_range["critic"][1]

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._arena = None   # .to()/.cuda() re-created the tensors: re-flatten lazily
        return r

    def _ensure_arena(self):
        p0 = next(self.parameters())
        if self._arena is not None and self._arena_device == p0.device and p0.data_ptr() == self._arena.data_ptr():
            return
        dev = p0.device
        arena = torch.zeros(self._arena_numel, dtype=torch.float32, device=dev)
        garena = torch.zeros(self._train_numel, dtype=torch.float32, device=dev)
        for g in GROUPS + ("target",):
            for p in self._group_params[g]:
                o = self._offsets[id(p)]
                v = arena[o:o + p.numel()].view(p.shape)
                v.copy_(p.data)
                p.data = v
                if g != "target" and id(p) not in self._frozen:
                    p.grad = garena[o:o + p.numel()].view(p.shape)
        self._arena, self._garena, self._arena_device = arena, garena, dev
        self._sarena = torch.zeros_like(arena)     # tf32-rounded shadow of the arena (GEMM operands)
        self._harena = torch.zeros(arena.shape, dtype=torch.float16, device=dev)   # fp16 shadow (forward-only GEMMs)
        self._ws = {}
        self._graphs = {}
        self._ops = None
        self._weights_dirty = True

    def _group_slice(self, gid, arena):
        a, b = self._group_range[gid]
        return arena[a:b]

    @property
    def ops(self):
        if self._ops is None:
            self._ops = _ops.get_ops(next(self.parameters()).device)
        return self._ops

    def _view(self, arena, p):
        o = self._offsets[id(p)]
        return arena[o:o + p.numel()].view(p.shape)

    def _deliver_grads(self, gid, grad_out):
        """backward() of one of the four losses: scale the group's precomputed gradients by grad_out (a device-side
        no-op when it is exactly 1, the plain `loss.backward()` of train.py:186-187; a GradScaler under amp or any
        `(k * loss).backward()` scales them) and make sure `.grad` of its parameters points at them."""
        g = self._group_slice(gid, self._garena)
        self.ops.scale_by(g, grad_out.reshape(1).to(device=g.device, dtype=g.dtype))
        for p in self._group_params[gid]:
            if id(p) in self._frozen:
                continue
            if p.grad is None or p.grad.data_ptr() != self._view(self._garena, p).data_ptr():
                p.grad = self._view(self._garena, p)

    def _note_new_grads(self):
        """Every training_step overwrites the gradient arena (it is never accumulated into).  A caller that runs two
        training steps without an optimizer step / zero_grad in between is accumulating gradients in the reference's
        semantics; that is not supported here and is said once instead of silently training on the last micro-batch."""
        if self._grads_pending and not self._warned_accum:
            warnings.warn("pydreamer_b200: training_step overwrites the gradients of the previous call (groups "
                          f"{sorted(self._grads_pending)} were neither stepped nor zero_grad()-ed): gradient accumulation "
                          "over several training_step calls is not supported")
            self._warned_accum = True
        self._grads_pending = set(GROUPS)

    _warned_accum = False
    # forward-only layers (imagination rollout, heads on dreamed features) use fp16 tensor-core operands: the same
    # 10-bit mantissa as TF32 at twice the MMA rate and half the operand traffic; no gradient flows through them.
    fp16_forward = os.environ.get("PD_B200_FP16_FORWARD", "1") != "0"
    # The decoder's deconvolution column matrices (GEMM output -> col2im fold; written once, read once, ~4 GB per step in fp32)
    # are stored in fp16 on the fp16-forward product path: half the HBM traffic of the two kernels either side of them.
    fp16_cols = os.environ.get("PD_B200_FP16_COLS", "0") != "0"
    # conv / deconv contractions gather their operand with TMA im2col-mode loads (pd_conv_gemm) instead of materialising
    # im2col matrices: encoder layers 2-4 (forward + weight gradient), deconv layers 2-3 (input + weight gradient).
    implicit_conv = os.environ.get("PD_B200_IMPLICIT_CONV", "1") != "0"

    # ------------------------------------------------------------------ reference API
    def init_optimizers(self, lr, lr_actor=None, lr_critic=None, eps=1e-5):
        self._ensure_arena()
        return (_FusedAdamW(self, "wm", lr, eps), _FusedAdamW(self, "probe", lr, eps),
                _FusedAdamW(self, "actor", lr_actor or lr, eps), _FusedAdamW(self, "critic", lr_critic or lr, eps))

    @torch.no_grad()
    def grad_clip(self, grad_clip, grad_clip_ac=None):
        """dreamer.py:73-87: per-group clip_grad_norm_, returns the pre-clip norms."""
        self._ensure_arena()
        if self._dp is not None:
            self._dp.allreduce_grads(self)
        ws = self._buf("clip", 8)
        self.ops.fill(ws, 0.0)
        keys = []
        for i, (gid, key, mx) in enumerate((("wm", "grad_norm", grad_clip), ("probe", "grad_norm_probe", grad_clip),
                                            ("actor", "grad_norm_actor", grad_clip_ac or grad_clip),
                                            ("critic", "grad_norm_critic", grad_clip_ac or grad_clip))):
            g = self._group_slice(gid, self._garena)
            self.ops.sumsq(g, ws[i:i + 1])
            self.ops.clip_scale(g, ws[i:i + 1], mx, ws[4 + i:5 + i])
            keys.append(key)
        norms = ws[4:8].clone()                 # the caller's own copy (the workspace is rewritten by the next call)
        return {k: norms[i] for i, k in enumerate(keys)}

    def init_state(self, batch_size):
        dev = next(self.parameters()).device
        return (torch.zeros((batch_size, self.d.D), device=dev), torch.zeros((batch_size, self.d.Z), device=dev))

    @torch.no_grad()
    def inference(self, obs, in_state):
        """dreamer.py:92-111: one posterior step (T=1) + actor / critic forward for the env-interaction policy.
        Returns (action distribution, out_state, {'policy_value'}) like the reference (generator.py:321-328)."""
        import torch.distributions as D

        assert "action" in obs, "Observation should contain previous action"
        act_shape = obs["action"].shape
        assert len(act_shape) == 3 and act_shape[0] == 1, f"Expected shape (1,B,A), got {act_shape}"
        self._ensure_arena()
        self._prepare_weights()
        d, B = self.d, act_shape[1]
        noise = self._buf("inf.noise", 1, B, d.Z).exponential_()
        if getattr(self, "_test_inference_noise", None) is not None:      # tests pin the sampling noise
            noise = self._test_inference_noise
        feat = self._buf("inf.feat", 1, B, d.F)
        out_state = self._wm_features(obs, in_state, 1, B, 1, noise, "inf.", feat).out_state
        f = feat.view(B, d.F)
        alog, val = self._buf("inf.alog", B, d.Aout), self._buf("inf.val", B, 1)
        self._mlp_fwd(self._mlp_params(self.ac.actor), f, alog)
        self._mlp_fwd(self._mlp_params(self.ac.critic), f, val)
        y = alog.view(1, B, d.Aout).clone()
        if self.conf.actor_dist == "onehot":
            dist = D.OneHotCategorical(logits=y)
        elif self.conf.actor_dist == "tanh_normal":                    # functions.py:69-78
            mean = 5 * torch.tanh(y[..., :d.A] / 5)
            std = torch.nn.functional.softplus(y[..., d.A:]) + 0.1
            normal = D.independent.Independent(D.normal.Normal(mean, std), 1)
            dist = D.TransformedDistribution(normal, [D.TanhTransform()])
            dist.entropy = normal.entropy
        else:                                                          # normal_tanh, functions.py:59-66
            mean = torch.tanh(y[..., :d.A])
            std = torch.sigmoid(y[..., d.A:]) + 0.01
            dist = D.independent.Independent(D.normal.Normal(mean, std), 1)
        return dist, out_state, dict(policy_value=val.mean())

    # ------------------------------------------------------------------ workspace
    def _buf(self, name, *shape, dtype=torch.float32, zero=False):
        key = (name, shape, dtype)
        t = self._ws.get(key)
        if t is None:
            dev = self._arena.device
            t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=dev)
            self._ws[key] = t
        return t

    # ------------------------------------------------------------------ weights
    def _w(self, p):      # rounded shadow (tensor-core operand)
        return self._view(self._sarena, p)

    def _wh(self, p):     # fp16 shadow (operand of forward-only GEMMs)
        return self._view(self._harena, p)

    def _raw(self, p):    # fp32 master (biases, LayerNorm affine)
        return self._view(self._arena, p)

    def _g(self, p):
        return self._view(self._garena, p)

    def _w2d(self, p):
        return self._w(p).view(p.shape[0], -1)

    def _prepare_weights(self):
        """Per optimizer step: tf32-round the whole arena into the shadow arena (one kernel) and build the
        conv / deconv weights in GEMM layout: conv (Cout,Cin,kh,kw)->(Cout,(kh,kw,Cin)); deconv
        (Cin,Cout,kh,kw)->((kh,kw,Cout),Cin)."""
        if not self._weights_dirty:
            return
        ops = self.ops
        ops.round_copy(self._arena, self._sarena, True)
        if self._fp16_forward_ok():
            ops.to_half(self._arena.view(1, -1), self._harena.view(1, -1))
        if self._conv:
            enc = self.wm.encoder.encoder_image.model
            self._encw = []
            for li, idx in enumerate((0, 2, 4, 6)):
                w = enc[idx].weight
                if li == 0:
                    self._encw.append(self._w(w).view(w.shape[0], -1))          # (c,kh,kw) order == native
                else:
                    co, ci, kh, kw = w.shape
                    sh = self._buf(f"encw{li}", co, kh, kw, ci)
                    ops.permute4(self._w(w), sh, (0, 2, 3, 1))
                    self._encw.append(sh.view(co, kh * kw * ci))
            dec = self.wm.decoder.image.model
            self._decw = []
            for li, idx in enumerate((2, 4, 6, 8)):
                w = dec[idx].weight
                ci, co, kh, kw = w.shape
                sh = self._buf(f"decw{li}", kh, kw, co, ci)
                ops.permute4(self._w(w), sh, (2, 3, 1, 0))
                self._decw.append(sh.view(kh * kw * co, ci))
        if self.persistent_rssm:      # z_mlp^T [Z, Hd] fp16: a one-hot latent selects rows (persistent unroll, phase A)
            wz = self.wm.core.cell.z_mlp.weight
            self._k1_wzT = self._buf("k1.wzT", wz.shape[1], wz.shape[0], dtype=torch.float16)
            ops.transpose_to_half(self._raw(wz), self._k1_wzT)
            d = self.d
            if d.L > 1 and self._fp16_forward_ok():
                # a stacked GRU's recurrent weights as the block-diagonal [3D, D] fp16 matrix the persistent unroll contracts
                # (row gate * D + u: unit u's row of its layer's W_hh in that layer's columns; the zeros are never written)
                self._k1_whh = self._buf("k1.whh_bd", 3 * d.D, d.D, dtype=torch.float16, zero=True)
                for l, g_ in enumerate(self.wm.core.cell.gru.layers):
                    cl = self._gru_cols(l)
                    for gate in range(3):
                        ops.to_half(self._raw(g_.weight_hh)[gate * d.Dl:(gate + 1) * d.Dl],
                                    self._k1_whh[gate * d.D + l * d.Dl:gate * d.D + (l + 1) * d.Dl, cl])
        if self.persistent_bptt and self.d.L == 1:     # transposed fp16 copies: operands of pd_rssm_unroll_bwd (one cell)
            cell = self.wm.core.cell
            gru = cell.gru.layers[0]
            self._k1b_w = {}
            for name, wgt in (("w_pmT16", cell.post_mlp.weight), ("w_phT16", cell.post_mlp_h.weight),
                              ("w_hhT16", gru.weight_hh), ("w_ihT16", gru.weight_ih), ("w_zT16", cell.z_mlp.weight)):
                buf = self._buf("k1b." + name, wgt.shape[1], wgt.shape[0], dtype=torch.float16)
                ops.transpose_to_half(self._raw(wgt), buf)
                self._k1b_w[name] = buf
        # a_mlp^T [A, Hd]: a one-hot action selects one row (imagination rollout, pd_gather_rows)
        wa = self.wm.core.cell.a_mlp.weight
        self._waT = self._buf("waT", wa.shape[1], wa.shape[0])
        ops.permute4(self._w(wa).view(wa.shape[0], wa.shape[1], 1, 1), self._waT.view(wa.shape[1], wa.shape[0], 1, 1),
                     (1, 0, 2, 3))
        self._weights_dirty = False

    def _mlp_params(self, mlp, off=0):
        """Layers of an MLP container: hidden layer l's Linear / LayerNorm at model[off + 3 l] / model[off + 3 l + 1], the
        output Linear at model[off + 3 L] (off = 1 for the dense image encoder, whose model[0] is a Flatten)."""
        seq = mlp.model
        L = mlp.hidden_layers
        return SimpleNamespace(L=L, lin=[seq[off + 3 * l] for l in range(L)], ln=[seq[off + 3 * l + 1] for l in range(L)],
                               out=seq[off + 3 * L], hid=mlp.hidden_dim, out_dim=mlp.out_dim, in_dim=mlp.in_dim)

    # ------------------------------------------------------------------ dense layers
    def _fgemm(self, x, w, out, f16, c_zeroed=False, **kw):
        """out = x·wᵀ (+ the epilogue in kw) with fp16 operands (x in fp16 and the fp16 shadow of w: forward-only layers)
        or tf32 ones.  c_zeroed (out is pre-cleared for split-K) only concerns the tf32 GEMM."""
        if f16:
            self.ops.gemm_f16(x, self._wh(w), out, **kw)
        else:
            self.ops.gemm(x, self._w(w), out, c_zeroed=c_zeroed, **kw)

    def _head_fwd(self, layers, h, y, p, m, r, out, f16=False, p16=None, res=None, r_div=1, c_zeroed=False):
        """out = Linear(LayerNorm+ELU(Linear(h) + res)): the prior or posterior logits of the RSSM (rssm.py:108-116).
        layers = (Linear, LayerNorm, Linear); y, p, m, r receive the pre-norm input, the ELU output and the LN statistics.
        f16: fp16 operands, h in fp16 and p16 receiving the fp16 copy of p."""
        l1, ln, l2 = layers
        self._fgemm(h, l1.weight, y, f16, bias=self._raw(l1.bias), res=res, r_div=r_div, c_zeroed=c_zeroed)
        self.ops.ln_elu_fwd(y, self._raw(ln.weight), self._raw(ln.bias), 1e-3, p, m, r, p16)
        self._fgemm(p16 if f16 else p, l2.weight, out, f16, bias=self._raw(l2.bias), c_zeroed=c_zeroed)

    # ------------------------------------------------------------------ MLP forward / backward
    def _mlp_saved(self, mp, tag, rows):
        """Workspace for what an MLP forward keeps for its backward: per hidden layer the pre-norm x, the post-ELU y and the
        LayerNorm mean / rstd of `rows` rows (buffers `tag.x0`, `tag.y0`, `tag.m0`, `tag.r0`, ...)."""
        b = self._buf
        return SimpleNamespace(x=[b(f"{tag}.x{l}", rows, mp.hid) for l in range(mp.L)],
                               y=[b(f"{tag}.y{l}", rows, mp.hid) for l in range(mp.L)],
                               m=[b(f"{tag}.m{l}", rows) for l in range(mp.L)],
                               r=[b(f"{tag}.r{l}", rows) for l in range(mp.L)])

    def _mlp_fwd(self, mp, x_in, out, saved=None, row0=0, x16=None, act=ACT_NONE):
        """out[rows, out_dim] = MLP(x_in).  With `saved` (from _mlp_saved) the activations the backward needs are kept in
        its rows [row0, row0+rows); otherwise they go to scratch buffers.
        x16 (optional, fp16 copy of x_in): run the hidden-layer GEMMs with fp16 operands (forward-only use).
        act: the activation after the output layer (ELU for the dense image encoder)."""
        ops, ns = self.ops, self._scratch_ns
        rows = x_in.shape[0]
        inp, inp16 = x_in, x16
        f16 = x16 is not None
        for l in range(mp.L):
            if saved is not None:
                x, y, mean, rstd = (s[l][row0:row0 + rows] for s in (saved.x, saved.y, saved.m, saved.r))
            else:
                x = self._buf(f"{ns}mlp.sx", rows, mp.hid)
                y = self._buf(f"{ns}mlp.sy{l % 2}", rows, mp.hid)
                mean = self._buf(f"{ns}mlp.sm", rows)
                rstd = self._buf(f"{ns}mlp.sr", rows)
            y16 = self._buf(f"{ns}mlp.h16_{l % 2}", rows, mp.hid, dtype=torch.float16) if f16 else None
            self._fgemm(inp16 if f16 else inp, mp.lin[l].weight, x, f16, bias=self._raw(mp.lin[l].bias))
            ops.ln_elu_fwd(x, self._raw(mp.ln[l].weight), self._raw(mp.ln[l].bias), 1e-3, y, mean, rstd, y16)
            inp, inp16 = y, y16
        ops.gemm(inp, self._w(mp.out.weight), out, bias=self._raw(mp.out.bias), act=act)   # narrow output layer: fp32 operands

    def _mlp_bwd(self, mp, x_in, dout, saved, din=None, din_accum=False):
        """Accumulates parameter grads of the MLP from the activations its forward kept in `saved` (first rows of it);
        optionally (+)= the input gradient into din."""
        ops = self.ops
        rows = x_in.shape[0]
        sv = lambda s, l: s[l][:rows]
        ops.gemm(dout, sv(saved.y, mp.L - 1) if mp.L else x_in, self._g(mp.out.weight), a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(dout, self._g(mp.out.bias))
        if mp.L == 0:                   # a head without hidden layers: one Linear
            if din is not None:
                ops.gemm(dout, self._w(mp.out.weight), din, b_mn=True, res=din if din_accum else None)
            return
        dy = self._buf(f"{self._scratch_ns}mlp.dy", rows, mp.hid)
        dx = self._buf(f"{self._scratch_ns}mlp.dx", rows, mp.hid)
        ops.gemm(dout, self._w(mp.out.weight), dy, b_mn=True)
        for l in reversed(range(mp.L)):
            ops.ln_elu_bwd(dy, sv(saved.x, l), sv(saved.y, l), self._raw(mp.ln[l].weight), sv(saved.m, l), sv(saved.r, l),
                           dx, self._g(mp.ln[l].weight), self._g(mp.ln[l].bias), self._g(mp.lin[l].bias))
            inp = x_in if l == 0 else sv(saved.y, l - 1)
            ops.gemm(dx, inp, self._g(mp.lin[l].weight), a_mn=True, b_mn=True, accumulate=True)
            if l > 0:
                ops.gemm(dx, self._w(mp.lin[l].weight), dy, b_mn=True)
            elif din is not None:
                ops.gemm(dx, self._w(mp.lin[0].weight), din, b_mn=True, res=din if din_accum else None)

    # ------------------------------------------------------------------ noise
    def _draw_noise(self, T, BI, N, H, image_pred=False, dream_log=False, B=0):
        """Exp(1) noise for the categorical samples in the reference's consumption order (SURVEY.md App. D);
        Gaussian noise for the tanh_normal and normal_tanh actors."""
        d, dev = self.d, self._arena.device
        post = self._buf("noise.post", T, BI, d.Z).exponential_()
        actor = self._buf("noise.actor", H, N, d.A)
        actor = actor.exponential_() if self.conf.actor_dist == "onehot" else actor.normal_()
        prior = self._buf("noise.prior", H, N, d.Z).exponential_()
        out = dict(post=post, actor=actor, prior=prior)
        if image_pred:
            out["image_pred"] = self._buf("noise.image_pred", N, d.Z).exponential_()
        if dream_log:
            la = self._buf("noise.dl_actor", T - 1, B, d.A)
            out["dream_log_actor"] = la.exponential_() if self.conf.actor_dist == "onehot" else la.normal_()
            out["dream_log_prior"] = self._buf("noise.dl_prior", T - 1, B, d.Z).exponential_()
        return out

    # ------------------------------------------------------------------ training step
    def training_step(self, obs, in_state, iwae_samples=None, imag_horizon=None, do_open_loop=False,
                      do_image_pred=False, do_dream_tensors=False, noise=None):
        """dreamer.py:113-186.  `noise` (optional, tests): dict(post=(T,BI,Z) Exp(1), actor=(H,N,A),
        prior=(H,N,Z) Exp(1)) replacing the internally drawn sampling noise."""
        assert "action" in obs, "`action` required in observation"
        assert "reward" in obs, "`reward` required in observation"
        assert "reset" in obs, "`reset` required in observation"
        assert "terminal" in obs, "`terminal` required in observation"
        I = int(iwae_samples or self.iwae_samples)
        H = int(imag_horizon or self.imag_horizon)
        _check_imag_horizon(H)
        T, B = obs["action"].shape[:2]
        if self.wm.ac_aux is not None:
            _check_aux_length(T)
        self._ensure_arena()
        want_grad = torch.is_grad_enabled()
        with torch.no_grad():
            if want_grad:
                self._note_new_grads()
                self._sync_target_critic()
                self._sync_aux_target()
            flags = (bool(do_open_loop), bool(do_image_pred), bool(do_dream_tensors and self.wm.decoder.image is not None))
            if flags[0] and want_grad:
                raise NotImplementedError("do_open_loop is the evaluation branch (train.py:353-359 runs it under no_grad)")
            graphed = self.use_cuda_graph and noise is None and want_grad and self._arena.is_cuda and not any(flags)
            if graphed:
                wm_out, ac_out = self._graphed_core(obs, in_state, T, B, I, H)
            else:                                   # logging / evaluation steps (~10 % of steps) are launched eagerly
                wm_out, ac_out = self._core(obs, in_state, T, B, I, H, noise, want_grad, flags=flags)
        loss_model, loss_probe = wm_out["loss_model"], self.probe_model.dummy.detach() ** 2
        loss_actor, loss_critic = ac_out["loss_actor"], ac_out["loss_critic"]
        if want_grad:
            gp = self._group_params
            loss_model = _AttachGrads.apply(loss_model, self, "wm", *gp["wm"])
            loss_probe = _AttachGrads.apply(loss_probe, self, "probe", *gp["probe"])
            loss_actor = _AttachGrads.apply(loss_actor, self, "actor", *gp["actor"])
            loss_critic = _AttachGrads.apply(loss_critic, self, "critic", *gp["critic"])
        metrics = dict(wm_out["metrics"]); metrics.update(ac_out["metrics"])
        # the step's scalars live in reused workspace / CUDA-graph buffers: hand the caller its own copy (one small gather
        # kernel), so metrics kept across steps (train.py:204-214 accumulates them for logging) stay what they were
        keys = list(metrics)
        snap = torch.stack([metrics[k].detach().reshape(()).to(torch.float32) for k in keys])
        metrics = {k: snap[i] for i, k in enumerate(keys)}
        tensors = dict(wm_out["tensors"])
        tensors.update(policy_value=ac_out["value"][0].reshape(T, B, I).mean(-1))
        if not graphed:
            # logging / evaluation steps (the ones whose tensors train.py actually reads) return private copies; on the
            # CUDA-graph steady-state path `tensors` stay views of the step workspace, valid until the next call
            tensors = {k: v.clone() for k, v in tensors.items()}
        return (loss_model, loss_probe, loss_actor, loss_critic), wm_out["out_state"], metrics, tensors, \
            ac_out.get("dream_tensors", {})

    def _core(self, obs, in_state, T, B, I, H, noise, want_grad, force_weights=False, flags=(False, False, False)):
        """The kernel schedule of one step: weights prep, WM forward (+backward), dream, actor-critic (+backward)."""
        if force_weights:
            self._weights_dirty = True
        self._prepare_weights()
        N = T * B * I
        open_loop, image_pred, dream_log = flags
        if noise is None:
            noise = self._draw_noise(T, B * I, N, H, image_pred, dream_log, B)
        if want_grad:
            self.ops.fill(self._garena, 0.0)
        mark = self._phase_timer.mark if self._phase_timer is not None else (lambda phase: None)
        mark("prepare+noise")
        par = self._ov(1)
        ac_box = {}
        feats = self._buf("feats", H + 1, N, self.d.F)     # feats[0] = world-model features, feats[1:] = dream

        def run_ac():
            dr = self._dream(feats, N, H, noise["actor"], noise["prior"], "")
            mark("dream")
            ac_box["out"] = self._actor_critic(feats, dr, N, H, want_grad, "")
            mark("actor_critic")

        def after_features():                       # the dream needs only the (detached) posterior features
            if par:
                self._scratch_ns = "ac."
                try:
                    with self._fork(1):
                        run_ac()
                finally:
                    self._scratch_ns = ""

        wm_out, fw = self._wm_forward(obs, in_state, feats, T, B, I, noise["post"], open_loop,
                                      noise["image_pred"] if image_pred else None, after_features=after_features)
        mark("wm_forward")
        if want_grad:
            self._wm_backward(obs, fw)
        mark("wm_backward")
        if par:
            self._join(1)
            cur = torch.cuda.current_stream(self._arena.device)
            for v in ac_box["out"]["metrics"].values():       # allocated on the side stream, consumed on this one
                v.record_stream(cur)
        else:
            run_ac()
        ac_out = ac_box["out"]
        if dream_log:
            ac_out["dream_tensors"] = self._dream_for_log(obs, feats[0], T, B, I, noise["dream_log_actor"],
                                                          noise["dream_log_prior"])
        return wm_out, ac_out

    _phase_timer = None       # bench.py installs a PhaseTimer (CUDA events between the phases of one eager step)

    def _sync_target_critic(self):
        """a2c.py:76-79: copy critic -> critic_target every target_interval calls (host-side counter)."""
        ac = self.ac
        if ac.train_steps % self.conf.target_interval == 0:
            self._group_slice("target", self._arena).copy_(self._group_slice("critic", self._arena))
            self._weights_dirty = True
        ac.train_steps += 1

    def _sync_aux_target(self):
        """a2c.py:76-79 for the world model's auxiliary critic: its own counter and target_interval_aux.  Like the main
        critic's, the counter advances on steps with gradients only."""
        aux = self.wm.ac_aux
        if aux is None:
            return
        if aux.train_steps % self.conf.target_interval_aux == 0:
            for pt, pc in zip(aux.critic_target.parameters(), aux.critic.parameters()):
                self._raw(pt).copy_(self._raw(pc))
            self._weights_dirty = True
        aux.train_steps += 1

    # set PD_B200_GRAPHS=0 to launch every kernel from Python instead of replaying a captured CUDA graph
    use_cuda_graph = os.environ.get("PD_B200_GRAPHS", "1") != "0"

    # Independent parts of the step are issued on side streams (parallel branches of the captured graph), so the
    # latency-bound M=B recurrent chains share the GPU with throughput-bound work instead of idling it.  Bit mask:
    #   1  dream + actor-critic (needs only the detached features) alongside decoder / losses / world-model backward
    #   2  the h·W_hh GEMM of the next step (and its transpose in BPTT) off the per-timestep critical path
    #   4  image-decoder weight gradients alongside the input-gradient chain and BPTT
    overlap = int(os.environ.get("PD_B200_OVERLAP", "3"))
    _scratch_ns = ""          # name space of the shared MLP scratch buffers (one per concurrent branch)

    # The posterior unroll runs as ONE cooperative kernel (csrc/pd_rssm_fwd3.cu) when the shape fits its limits
    # (B*I <= 256 rows, ...); PD_B200_PERSISTENT_RSSM=0 selects the chain of 9 launches per timestep instead.
    persistent_rssm = os.environ.get("PD_B200_PERSISTENT_RSSM", "1") != "0"

    # BPTT through the posterior unroll as ONE cooperative kernel (csrc/pd_rssm_bptt.cu): opt-in with PD_B200_PERSISTENT_BPTT=1
    # (faster than the default chain of ~12 launches per timestep in the Atari and DMC steps on the H100: README, Numbers).
    persistent_bptt = os.environ.get("PD_B200_PERSISTENT_BPTT", "0") != "0"

    def _persistent_bptt_ok(self, BI):
        d, P = self.d, _persistent_sms(self, self.persistent_bptt and getattr(self, "_k1b_w", None))
        if P is None or getattr(d, "L", 1) > 1:         # the kernel contracts one GRU cell (d without L: one cell)
            return False
        Z = d.G * d.C
        ks2 = 4 if Z % 256 == 0 and P >= 4 else 1
        ks6 = 4 if (3 * d.D) % 256 == 0 and P >= 4 else 1
        R = max(1, min(4, P // d.G))
        cd = lambda a_, b_: -(-a_ // b_)
        return (BI <= min(64, P) and d.Hd <= 1024 and d.Hd % 8 == 0 and d.D % 8 == 0 and Z % 8 == 0 and d.C <= 32 and d.G <= P and
                cd(BI, R) <= 16 and cd(d.D, P) <= 16 and cd(d.Hd, P // ks2) <= 32 and cd(d.D, P // ks6) <= 64 and
                cd(d.Hd, P // ks6) <= 32)

    def _persistent_rssm_ok(self, BI):
        d = self.d
        P = _persistent_sms(self, self.persistent_rssm and _fp16_path_ok(self) and getattr(self, "_k1_wzT", None) is not None)
        if P is None:
            return False
        ks = 4 if d.D % 256 == 0 and P >= 4 else 1
        cd = lambda a_, b_: -(-a_ // b_)
        # a stacked GRU: up to 4 layers of Dl = D / L units, Dl a multiple of 8 (the fp16 TMA maps of its column slices);
        # phase B spreads one layer's units over the P CTAs (d without L: one cell)
        L, Dl = getattr(d, "L", 1), getattr(d, "Dl", d.D)
        # batch rows (B x iwae_samples) beyond one 64-row MMA operand are taken in blocks by the kernel, up to 256; at most
        # 256 latent groups (MAXG of csrc/pd_rssm_fwd3.cu)
        return (BI <= 256 and d.Hd <= 1024 and d.Hd % 8 == 0 and d.D % 8 == 0 and d.C <= 32 and d.G <= min(P, 256) and
                L <= 4 and Dl % 8 == 0 and cd(Dl, P) <= 16 and cd(d.D, P // ks) <= 64 and cd(d.Hd, P // ks) <= 32)

    def _fp16_forward_ok(self):
        # a stacked GRU's layers read and write column slices of D / L units: D / L too must be a multiple of 8 halves
        return _fp16_path_ok(self) and self.d.Dl % 8 == 0

    def _implicit_conv_ok(self):
        """The implicit-GEMM convolutions (pd_conv_gemm) run when switched on and every activation they read or write has
        16-byte rows: channel counts cnn_depth x {1, 2, 4, 8} multiples of 4 floats."""
        return self.implicit_conv and self.d.cd % 4 == 0

    def _ov(self, bit):
        # (the eager phase timer of bench.py needs one stream)
        return bool(self.overlap & bit) and self._arena.is_cuda and self._phase_timer is None

    def _side(self, k):
        key = (k, torch.cuda.current_stream(self._arena.device).cuda_stream)     # one side stream per (purpose, parent)
        st = self.__dict__.setdefault("_side_streams", {})
        if key not in st:
            st[key] = torch.cuda.Stream(device=self._arena.device)
        return st[key]

    def _fork(self, k):
        """Context manager: the block is issued on side stream k, ordered after everything issued so far."""
        s = self._side(k)
        s.wait_stream(torch.cuda.current_stream(self._arena.device))
        return torch.cuda.stream(s)

    def _join(self, k):
        torch.cuda.current_stream(self._arena.device).wait_stream(self._side(k))

    def _graphed_core(self, obs, in_state, T, B, I, H):
        """CUDA-graph replay of `_core` (the ~1 400 kernel launches of a step are issued by one cudaGraphLaunch).
        Calls 1-2 for a shape run eagerly (allocates the workspace, loads the kernels); call 3 captures."""
        key = (T, B, I, H) + tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(obs.items()))
        st = self._graphs.setdefault(key, dict(calls=0, graph=None))
        st["calls"] += 1
        if st["graph"] is None and (st["calls"] <= 2 or st.get("failed")):
            return self._core(obs, in_state, T, B, I, H, None, True)
        if st["graph"] is None:
            st["obs"] = {k: torch.empty_like(v) for k, v in obs.items()}
            st["state"] = tuple(torch.empty_like(s_) for s_ in in_state)
            for k, v in obs.items():
                st["obs"][k].copy_(v)
            for d_, s_ in zip(st["state"], in_state):
                d_.copy_(s_)
            torch.cuda.synchronize()
            try:
                g = torch.cuda.CUDAGraph()
                k0 = self.ops.launch_count()
                with torch.cuda.graph(g):
                    st["out"] = self._core(st["obs"], st["state"], T, B, I, H, None, True, force_weights=True)
                st["kernels"] = self.ops.launch_count() - k0      # kernel nodes of this library in the graph
                st["graph"] = g
            except Exception as e:                           # keep running eagerly (same kernels), say so once
                st["failed"] = True
                warnings.warn(f"pydreamer_b200: CUDA graph capture failed ({e}); continuing with eager launches")
                torch.cuda.synchronize()
                return self._core(obs, in_state, T, B, I, H, None, True)
        else:
            for k, v in obs.items():
                st["obs"][k].copy_(v, non_blocking=True)
            for d_, s_ in zip(st["state"], in_state):
                d_.copy_(s_, non_blocking=True)
        st["graph"].replay()
        wm_out, ac_out = st["out"]
        # the captured out_state lives in the graph's memory pool and every replay rewrites it; the caller keeps it as a data
        # worker's carried state (train.py:177-178, no copy), so it gets its own, as the eager path's clones are
        return dict(wm_out, out_state=tuple(s_.clone() for s_ in wm_out["out_state"])), ac_out

    # ------------------------------------------------------------------ world model forward
    def _gru_cols(self, l):
        """The units of GRU layer l in a D-wide state row (rnn.py:63, state.chunk(num_layers, -1))."""
        return slice(l * self.d.Dl, (l + 1) * self.d.Dl)

    def _rssm_head(self, prior):
        """(Linear, LayerNorm, Linear) computing the prior logits (from h) or the posterior ones (from h and the embedding)."""
        c = self.wm.core.cell
        return (c.prior_mlp_h, c.prior_norm, c.prior_mlp) if prior else (c.post_mlp_h, c.post_norm, c.post_mlp)

    def _wm_features(self, obs, in_state, T, B, I, noise_post, tag, feat, open_loop=False):
        """Encoder + posterior unroll (forward only).  `feat` (T, B*I, F) receives cat(h, z).  Returns a namespace of every
        intermediate the backward reads (workspace buffers named `tag + ...`) and the out_state."""
        ops, d = self.ops, self.d
        NB, BI = T * B, B * I
        b = lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)
        cell = self.wm.core.cell
        gru = cell.gru.layers[0]                # layer 0 (the only one of a single cell)
        ea = b("rssm.ea", NB, d.Hd)
        w_pe = self._w(cell.post_mlp_e.weight)         # [Hd, E]: columns [0, Ei) meet the image part, [Ei, E) the vecobs part
        img = embed = enc_in = denc = None
        acts, cols = [], []
        if self._dense:
            # ---- dense encoder of grid images (encoders.py:50-60, 99-125): the one-hot image rows, with reward_input
            # followed by reward and terminal planes; rows of (C+2) H W floats need not be 16-byte multiples, so the first
            # GEMM (and that layer's weight gradient) take the generic GEMM route
            ep = self._mlp_params(self.wm.encoder.encoder_image, off=1)
            img = obs["image"].reshape(NB, d.CP)
            if self._reward_input:
                enc_in = b("enc.gin", NB, (d.IC + 2) * d.P)
                ops.grid_enc_input(img.view(NB, d.IC, d.P, 1), obs["reward"].reshape(NB), obs["terminal"].reshape(NB),
                                   enc_in)
            else:
                enc_in = img
            embed = b("enc.embed", NB, d.Ei)
            denc = self._mlp_saved(ep, tag + "denc", NB)
            self._mlp_fwd(ep, enc_in, embed, denc, act=ACT_ELU)
            ops.gemm(embed, w_pe[:, :d.Ei], ea)                            # hoisted over T
        elif self._image:
            # ---- encoder (encoders.py:72-96): im2col -> tensor-core GEMM (+bias+ELU) x4, NHWC activations
            enc = self.wm.encoder.encoder_image.model
            img = obs["image"].reshape(NB, d.IC, 64, 64)
            embed = b("enc.embed", NB, d.Ei)
            x4 = img.permute(0, 2, 3, 1)
            for li, (_, hout, ci, co) in enumerate(self._enc_geo):
                act, col = b(f"enc.a{li}", NB * hout * hout, co), None
                if li > 0 and self._implicit_conv_ok():
                    ops.conv_gemm(1, x4, 4, self._encw[li], act, bias=self._raw(enc[2 * li].bias), act=ACT_ELU, round_out=True)
                else:
                    col = b(f"enc.col{li}", NB * hout * hout, 16 * ci)
                    ops.im2col(x4, 4, 1 if li == 0 else 0, col, round_out=True)
                    ops.gemm(col, self._encw[li], act, bias=self._raw(enc[2 * li].bias), act=ACT_ELU, round_out=True)
                acts.append(act)
                cols.append(col)
                x4 = act.view(NB, hout, hout, co)
            ops.permute4(x4.view(NB, 4, 8 * d.cd, 1), embed.view(NB, 8 * d.cd, 4, 1), (0, 2, 1, 3),
                         round_out=True)                                   # (h,w,c) -> reference (c,h,w) flatten
            ops.gemm(embed, w_pe[:, :d.Ei], ea)                            # hoisted over T
        vec_in = vembed = venc = None
        if d.Ev:
            # ---- vector-observation MLP (encoders.py:33-34, 64-66); its rows of K floats need not be 16-byte multiples,
            # so its first GEMM (and that layer's weight gradient) take the generic GEMM route
            vp = self._mlp_params(self.wm.encoder.encoder_vecobs)
            vec_in = obs["vecobs"].reshape(NB, d.K)
            vembed = b("enc.vembed", NB, d.Ev)
            venc = self._mlp_saved(vp, tag + "venc", NB)
            self._mlp_fwd(vp, vec_in, vembed, venc)
            ops.gemm(vembed, w_pe[:, d.Ei:], ea, res=ea if self._image else None)     # + the image part's product

        # ---- RSSM posterior unroll (rssm.py:21-78, 125-153)
        mask = b("rssm.mask", T, BI)
        ops.reset_mask(obs["reset"], I, mask)
        action = obs["action"].reshape(NB, d.A)
        aa = b("rssm.aa", NB, d.Hd); ops.gemm(action, self._w(cell.a_mlp.weight), aa)
        hin, zin = b("rssm.hin", T, BI, d.D), b("rssm.zin", T, BI, d.Z)
        ops.mask_rows(in_state[0], mask[0], hin[0]); ops.mask_rows(in_state[1], mask[0], zin[0])
        x1, za = b("rssm.x1", T, BI, d.Hd), b("rssm.za", T, BI, d.Hd)
        m1, r1 = b("rssm.m1", T, BI), b("rssm.r1", T, BI)
        gates = b("rssm.gates", T, BI, 4 * d.D)
        y2, pin = b("rssm.y2", T, BI, d.Hd), b("rssm.pin", T, BI, d.Hd)
        m2, r2 = b("rssm.m2", T, BI), b("rssm.r2", T, BI)
        post = b("rssm.post", T, BI, d.Z)
        idx = b("rssm.idx", T, BI, d.G, dtype=torch.int32)
        fw = SimpleNamespace(T=T, B=B, I=I, img=img, embed=embed, enc_act=acts, enc_col=cols, enc_in=enc_in, denc=denc,
                             vec_in=vec_in,
                             vembed=vembed, venc=venc, mask=mask, hin=hin, zin=zin, x1=x1, za=za, m1=m1, r1=r1,
                             gates=gates, y2=y2, pin=pin, m2=m2, r2=r2, post=post, idx=idx)
        head = self._rssm_head(prior=open_loop)     # open loop (rssm.py:52-53): the "posterior" is the prior, no embed
        W = self._w
        if self._persistent_rssm_ok(BI):
            try:
                # one cooperative kernel for all T steps (csrc/pd_rssm_fwd3.cu); step 0's pre-norm input is formed
                # here because the incoming z need not be one-hot
                Wh, h16 = self._wh, torch.float16
                ops.gemm(zin[0], W(cell.z_mlp.weight), x1[0], bias=self._raw(cell.z_mlp.bias), res=aa[:B], r_div=I)
                ph, pn, pm = head
                grus = cell.gru.layers
                ops.rssm_unroll_fwd(
                    dict(T=T, BI=BI, I=I, D=d.D, Hd=d.Hd, G=d.G, C=d.C, layers=d.L if d.L > 1 else 0), 1e-3,
                    w_z16=Wh(cell.z_mlp.weight), w_ih16=Wh(gru.weight_ih),
                    w_hh16=Wh(gru.weight_hh) if d.L == 1 else self._k1_whh, w_ph16=Wh(ph.weight),
                    w_ih16_l=[Wh(g_.weight_ih) for g_ in grus[1:]], b_ih_l=[self._raw(g_.bias_ih) for g_ in grus[1:]],
                    b_hh_l=[self._raw(g_.bias_hh) for g_ in grus[1:]],
                    w_pm16=Wh(pm.weight), b_z=self._raw(cell.z_mlp.bias), ln1_g=self._raw(cell.in_norm.weight),
                    ln1_b=self._raw(cell.in_norm.bias), b_ih=self._raw(gru.bias_ih), b_hh=self._raw(gru.bias_hh),
                    b_ph=self._raw(ph.bias), ln2_g=self._raw(pn.weight), ln2_b=self._raw(pn.bias), b_pm=self._raw(pm.bias),
                    aa=aa, ea=None if open_loop else ea, mask=mask, noise=noise_post, x1=x1, za=za, m1=m1, r1=r1,
                    gates=gates, feat=feat, hin=hin, zin=zin, y2=y2, pin=pin, m2=m2, r2=r2, post=post, idx=idx,
                    ws_wzT16=self._k1_wzT, ws_za16=b("k1.za16", BI, d.Hd, dtype=h16),
                    ws_h16=b("k1.h16", BI, d.D, dtype=h16), ws_pin16=b("k1.pin16", BI, d.Hd, dtype=h16),
                    ws_barrier=b("k1.bar", 16, dtype=torch.int32), ws_ghpart=b("k1.ghpart", 4, BI, 3 * d.D),
                    ws_y2part=b("k1.y2part", 4, BI, d.Hd))
                fw.out_state = (feat[T - 1, :, :d.D].clone(), feat[T - 1, :, d.D:].clone())
                return fw
            except RuntimeError as e:        # e.g. cooperative launch refused (SMs reserved by MPS / green contexts)
                warnings.warn(f"pydreamer_b200: persistent RSSM kernel unavailable ({e}); using the per-timestep chain")
                self.persistent_rssm = False

        gi, gh = b("rssm.gi", T, BI, 3 * d.D), b("rssm.gh", T, BI, 3 * d.D)
        skinny = BI <= 128                      # the per-timestep GEMMs split K and reduce into C: clear all T slices at once
        if skinny:
            for buf_ in (x1, gi, gh, y2, post):
                ops.fill(buf_, 0.0)
        par = self._ov(2)
        # GRU layer l (rnn.py:60-67) owns the units col(l) of the state rows; its gates / products are rows [l, t] of the
        # (L, T, BI, ·) views (the (T, BI, ·) buffers themselves when L = 1)
        grus, col = cell.gru.layers, self._gru_cols
        gil, ghl, gatesl = (x.view(d.L, T, BI, -1) for x in (gi, gh, gates))
        gh_gemm = lambda t, l: ops.gemm(hin[t][:, col(l)], W(grus[l].weight_hh), ghl[l, t], bias=self._raw(grus[l].bias_hh),
                                        c_zeroed=skinny)
        if par:
            with self._fork(2):
                for l in range(d.L):
                    gh_gemm(0, l)
        for t in range(T):
            last = t == T - 1
            ops.gemm(zin[t], W(cell.z_mlp.weight), x1[t], bias=self._raw(cell.z_mlp.bias), res=aa[t * B:(t + 1) * B],
                     r_div=I, c_zeroed=skinny)
            ops.ln_elu_fwd(x1[t], self._raw(cell.in_norm.weight), self._raw(cell.in_norm.bias), 1e-3, za[t], m1[t], r1[t])
            for l in range(d.L):                    # layer l > 0 reads layer l - 1's new state
                ops.gemm(za[t] if l == 0 else feat[t, :, col(l - 1)], W(grus[l].weight_ih), gil[l, t],
                         bias=self._raw(grus[l].bias_ih), c_zeroed=skinny)
                if not par:
                    gh_gemm(t, l)
                elif l == 0:
                    self._join(2)
                ops.gru_fwd(gil[l, t], ghl[l, t], hin[t][:, col(l)], feat[t, :, col(l)],
                            None if last else hin[t + 1][:, col(l)], None if last else mask[t + 1], gatesl[l, t])
                if par and not last:                # h_{t+1} of this layer is known: its W_hh product overlaps what follows
                    with self._fork(2):
                        gh_gemm(t + 1, l)
            self._head_fwd(head, feat[t, :, :d.D], y2[t], pin[t], m2[t], r2[t], post[t],
                           res=None if open_loop else ea[t * B:(t + 1) * B], r_div=1 if open_loop else I, c_zeroed=skinny)
            ops.cat_sample(post[t], noise_post[t], d.G, d.C, feat[t, :, d.D:], None if last else zin[t + 1],
                           None if last else mask[t + 1], idx[t])
        fw.out_state = (feat[T - 1, :, :d.D].clone(), feat[T - 1, :, d.D:].clone())
        return fw

    def _wm_forward(self, obs, in_state, feats, T, B, I, noise_post, open_loop=False, noise_image_pred=None,
                    after_features=None):
        """World-model forward; the posterior features go to feats[0] (N, F).  Returns the losses / metrics / tensors of the
        step and the namespace of everything _wm_backward reads."""
        ops, d, conf = self.ops, self.d, self.conf
        NB, BI = T * B, B * I
        N = NB * I
        b = self._buf
        fw = self._wm_features(obs, in_state, T, B, I, noise_post, "", feats[0].view(T, BI, d.F), open_loop)
        if after_features is not None:
            after_features()
        fw.featN = featN = feats[0]                        # (N, F)
        # batched prior (rssm.py:186-193)
        fw.yp, fw.ppin = b("rssm.yp", N, d.Hd), b("rssm.ppin", N, d.Hd)
        fw.m3, fw.r3 = b("rssm.m3", N), b("rssm.r3", N)
        prior = b("rssm.prior", N, d.Z)
        self._head_fwd(self._rssm_head(prior=True), featN[:, :d.D], fw.yp, fw.ppin, fw.m3, fw.r3, prior)

        # ---- image decoder + reward / terminal heads on the posterior features
        fw.dec = dd = self._decode_all(featN, fw.img, obs, N, NB, I, "")
        aux = self._aux_critic_fwd(obs, fw) if self.wm.ac_aux is not None else None

        # ---- KL + loss assembly (dreamer.py:328-379)
        l_kl, kl_exact = b("loss.kl", N), b("loss.klx", N)
        ent_post, ent_prior = b("loss.entq", N), b("loss.entp", N)
        fw.dpost_u, fw.dprior = b("kl.dpost", N, d.Z), b("kl.dprior", N, d.Z)
        ops.kl(fw.post.view(N, d.Z), prior, fw.idx.view(N, d.G), 0 if I == 1 else 1, kl_balance_arg(conf.kl_balance), d.G,
               d.C, l_kl, kl_exact, ent_post, ent_prior, fw.dpost_u, fw.dprior)
        fw.w, tb = b("loss.w", N), b("loss.tb", NB, 8)
        vec = dict(l_vec=dd.l_vec, w_vec=conf.vecobs_weight) if d.K else {}
        ops.wm_loss(NB, I, conf.kl_weight, conf.image_weight, conf.reward_weight, conf.terminal_weight, dd.l_img, dd.l_rew,
                    dd.l_term, l_kl, kl_exact, ent_prior, ent_post, fw.w, tb, **vec)
        means = b("loss.means", 8)
        ops.colmean(tb, means)
        tbv = tb.view(T, B, 8)
        metrics = dict(loss_image=means[1]) if self._image else {}
        metrics.update(loss_reward=means[2], loss_terminal=means[3], loss_model=means[0],
                       loss_kl=means[4], entropy_prior=means[5], entropy_post=means[6])
        tensors = dict(loss_image=tbv[..., 1], image_rec=self._image_out(dd, T, B, I)) if self._image else {}
        tensors.update(loss_reward=tbv[..., 2], reward_rec=self._sel(dd.rec_r, T, B, I), loss_terminal=tbv[..., 3],
                       terminal_rec=self._sel(dd.rec_t, T, B, I), loss_kl=tbv[..., 4], entropy_prior=tbv[..., 5],
                       entropy_post=tbv[..., 6])
        if d.K:
            metrics.update(loss_vecobs=means[7])
            tensors.update(loss_vecobs=tbv[..., 7], vecobs_rec=self._sel(dd.yv, T, B, I))
        loss_model = means[0]
        if aux is not None:                 # dreamer.py:351-365, 369: loss_model stays the metric, the aux term joins the loss
            loss_model = loss_model + conf.aux_critic_weight * aux["loss"]
            metrics.update(loss_critic_aux=aux["loss"], policy_value_aux=aux["value_mean"])
            tensors.update(policy_value_aux=aux["value"])
        if noise_image_pred is not None:
            self._image_pred(obs, fw, prior, noise_image_pred, metrics, tensors)
        return dict(loss_model=loss_model, out_state=fw.out_state, metrics=metrics, tensors=tensors), fw

    def _aux_critic_fwd(self, obs, fw):
        """a2c.py:81-116 for the auxiliary critic (dreamer.py:347-365): the target critic and the critic on the posterior
        features of importance sample 0 (rows t*B*I + b*I of featN, a strided view), then the return scan over the observed
        rewards and terminals.  Keeps in fw what _wm_backward reads: the critic's activations and dv = aux_critic_weight *
        d loss_critic_aux / d value[:-1]."""
        ops, conf, b = self.ops, self.conf, self._buf
        T, B, I = fw.T, fw.B, fw.I
        aux = self.wm.ac_aux
        cp = self._mlp_params(aux.critic)
        x = fw.featN[::I]                                          # (T*B, F)
        vt, v = b("aux.vt", T * B, 1), b("aux.v", T * B, 1)
        fw.aux_critic = self._mlp_saved(cp, "aux.critic", T * B)
        self._mlp_fwd(self._mlp_params(aux.critic_target), x, vt)
        self._mlp_fwd(cp, x, v, fw.aux_critic)
        fw.aux_dv = b("aux.dv", (T - 1) * B, 1)
        sums = b("aux.sums", 2, dtype=torch.float64)
        ops.fill(sums.view(torch.float32), 0.0)
        ops.gae_critic_obs(T, B, conf.gamma_aux, conf.lambda_gae_aux, vt, v, obs["reward"].reshape(T * B),
                           obs["terminal"].reshape(T * B), conf.aux_critic_weight, fw.aux_dv, sums)
        hb = float((T - 1) * B)
        return dict(loss=(sums[0] / hb).to(torch.float32), value_mean=(sums[1] / hb).to(torch.float32), value=v.view(T, B))

    def _image_out(self, dd, T, B, I):
        """The decoded image (T, B, C, H, W) of a _decode_all namespace: the conv decoder's output averaged over the importance
        samples, or the categorical decoder's normalised log-probabilities aggregated over them (decoders.py:247-250)."""
        if self._dense:
            s = self.conf.image_size
            return dd.rec.view(T, B, self.d.IC, s, s)
        return self._sel(dd.image, T, B, I)

    @staticmethod
    def _sel(x, T, B, I):
        """Per-row values (T*B*I, ...) -> (T, B, ...): the value itself, or with importance samples their mean."""
        x = x.view(T, B, I, *x.shape[1:])
        return x[:, :, 0] if I == 1 else x.mean(2)

    def _image_pred(self, obs, fw, prior, noise, metrics, tensors):
        """dreamer.py:383-394: decode from a PRIOR sample (what the model predicts before seeing the observation);
        reports the reconstruction losses as logprob_* and the decoded tensors as *_pred.  Logging branch."""
        ops, d, b = self.ops, self.d, self._buf
        T, B, I = fw.T, fw.B, fw.I
        NB, N = T * B, T * B * I
        featP = b("p.feat", N, d.F)
        featP[:, :d.D].copy_(fw.featN[:, :d.D])
        ops.cat_sample(prior, noise, d.G, d.C, featP[:, d.D:])
        dd = self._decode_all(featP, fw.img, obs, N, NB, I, "p.")
        zeros = b("p.zeros", N, zero=True)
        w, tb = b("p.loss.w", N), b("p.loss.tb", NB, 8)
        vec = dict(l_vec=dd.l_vec, w_vec=1.0) if d.K else {}
        ops.wm_loss(NB, I, 0.0, 1.0, 1.0, 1.0, dd.l_img, dd.l_rew, dd.l_term, zeros, zeros, zeros, zeros, w, tb, **vec)
        tbv = tb.view(T, B, 8)
        lp_img, lp_rew, lp_term = tbv[..., 1], tbv[..., 2], tbv[..., 3]
        nanmean = lambda x: torch.nansum(x) / (~torch.isnan(x)).sum()                # functions.py:150-151
        extra_t = {}
        if self._catreward:                                                          # decoders.py:85-92: per support bucket
            kr = dd.kr.view(T, B, I)[:, :, 0]
            for i in range(d.S):
                m = kr == i
                extra_t[f"logprob_reward{i}"] = lp_rew * m / m
        else:
            for sig in (-1, 1):                                                      # decoders.py:96-101
                m = torch.sign(obs["reward"]) == sig
                extra_t[f"logprob_reward{sig}"] = lp_rew * m / m
        m = obs["terminal"] > 0                                                      # decoders.py:103-106
        extra_t["logprob_terminal1"] = lp_term * m / m
        if self._image:
            metrics.update(logprob_image=lp_img.mean())
            tensors.update(logprob_image=lp_img, image_pred=self._image_out(dd, T, B, I))
        metrics.update(logprob_reward=lp_rew.mean(), logprob_terminal=lp_term.mean(),
                       **{k: nanmean(v) for k, v in extra_t.items()})
        tensors.update(logprob_reward=lp_rew, logprob_terminal=lp_term, **extra_t,
                       reward_pred=self._sel(dd.rec_r, T, B, I), terminal_pred=self._sel(dd.rec_t, T, B, I))
        if d.K:
            lp_vec = tbv[..., 7]
            metrics.update(logprob_vecobs=lp_vec.mean())
            tensors.update(logprob_vecobs=lp_vec, vecobs_pred=self._sel(dd.yv, T, B, I))

    def _cols_dtype(self, ncols):
        """Column matrices of the transposed convolutions are written once and read once: fp16 halves that traffic.  The GEMM's
        fp16 TMA store needs 16-byte rows (ncols % 8 == 0); the last layer (k*k*3 columns) stays fp32."""
        return torch.float16 if (self._fp16_forward_ok() and self.fp16_cols and ncols % 8 == 0) else torch.float32

    def _image_decoder(self, featN, N, tag, img=None, I=1):
        """ConvDecoder forward (decoders.py:111-161) on features (N,F): Linear, then each deconvolution as a GEMM into column
        form + a col2im gather with bias (+ELU).  Given the target images `img` (each the target of I feature rows), the last
        gather also computes the image loss and its gradient seeds; without, it writes the decoded image."""
        ops, d = self.ops, self.d
        b = lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)
        dec = self.wm.decoder.image.model
        x0 = b("dec.x0", N, 32 * d.cd)
        ops.gemm(featN, self._w(dec[0].weight), x0, bias=self._raw(dec[0].bias), round_out=True)
        out = SimpleNamespace(xin=[x0], image=b("dec.image", N, d.IC, 64, 64))     # xin[li]: (rows, ci) input of deconv li
        for li, (hi, ho, k, ci, co) in enumerate(self._dec_geo):
            cols = b(f"dec.cols{li}", N * hi * hi, k * k * co, dtype=self._cols_dtype(k * k * co))
            ops.gemm(out.xin[li], self._decw[li], cols)
            bias = self._raw(dec[2 + 2 * li].bias)
            if li < 3:
                a = b(f"dec.d{li}", N, ho, ho, co)
                ops.col2im(cols, hi, hi, k, bias, ACT_ELU, a, round_out=True)
                out.xin.append(a.view(N * ho * ho, co))
            elif img is not None:
                out.diff, out.l_img, out.csum = b("dec.diff", N, d.IC, 64, 64), b("loss.img", N), b("dec.csum", N, d.IC)
                ops.col2im_imgloss(cols, N, hi, hi, d.IC, k, bias, img, I, out.image, out.diff, out.l_img, out.csum)
            else:
                ops.col2im(cols, hi, hi, k, bias, ACT_NONE, out.image.permute(0, 2, 3, 1), round_out=False)
        return out

    def _cat_image_decoder(self, featN, N, tag, img, I):
        """CatImageDecoder.training_step forward (decoders.py:183-254) on features (N,F): the MLP to C*H*W logits, then the
        per-row loss, its gradient seed and the decoded image of each (t, b) (pd_cat_image_loss against the one-hot target
        rows `img` (N / I, C*H*W))."""
        d = self.d
        b = lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)
        dp = self._mlp_params(self.wm.decoder.image)
        out = SimpleNamespace(logits=b("gdec.y", N, d.CP), mlp=self._mlp_saved(dp, tag + "gdec", N))
        self._mlp_fwd(dp, featN, out.logits, out.mlp)
        out.l_img, out.diff, out.rec = b("loss.img", N), b("gdec.dy", N, d.CP), b("gdec.rec", N // I, d.CP)
        self.ops.cat_image_loss(out.logits, d.IC, img, I, self.conf.image_decoder_min_prob, out.l_img, out.diff, out.rec)
        return out

    def _decode_all(self, featN, img, obs, N, NB, I, tag):
        """MultiDecoder.training_step forward (decoders.py:50-108) on features (N,F): the image decoder with its loss and the
        reward / terminal MLP heads with theirs.  Buffers are named `tag + ...` (tag "" = the training pass the backward
        reads); returns the image decoder's namespace extended by the heads'."""
        ops, d = self.ops, self.d
        b = lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)
        if self._dense:
            dd = self._cat_image_decoder(featN, N, tag, img, I)
        else:
            dd = self._image_decoder(featN, N, tag, img, I) if self._image else SimpleNamespace(l_img=None)
        # reward / terminal heads (decoders.py:257-319)
        rp, tp = self._mlp_params(self.wm.decoder.reward.model), self._mlp_params(self.wm.decoder.terminal.model)
        yr, yt = b("head.yr", N, d.Sp)[:, :d.S], b("head.yt", N, 1)     # reward logits: S per row at pitch Sp
        dd.rew, dd.term = self._mlp_saved(rp, tag + "rew", N), self._mlp_saved(tp, tag + "term", N)
        self._mlp_fwd(rp, featN, yr, dd.rew)
        self._mlp_fwd(tp, featN, yt, dd.term)
        dd.l_rew, dd.dyr, dd.rec_r = b("loss.rew", N), b("head.dyr", N, d.Sp)[:, :d.S], b("head.rec_r", N)
        dd.l_term, dd.dyt, dd.rec_t = b("loss.term", N), b("head.dyt", N, 1), b("head.rec_t", N)
        if self._catreward:                  # decoders.py:338-362; dd.kr: each row's target bucket (logging masks)
            dd.kr = b("head.kr", N, dtype=torch.int32)
            ops.support_head(yr, self._raw(self.wm.decoder.reward._support), obs["reward"].reshape(NB), I, dd.rec_r,
                             dd.l_rew, dd.dyr, dd.kr)
        else:
            ops.scalar_head_loss(0, yr, obs["reward"].reshape(NB), I, dd.l_rew, dd.dyr, dd.rec_r)
        ops.scalar_head_loss(1, yt, obs["terminal"].reshape(NB), I, dd.l_term, dd.dyt, dd.rec_t)
        if d.K:                              # vector-observation head (decoders.py:66-69, 290-319)
            vp = self._mlp_params(self.wm.decoder.vecobs.model)
            dd.yv, dd.vec = b("head.yv", N, d.K), self._mlp_saved(vp, tag + "vec", N)
            self._mlp_fwd(vp, featN, dd.yv, dd.vec)
            dd.l_vec, dd.dyv = b("loss.vec", N), b("head.dyv", N, d.K)
            ops.vec_head_loss(dd.yv, obs["vecobs"].reshape(NB, d.K), I, dd.l_vec, dd.dyv)
        return dd

    # ------------------------------------------------------------------ world model backward
    def _wm_backward(self, obs, fw):
        """Gradients of the world-model loss into the arena, from the intermediates `fw` that _wm_forward returned."""
        ops, d, conf = self.ops, self.d, self.conf
        T, B, I = fw.T, fw.B, fw.I
        NB, BI = T * B, B * I
        N = NB * I
        b, W, G = self._buf, self._w, self._g
        cell = self.wm.core.cell
        featN, w, dd = fw.featN, fw.w, fw.dec
        dfeat = b("bwd.dfeat", N, d.F)
        par_w = self._conv and self._ov(4)      # image weight gradients leave the dfeat -> BPTT critical path (joined at the end)
        if self._dense:                         # categorical image decoder: the first writer of dfeat
            ops.rowscale(dd.diff, w, 1, conf.image_weight)
            self._mlp_bwd(self._mlp_params(self.wm.decoder.image), featN, dd.diff, dd.mlp, din=dfeat)
        elif self._image:
            self._image_decoder_bwd(fw, dfeat, par_w)

        # ---- reward / terminal heads (without an image decoder the reward head is the first writer of dfeat)
        rp, tp = self._mlp_params(self.wm.decoder.reward.model), self._mlp_params(self.wm.decoder.terminal.model)
        ops.rowscale(dd.dyr, w, 1, conf.reward_weight)
        ops.rowscale(dd.dyt, w, 1, conf.terminal_weight)
        self._mlp_bwd(rp, featN, dd.dyr, dd.rew, din=dfeat, din_accum=self._image)
        self._mlp_bwd(tp, featN, dd.dyt, dd.term, din=dfeat, din_accum=True)
        if d.K:
            ops.rowscale(dd.dyv, w, 1, conf.vecobs_weight)
            self._mlp_bwd(self._mlp_params(self.wm.decoder.vecobs.model), featN, dd.dyv, dd.vec, din=dfeat, din_accum=True)
        if self.wm.ac_aux is not None:      # auxiliary critic: into the sample-0 rows of the first T-1 steps
            rows = (T - 1) * B
            self._mlp_bwd(self._mlp_params(self.wm.ac_aux.critic), featN[::I][:rows], fw.aux_dv, fw.aux_critic,
                          din=dfeat[::I][:rows], din_accum=True)

        # ---- prior branch (batch_prior): dprior = kl_weight * w[n] * dKL/dprior
        dprior = fw.dprior
        ops.rowscale(dprior, w, 1, conf.kl_weight)
        dpp, dyp = b("bwd.dpp", N, d.Hd), b("bwd.dyp", N, d.Hd)
        ops.gemm(dprior, fw.ppin, G(cell.prior_mlp.weight), a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(dprior, G(cell.prior_mlp.bias))
        ops.gemm(dprior, W(cell.prior_mlp.weight), dpp, b_mn=True)
        ops.ln_elu_bwd(dpp, fw.yp, fw.ppin, self._raw(cell.prior_norm.weight), fw.m3, fw.r3, dyp,
                       G(cell.prior_norm.weight), G(cell.prior_norm.bias), G(cell.prior_mlp_h.bias))
        ops.gemm(dyp, featN[:, :d.D], G(cell.prior_mlp_h.weight), a_mn=True, b_mn=True, accumulate=True)
        ops.gemm(dyp, W(cell.prior_mlp_h.weight), dfeat[:, :d.D], b_mn=True, res=dfeat[:, :d.D])

        # ---- BPTT through the posterior unroll
        dfeat3 = dfeat.view(T, BI, d.F)
        mask, post, pin, y2, m2, r2 = fw.mask, fw.post, fw.pin, fw.y2, fw.m2, fw.r2
        x1, za, m1, r1, gates, hin, zin = fw.x1, fw.za, fw.m1, fw.r1, fw.gates, fw.hin, fw.zin
        dpost_u = fw.dpost_u.view(T, BI, d.Z)
        w3 = w.view(T, BI)
        dpost = b("bwd.dpost", T, BI, d.Z)
        dy2, dx1 = b("bwd.dy2", T, BI, d.Hd), b("bwd.dx1", T, BI, d.Hd)
        dgi, dgh = b("bwd.dgi", T, BI, 3 * d.D), b("bwd.dgh", T, BI, 3 * d.D)
        dpin, dza = b("bwd.dpin", T, BI, d.Hd), b("bwd.dza", T, BI, d.Hd)
        dhp, dhc = b("bwd.dhp", T, BI, d.D), b("bwd.dhc", BI, d.D)
        dhin, dzin = b("bwd.dhin", T, BI, d.D), b("bwd.dzin", T, BI, d.Z)
        grus, col = cell.gru.layers, self._gru_cols
        gatesl, dgil, dghl = (x.view(d.L, T, BI, -1) for x in (gates, dgi, dgh))
        done = False
        if self._persistent_bptt_ok(BI):
            try:
                ops.rssm_unroll_bwd(
                    dict(T=T, BI=BI, D=d.D, Hd=d.Hd, G=d.G, C=d.C), conf.kl_weight, True,
                    ln2_g=self._raw(cell.post_norm.weight), ln1_g=self._raw(cell.in_norm.weight), post=post, pin=pin, y2=y2,
                    m2=m2, r2=r2, x1=x1, za=za, m1=m1, r1=r1, gates=gates, hin=hin, mask=mask, dfeat=dfeat3,
                    dpost_u=dpost_u, w=w3, dpost=dpost, dy2=dy2, dgi=dgi, dgh=dgh, dx1=dx1,
                    g_ln2_g=G(cell.post_norm.weight), g_ln2_b=G(cell.post_norm.bias), g_b_ph=G(cell.post_mlp_h.bias),
                    g_ln1_g=G(cell.in_norm.weight), g_ln1_b=G(cell.in_norm.bias), g_b_z=G(cell.z_mlp.bias),
                    ws_part2=b("k1b.part2", 4, BI, d.Hd), ws_part6=b("k1b.part6", 4, BI, d.D),
                    ws_part7=b("k1b.part7", 4, BI, d.Hd), ws_barrier=b("k1b.bar", 16, dtype=torch.int32), **self._k1b_w)
                done = True
            except RuntimeError as e:        # e.g. cooperative launch refused
                warnings.warn(f"pydreamer_b200: persistent BPTT kernel unavailable ({e}); using the per-timestep chain")
                self.persistent_bptt = False
        par = self._ov(2) and not done
        for t in (() if done else reversed(range(T))):
            nxt = t < T - 1
            ops.cat_st_bwd(post[t], d.G, d.C, dfeat3[t, :, d.D:], dzin[t + 1] if nxt else None,
                           mask[t + 1] if nxt else None, dpost_u[t], w3[t], conf.kl_weight, dpost[t])
            ops.gemm(dpost[t], W(cell.post_mlp.weight), dpin[t], b_mn=True)
            ops.ln_elu_bwd(dpin[t], y2[t], pin[t], self._raw(cell.post_norm.weight), m2[t], r2[t], dy2[t],
                           G(cell.post_norm.weight), G(cell.post_norm.bias), G(cell.post_mlp_h.bias))
            ops.gemm(dy2[t], W(cell.post_mlp_h.weight), dhp[t], b_mn=True, res=dfeat3[t, :, :d.D])
            if par and nxt:
                self._join(2)                       # dhin[t + 1]
            for l in reversed(range(d.L)):          # layer l's input gradient joins layer l - 1's output gradient
                c = col(l)
                ops.gru_bwd(dhp[t][:, c], dhin[t + 1][:, c] if nxt else None, mask[t + 1] if nxt else None, gatesl[l, t],
                            hin[t][:, c], dgil[l, t], dghl[l, t], dhc[:, c])
                with self._fork(2) if par else contextlib.nullcontext():
                    ops.gemm(dghl[l, t], W(grus[l].weight_hh), dhin[t][:, c], b_mn=True, res=dhc[:, c])
                if l > 0:
                    dx = dhp[t][:, col(l - 1)]
                    ops.gemm(dgil[l, t], W(grus[l].weight_ih), dx, b_mn=True, res=dx)
                else:
                    ops.gemm(dgil[0, t], W(grus[0].weight_ih), dza[t], b_mn=True)
            ops.ln_elu_bwd(dza[t], x1[t], za[t], self._raw(cell.in_norm.weight), m1[t], r1[t], dx1[t],
                           G(cell.in_norm.weight), G(cell.in_norm.bias), G(cell.z_mlp.bias))
            ops.gemm(dx1[t], W(cell.z_mlp.weight), dzin[t], b_mn=True)
        if par:
            self._join(2)
        # batched weight gradients over all T*BI rows
        f2 = lambda x: x.view(N, x.shape[-1])
        ops.gemm(f2(dpost), f2(pin), G(cell.post_mlp.weight), a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(f2(dpost), G(cell.post_mlp.bias))
        ops.gemm(f2(dy2), featN[:, :d.D], G(cell.post_mlp_h.weight), a_mn=True, b_mn=True, accumulate=True)
        for l, g_ in enumerate(grus):               # layer l's rows of dgi / dgh, its column slices of hin / h'
            ops.gemm(dghl[l].reshape(N, -1), f2(hin)[:, col(l)], G(g_.weight_hh), a_mn=True, b_mn=True, accumulate=True)
            ops.colsum(dghl[l].reshape(N, -1), G(g_.bias_hh))
            ops.gemm(dgil[l].reshape(N, -1), f2(za) if l == 0 else featN[:, col(l - 1)], G(g_.weight_ih), a_mn=True,
                     b_mn=True, accumulate=True)
            ops.colsum(dgil[l].reshape(N, -1), G(g_.bias_ih))
        ops.gemm(f2(dx1), f2(zin), G(cell.z_mlp.weight), a_mn=True, b_mn=True, accumulate=True)
        if I == 1:
            dea, daa = f2(dy2), f2(dx1)
        else:
            dea, daa = b("bwd.dea", NB, d.Hd), b("bwd.daa", NB, d.Hd)
            ops.group_sum(f2(dy2), I, dea); ops.group_sum(f2(dx1), I, daa)
        g_pe, w_pe = G(cell.post_mlp_e.weight), W(cell.post_mlp_e.weight)     # [Hd, E]: image columns, then vecobs columns
        if self._image:
            ops.gemm(dea, fw.embed, g_pe[:, :d.Ei], a_mn=True, b_mn=True, accumulate=True)
        if d.Ev:
            ops.gemm(dea, fw.vembed, g_pe[:, d.Ei:], a_mn=True, b_mn=True, accumulate=True)
        ops.gemm(daa, obs["action"].reshape(NB, d.A), G(cell.a_mlp.weight), a_mn=True, b_mn=True, accumulate=True)

        # ---- encoder backward
        if self._dense:
            dea_c = self._dea_c(fw, dy2)
            dembed = b("bwd.dembed", NB, d.Ei)
            # through the encoder's output ELU in the GEMM epilogue (its bias gradient: _mlp_bwd)
            ops.gemm_actbwd(dea_c, w_pe[:, :d.Ei], dembed, fw.embed, None, b_mn=True)
            self._mlp_bwd(self._mlp_params(self.wm.encoder.encoder_image, off=1), fw.enc_in, dembed, fw.denc)
        else:
            dea_c = self._image_encoder_bwd(fw, dy2, w_pe[:, :d.Ei]) if self._image else self._dea_c(fw, dy2)
        if d.Ev:
            dembed_v = b("bwd.dembed_v", NB, d.Ev)
            ops.gemm(dea_c, w_pe[:, d.Ei:], dembed_v, b_mn=True)
            self._mlp_bwd(self._mlp_params(self.wm.encoder.encoder_vecobs), fw.vec_in, dembed_v, fw.venc)
        if par_w:
            self._join(4)

    def _dea_c(self, fw, dy2):
        """Gradient of the hoisted embedding product ea [T*B, Hd]: dy2 summed over the importance samples."""
        if fw.I == 1:
            return dy2.view(-1, self.d.Hd)
        dea_c = self._buf("bwd.dea_c", fw.T * fw.B, self.d.Hd)
        self.ops.group_sum(dy2.view(-1, self.d.Hd), fw.I, dea_c)
        return dea_c

    def _image_encoder_bwd(self, fw, dy2, w_pe_img):
        """ConvEncoder backward through W_pe's image columns; returns the gradient of ea (_dea_c) it started from."""
        ops, d = self.ops, self.d
        NB = fw.T * fw.B
        b, G = self._buf, self._g
        enc = self.wm.encoder.encoder_image.model
        geo = self._enc_geo
        implicit = self._implicit_conv_ok()
        cpad = [(ci + 31) // 32 * 32 if implicit else ci for _, _, ci, _ in geo]   # implicit: 32 channels per tap
        encgw = {li: b(("bwd.gencwp" if implicit else "bwd.gencw") + str(li), geo[li][3], 16 * cpad[li])
                 for li in (1, 2, 3)}
        for li in (1, 2, 3):
            ops.fill(encgw[li], 0.0)
        dea_c = self._dea_c(fw, dy2)
        dembed = b("bwd.dembed", NB, d.Ei)
        ops.gemm(dea_c, w_pe_img, dembed, b_mn=True)
        da = b("bwd.da3", NB * 4, 8 * d.cd)
        ops.permute4(dembed.view(NB, 8 * d.cd, 4, 1), da.view(NB, 4, 8 * d.cd, 1), (0, 2, 1, 3))
        ops.bias_act_bwd(da, fw.enc_act[3], ACT_ELU, G(enc[6].bias))
        for li in (3, 2, 1):                # (the ELU / bias of layers 2..0: done by the col2im that produced their gradient)
            hin_, hout, ci, co = geo[li]
            act_prev = fw.enc_act[li - 1]
            if implicit:
                ops.conv_gemm(3, act_prev.view(NB, hin_, hin_, ci), 4, da, encgw[li])
            else:
                ops.gemm(da, fw.enc_col[li], encgw[li], a_mn=True, b_mn=True, accumulate=True)
            dcol = b(f"bwd.dcol{li}", NB * hout * hout, 16 * ci)
            ops.gemm(da, self._encw[li], dcol, b_mn=True)
            da_prev = b(f"bwd.da{li - 1}", NB * hin_ * hin_, ci)
            # fold the column-form gradient back AND go through the ELU / bias of the layer below in the same pass
            ops.col2im_actbwd(dcol, hout, hout, 4, act_prev, G(enc[2 * (li - 1)].bias), da_prev.view(NB, hin_, hin_, ci))
            da = da_prev
        ops.gemm(da, fw.enc_col[0], G(enc[0].weight).view(geo[0][3], 16 * geo[0][2]), a_mn=True, b_mn=True, accumulate=True)
        for li in (1, 2, 3):
            _, _, ci, co = geo[li]
            ops.permute4(encgw[li].view(co, 4, 4, cpad[li])[..., :ci], G(enc[2 * li].weight), (0, 3, 1, 2))
        return dea_c

    def _image_decoder_bwd(self, fw, dfeat, par_w):
        """ConvDecoder backward: the image-loss seeds w[n] * image_weight * (dec - target) back to the first write of dfeat;
        with par_w the weight gradients go to side stream 4 (joined by the caller)."""
        ops, d, conf = self.ops, self.d, self.conf
        N = fw.T * fw.B * fw.I
        b, W, G = self._buf, self._w, self._g
        dec = self.wm.decoder.image.model
        featN, w, dd = fw.featN, fw.w, fw.dec
        ops.rowscale(dd.diff.view(N, d.IC * 4096), w, 1, conf.image_weight)
        ops.rowscale(dd.csum, w, 1, conf.image_weight)
        ops.colsum(dd.csum, G(dec[8].bias))
        dgeo = self._dec_geo
        impl = [self._implicit_conv_ok() and li in (1, 2) for li in range(4)]   # deconv 2,3: 32-channel-aligned NHWC gradients
        copad = [(co + 31) // 32 * 32 if impl[li] else co for li, (_, _, _, _, co) in enumerate(dgeo)]
        gdec = [b(("bwd.gdecwp" if impl[li] else "bwd.gdecw") + str(li), k * k * copad[li], ci)
                for li, (_, _, k, ci, _) in enumerate(dgeo)]                 # rows (tap, co padded), as self._decw
        for g_ in gdec:
            ops.fill(g_, 0.0)
        side = (lambda: self._fork(4)) if par_w else contextlib.nullcontext
        dout4 = dd.diff.permute(0, 2, 3, 1)                    # [n,y,x,c] view of the NCHW diff
        for li in (3, 2, 1, 0):
            hi, ho, k, ci, co = dgeo[li]
            xin = dd.xin[li]
            dxin = b(f"bwd.dd{li}", N * hi * hi, ci)
            # (li > 0: the ELU backward and the bias gradient of the deconv below ride in the input-gradient GEMM's epilogue)
            below_bias = G(dec[2 * li].bias) if li > 0 else None
            if impl[li]:
                with side():
                    ops.conv_gemm(2, dout4, k, xin, gdec[li])                          # weight gradient
                ops.conv_gemm_actbwd(dout4, k, self._decw[li], dxin, xin, below_bias, o_mn=True)   # input gradient
            else:
                if li == 0:
                    dcols = dout4.reshape(N, k * k * co)       # 5x5 input of a 5x5 kernel: im2col is the identity
                else:
                    dcols = b(f"bwd.dcols{li}", N * hi * hi, k * k * co)
                    ops.im2col(dout4, k, 0, dcols, round_out=True)
                with side():
                    ops.gemm(dcols, xin, gdec[li], a_mn=True, b_mn=True, accumulate=True)
                if li > 0:
                    ops.gemm_actbwd(dcols, self._decw[li], dxin, xin, below_bias, b_mn=True)
                else:
                    ops.gemm(dcols, self._decw[li], dxin, b_mn=True, round_out=True)
            dout4 = dxin.view(N, hi, hi, ci)
        dx0 = dxin
        with side():
            for li, idx_ in enumerate((2, 4, 6, 8)):          # back to ConvTranspose2d layout (Cin,Cout,kh,kw)
                wt = dec[idx_].weight
                ci, co, kh, kw = wt.shape
                ops.permute4(gdec[li].view(kh, kw, copad[li], ci)[:, :, :co], G(wt), (3, 2, 0, 1))
            ops.gemm(dx0, featN, G(dec[0].weight), a_mn=True, b_mn=True, accumulate=True)
            ops.colsum(dx0, G(dec[0].bias))
        ops.gemm(dx0, W(dec[0].weight), dfeat, b_mn=True)                      # first writer of dfeat

    # ------------------------------------------------------------------ imagination rollout
    def _dream(self, feats, N, H, noise_actor, noise_prior, tag):
        """dreamer.py:188-216: H x { actor -> sample action -> forward_prior }, forward only (reinforce).
        feats (H+1, N, F): feats[0] holds the start states; rows 1..H are written here.  Returns what the actor-critic
        reads: the actor outputs `alog`, its saved activations `actor`, the sampled `actions` and `feats16`, the fp16 copy
        of feats on the fp16-forward path (else None)."""
        ops, d, conf = self.ops, self.d, self.conf
        b, W = (lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)), self._w
        cell = self.wm.core.cell
        grus, col = cell.gru.layers, self._gru_cols
        ap = self._mlp_params(self.ac.actor)
        f16 = self._fp16_forward_ok()
        dr = SimpleNamespace(alog=b("dream.alog", H, N, d.Ap)[..., :d.Aout], actions=b("dream.actions", H, N, d.A),
                             actor=self._mlp_saved(ap, tag + "actor", H * N),
                             feats16=b("feats16", H + 1, N, d.F, dtype=torch.float16) if f16 else None)
        aidx = b("dream.aidx", N, 1, dtype=torch.int32)
        aa, x, za = b("dream.aa", N, d.Hd), b("dream.x", N, d.Hd), b("dream.za", N, d.Hd)
        mm, rr = b("dream.m", N), b("dream.r", N)
        gi, gh = (b(n_, N, 3 * d.D).view(d.L, N, 3 * d.Dl) for n_ in ("dream.gi", "dream.gh"))     # [l]: GRU layer l
        yp, pp, prior = b("dream.yp", N, d.Hd), b("dream.pp", N, d.Hd), b("dream.prior", N, d.Z)
        za16, pp16 = (b("dream.za16", N, d.Hd, dtype=torch.float16), b("dream.pp16", N, d.Hd, dtype=torch.float16)) if f16 \
            else (None, None)
        fx = dr.feats16 if f16 else feats          # GEMM operand copy of the features
        if f16:
            ops.to_half(feats[0], fx[0])
        par = self._ov(2)
        gh_gemm = lambda i, l: self._fgemm(fx[i][:, col(l)], grus[l].weight_hh, gh[l], f16, bias=self._raw(grus[l].bias_hh))
        if par:
            with self._fork(2):
                for l in range(d.L):
                    gh_gemm(0, l)
        for i in range(H):
            f, fn, xn = feats[i], feats[i + 1], fx[i + 1]
            self._mlp_fwd(ap, f, dr.alog[i], dr.actor, row0=i * N, x16=fx[i] if f16 else None)
            onehot = conf.actor_dist == "onehot"
            if onehot:
                ops.cat_sample(dr.alog[i], noise_actor[i], 1, d.A, dr.actions[i], idx=aidx)
            elif conf.actor_dist == "tanh_normal":
                ops.tanh_normal_sample(dr.alog[i], noise_actor[i], dr.actions[i])
            else:
                ops.normal_tanh_sample(dr.alog[i], noise_actor[i], dr.actions[i])
            if onehot and d.Hd % 4 == 0:
                ops.gather_rows(aidx, self._waT, aa)                 # a_mlp(one-hot) = one row of a_mlp^T
            else:
                ops.gemm(dr.actions[i], W(cell.a_mlp.weight), aa)
            self._fgemm(fx[i][:, d.D:], cell.z_mlp.weight, x, f16, bias=self._raw(cell.z_mlp.bias), res=aa)
            ops.ln_elu_fwd(x, self._raw(cell.in_norm.weight), self._raw(cell.in_norm.bias), 1e-3, za, mm, rr, za16)
            for l in range(d.L):                # layer l > 0 reads layer l - 1's new state (its fp16 copy on the fp16 path)
                xl = (za16 if f16 else za) if l == 0 else (xn if f16 else fn)[:, col(l - 1)]
                self._fgemm(xl, grus[l].weight_ih, gi[l], f16, bias=self._raw(grus[l].bias_ih))
                if not par:
                    gh_gemm(i, l)
                elif l == 0:
                    self._join(2)
                ops.gru_fwd(gi[l], gh[l], f[:, col(l)], fn[:, col(l)], h16=xn[:, col(l)] if f16 else None)
                if par and i + 1 < H:           # next step's h·W_hh overlaps prior MLP, sampling and the actor
                    with self._fork(2):
                        gh_gemm(i + 1, l)
            self._head_fwd(self._rssm_head(prior=True), xn[:, :d.D], yp, pp, mm, rr, prior, f16, pp16)
            ops.cat_sample(prior, noise_prior[i], d.G, d.C, fn[:, d.D:], z16=xn[:, d.D:] if f16 else None)
        return dr

    # ------------------------------------------------------------------ actor critic
    def _actor_critic(self, feats, dr, N, H, want_grad, tag):
        """a2c.py:61-149 on the dreamed features and what _dream returned with them (all inputs detached,
        dreamer.py:153-157)."""
        ops, d, conf, ac = self.ops, self.d, self.conf, self.ac
        J = H + 1
        b = lambda name, *shape, **kw: self._buf(tag + name, *shape, **kw)
        fall = feats.view(J * N, d.F)
        rp, tp = self._mlp_params(self.wm.decoder.reward.model), self._mlp_params(self.wm.decoder.terminal.model)
        cp, ctp, ap = self._mlp_params(ac.critic), self._mlp_params(ac.critic_target), self._mlp_params(ac.actor)
        rew, tlog = b("ac.rew", J * N, 1), b("ac.tlog", J * N, 1)
        vt, v = b("ac.vt", J * N, 1), b("ac.v", J * N, 1)
        fall16 = dr.feats16.view(J * N, d.F) if dr.feats16 is not None else None
        critic = self._mlp_saved(cp, tag + "critic", J * N)
        if self._catreward:                  # the actor-critic learns from the expected reward (dreamer.py:156, common.py:84)
            rlog = b("ac.rlog", J * N, d.Sp)[:, :d.S]
            self._mlp_fwd(rp, fall, rlog, x16=fall16)
            ops.support_head(rlog, self._raw(self.wm.decoder.reward._support), None, 1, rew)
        else:
            self._mlp_fwd(rp, fall, rew, x16=fall16)
        self._mlp_fwd(tp, fall, tlog, x16=fall16)
        self._mlp_fwd(ctp, fall, vt, x16=fall16)
        self._mlp_fwd(cp, fall, v, critic, x16=fall16)
        term = b("ac.term", J, N)
        adv, agae, target = b("ac.adv", H, N), b("ac.agae", H, N), b("ac.target", H, N)
        weight, dv = b("ac.weight", H, N), b("ac.dv", H * N, 1)
        sums = b("ac.sums", 8, dtype=torch.float64)
        ops.fill(sums.view(torch.float32), 0.0)
        ops.gae_critic(H, N, conf.gamma, conf.lambda_gae, vt, v, rew, tlog, term, adv, agae, target, weight, dv, sums)
        alog, actions = dr.alog.view(H * N, d.Aout), dr.actions.view(H * N, d.A)
        dal = b("ac.dalog", H * N, d.Ap)[:, :d.Aout]
        if conf.actor_dist == "onehot":
            ops.actor_loss_onehot(conf.entropy, alog, actions, agae, weight, dal, sums[5:7])
        elif conf.actor_dist == "tanh_normal":
            ops.actor_loss_tanh_normal(conf.entropy, alog, actions, agae, weight, dal, sums[5:7])
        else:
            ops.actor_loss_normal_tanh(conf.entropy, alog, actions, agae, weight, dal, sums[5:7])
        if want_grad:
            fH = fall[:H * N]
            self._mlp_bwd(cp, fH, dv, critic)
            self._mlp_bwd(ap, fH, dal, dr.actor)
        hm = float(H * N)
        s = sums
        r_mean = s[3] / hm
        r_var = torch.clamp((s[4] - s[3] * s[3] / hm) / (hm - 1.0), min=0.0)
        f32 = lambda x: x.to(torch.float32)
        metrics = dict(loss_critic=f32(s[0] / hm), loss_actor=f32(s[5] / hm), policy_entropy=f32(s[6] / hm),
                       policy_value=f32(s[1] / float(N)), policy_value_im=f32(s[2] / hm), policy_reward=f32(r_mean),
                       policy_reward_std=f32(r_var.sqrt()))
        return dict(loss_actor=metrics["loss_actor"], loss_critic=metrics["loss_critic"], metrics=metrics,
                    value=v.view(J, N), rew=rew.view(J, N), term=term,
                    tensors=dict(value=v.view(J, N), value_target=target, value_advantage=adv,
                                 value_advantage_gae=agae, value_weight=weight))

    def _dream_for_log(self, obs, featN, T, B, I, noise_actor, noise_prior):
        """dreamer.py:165-180 (do_dream_tensors): dream T-1 steps from the first posterior state of every sequence (rows of
        this step's posterior features featN), decode the imagined images, evaluate the critic (log_only).  Logging
        branch, no gradients."""
        d = self.d
        Hl, BI = T - 1, B * I
        fl = self._buf("dl.feats", Hl + 1, B, d.F)
        fl[0].copy_(featN[0:BI:I])                                       # states[0, :, 0]
        dr = self._dream(fl, B, Hl, noise_actor, noise_prior, "dl.")
        ac = self._actor_critic(fl, dr, B, Hl, False, "dl.")
        rows = (Hl + 1) * B
        if self._dense:                      # decoders.py:200-203: CatImageDecoder.forward, the raw logits
            img = self._buf("dl.gdec.y", rows, d.CP)
            self._mlp_fwd(self._mlp_params(self.wm.decoder.image), fl.view(rows, d.F), img)
        else:
            img = self._image_decoder(fl.view(rows, d.F), rows, "dl.").image
        s = self.conf.image_size
        t = ac["tensors"]
        return dict(action_pred=torch.cat([obs["action"][:1], dr.actions]), reward_pred=ac["rew"], terminal_pred=ac["term"],
                    image_pred=img.view(T, B, d.IC, s, s), value=t["value"], value_target=t["value_target"],
                    value_advantage=t["value_advantage"], value_advantage_gae=t["value_advantage_gae"],
                    value_weight=t["value_weight"])

    def __str__(self):
        n = sum(p.numel() for p in self.parameters())
        return f"Model: {n} parameters (pydreamer_b200: sm_90a kernels behind the pydreamer Dreamer API)"

"""Configuration namespaces with the reference's key names.

The reference builds an argparse.Namespace by dict-unioning YAML sections (launch.py:24-41) and
passes it to Dreamer(conf) (dreamer.py:21).  The drop-in keeps that contract: any object with these
attributes works, including one produced by the reference's own launcher.  The values below restate
the hot-path keys of config/defaults.yaml (`defaults`:1-120, `atari`:188-201, `dmc`:203-213) so that
benchmarks and tests do not need the reference checkout at run time.
"""
from argparse import Namespace

# config/defaults.yaml `defaults` section, hot-path keys only (SURVEY.md App. E)
DEFAULTS = dict(
    # features
    image_key="image", image_size=64, image_channels=3, image_categorical=False, action_dim=0, clip_rewards=None,
    map_key=None, map_size=0, map_channels=0, map_categorical=True, goals_size=0,
    # training
    reset_interval=200, iwae_samples=1, kl_balance=0.8, kl_weight=1.0, image_weight=1.0, vecobs_weight=1.0,
    reward_weight=1.0, terminal_weight=1.0, adam_lr=3.0e-4, adam_lr_actor=1.0e-4, adam_lr_critic=1.0e-4,
    adam_eps=1.0e-5, keep_state=True, batch_length=48, batch_size=32, device="cuda:0", grad_clip=200,
    grad_clip_ac=200, image_decoder_min_prob=0, amp=False, probe_gradients=False,
    # model
    model="dreamer", deter_dim=2048, stoch_dim=32, stoch_discrete=32, hidden_dim=1000, gru_layers=1, gru_type="gru",
    layer_norm=True, vecobs_size=0, image_encoder="cnn", cnn_depth=48, image_encoder_layers=0, image_decoder="cnn",
    image_decoder_layers=0, reward_input=False, reward_decoder_layers=4, reward_decoder_categorical=None,
    terminal_decoder_layers=4,
    # probe
    probe_model="none", map_decoder="dense", map_hidden_layers=4, map_hidden_dim=1024,
    # actor critic
    gamma=0.995, lambda_gae=0.95, entropy=0.003, target_interval=100, imag_horizon=15, actor_grad="reinforce",
    actor_dist="onehot",
    # auxiliary critic
    aux_critic=False, aux_critic_weight=1.0, gamma_aux=0.99, lambda_gae_aux=0.95, target_interval_aux=1000,
)

SECTIONS = {
    # config/defaults.yaml:188-201
    "atari": dict(action_dim=18, clip_rewards="tanh", deter_dim=1024, kl_weight=0.1, gamma=0.99, entropy=0.001),
    # config/defaults.yaml:203-213
    "dmc": dict(action_dim=12, entropy=1.0e-4, actor_grad="dynamics", actor_dist="tanh_normal", clip_rewards="tanh"),
    # config/defaults.yaml:236-242 (CartPole: a 4-float state vector, no image)
    "vectorenv": dict(env_id="CartPole-v0", action_dim=2, vecobs_size=4, image_key=None, image_encoder=None,
                      image_decoder=None),
    # config/defaults.yaml:244-248 (64x64x3 image + a 27-float vector)
    "minecraft": dict(env_id="Embodied-minecraft_diamond", action_dim=29, vecobs_size=27, clip_rewards="log1p"),
    # config/defaults.yaml:122-141 (7x7 grid of 4 object categories, one-hot encoded; reward / terminal planes appended to
    # the encoder input; dense image encoder and categorical image decoder; the map probe)
    "minigrid": dict(env_id="MiniGrid-MazeS11N-v0", image_key="image", image_size=7, image_channels=4, image_categorical=True,
                     map_key="map", map_size=11, map_channels=4, map_categorical=True, action_dim=7, reward_input=True,
                     image_encoder="dense", image_encoder_layers=3, image_decoder="dense", image_decoder_layers=2,
                     probe_model="map", imag_horizon=1),
}

# BASELINE.json configs (SURVEY.md §0.4: the shipped YAML differs from BASELINE's wording, so the
# overrides are explicit).  DMC: the shipped actor_grad=dynamics asserts at a2c.py:131 upstream
# (SURVEY.md §0.5) -> graded variant is reinforce + tanh_normal.
PRESETS = {
    "atari": (("atari",), dict(deter_dim=2048, batch_size=50, batch_length=50)),
    "atari_iwae": (("atari",), dict(deter_dim=2048, batch_size=50, batch_length=50, iwae_samples=4)),
    "dmc": (("dmc",), dict(deter_dim=1024, batch_size=50, batch_length=50, actor_grad="reinforce")),
    "atari_shipped": (("atari",), dict()),
    # small shapes for tests / smoke (same structure, every dimension shrunk)
    "tiny": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4, action_dim=5,
                              batch_size=3, batch_length=4, imag_horizon=3)),
    "tiny_dmc": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4, action_dim=3,
                                batch_size=3, batch_length=4, imag_horizon=3, actor_grad="reinforce")),
    # vector observations as shipped: `vectorenv` has no image encoder / decoder, `minecraft` has both plus the vector
    "vectorenv": (("vectorenv",), dict()),
    "minecraft": (("minecraft",), dict()),
    "tiny_vecobs": (("minecraft",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                         action_dim=5, vecobs_size=27, batch_size=3, batch_length=4, imag_horizon=3)),
    "tiny_vecobs_iwae3": (("minecraft",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                               action_dim=5, vecobs_size=27, batch_size=3, batch_length=4, imag_horizon=3,
                                               iwae_samples=3)),
    "tiny_vector": (("vectorenv",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, action_dim=3,
                                         batch_size=3, batch_length=4, imag_horizon=3)),
    # the categorical reward head (reward_decoder_categorical): Atari's [-1, 0, 1] through tanh clipping, S = 3
    "atari_catreward": (("atari",), dict(deter_dim=2048, batch_size=50, batch_length=50,
                                         reward_decoder_categorical=[-1.0, 0.0, 1.0])),
    "tiny_catreward": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                        action_dim=5, batch_size=3, batch_length=4, imag_horizon=3,
                                        reward_decoder_categorical=[-1.0, 0.0, 1.0])),
    "tiny_catreward_iwae3": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                              action_dim=5, batch_size=3, batch_length=4, imag_horizon=3, iwae_samples=3,
                                              reward_decoder_categorical=[-1.0, 0.0, 1.0])),
    "tiny_dmc_catreward": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                          action_dim=3, batch_size=3, batch_length=4, imag_horizon=3,
                                          actor_grad="reinforce", clip_rewards=None, reward_decoder_categorical=[0, 1])),
    # 33 unsorted support values (a row pitch of 36), every value in [-1, 0.875] listed twice: the target bucket of almost
    # every reward is a tie that the first index wins
    "tiny_catreward_wide": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                             action_dim=5, batch_size=3, batch_length=4, imag_horizon=3, clip_rewards=None,
                                             reward_decoder_categorical=[((5 * i) % 17 - 8) / 8 for i in range(17)] +
                                             [((3 * i) % 16 - 8) / 8 for i in range(16)])),
    # the world model's auxiliary critic (aux_critic): a critic of the observed rewards on the posterior features, trained
    # with the world model
    "atari_auxcritic": (("atari",), dict(deter_dim=2048, batch_size=50, batch_length=50, aux_critic=True)),
    "tiny_auxcritic": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                        action_dim=5, batch_size=3, batch_length=4, imag_horizon=3, aux_critic=True)),
    "tiny_auxcritic_iwae3": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                              action_dim=5, batch_size=3, batch_length=4, imag_horizon=3, iwae_samples=3,
                                              aux_critic=True)),
    "tiny_dmc_auxcritic": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                          action_dim=3, batch_size=3, batch_length=4, imag_horizon=3,
                                          actor_grad="reinforce", aux_critic=True)),
    "tiny_vector_auxcritic": (("vectorenv",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, action_dim=3,
                                                   batch_size=3, batch_length=4, imag_horizon=3, aux_critic=True)),
    # categorical grid images (the `minigrid` section) without the map probe: as shipped otherwise (B = 32, T = 48, deter
    # 2048, H = 1), then tiny shapes: 7x7x4 with reward input, importance samples, the uniform mix of image_decoder_min_prob,
    # MLPs without hidden layers, a 5x5x3 image without planes (C*H*W = 75 is not a multiple of 4) and a 27-float vector
    "minigrid": (("minigrid",), dict(probe_model="none")),
    "tiny_grid": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                      batch_size=3, batch_length=4, imag_horizon=3)),
    "tiny_grid_iwae3": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                            batch_size=3, batch_length=4, imag_horizon=3, iwae_samples=3)),
    "tiny_grid_minprob": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                              batch_size=3, batch_length=4, imag_horizon=3, image_decoder_min_prob=0.1)),
    "tiny_grid_layers0": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                              batch_size=3, batch_length=4, imag_horizon=3, image_encoder_layers=0,
                                              image_decoder_layers=0)),
    "tiny_grid_plain": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                            batch_size=3, batch_length=4, imag_horizon=3, reward_input=False, image_size=5,
                                            image_channels=3)),
    "tiny_grid_vecobs": (("minigrid",), dict(probe_model="none", deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40,
                                             batch_size=3, batch_length=4, imag_horizon=3, vecobs_size=27)),
    # a stacked GRU in the RSSM (gru_layers = L: L cells of deter_dim / L units, layer l > 0 reading layer l - 1's new
    # state): tiny shapes with L = 2, with L = 4 and three importance samples, with the tanh_normal actor, without an image,
    # and deter 66 in three 22-unit layers (column offsets off the 16-byte multiples); then the Atari benchmark shape
    "tiny_gru2": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4, action_dim=5,
                                   batch_size=3, batch_length=4, imag_horizon=3, gru_layers=2)),
    "tiny_gru4_iwae3": (("atari",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                         action_dim=5, batch_size=3, batch_length=4, imag_horizon=3, iwae_samples=3,
                                         gru_layers=4)),
    "tiny_dmc_gru2": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4, action_dim=3,
                                     batch_size=3, batch_length=4, imag_horizon=3, actor_grad="reinforce", gru_layers=2)),
    "tiny_vector_gru2": (("vectorenv",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, action_dim=3,
                                              batch_size=3, batch_length=4, imag_horizon=3, gru_layers=2)),
    "tiny_gru3_odd": (("atari",), dict(deter_dim=66, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4, action_dim=5,
                                       batch_size=3, batch_length=4, imag_horizon=3, gru_layers=3)),
    "atari_gru2": (("atari",), dict(deter_dim=2048, batch_size=50, batch_length=50, gru_layers=2)),
    # the normal_tanh actor (Normal(tanh(m), sigmoid(s) + 0.01), actions not bounded): tiny DMC shapes, with three importance
    # samples, without an image; then the DMC benchmark shape
    "tiny_dmc_normaltanh": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                           action_dim=3, batch_size=3, batch_length=4, imag_horizon=3,
                                           actor_grad="reinforce", actor_dist="normal_tanh")),
    "tiny_dmc_normaltanh_iwae3": (("dmc",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, cnn_depth=4,
                                                 action_dim=3, batch_size=3, batch_length=4, imag_horizon=3, iwae_samples=3,
                                                 actor_grad="reinforce", actor_dist="normal_tanh")),
    "tiny_vector_normaltanh": (("vectorenv",), dict(deter_dim=64, stoch_dim=4, stoch_discrete=8, hidden_dim=40, action_dim=3,
                                                    batch_size=3, batch_length=4, imag_horizon=3, actor_dist="normal_tanh")),
    "dmc_normaltanh": (("dmc",), dict(deter_dim=1024, batch_size=50, batch_length=50, actor_grad="reinforce",
                                      actor_dist="normal_tanh")),
}


def make_conf(preset="atari", **overrides):
    sections, over = PRESETS[preset]
    d = dict(DEFAULTS)
    for s in sections:
        d.update(SECTIONS[s])
    d.update(over)
    d.update(overrides)
    return Namespace(**d)

"""Synthetic replay batches in the layout the reference's Preprocessor emits (SURVEY.md §8d).

  image    (T,B,C,64,64) fp32 U[-0.5,0.5)          preprocessing.py:21-29 (uint8/255 - 0.5, CHW)
           with image_categorical: the one-hot (T,B,C,H,W) of the argmax over C of that draw (preprocessing.py:10-19)
  action   (T,B,A)       one-hot fp32 / U[-1,1)     preprocessing.py:135-138, wrappers.py:54-60
  reward   (T,B)         tanh(N(0,1))               clip_rewards: tanh (defaults.yaml:196)
  terminal (T,B)         Bernoulli(0.01) as 0./1.   preprocessing.py:148
  reset    (T,B) bool    reset[0]=True on the first batch, Bernoulli(1/200) elsewhere (data.py:255,284-304)
  vecobs   (T,B,K)       N(0,1) fp32 when vecobs_size = K > 0  preprocessing.py:160-163
`image` is left out for a model without an image encoder.  The vecobs draw comes after every other draw, so batches of
image-only configurations are the same with or without it.
"""
import torch


def synthetic_batch(conf, seed=1234, T=None, B=None, first=True, device="cpu", pin=False):
    T = T or conf.batch_length
    B = B or conf.batch_size
    g = torch.Generator().manual_seed(seed)
    A = conf.action_dim
    img = torch.rand(T, B, conf.image_channels, conf.image_size, conf.image_size, generator=g) - 0.5
    if getattr(conf, "image_categorical", False):        # the one-hot of a uniformly drawn category per pixel
        img = torch.nn.functional.one_hot(img.argmax(2), conf.image_channels).movedim(-1, 2).float().contiguous()
    if conf.actor_dist == "onehot":
        action = torch.nn.functional.one_hot(torch.randint(0, A, (T, B), generator=g), A).float()
    else:
        action = torch.rand(T, B, A, generator=g) * 2 - 1
    reward = torch.tanh(torch.randn(T, B, generator=g))
    terminal = (torch.rand(T, B, generator=g) < 0.01).float()
    reset = torch.rand(T, B, generator=g) < (1.0 / 200)
    if first:
        reset[0] = True
    obs = dict(image=img, action=action, reward=reward, terminal=terminal, reset=reset)
    if getattr(conf, "vecobs_size", 0):
        obs["vecobs"] = torch.randn(T, B, conf.vecobs_size, generator=g)
    if not conf.image_encoder:
        del obs["image"]
    if pin and torch.cuda.is_available():
        obs = {k: v.pin_memory() for k, v in obs.items()}
    if str(device) != "cpu":
        obs = {k: v.to(device, non_blocking=True) for k, v in obs.items()}
    return obs


def obs_bytes(obs):
    return int(sum(v.numel() * v.element_size() for v in obs.values()))

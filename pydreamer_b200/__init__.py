"""pydreamer_b200 — H100-native (sm_90a) drop-in for the hot path of jurgisp/pydreamer:
`Dreamer.training_step` (world-model step + imagination rollout + actor-critic losses), its gradients,
grad-clip and AdamW — hand-written CUDA kernels behind the reference's own module API."""
from .config import make_conf  # noqa: F401
from .dreamer import Dreamer  # noqa: F401
from .replay import synthetic_batch  # noqa: F401

__all__ = ["Dreamer", "make_conf", "synthetic_batch"]

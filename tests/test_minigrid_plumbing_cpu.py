"""BASELINE.json configs[0]: `--configs defaults minigrid`, batch 10 x seq 10.  This configuration (dense image encoder /
decoder, categorical 7x7 observations, reward input, map probe) is OUTSIDE the accelerated hot path (SURVEY.md §2 rows 4,
5, 9; §8f): the drop-in module refuses it loudly at construction (no silent partial support).
"""
from argparse import Namespace

import pytest

from pydreamer_b200.config import DEFAULTS
from pydreamer_b200.dreamer import Dreamer

# config/defaults.yaml:122-141 (`minigrid` section), hot-path keys
MINIGRID = dict(image_key="image", image_size=7, image_channels=4, image_categorical=True, map_key="map", map_size=11,
                map_channels=4, map_categorical=True, action_dim=7, reward_input=True, image_encoder="dense",
                image_encoder_layers=3, image_decoder="dense", image_decoder_layers=2, probe_model="map", imag_horizon=1)


def minigrid_conf(**over):
    d = dict(DEFAULTS)
    d.update(MINIGRID)
    d.update(batch_size=10, batch_length=10, device="cpu")
    d.update(over)
    return Namespace(**d)


def test_dropin_module_refuses_the_minigrid_config():
    with pytest.raises(NotImplementedError):
        Dreamer(minigrid_conf())

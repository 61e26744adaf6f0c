"""Generates tests/golden/reference_preprocess.npz from the unmodified reference (jurgisp/pydreamer): its
Preprocessor.apply of tests/test_preprocess.py:raw_batch() (image: a fixed sample of 4096 values; action / reward /
terminal in full).

    python tests/golden/make_reference_io.py <path of a reference checkout>
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.abspath(sys.argv[1]))

from pydreamer.preprocessing import Preprocessor  # noqa: E402

from tests.test_preprocess import IMAGE_SAMPLE, raw_batch  # noqa: E402


def preprocess():
    pp = Preprocessor(image_categorical=None, image_key="image", map_categorical=None, map_key=None, action_dim=18,
                      clip_rewards="tanh", amp=False)
    want = pp.apply({k: v.copy() for k, v in raw_batch().items()})
    np.savez_compressed(os.path.join(HERE, "reference_preprocess.npz"), image=want["image"].reshape(-1)[IMAGE_SAMPLE()],
                        action=want["action"], reward=want["reward"], terminal=want["terminal"])


if __name__ == "__main__":
    preprocess()

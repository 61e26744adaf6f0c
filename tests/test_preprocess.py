"""GpuPreprocessor (SURVEY.md §8f N3) against the numpy restatement of the reference Preprocessor; the restatement itself
is checked against stored outputs of the real `pydreamer.preprocessing.Preprocessor` (CPU test)."""
import os

import numpy as np
import pytest
import torch

from oracle import preprocess_oracle as P
from pydreamer_b200.config import make_conf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def raw_batch(T=5, B=4, A=18, seed=0):
    r = np.random.RandomState(seed)
    return dict(image=r.randint(0, 256, (T, B, 64, 64, 3)).astype(np.uint8), action=r.randint(0, A, (T, B)).astype(np.int64),
                reward=(r.randn(T, B) * 3).astype(np.float32), terminal=(r.rand(T, B) < 0.1).astype(np.float32),
                reset=r.rand(T, B) < 0.1)


def IMAGE_SAMPLE():
    """Fixed sample of flat indices into the (5, 4, 64, 64, 3) image of raw_batch(), stored with the golden vectors."""
    return np.sort(np.random.RandomState(1).choice(5 * 4 * 64 * 64 * 3, 4096, replace=False))


def test_restatement_matches_reference_preprocessor():
    """Against the reference's Preprocessor.apply on the same raw batch (tests/golden/reference_preprocess.npz, written by
    tests/golden/make_reference_io.py)."""
    want = np.load(os.path.join(ROOT, "tests", "golden", "reference_preprocess.npz"))
    got = P.apply(raw_batch(), 18, "tanh")
    image = np.ascontiguousarray(got["image"]).reshape(-1)[IMAGE_SAMPLE()]
    assert image.dtype == want["image"].dtype and np.array_equal(image, want["image"])
    for k in ("action", "reward", "terminal"):
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k


@pytest.mark.gpu
def test_gpu_preprocessor_matches_restatement():
    from pydreamer_b200.preprocess import GpuPreprocessor

    conf = make_conf("atari", device="cuda:0")
    raw = raw_batch(T=6, B=5)
    want = P.apply(raw, conf.action_dim, "tanh")
    got = GpuPreprocessor(conf, "cuda:0").apply({k: torch.from_numpy(v) for k, v in raw.items()})
    assert torch.equal(got["image"].cpu(), torch.from_numpy(np.ascontiguousarray(want["image"])))     # bit-exact x/255-0.5
    assert torch.equal(got["action"].cpu(), torch.from_numpy(want["action"]))
    assert torch.equal(got["terminal"].cpu(), torch.from_numpy(want["terminal"]))
    assert torch.equal(got["reset"].cpu(), torch.from_numpy(want["reset"]))
    assert torch.allclose(got["reward"].cpu(), torch.from_numpy(want["reward"]), rtol=1e-6, atol=1e-7)  # tanh: 1 ulp

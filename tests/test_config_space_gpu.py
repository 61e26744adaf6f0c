"""The rows of tests/test_config_space_cpu.py through the native kernels.

Per accepted row:
  * the product arm with its defaults (TF32 tensor cores, fp16 forward, implicit convolutions, overlap 3, the persistent
    forward kernel; the opt-in persistent BPTT kernel switched on) selects the paths the row declares, warns nothing, and
    passes the teacher-forced oracle comparison of tests/test_vecobs_gpu.py (3e-3 on world-model gradients, 3e-2 on the
    actor-critic's, which come from fp16-operand dreams) at twice its tolerances: a bias gradient is a signed sum over
    every row, and the TF32 errors of its terms do not cancel as the terms do (measured on an H100 at 700 W: the
    reward-head output bias of `dmc_a1` at 1.75x the world-model bound, the critic output bias of `d520` at 0.62x the
    actor-critic one; every loss and metric within 1x);
  * the exact arm (SIMT fp32, no operand rounding) reproduces the reference's committed outputs where the row has them;
  * one CUDA-graph replay of the product arm equals the same step launched eagerly on one stream, bit for bit
    (the comparison of tests/test_step_schedule_gpu.py)."""
import time
import warnings
import weakref

import pytest
import torch

from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.test_config_space_cpu import ACCEPTED, ROWS, SEEDS, build_row, check_against_oracle, expected, predicates
from tests.test_dreamer_gpu import check_exact_arm, run_gpu
from tests.test_step_schedule_gpu import assert_graph_ran, assert_identical, drawn_noise, released, train_step
from tests.util import seeded_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("name", ACCEPTED)
def test_product_arm_matches_the_oracle(name):
    fx, conf, obs, state, noise = build_row(name, DEV)
    model = Dreamer(conf).to(DEV)
    model.persistent_bptt = True
    model.load_state_dict(seeded_weights(model.state_dict(), dict(seeds=SEEDS)))
    model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        n0 = model.ops.launch_count()
        losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
        for l in losses:
            l.backward()
        torch.cuda.synchronize()
    assert not [str(w.message) for w in caught], name
    assert model.ops.launch_count() - n0 > 100                      # the native kernels really ran
    assert predicates(model, conf.batch_size * conf.iwae_samples) == expected(ROWS[name], on_gpu=True)
    check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, 2.0)


@pytest.mark.parametrize("name", [n for n in ACCEPTED if ROWS[n].golden])
def test_exact_arm_matches_reference_golden(name):
    fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors = run_gpu(ROWS[name].golden, impl=1,
                                                                                      rounding=False)
    check_exact_arm(fx, conf, model, losses, metrics, tensors)


@pytest.mark.parametrize("name", ACCEPTED)
def test_graph_replay_equals_the_eager_one_stream_step(name):
    """Three calls per arm: calls 1-2 eager, call 3 captures and replays (graphed arm, overlap 3); the eager arm (overlap 0)
    is fed the noise the graphed arm drew."""
    t0, calls = time.time(), 3
    row = ROWS[name]
    conf = make_conf(row.preset, device=DEV, **row.over)
    obs = [synthetic_batch(conf, seed=100 + i, first=(i == 0), device=DEV) for i in range(calls)]
    BI = conf.batch_size * conf.iwae_samples
    recs = {}
    for graphs in (True, False):
        torch.manual_seed(0)
        torch.cuda.manual_seed(0)
        m = Dreamer(conf).to(DEV)
        m.load_state_dict(seeded_state_dict(m.state_dict(), 11))
        m.use_cuda_graph, m.overlap = graphs, Dreamer.overlap if graphs else 0
        opts = m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
        state, recs[graphs] = m.init_state(BI), []
        for i in range(calls):
            rec, state, _, warned = train_step(m, opts, conf, obs[i], state,
                                               noise=None if graphs else recs[True][i][1])
            assert not warned, f"[{name}] graphs {graphs} call {i + 1}: {warned}"
            recs[graphs].append((rec, drawn_noise(m, conf, obs[i], False) if graphs else None))
        if graphs:
            kernels = assert_graph_ran(name, m, [])
        assert predicates(m, BI)["prssm"] == expected(row, on_gpu=True)["prssm"]
        ref = weakref.ref(m)
        del m, opts
        released(ref)
    for i in range(calls):
        assert_identical(f"[{name}] call {i + 1}", recs[False][i][0], recs[True][i][0])
    print(f"[{name}] {kernels} graph kernel nodes: replay == one-stream eager ({time.time() - t0:.1f} s)")

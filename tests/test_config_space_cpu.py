"""The training step across the model shapes `Dreamer(conf)` accepts, on the reference op table (oracle/ref_ops.py).

The kernel tests check each kernel at the shapes of the shipped steps; this file checks the host schedule of
pydreamer_b200/dreamer.py at the other shapes: dimensions off the multiples of 8 / 4 the tensor-core paths need, heads
without hidden layers, the widest LayerNorm, batch rows on either side of the persistent kernels' limits, and the configs
past a kernel limit, which the constructor refuses.  The op table refuses every call its native entry point refuses, so
a row that completes here passes the native host checks too (tests/test_config_space_gpu.py runs the same rows on the
GPU).

Each accepted row runs twice:
  * fp32 forward, persistent kernels off: the oracle (teacher-forced on the step's samples) at 2e-4 (2e-3 on the
    actor-critic gradients, signed sums over the dreamed rows), and the reference's committed outputs where the row has
    a fixture;
  * the fp16-forward and persistent-kernel stand-ins switched on: the shape predicates select what the row declares, the
    step completes without a warning (a refused persistent kernel would warn and fall back) and its losses stay within
    the 5e-3 of the fp16 emulation (tests/test_dreamer_cpu.py) of the fp32 step's."""
import warnings
from collections import namedtuple

import pytest
import torch

from oracle.vecobs_ops import VecRefOps
from pydreamer_b200 import ops as pd_ops
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from tests.test_dreamer_cpu import check_golden
from tests.util import build_case, load_fixture, seeded_weights

# the seeds of tests/golden/make_golden.py: a row with a fixture is built exactly as the fixture was
SEEDS = dict(noise=4321, data=1234, weights=7, state=99)

# fp16 / implicit / prssm / pbptt: what _fp16_forward_ok, _implicit_conv_ok, _persistent_rssm_ok and _persistent_bptt_ok
# return with every switch on, on an H100 (132 SMs).  cpu: the same where the reference op table, whose persistent
# stand-ins assume 148 SMs, differs.  refuse: the NotImplementedError message of a config past a kernel limit.
Row = namedtuple("Row", "why preset over golden fp16 implicit prssm pbptt cpu refuse",
                 defaults=(None, True, True, True, True, None, None))
SMALL = dict(batch_length=2, imag_horizon=2)
ROWS = {
    "heads0": Row("reward / terminal heads without hidden layers (_mlp_fwd / _mlp_bwd with L = 0)", "tiny",
                  dict(reward_decoder_layers=0, terminal_decoder_layers=0), golden="tiny_heads0"),
    "odd_dims": Row("Hd 42, D 70, Z 35, cnn_depth 6, one image channel: fp16 forward and implicit convolutions off", "tiny",
                    dict(hidden_dim=42, deter_dim=70, stoch_dim=5, stoch_discrete=7, cnn_depth=6, image_channels=1),
                    golden="tiny_odd_dims", fp16=False, implicit=False, prssm=False, pbptt=False),
    "z2": Row("Z = 2 < 8 (one group of two classes), T = H = 1: fp16 forward off", "tiny",
              dict(stoch_dim=1, stoch_discrete=2, batch_length=1, imag_horizon=1), golden="tiny_z2", fp16=False,
              prssm=False, pbptt=False),
    "hd44": Row("Hd % 8 != 0, % 4 == 0: fp16 forward off, a_mlp by pd_gather_rows", "tiny", dict(hidden_dim=44),
                fp16=False, prssm=False, pbptt=False),
    "hd42": Row("Hd % 4 != 0: pd_gather_rows off, CUDA-core GEMM routes", "tiny", dict(hidden_dim=42), fp16=False,
                prssm=False, pbptt=False),
    "hd1024": Row("the widest LayerNorm row (1024)", "tiny", dict(hidden_dim=1024)),
    "stoch32x32_d256": Row("32 groups of 32 classes at D = 256 (k-split 4 in both persistent kernels)", "tiny",
                           dict(deter_dim=256, stoch_dim=32, stoch_discrete=32)),
    "d512": Row("D % 256 == 0: persistent forward k-split 4", "tiny", dict(deter_dim=512)),
    "d520": Row("D % 256 != 0: persistent forward k-split 1", "tiny", dict(deter_dim=520)),
    "d2176": Row("cdiv(D, SMs) = 17 > 16 on 132 SMs: both persistent kernels off (15 on the 148 SMs RefOps assumes)",
                 "tiny", dict(deter_dim=2176, **SMALL), prssm=False, pbptt=False, cpu=dict(prssm=True, pbptt=True)),
    "cnn32": Row("cnn_depth 32 (the implicit convolutions' 32-channel blocks)", "tiny", dict(cnn_depth=32)),
    "bi65": Row("B*I = 65: persistent BPTT off (> 64 rows), persistent forward in row blocks (MULTI)", "tiny",
                dict(batch_size=65, **SMALL), pbptt=False),
    "bi129": Row("B*I = 129: the per-timestep chain is no longer skinny (> 128 rows)", "tiny",
                 dict(batch_size=43, iwae_samples=3, **SMALL), pbptt=False),
    "bi257": Row("B*I = 257: persistent forward off (> 256 rows)", "tiny", dict(batch_size=257, **SMALL), prssm=False,
                 pbptt=False),
    "heads1": Row("reward / terminal heads with one hidden layer", "tiny",
                  dict(reward_decoder_layers=1, terminal_decoder_layers=1)),
    "heads2": Row("reward / terminal heads with two hidden layers", "tiny",
                  dict(reward_decoder_layers=2, terminal_decoder_layers=2)),
    "dmc_a1": Row("tanh_normal actor with one action (two actor outputs)", "tiny_dmc", dict(action_dim=1)),
    "onehot_a32": Row("one-hot actor at the 32-class limit", "tiny", dict(action_dim=32)),
    # (one value is not a case: the reference's 1-wide head output flattens across the batch and fails to broadcast)
    "vector_k2": Row("the narrowest vector observation the reference trains, no image", "tiny_vector",
                     dict(vecobs_size=2)),
    # just past each hard kernel limit: refused at construction
    "hd1032": Row("LayerNorm rows past 1024", "tiny", dict(hidden_dim=1032), refuse="hidden_dim=1032"),
    "onehot_a33": Row("one-hot actor past 32 classes", "tiny", dict(action_dim=33), refuse="action_dim=33"),
    "vecobs4097": Row("vector observation past 4096 values", "tiny_vecobs", dict(vecobs_size=4097),
                      refuse="vecobs_size=4097"),
    "channels17": Row("image past 16 channels", "tiny", dict(image_channels=17), refuse="image_channels=17"),
    "horizon128": Row("imagination horizon past 127 steps", "tiny", dict(imag_horizon=128), refuse="imag_horizon=128"),
}
ACCEPTED = [n for n, r in ROWS.items() if r.refuse is None]
REFUSED = [n for n, r in ROWS.items() if r.refuse is not None]


def expected(row, on_gpu):
    e = dict(fp16=row.fp16, implicit=row.implicit, prssm=row.prssm, pbptt=row.pbptt)
    if not on_gpu:
        e.update(row.cpu or {})
    return e


def build_row(name, device="cpu"):
    """-> (fixture or None, conf, obs, in_state, noise) of a row, seeded as the committed fixtures are."""
    row = ROWS[name]
    fx = load_fixture(row.golden) if row.golden else dict(preset=row.preset, overrides=row.over, seeds=SEEDS)
    assert (fx["preset"], fx["overrides"]) == (row.preset, row.over), name
    out = build_case(row.golden, device, fx)
    return (fx if row.golden else None,) + out[1:]


def predicates(model, BI):
    return dict(fp16=model._fp16_forward_ok(), implicit=model._implicit_conv_ok(), prssm=model._persistent_rssm_ok(BI),
                pbptt=model._persistent_bptt_ok(BI))


def check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, tol):
    """The teacher-forced oracle comparison of tests/test_vecobs_gpu.py (its oracle covers models with and without an image
    and a vector observation); tol scales its TF32 product-arm bounds."""
    from tests.test_vecobs_gpu import check_against_oracle as check
    check(conf, obs, state, noise, model, losses, metrics, tensors, tol=tol)


@pytest.fixture()
def ref_ops():
    pd_ops.set_ops_for_testing(VecRefOps("cpu"))
    yield
    pd_ops.set_ops_for_testing(None)


def run_row(name, fp16_and_persistent):
    fx, conf, obs, state, noise = build_row(name)
    model = Dreamer(conf)
    model.fp16_forward = model.persistent_rssm = model.persistent_bptt = fp16_and_persistent
    model.load_state_dict(seeded_weights(model.state_dict(), dict(seeds=SEEDS)))
    model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        losses, out_state, metrics, tensors, _ = model.training_step(obs, state, noise=noise)
        for l in losses:
            l.backward()
    assert not [str(w.message) for w in caught], name
    return fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors


# 2e-4 (the reference goldens' bound) over the 3e-3 world-model bound of the GPU product arm the oracle comparison is
# written for
FP32_TOL = 2e-4 / 3e-3


@pytest.mark.parametrize("name", ACCEPTED)
def test_fp32_step_matches_the_oracle_and_the_reference(ref_ops, name):
    fx, conf, obs, state, noise, model, losses, out_state, metrics, tensors = run_row(name, False)
    BI = conf.batch_size * conf.iwae_samples
    assert predicates(model, BI) == dict(fp16=False, implicit=ROWS[name].implicit, prssm=False, pbptt=False)
    check_against_oracle(conf, obs, state, noise, model, losses, metrics, tensors, FP32_TOL)
    if fx is not None:
        check_golden(fx, model, losses, out_state, metrics, tensors)


@pytest.mark.parametrize("name", ACCEPTED)
def test_fp16_forward_and_persistent_stand_ins_take_the_shape(ref_ops, name):
    conf, model, losses = (run_row(name, True)[i] for i in (1, 5, 6))
    assert predicates(model, conf.batch_size * conf.iwae_samples) == expected(ROWS[name], on_gpu=False)
    for i, (got, want) in enumerate(zip(losses, run_row(name, False)[6])):
        got, want = float(got.detach().reshape(-1)[0]), float(want.detach().reshape(-1)[0])
        assert abs(got - want) <= 5e-3 * max(1.0, abs(want)), (i, got, want)


@pytest.mark.parametrize("name", REFUSED)
def test_configs_past_a_kernel_limit_are_refused_at_construction(name):
    row = ROWS[name]
    with pytest.raises(NotImplementedError, match=row.refuse):
        Dreamer(make_conf(row.preset, device="cpu", **row.over))


def test_imag_horizon_argument_past_the_limit_is_refused(ref_ops):
    fx, conf, obs, state, noise = build_row("heads1")
    model = Dreamer(conf)
    with pytest.raises(NotImplementedError, match="imag_horizon=128"):
        model.training_step(obs, state, imag_horizon=128)

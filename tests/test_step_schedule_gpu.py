"""The training step as a training run executes it, bit for bit against the same step launched eagerly on one stream.

`training_step` replays a captured CUDA graph from the third call of a shape on (noise drawn inside the step, no logging
flags), and its schedule issues independent branches on side streams (`Dreamer.overlap`).  The reference here is the
same step with `use_cuda_graph = False` and `overlap = 0`, fed the sampling noise the tested arm drew (read back from its
noise buffers after each call).  The eager step is tied to the oracle by tests/test_dreamer_gpu.py; every sum of the step
is added in a fixed order, so anything short of bit identity is a race, a stale buffer or an arrival-order sum.

The arms run one after the other (graphed arm first, then freed), never side by side.  Every compared tensor is copied on
the device right after the call that produced it, in step order: the 4 losses, the metrics, the `tensors` and dream
tensors, `out_state`, every parameter gradient, the 4 `grad_clip` norms, and after the optimizer step every parameter
(critic target included) and the AdamW moments."""
import gc
import time
import warnings
import weakref

import pytest
import torch

from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.replay import synthetic_batch
from tests.util import tf32_rna

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# preset, overrides; target_interval = 2 syncs the target critic between replays
CASES = {"tiny": ("tiny", {}), "tiny_dmc": ("tiny_dmc", {}), "tiny_iwae3": ("tiny", dict(iwae_samples=3)),
         "atari": ("atari", {})}
LOSSES = ("model", "probe", "actor", "critic")


# ----------------------------------------------------------------------------------------------------------- harness
def make_model(case, graphs, overlap, prssm=True, pbptt=False):
    preset, over = CASES[case]
    conf = make_conf(preset, device=DEV, target_interval=2, **over)
    torch.manual_seed(0)                 # the noise a graphed arm draws, so every run of the file sees the same steps
    torch.cuda.manual_seed(0)
    m = Dreamer(conf).to(DEV)
    m.load_state_dict(seeded_state_dict(m.state_dict(), 11))
    configure(m, graphs, overlap, prssm, pbptt)
    opts = m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    return conf, m, opts


def configure(m, graphs, overlap, prssm, pbptt):
    m.use_cuda_graph, m.overlap, m.persistent_rssm, m.persistent_bptt = graphs, overlap, prssm, pbptt


def batches(conf, n, seed=100):
    return [synthetic_batch(conf, seed=seed + i, first=(i == 0), device=DEV) for i in range(n)]


def ws(m, name, *shape, dtype=torch.float32):
    """A workspace buffer the step already wrote (never a fresh one: _buf would allocate a missing key)."""
    assert (name, shape, dtype) in m._ws, f"no workspace buffer {name} {shape}"
    return m._buf(name, *shape, dtype=dtype)


def drawn_noise(m, conf, obs, log):
    """The sampling noise the last call drew (the buffers `_draw_noise` fills), as `training_step(noise=...)` takes it."""
    d, (T, B) = m.d, obs["action"].shape[:2]
    I, H = conf.iwae_samples, conf.imag_horizon
    N = T * B * I
    nz = dict(post=ws(m, "noise.post", T, B * I, d.Z), actor=ws(m, "noise.actor", H, N, d.A),
              prior=ws(m, "noise.prior", H, N, d.Z))
    if log:
        nz.update(image_pred=ws(m, "noise.image_pred", N, d.Z), dream_log_actor=ws(m, "noise.dl_actor", T - 1, B, d.A),
                  dream_log_prior=ws(m, "noise.dl_prior", T - 1, B, d.Z))
    return {k: v.clone() for k, v in nz.items()}


def arena_views(m, arena, prefix, names):
    """(prefix.name, view) of every parameter in a copy of one of the model's flat arenas."""
    return [(f"{prefix}.{n}", arena[m._offsets[id(p)]:m._offsets[id(p)] + p.numel()].view(p.shape)) for n, p in names]


def train_step(m, opts, conf, obs, state, noise=None, log=False, returned=None, optimize=True, after_backward=None):
    """One iteration of the reference training loop (train.py:160-197): training_step, zero_grad x4, backward x4,
    grad_clip, step x4 (without `optimize`: up to the backward calls).  Returns (records, new_state, the call's library
    launches, this library's warnings).  `returned` (a list) receives the losses and metrics objects the call returned;
    after_backward(losses, metrics, tensors) runs between the backward calls and grad_clip."""
    rec = []
    add = lambda name, t: rec.append((name, t.detach().clone()))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        k0 = m.ops.launch_count()
        losses, new_state, metrics, tensors, dream = m.training_step(obs, state, noise=noise, do_image_pred=log,
                                                                     do_dream_tensors=log)
        launches = m.ops.launch_count() - k0
        for n, l in zip(LOSSES, losses):
            add(f"loss_{n}", l)
        for k, v in metrics.items():
            add(f"metric.{k}", v)
        if returned is not None:
            returned += [(f"loss_{n}", l) for n, l in zip(LOSSES, losses)] + [(f"metric.{k}", v) for k, v in metrics.items()]
        for k, v in tensors.items():
            add(f"tensors.{k}", v)
        for k, v in dream.items():
            add(f"dream.{k}", v)
        add("out_state.h", new_state[0])
        add("out_state.z", new_state[1])
        for o in opts:
            o.zero_grad()
        for l in losses:
            l.backward()
        names = [(n, p) for n, p in m.named_parameters()]
        rec += arena_views(m, m._garena.clone(), "grad", [(n, p) for n, p in names if p.grad is not None])
        if after_backward is not None:
            after_backward(losses, metrics, tensors)
        if optimize:
            for k, v in m.grad_clip(conf.grad_clip, conf.grad_clip_ac).items():
                add(k, v)
            for o in opts:
                o.step()
            rec += arena_views(m, m._arena.clone(), "param", names)
            for i, o in enumerate(opts):
                add(f"opt{i}.exp_avg", o.exp_avg)
                add(f"opt{i}.exp_avg_sq", o.exp_avg_sq)
        torch.cuda.synchronize()
    ours = [str(w.message) for w in caught if "pydreamer_b200" in str(w.message)]
    return rec, new_state, launches, ours


def _ordered(t):
    """Bit patterns of a float tensor as integers that order like the values (adjacent floats differ by 1)."""
    i = t.view({torch.float32: torch.int32, torch.float16: torch.int16, torch.float64: torch.int64}[t.dtype]).long()
    return torch.where(i < 0, -(i & (2 ** (8 * t.element_size() - 1) - 1)), i)


# logging outputs that are NaN by definition where their mask is empty (decoders.py:96-106: `x * m / m`, then nanmean)
MASKED = ("logprob_reward-1", "logprob_reward1", "logprob_terminal1")


def assert_identical(label, ref, got):
    """torch.equal on every tensor of two record lists, in order.  The first difference is reported with its element count
    and the largest difference in ulps.  A NaN fails, except in the masked logging outputs, whose NaNs must sit at the
    same elements in both arms."""
    assert [n for n, _ in ref] == [n for n, _ in got], f"{label}: the two arms returned different outputs"
    for (name, a), (_, b) in zip(ref, got):
        assert a.shape == b.shape and a.dtype == b.dtype, f"{label}: {name} {a.shape}/{a.dtype} vs {b.shape}/{b.dtype}"
        if a.is_floating_point() and name.split(".")[-1] in MASKED:
            assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{label}: {name} has NaNs at different elements"
            a, b = torch.nan_to_num(a, nan=0.0), torch.nan_to_num(b, nan=0.0)
        for arm, t in (("reference", a), ("tested", b)):
            assert not (t.is_floating_point() and torch.isnan(t).any()), f"{label}: {name} has NaNs in the {arm} arm"
        if not torch.equal(a, b):
            n = int((a != b).sum())
            if a.is_floating_point():
                worst = f"{int((_ordered(a) - _ordered(b)).abs().max())} ulp"
            else:
                worst = f"{float((a.double() - b.double()).abs().max()):g}"
            raise AssertionError(f"{label}: first differing tensor {name}: {n}/{a.numel()} elements differ, "
                                 f"largest difference {worst}")


def graph_state(m):
    (st,) = m._graphs.values()
    return st


def assert_graph_ran(label, m, warned):
    st = graph_state(m)
    assert st["graph"] is not None and not st.get("failed"), f"{label}: the step was not captured"
    assert not warned, f"{label}: {warned}"
    return st["kernels"]


def released(ref):
    """After the caller dropped every name of an arm's model: the model, its captured graph and the graph's memory pool
    are gone before the next arm is built."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert ref() is None, "the previous arm's model is still referenced"


def assert_shadows_fresh(label, m, rounding=True):
    """The operand shadows the step just read were rebuilt from the weights it trained on: the tf32 (rna; a plain copy
    with operand rounding off) and the fp16 copy of the whole arena, the critic target included, and the transposed fp16
    z_mlp of the persistent unroll."""
    a = m._arena
    assert torch.equal(m._sarena.double(), tf32_rna(a) if rounding else a.double()), f"{label}: stale tf32 shadow"
    if m.fp16_forward:
        assert torch.equal(m._harena, a.half()), f"{label}: stale fp16 shadow"
    if m.persistent_rssm:
        wz = m.wm.core.cell.z_mlp.weight
        assert torch.equal(m._k1_wzT, m._raw(wz).t().half()), f"{label}: stale transposed z_mlp"


# ------------------------------------------------------------------------------------- (a) graph replay == eager step
STEPS, LOG_STEP = 7, 4          # calls 1-2 eager, 3 captures, 4 / 6 / 7 replay; call 5 is an eager logging step


@pytest.mark.parametrize("case", list(CASES))
def test_graph_replay_equals_eager_one_stream_step_by_step(case):
    t0 = time.time()
    conf, m, opts = make_model(case, graphs=True, overlap=Dreamer.overlap)
    obs = batches(conf, STEPS)
    B, I = conf.batch_size, conf.iwae_samples
    state = m.init_state(B * I)
    graphed, noises = [], []
    for i in range(STEPS):
        fresh = lambda *_, i=i: assert_shadows_fresh(f"[{case}] call {i + 1}", m)
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state, log=i == LOG_STEP, after_backward=fresh)
        noises.append(drawn_noise(m, conf, obs[i], i == LOG_STEP))
        graphed.append(rec)
        assert not warned, f"[{case}] call {i + 1}: {warned}"
    kernels = assert_graph_ran(case, m, [])
    assert graph_state(m)["calls"] == STEPS - 1
    ref = weakref.ref(m)
    del m, opts, fresh
    released(ref)
    conf, m, opts = make_model(case, graphs=False, overlap=0)
    state = m.init_state(B * I)
    for i in range(STEPS):
        rec, state, n, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i], log=i == LOG_STEP)
        assert not warned, f"[{case}] eager call {i + 1}: {warned}"
        assert_identical(f"[{case}] step {i + 1}", rec, graphed[i])
        if i == 2:
            assert kernels == n, f"[{case}] the graph holds {kernels} kernel nodes, the eager step launched {n}"
    del m, opts
    print(f"[{case}] graph replay vs one-stream eager, {STEPS} steps: {kernels} graph kernel nodes, bit-identical "
          f"({time.time() - t0:.1f} s)")


# --------------------------------------------------------------- (e) a replay on trained weights against the oracle
@pytest.mark.parametrize("case", [c for c in CASES if c != "atari"])
def test_replay_on_trained_weights_matches_the_oracle(case):
    """The graph replays of (a)'s loop, on weights up to 6 AdamW updates from the seed (operand shadows rebuilt inside the
    graph, the target critic synced between replays), against the teacher-forced oracle of tests/test_dreamer_gpu.py.
    (a) cannot see a wrong shadow refresh or target sync: both of its arms run that code.

    It runs the exact arm (plain fp32 SIMT GEMM, no operand rounding, fp32 forward, explicit im2col), where the step and
    the oracle differ only in the order of fp32 sums, so the oracle's bounds can be 10x tighter than the TF32 product arm's.
    On moved weights the product arm's TF32 / fp16 operand rounding alone comes within ~10% of those product-arm bounds,
    so a test of the product arm there could not tell rounding from a bug; its shadows are checked exactly by (a)."""
    from tests.test_dreamer_gpu import check_teacher_forced_against_oracle

    conf, m, opts = make_model(case, graphs=True, overlap=Dreamer.overlap, prssm=False)
    m.fp16_forward = m.implicit_conv = False
    m.ops.set_gemm_impl(1)
    m.ops.set_round_operands(False)
    obs = batches(conf, STEPS)
    state = m.init_state(conf.batch_size * conf.iwae_samples)
    checked = []
    for i in range(STEPS):
        def oracle(losses, metrics, tensors, state=state, i=i):
            assert_shadows_fresh(f"[{case}] call {i + 1}", m, rounding=False)
            if i in (3, STEPS - 1):          # call 4: the target lags the critic by one update; call 7: just synced
                check_teacher_forced_against_oracle(f"{case} exact arm, replay {i + 1}", conf, obs[i], state,
                                                    drawn_noise(m, conf, obs[i], False), m, losses, metrics, tensors,
                                                    target_synced=i % conf.target_interval == 0, tol=0.1)
                checked.append(i + 1)

        _, state, _, warned = train_step(m, opts, conf, obs[i], state, log=i == LOG_STEP, after_backward=oracle)
        assert not warned, f"[{case}] call {i + 1}: {warned}"
    kernels = assert_graph_ran(case, m, [])
    assert checked == [4, STEPS]
    print(f"[{case}] exact arm, {kernels} graph kernel nodes: replays 4 and {STEPS} on trained weights match the oracle "
          f"at 1/10 of the product arm's tolerances")


# --------------------------------------------------------------------- (b) carried state across interleaved data workers
def test_carried_state_of_interleaved_data_workers_is_caller_owned():
    """train.py:168-178 keeps `states[wid] = new_state` without a copy and alternates data workers.  The graphed arm must
    compute what the eager one does, and what a call returned (losses, metrics, out_state) must not change under the
    next call.  `tensors` are views of the workspace on the graph path: they are compared right after their call."""
    case, calls = "tiny", 8
    conf, m, opts = make_model(case, graphs=True, overlap=Dreamer.overlap)
    B, I = conf.batch_size, conf.iwae_samples
    obs = [synthetic_batch(conf, seed=200 + 10 * (i % 2) + i // 2, first=i < 2, device=DEV) for i in range(calls)]
    states, graphed, noises, held = {}, [], [], None
    for i in range(calls):
        wid = i % 2
        state = states.get(wid) or m.init_state(B * I)
        ret = []
        rec, new_state, _, warned = train_step(m, opts, conf, obs[i], state, returned=ret)
        assert not warned, warned
        states[wid] = new_state                                   # no copy, as train.py:177-178
        if held is not None:                                      # the previous call's outputs, as that call returned them
            assert_identical(f"call {i}'s outputs after call {i + 1}", held[0], [(n, t.detach().clone()) for n, t in held[1]])
        ret += [("out_state.h", new_state[0]), ("out_state.z", new_state[1])]
        held = ([(n, t.detach().clone()) for n, t in ret], ret)
        noises.append(drawn_noise(m, conf, obs[i], False))
        graphed.append(rec)
    assert_graph_ran(case, m, [])
    ref = weakref.ref(m)
    del m, opts, held, ret                      # (the returned losses keep their module alive)
    released(ref)
    conf, m, opts = make_model(case, graphs=False, overlap=0)
    states = {}
    for i in range(calls):
        wid = i % 2
        state = states.get(wid) or m.init_state(B * I)
        rec, states[wid], _, warned = train_step(m, opts, conf, obs[i], state, noise=noises[i])
        assert not warned, warned
        assert_identical(f"call {i + 1} (data worker {wid})", rec, graphed[i])
    print(f"[{case}] {calls} calls alternating two data workers: graph replay == one-stream eager, returned outputs kept")


# ------------------------------------------------------------------------ (c) every concurrency mask, graphs off and on
def reset(m, conf, sd0):
    """Back to the seeded weights with fresh optimizers, no captured graph and the target-sync counter at 0."""
    m.load_state_dict(sd0)
    m.ac.train_steps = 0
    m._graphs = {}
    m._grads_pending = set()
    return m.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)


ALL = tuple((ov, g) for g in (False, True) for ov in range(8))
MASK_CASES = [pytest.param(case, prssm, pbptt, ALL, id=f"{case}-{'prssm' if prssm else 'chain'}-{'pbptt' if pbptt else 'bptt_chain'}")
              for case in ("tiny",) for prssm in (True, False) for pbptt in (False, True)]
# full size: the masks and switches a run can take, trimmed to keep the file within a few minutes
MASK_CASES += [pytest.param("atari", True, False, ((1, False), (3, False), (7, False), (0, True), (3, True), (4, True), (7, True)),
                            id="atari-prssm-bptt_chain"),
               pytest.param("atari", True, True, ((3, False), (3, True), (7, True)), id="atari-prssm-pbptt"),
               pytest.param("atari", False, False, ((3, True),), id="atari-chain-bptt_chain")]


@pytest.mark.parametrize("case,prssm,pbptt,masks", MASK_CASES)
def test_every_concurrency_mask_computes_the_one_stream_step(case, prssm, pbptt, masks):
    """`overlap` bit 1 (dream + actor-critic), 2 (the next h.W_hh product) and 4 (image-decoder weight gradients) each move
    work to a side stream; with graphs off and on, every mask must compute the overlap = 0 eager step bit for bit, and
    with graphs on the capture must succeed."""
    t0 = time.time()
    calls = 4 if case != "atari" else 3                  # graphs on: calls 1-2 eager, 3 captures and replays, 4 replays
    conf, m, _ = make_model(case, graphs=False, overlap=0, prssm=prssm, pbptt=pbptt)
    B, I = conf.batch_size, conf.iwae_samples
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    obs = batches(conf, calls, seed=300)
    refs = []                                            # (noise, records) of overlap-0 one-stream eager runs

    def run(ov, graphs, noise=None):
        opts = reset(m, conf, sd0)
        configure(m, graphs, ov, prssm, pbptt)
        torch.cuda.manual_seed(17)
        state, recs, drawn = m.init_state(B * I), [], []
        for i in range(calls):
            rec, state, _, warned = train_step(m, opts, conf, obs[i], state, noise=None if graphs else noise[i])
            assert not warned, f"overlap {ov} graphs {graphs}: {warned}"
            recs.append(rec)
            drawn.append(drawn_noise(m, conf, obs[i], False) if graphs else noise[i])
        assert m._persistent_rssm_ok(B * I) == prssm and m._persistent_bptt_ok(B * I) == pbptt
        return recs, drawn, assert_graph_ran(f"overlap {ov}", m, []) if graphs else None

    def reference(noise):
        for nz, recs in refs:
            if all(torch.equal(a[k], b[k]) for a, b in zip(nz, noise) for k in a):
                return recs
        refs.append((noise, run(0, False, noise)[0]))
        return refs[-1][1]

    noise0 = None
    for ov, graphs in sorted(masks, key=lambda mg: not mg[1]):       # graphed runs first: one of them draws the noise
        recs, drawn, kernels = run(ov, graphs, noise0)
        noise0 = noise0 or drawn
        ref = reference(drawn)
        for i in range(calls):
            assert_identical(f"[{case} prssm={prssm} pbptt={pbptt}] overlap {ov} graphs {'on' if graphs else 'off'}, call {i + 1}",
                             ref[i], recs[i])
        nodes = f"{kernels} graph kernel nodes" if graphs else "eager"
        print(f"[{case} prssm={int(prssm)} pbptt={int(pbptt)}] overlap {ov} graphs {'on ' if graphs else 'off'}: {nodes}, "
              f"bit-identical to one-stream eager over {calls} calls")
    print(f"[{case} prssm={int(prssm)} pbptt={int(pbptt)}] {len(masks)} schedules, {len(refs)} reference run(s), "
          f"{time.time() - t0:.1f} s")


# ----------------------------------------------------------------------------------------------------- (d) run to run
@pytest.mark.parametrize("pbptt", (False, True), ids=("bptt_chain", "persistent_bptt"))
def test_full_size_eager_step_is_identical_run_to_run(pbptt):
    """Three eager steps at full Atari size on the same weights, batch and noise: every output and gradient identical.
    This checks the order of the floating-point sums only (concurrent branches, split-K, block reductions)."""
    conf, m, opts = make_model("atari", graphs=False, overlap=Dreamer.overlap, pbptt=pbptt)
    T, B, H = conf.batch_length, conf.batch_size, conf.imag_horizon
    D, Z, A, N = conf.deter_dim, conf.stoch_dim * conf.stoch_discrete, conf.action_dim, T * B
    obs = batches(conf, 1, seed=400)[0]
    g = torch.Generator(device=DEV).manual_seed(5)
    state = (torch.tanh(torch.randn(B, D, device=DEV, generator=g)), torch.zeros(B, Z, device=DEV))
    noise = dict(post=torch.empty(T, B, Z, device=DEV).exponential_(generator=g),
                 actor=torch.empty(H, N, A, device=DEV).exponential_(generator=g),
                 prior=torch.empty(H, N, Z, device=DEV).exponential_(generator=g))
    runs = []
    for _ in range(3):
        rec, _, _, warned = train_step(m, opts, conf, obs, state, noise=noise, optimize=False)
        assert not warned, warned
        runs.append(rec)
    assert m._persistent_bptt_ok(B) == pbptt
    for r in (1, 2):
        assert_identical(f"[atari pbptt={pbptt}] run {r + 1} vs run 1", runs[0], runs[r])
    print(f"[atari pbptt={int(pbptt)}] 3 eager steps on the same inputs: bit-identical")

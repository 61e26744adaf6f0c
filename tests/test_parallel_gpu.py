"""Data parallelism on real GPUs over NCCL (skipped with fewer than 2 devices): 2 ranks x the native kernels with the FULL
one-GPU schedule (side-stream branches, persistent RSSM kernels) on halves of a global batch.  After the single flat
all-reduce the clipped-gradient norms must equal a single-GPU run of the concatenated batch (SURVEY.md §8e) and both
ranks must hold bit-identical parameters after the optimizer step.  Tolerance 2e-3: the exact-index arm (SIMT fp32 GEMM)
keeps the categorical samples identical between the sharded and the global run."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import dreamer_oracle as O
from oracle.weights import seeded_state_dict
from pydreamer_b200.config import make_conf
from pydreamer_b200.dreamer import Dreamer
from pydreamer_b200.parallel import GradAllReduce
from pydreamer_b200.replay import synthetic_batch
from tests.test_parallel_cpu import BG, WORLD, _inputs, _shard

pytestmark = pytest.mark.gpu


def _run(model, conf, obs, noise, B, steps=1):
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    norms = None
    for _ in range(steps):
        losses, *_ = model.training_step(obs, model.init_state(B), noise=noise)
        for l in losses:
            l.backward()
        norms = model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
        for o in opts:
            o.step()
    torch.cuda.synchronize()
    return {k: float(v) for k, v in norms.items()}


def _worker(rank, port, out):
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=WORLD,
                            device_id=torch.device(dev))
    conf, obs, noise = _inputs()
    lconf = make_conf("tiny", device=dev, batch_size=BG // WORLD)
    model = Dreamer(lconf).to(dev)
    model.fp16_forward = False
    model.implicit_conv = False
    if rank == 0:
        model.load_state_dict(seeded_state_dict(model.state_dict(), 3))
    model._ensure_arena()
    model.ops.set_gemm_impl(1)
    model.ops.set_round_operands(False)
    model._dp = GradAllReduce(WORLD)
    model._dp.broadcast_params(model)
    o, n = _shard(conf, obs, noise, rank)
    mv = lambda d: {k: v.to(dev) for k, v in d.items()}
    norms = _run(model, lconf, mv(o), mv(n), BG // WORLD)
    flat = model._arena.detach().clone()
    gathered = [torch.empty_like(flat) for _ in range(WORLD)]
    dist.all_gather(gathered, flat)
    same = all(torch.equal(gathered[0], g) for g in gathered)
    maxdiff = max(float((gathered[0] - g).abs().max()) for g in gathered)
    if rank == 0:
        torch.save(dict(norms=norms, same=same, maxdiff=maxdiff, params={k: v.cpu().clone() for k, v in model.state_dict().items()}), out)
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_matches_single_gpu_global_batch(tmp_path):
    out = str(tmp_path / "dp.pt")
    port = 29600 + os.getpid() % 2000
    mp.spawn(_worker, args=(port, out), nprocs=WORLD, join=True)
    got = torch.load(out)
    assert got["same"], f"ranks diverged after one data-parallel step (max |delta| {got['maxdiff']:.3e})"
    dev = "cuda:0"
    conf, obs, noise = _inputs()
    conf = make_conf("tiny", device=dev, batch_size=BG)
    model = Dreamer(conf).to(dev)
    model.fp16_forward = False
    model.implicit_conv = False
    model.load_state_dict(seeded_state_dict(model.state_dict(), 3))
    model._ensure_arena()
    model.ops.set_gemm_impl(1)
    model.ops.set_round_operands(False)
    mv = lambda d: {k: v.to(dev) for k, v in d.items()}
    norms = _run(model, conf, mv(obs), mv(noise), BG)
    for k, v in norms.items():
        assert abs(got["norms"][k] - v) <= 2e-3 * max(abs(v), 1e-6), (k, got["norms"][k], v)
    for k, v in model.state_dict().items():
        assert torch.allclose(got["params"][k], v.cpu(), rtol=2e-3, atol=1e-5), k

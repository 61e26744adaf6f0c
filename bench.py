#!/usr/bin/env python
"""bench.py — gradient-steps/sec (and imagined-samples/sec) of the Dreamer training step on H100.

  python bench.py --gpus N --steps K --warmup W            # our arm (hand-written sm_90a kernels)
  python bench.py --impl reference --gpus N ...            # the reference's own CPU path (rank 0 only)

One "step" = Dreamer.training_step + 4x backward + grad_clip(200,200) + 4x AdamW on one synthetic replay batch
(BASELINE.json configs[1]: Atari shape, deter 2048, stoch 32x32, batch 50 x seq 50, imag_horizon 15, 64x64x3) —
the reference's own `train/fps` (train.py:243-246) minus data loading.  Prints ONE JSON line (rank 0).

  value : steps/s with the batch already resident in HBM (CUDA events, max over ranks)
  e2e   : the same through the public module API with the batch copied from pinned host memory every step and
          the four losses read back to the host inside the timed region
  roofline : the dominant kernel (pd_gemm_tf32_kernel: TMA-fed wgmma / mma.sync GEMM, tf32 and fp16 launches) — algorithmic
          FLOPs of every launch in one step / their CUDA-event durations, against MEASURED_PEAKS.json; split per operand
          kind, plus the top HBM-bound kernels (algorithmic bytes / CUDA-event time vs the measured copy bandwidth)
  cpu_baseline : the unmodified reference on this box's host cores at the FULL batch (rank 0, N=1): 1 small warm-up +
          2 timed steps
  reference_gpu_eager : the unmodified reference (eager PyTorch fp32, cudnn.benchmark, train.py:30-31,143,166) on the same
          GPU, CUDA events, its own clock record — the denominator of north_star's 20x target (rank 0, N=1)

`--impl reference` times the reference's CPU path at the full batch; a CPU step takes ~15 s, so it times
min(K, 3) steps after min(W, 1) warm-up and reports THOSE counts in `steps` / `warmup`.

`--dump-outputs DIR` writes what the last timed step returned (the four losses, the output state, the metrics and the
per-timestep tensors) as DIR/<name>.npy in float32; an array above 2**20 elements is replaced by a fixed, seeded sample of
its flattened values.  Weights, batch and sampling noise are seeded, so two builds run with the same arguments can be
compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# FLOPs of one gradient step at the Atari shape, counted with torch.utils.flop_counter on the reference
# (SURVEY.md §8a row a17): 3113.3 G forward + 1519.7 G backward.
ALGO_FLOPS_ATARI = 4.633e12


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="atari")
    ap.add_argument("--gemm", default="tc", choices=["tc", "simt"])
    ap.add_argument("--dump-outputs", default="", metavar="DIR", help="write the last timed step's outputs here as .npy")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-ref-gpu", action="store_true", help="skip the reference-eager-on-this-GPU measurement")
    ap.add_argument("--ref-device", default="cpu", help="device of the --impl reference arm (cpu per the contract)")
    ap.add_argument("--ref-batch", type=int, default=0, help="sequences per reference sample step (0 = auto)")
    ap.add_argument("--dump-gemm-profile", default="", help="write the per-shape GEMM timing table of one step here")
    ap.add_argument("--cpu-threads", type=int, default=0, help="threads for the CPU reference (0 = calibrate)")
    ap.add_argument("--watchdog", type=int, default=int(os.environ.get("PD_BENCH_WATCHDOG", "0")),
                    help="dump all Python stacks to stderr and exit after this many seconds (0 = off)")
    a = ap.parse_args()
    if a.watchdog > 0:
        import faulthandler
        faulthandler.dump_traceback_later(a.watchdog, exit=True)
    return a


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return dict(hbm_gbs=d["hbm_gbs"], bf16_burst=d["bf16_tflops"], bf16_sustained=d["bf16_tflops_sustained"],
                    source="measured (MEASURED_PEAKS.json)")
    # not measured: NVIDIA's H100 SXM data sheet (dense BF16, 700 W card); a power-limited card reaches less
    return dict(hbm_gbs=3350.0, bf16_burst=989.0, bf16_sustained=989.0, source="H100 SXM data sheet (not measured)")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index
        self.t0 = self.t1 = None

    # nvidia-smi can take about a second to come up — longer than a 20-step timed region — so the sampler is
    # started before the warm-up steps and begin() / end() bracket the timed region: summary() keeps the rows that
    # arrived inside it (plus one sampling period either side; the GPU runs the same steps there).
    def begin(self):
        self.t0 = time.time()

    def end(self):
        self.t1 = time.time()

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([time.time()] + [x.strip() for x in line.split(",")])

    def __exit__(self, *a):
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                pass

    def summary(self):
        sm, mx, reasons = [], 0.0, set()
        names = ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap")
        for ts, *r in self.rows:
            if self.t0 is not None and not (self.t0 - 0.12 <= ts <= (self.t1 or time.time()) + 0.12):
                continue
            try:
                sm.append(float(r[0])); mx = max(mx, float(r[1]))
                for n, v in zip(names, r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                pass
        sm.sort()
        return dict(sm_mhz=sm[len(sm) // 2] if sm else None, sm_max_mhz=mx or None, reasons=sorted(reasons),
                    samples=len(sm))


# ----------------------------------------------------------------------------------------------------------------------
def reference_module():
    """(Dreamer class, kind): the unmodified reference installed under baseline/_ref if present (it is git-ignored), else
    the oracle port."""
    ref_path = os.path.join(ROOT, "baseline", "_ref")
    if os.path.isdir(os.path.join(ref_path, "pydreamer")):
        sys.path.insert(0, ref_path)
        try:
            from pydreamer.models import Dreamer as RefDreamer  # the reference's own module

            return RefDreamer, "reference"
        except Exception:
            pass
    return None, "port"


def host_cores():
    """Cores this process may really use: affinity mask capped by the cgroup CPU quota."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            q, per = f.read().split()
        if q != "max":
            n = max(1, min(n, int(float(q) / float(per) + 0.5)))
    except Exception:
        pass
    return n


def pick_cpu_threads(conf, requested=0):
    """The eager CPU path does not scale to arbitrarily many threads at these tensor sizes (and oversubscribing a
    cgroup-limited box is catastrophic), so probe a few thread counts on a 1-sequence step and keep the fastest."""
    if requested:
        torch.set_num_threads(requested)
        return requested
    avail = host_cores()
    cands = sorted({c for c in (avail, 64, 32, 16, 8) if c <= avail}, reverse=True) or [1]
    best, best_t = cands[-1], float("inf")
    for c in reversed(cands):                       # ascending
        torch.set_num_threads(c)
        t, _ = time_reference(conf, "cpu", 1, 1, 1)
        if t < best_t * 0.95:
            best, best_t = c, t
        else:
            break
    torch.set_num_threads(best)
    return best


def time_reference(conf, device, B, steps, warmup):
    """Seconds per gradient step of the reference path at batch B (its own Dreamer if installed, else the oracle).
    CPU: wall clock per step.  GPU: CUDA events around the timed steps (eager launches are asynchronous)."""
    from pydreamer_b200.replay import synthetic_batch

    torch.distributions.Distribution.set_default_validate_args(False)       # train.py:30
    RefDreamer, kind = reference_module()
    obs = synthetic_batch(conf, seed=1234, B=B, device=device)
    on_gpu = str(device) != "cpu"
    if kind == "reference":
        if on_gpu:
            torch.backends.cudnn.benchmark = True                            # train.py:31
        model = RefDreamer(conf).to(device)
        opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
        st = {"s": model.init_state(B * conf.iwae_samples)}

        def one():
            losses, st["s"], *_ = model.training_step(obs, st["s"])
            for o in opts:
                o.zero_grad()
            for l in losses:
                l.backward()
            model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
            for o in opts:
                o.step()
    else:
        from oracle import dreamer_oracle as O
        from pydreamer_b200.dreamer import Dreamer

        sd = {k: v.to(device).requires_grad_(not k.startswith("ac.critic_target"))
              for k, v in Dreamer(conf).state_dict().items()}
        params = [v for v in sd.values() if v.requires_grad]
        opt = torch.optim.AdamW(params, lr=conf.adam_lr, eps=conf.adam_eps)
        st = {"s": (torch.zeros(B, conf.deter_dim, device=device),
                    torch.zeros(B, conf.stoch_dim * conf.stoch_discrete, device=device))}

        def one():
            noise = O.draw_noise(conf, conf.batch_length, B, device=device)
            res = O.training_step(sd, conf, obs, st["s"], noise)
            opt.zero_grad()
            for l in res["losses"]:
                l.backward()
            torch.nn.utils.clip_grad_norm_(params, conf.grad_clip)
            opt.step()
            st["s"] = res["out_state"]

    for _ in range(warmup):
        one()
    if on_gpu:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            one()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1000.0 / steps, kind
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    return (time.perf_counter() - t0) / steps, kind


def time_reference_cpu_full(conf, threads_requested=0, steps=2):
    """The reference's CPU path at the FULL benchmark batch: thread-count calibration on 1-sequence steps, one 5-sequence
    warm-up (allocator / oneDNN primitive caches), then `steps` timed full-batch steps.  -> (s/step, kind, cores, sample)"""
    cores = pick_cpu_threads(conf, threads_requested)
    time_reference(conf, "cpu", max(1, conf.batch_size // 10), 1, 0)
    sec, kind = time_reference(conf, "cpu", conf.batch_size, steps, 0)
    sample = (f"full batch: {conf.batch_size} sequences x T={conf.batch_length}, H={conf.imag_horizon}, I={conf.iwae_samples}; "
              f"1 warm-up step at {max(1, conf.batch_size // 10)} sequences + {steps} timed full-batch steps ({sec:.1f} s each) "
              f"on {cores} threads")
    return sec, kind, cores, sample


def run_reference(args):
    from pydreamer_b200.config import make_conf

    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return                               # rank 0 alone times the CPU reference; the others exit without touching CUDA
    conf = make_conf(args.config, device=args.ref_device)
    full_B = conf.batch_size
    T, I, H = conf.batch_length, conf.iwae_samples, conf.imag_horizon
    if args.ref_device == "cpu":
        # a full-batch CPU step is ~15 s: time min(K,3) of them after min(W,1) warm-up and SAY so in steps / warmup
        steps, warmup = max(1, min(args.steps, 3)), min(args.warmup, 1)
        cores = pick_cpu_threads(conf, args.cpu_threads)
        B = args.ref_batch or full_B
        if warmup:
            time_reference(conf, "cpu", max(1, B // 10), 1, 0)
        sec, kind = time_reference(conf, "cpu", B, steps, 0)
        clocks = None
        sample = (f"{B} of {full_B} sequences x T={T}, H={H} per step on cpu, {cores} threads; {steps} timed steps after "
                  f"{warmup} warm-up step (at {max(1, B // 10)} sequences); requested --steps {args.steps} --warmup {args.warmup}")
    else:
        steps, warmup, cores, B = args.steps, max(args.warmup, 3), 0, args.ref_batch or full_B
        with ClockSampler(0) as cs:
            sec, kind = time_reference(conf, args.ref_device, B, steps, warmup)
        clocks = cs.summary()
        sample = f"{B} of {full_B} sequences x T={T}, H={H} per step on {args.ref_device} (eager PyTorch fp32, cudnn.benchmark)"
    scale = full_B / B                      # 1 unless --ref-batch asks for a sub-batch
    sps = 1.0 / (sec * scale)
    line = dict(metric="grad_steps_per_sec", value=sps, unit="steps/s", impl="reference", n_gpus=args.gpus,
                steps=steps, warmup=warmup, ms_per_step=1000.0 * sec * scale, higher_is_better=True,
                scaling="weak", vs_baseline=None, dtype="f32", data="synthetic",
                imagined_samples_per_sec=sps * T * full_B * I * H,
                config=dict(workload=f"{args.config}: Dreamer.training_step+4x backward+grad_clip+4x AdamW, per-GPU B={full_B} "
                                     f"T={T} H={H} I={I} deter={conf.deter_dim} stoch={conf.stoch_dim}x{conf.stoch_discrete} "
                                     f"image 64x64x3", global_batch=full_B, seq_len=T, parallelism="cpu" if cores else "1 gpu eager",
                            ref_device=args.ref_device),
                cpu_baseline=dict(value=sps, unit="steps/s", cores=cores, kind=kind, sample=sample),
                e2e=dict(value=sps, unit="steps/s", h2d_bytes_per_step=0, d2h_bytes_per_step=0))
    if clocks is not None:
        line["clocks"] = clocks
    print(json.dumps(line))


# ----------------------------------------------------------------------------------------------------------------------
DUMP_MAX_ELEMS = 1 << 20       # per array; with the step's ~30 outputs the dump stays far below 64 MB


def dump_outputs(d, last):
    """Write the outputs of the last timed step (see the module docstring) as float32 .npy files under `d`."""
    import numpy as np

    os.makedirs(d, exist_ok=True)
    arrays = {f"loss_{n}": l for n, l in zip(("model", "probe", "actor", "critic"), last["losses"])}
    arrays.update(state_h=last["state"][0], state_z=last["state"][1])
    arrays.update({f"metric_{k}": v for k, v in last["metrics"].items()})
    arrays.update({f"tensor_{k}": v for k, v in last["tensors"].items()})
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy() if torch.is_tensor(t) else np.asarray(t, np.float32)
        if a.size > DUMP_MAX_ELEMS:
            a = a.reshape(-1)[np.sort(np.random.default_rng(0).choice(a.size, DUMP_MAX_ELEMS, replace=False))]
        np.save(os.path.join(d, name + ".npy"), a.astype(np.float32))


def run_ours(args):
    import torch.distributed as dist

    from pydreamer_b200.config import make_conf
    from pydreamer_b200.dreamer import Dreamer
    from pydreamer_b200.replay import obs_bytes, synthetic_batch

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        import datetime
        # a stuck collective aborts the job after 3 minutes instead of wedging the box (NCCL watchdog), and so does the
        # Python-level watchdog below if the device itself stops answering
        dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=180))
        if args.watchdog <= 0:
            import faulthandler
            faulthandler.dump_traceback_later(900, exit=True)
    conf = make_conf(args.config, device=str(dev))
    T, B, I, H = conf.batch_length, conf.batch_size, conf.iwae_samples, conf.imag_horizon
    torch.manual_seed(1234 + rank)                                     # same weights and sampling noise on every run
    model = Dreamer(conf).to(dev)
    model._ensure_arena()
    if args.gemm == "simt":
        model.ops.set_gemm_impl(1)
    if world > 1:
        from pydreamer_b200.parallel import GradAllReduce

        model._dp = GradAllReduce(world)
        model._dp.broadcast_params(model)
    opts = model.init_optimizers(conf.adam_lr, conf.adam_lr_actor, conf.adam_lr_critic, conf.adam_eps)
    host = synthetic_batch(conf, seed=1234 + rank, pin=True)           # per-rank shard of the global batch (weak scaling)
    dev_obs = {k: v.to(dev) for k, v in host.items()}
    state = {"s": model.init_state(B * I)}
    host_loss = torch.empty(4, pin_memory=True)
    last = {}

    def step(obs):
        losses, state["s"], metrics, tensors, _ = model.training_step(obs, state["s"])
        last.update(losses=losses, state=state["s"], metrics=metrics, tensors=tensors)
        for o in opts:
            o.zero_grad()
        for l in losses:
            l.backward()
        model.grad_clip(conf.grad_clip, conf.grad_clip_ac)
        for o in opts:
            o.step()
        return losses

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, k):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()

    n0 = model.ops.launch_count()
    step(dev_obs)                                    # first call of a shape is always launched kernel by kernel
    launches = model.ops.launch_count() - n0         # this library's kernels in one eagerly launched step
    with ClockSampler(local) as cs:                  # (started before the warm-up: see ClockSampler.begin)
        for _ in range(max(args.warmup, 3) - 1):
            step(dev_obs)
        n1 = model.ops.launch_count()
        cs.begin()
        ms = timed(lambda: step(dev_obs), args.steps)
        cs.end()
    clocks = cs.summary()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last)          # before later steps reuse the step's output buffers
    # kernels of this library that ran in the timed region: the ones launched from Python (gradient hand-over, clip, AdamW)
    # plus, per replay, the kernel nodes the step's CUDA graph re-issues (counted when it was captured)
    eager_in_region = model.ops.launch_count() - n1
    graph_nodes = max([g.get("kernels", 0) for g in model._graphs.values() if g.get("graph") is not None] or [0])
    launches_timed = eager_in_region + graph_nodes * args.steps

    # End to end through the public API: every step's batch travels from pinned host memory to the device inside the
    # timed region and its four losses travel back.  Like any input pipeline (the reference uses DataLoader workers +
    # `.to(device)`, train.py:160-161) the copy of batch k+1 runs on a side stream while step k computes.
    copy_stream = torch.cuda.Stream(device=dev)
    dbuf = [{k: torch.empty_like(v, device=dev) for k, v in host.items()} for _ in range(2)]
    ready = [torch.cuda.Event(), torch.cuda.Event()]
    consumed = [torch.cuda.Event(), torch.cuda.Event()]
    st = {"k": 0}

    def upload(slot):
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[slot])                       # previous user of this buffer is done
            for k, v in host.items():
                dbuf[slot][k].copy_(v, non_blocking=True)
            ready[slot].record(copy_stream)

    for e in consumed:
        e.record()
    upload(0)

    def e2e_step():
        slot = st["k"] & 1
        upload(slot ^ 1)                                                 # prefetch the next step's batch
        torch.cuda.current_stream().wait_event(ready[slot])
        losses = step(dbuf[slot])
        consumed[slot].record()
        host_loss.copy_(torch.stack([l.detach().reshape(-1)[0] for l in losses]), non_blocking=True)
        torch.cuda.current_stream().synchronize()                      # the caller consumes the losses every step
        st["k"] += 1

    e2e_step()
    ms_e2e = timed(e2e_step, args.steps)

    # Same, but the batch crosses PCIe in the replay's own format (uint8 HWC images, integer actions) and is converted on
    # the device by pydreamer_b200.preprocess.GpuPreprocessor (SURVEY.md §8f N3): 4x fewer bytes per step.
    e2e_u8 = None
    if conf.actor_dist == "onehot":
        from pydreamer_b200.preprocess import GpuPreprocessor

        gp = GpuPreprocessor(conf, dev)
        raw = dict(image=((host["image"] + 0.5) * 255).round().clamp(0, 255).to(torch.uint8).permute(0, 1, 3, 4, 2).contiguous().pin_memory(),
                   action=host["action"].argmax(-1).pin_memory(), reward=host["reward"].clone().pin_memory(),
                   terminal=host["terminal"].clone().pin_memory(), reset=host["reset"].clone().pin_memory())
        rbuf = [{k: torch.empty_like(v, device=dev) for k, v in raw.items()} for _ in range(2)]

        def upload_raw(slot):
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(consumed[slot])
                for k, v in raw.items():
                    rbuf[slot][k].copy_(v, non_blocking=True)
                ready[slot].record(copy_stream)

        torch.cuda.synchronize()
        for e in consumed:
            e.record()
        st["k"] = 0
        upload_raw(0)

        def e2e_u8_step():
            slot = st["k"] & 1
            upload_raw(slot ^ 1)
            torch.cuda.current_stream().wait_event(ready[slot])
            obs = gp.apply(rbuf[slot])
            consumed[slot].record()
            losses = step(obs)
            host_loss.copy_(torch.stack([l.detach().reshape(-1)[0] for l in losses]), non_blocking=True)
            torch.cuda.current_stream().synchronize()
            st["k"] += 1

        e2e_u8_step()
        ms_u8 = timed(e2e_u8_step, args.steps)
        e2e_u8 = dict(value=world * args.steps / (ms_u8 / 1000.0), unit="steps/s", h2d_bytes_per_step=obs_bytes(raw),
                      d2h_bytes_per_step=16, ms_per_step=ms_u8 / args.steps,
                      note="raw replay format (uint8 HWC image, int64 action) + device-side preprocessing")

    # ---- roofline of the dominant kernel: every pd_gemm launch of one step, CUDA-event timed
    graphs_on, model.use_cuda_graph = model.use_cuda_graph, False      # per-launch events need eager launches
    overlap_on, model.overlap = model.overlap, 0                       # ... on ONE stream: concurrent branches would stretch them
    step(dev_obs)                                                      # warm-up of this schedule (allocates its scratch buffers)
    torch.cuda.synchronize()
    model.ops.gemm_profile = []
    # the HBM-bound kernels with the most traffic: CUDA events around each launch + their ALGORITHMIC bytes (every operand
    # read once, every result written once)
    hbm_prof = {}

    def timed_op(name, nbytes):
        orig = getattr(model.ops, name)

        def wrapper(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r = orig(*a, **k); e1.record()
            hbm_prof.setdefault(name, []).append((e0, e1, nbytes(*a, **k)))
            return r
        setattr(model.ops, name, wrapper)
        return lambda: delattr(model.ops, name)

    nb = lambda *ts: float(sum(t.numel() * t.element_size() for t in ts if t is not None))
    undo = [
        # (col, NB, Hin, Win, Cc, k, bias, target, tgt_div, dec, diff, loss, csum)
        timed_op("col2im_imgloss", lambda col, NB, Hin, Win, Cc, k, bias, target, div, dec, diff, loss, csum:
                 nb(col, dec, diff) + nb(target) / max(1, conf.iwae_samples)),
        timed_op("ln_elu_fwd", lambda x, g, b_, eps, y, mean, rstd, y16=None: nb(x, y, y16)),
        timed_op("adamw", lambda p_, g, m, v, *a: 7.0 * nb(p_)),       # read p,g,m,v + write p,m,v
        timed_op("col2im", lambda col, Hin, Win, k, bias, act, out, round_out=True: nb(col, out)),
        timed_op("im2col", lambda inp, k, korder, col, round_out=True: nb(col) + float(inp.numel() * 4)),
        # (col, Hin, Win, k, dact, dbias, out): column matrix + saved activation read, gradient image written
        timed_op("col2im_actbwd", lambda col, Hin, Win, k, dact, dbias, out: nb(col, dact, out)),
        timed_op("gru_fwd", lambda gi, gh, hprev, hout, *a, **k: nb(gi, gh, hprev, hout) + 4.0 * nb(hout)),   # + gates (4 D per row)
        timed_op("ln_elu_bwd", lambda dy, x, y, *a, **k: 4.0 * nb(dy)),                                      # dy, x, y read, dx written
    ]
    step(dev_obs)
    torch.cuda.synchronize()
    for u in undo:
        u()
    prof, model.ops.gemm_profile = model.ops.gemm_profile, None

    class PhaseTimer:
        def __init__(self):
            self.ev = [("start", torch.cuda.Event(enable_timing=True))]
            self.ev[0][1].record()

        def mark(self, name):
            e = torch.cuda.Event(enable_timing=True); e.record(); self.ev.append((name, e))

    model._phase_timer = pt = PhaseTimer()
    step(dev_obs)
    pt.mark("backward()+clip+adamw")
    torch.cuda.synchronize()
    model._phase_timer = None
    phases = {n: round(a[1].elapsed_time(b), 3) for a, (n, b) in zip(pt.ev[:-1], pt.ev[1:])}
    model.use_cuda_graph = graphs_on
    model.overlap = overlap_on
    if args.dump_gemm_profile and rank == 0:
        agg = {}
        for e0, e1, f, shp in prof:
            a = agg.setdefault(shp, [0, 0.0, 0.0])
            a[0] += 1; a[1] += e0.elapsed_time(e1); a[2] += f
        rows = sorted(([list(k), v[0], v[1], v[2], v[2] / max(v[1], 1e-9) / 1e9] for k, v in agg.items()), key=lambda r: -r[2])
        with open(args.dump_gemm_profile, "w") as f:
            json.dump(dict(columns=["(M,N,K,a_mn,b_mn,acc)", "launches", "ms", "flops", "TFLOP/s"], rows=rows), f, indent=0)
    gemm_ms = sum(e0.elapsed_time(e1) for e0, e1, _, _ in prof)
    gemm_flops = sum(f for _, _, f, _ in prof)
    pk = peaks()
    # per operand kind: fp16 launches (pd_gemm_f16) carry "f16" in their shape key, everything else runs tf32
    buckets = {}
    for e0, e1, f, shp in prof:
        kind = "f16" if shp[3] == "f16" else "tf32"
        bk = buckets.setdefault(kind, dict(launches=0, ms=0.0, flops=0.0))
        bk["launches"] += 1; bk["ms"] += e0.elapsed_time(e1); bk["flops"] += f
    for kind, bk in buckets.items():
        bk["tflops"] = bk["flops"] / max(bk["ms"], 1e-9) / 1e9
        # denominator: the bf16 rate (16-bit operands); TF32's MMA rate is half of the 16-bit rate
        bk["peak"] = pk["bf16_sustained"] * (1.0 if kind == "f16" else 0.5)
        bk["frac"] = bk["tflops"] / bk["peak"]
        bk["share_of_gemm_flops"] = bk["flops"] / max(gemm_flops, 1.0)
    hbm_kernels = []
    for name, rows in hbm_prof.items():
        ms_k = sum(a.elapsed_time(b) for a, b, _ in rows)
        by = sum(c for _, _, c in rows)
        hbm_kernels.append(dict(kernel=name, launches=len(rows), ms=round(ms_k, 4), algorithmic_bytes=by,
                                achieved_gbs=by / max(ms_k, 1e-9) / 1e6, frac=by / max(ms_k, 1e-9) / 1e6 / pk["hbm_gbs"]))
    hbm_kernels.sort(key=lambda r: -r["ms"])
    steps_per_s = world * args.steps / (ms / 1000.0)
    e2e_per_s = world * args.steps / (ms_e2e / 1000.0)
    per_step_samples = T * B * I * H
    achieved = gemm_flops / (gemm_ms / 1000.0) / 1e12 if gemm_ms > 0 else 0.0
    line = dict(
        metric="grad_steps_per_sec", value=steps_per_s, unit="steps/s", n_gpus=world, steps=args.steps,
        global_steps_per_sec=steps_per_s / world,
        warmup=max(args.warmup, 3), ms_per_step=ms / args.steps, higher_is_better=True, scaling="weak",
        vs_baseline=None, dtype="tf32 (fp32 storage + accumulate); fp16 operands on forward-only layers" if model.fp16_forward else "tf32 (fp32 storage + accumulate)", data="synthetic",
        imagined_samples_per_sec=steps_per_s * per_step_samples,
        config=dict(workload=f"{args.config}: Dreamer.training_step+4x backward+grad_clip+4x AdamW, per-GPU B={B} T={T} H={H} "
                             f"I={I} deter={conf.deter_dim} stoch={conf.stoch_dim}x{conf.stoch_discrete} image 64x64x3",
                    global_batch=B * world, seq_len=T, parallelism=f"dp{world}",
                    l2="per-step working set (GBs of activations) is far larger than the 50 MB L2; no flush needed"),
        e2e=dict(value=e2e_per_s, unit="steps/s", h2d_bytes_per_step=obs_bytes(host), d2h_bytes_per_step=16,
                 ms_per_step=ms_e2e / args.steps),
        e2e_uint8=e2e_u8,
        gpu_launches=int(launches_timed),
        gpu_launches_note=f"{graph_nodes} kernel nodes per CUDA-graph replay x {args.steps} steps + {eager_in_region} launched from "
                          f"Python in the timed region (gradient hand-over, clip, AdamW); one eagerly launched step = {int(launches)}",
        phases_ms_eager=phases,
        launches_per_step=int(launches),
        clocks=clocks,
        roofline=dict(bound="tensor", kernel="pd_gemm_tf32_kernel (TMA + wgmma / mma.sync, tf32 and fp16 launches)",
                      achieved=achieved, peak=pk["bf16_sustained"], unit="TFLOP/s", frac=achieved / pk["bf16_sustained"],
                      peak_source=pk["source"] + ": bf16 dense; tf32 launches can reach half of it",
                      by_operand_kind=buckets,
                      gemm_launches_per_step=len(prof), gemm_ms_per_step=gemm_ms,
                      gemm_share_of_step=gemm_ms / (ms / args.steps), gemm_flops_per_step=gemm_flops,
                      step_algorithmic_tflop=ALGO_FLOPS_ATARI / 1e12 if args.config == "atari" else None,
                      step_tflops=(ALGO_FLOPS_ATARI / 1e12) / (ms / args.steps / 1000.0) if args.config == "atari" else None,
                      hbm_kernels=hbm_kernels[:8], hbm_peak_gbs=pk["hbm_gbs"]),
    )
    if rank == 0 and world == 1 and not args.no_ref_gpu:
        # the denominator of north_star's ">= 20x the reference's 1-GPU PyTorch steps/s": the unmodified reference, eager fp32
        # on this same GPU (train.py:30-31,143,166), after our own measurement so nothing of it overlaps ours
        try:
            model._ws.clear(); model._graphs.clear()
            torch.cuda.empty_cache()
            gconf = make_conf(args.config, device=str(dev))
            with ClockSampler(local) as cs2:
                sec_g, kind_g = time_reference(gconf, str(dev), B, 20, 5)
            if kind_g == "reference":
                line["reference_gpu_eager"] = dict(value=1.0 / sec_g, unit="steps/s", ms_per_step=1000.0 * sec_g, steps=20,
                                                   warmup=5, clocks=cs2.summary(),
                                                   how="unmodified reference Dreamer on the same GPU: eager PyTorch fp32, "
                                                       "cudnn.benchmark, TF32 matmul off (torch default), CUDA events")
                line["vs_reference_gpu_eager"] = dict(ratio=steps_per_s * sec_g, e2e_ratio=e2e_per_s * sec_g, target=20.0)
        except Exception as e:                   # the reference arm must never take the headline down with it
            line["reference_gpu_eager"] = dict(unavailable=f"{type(e).__name__}: {e}"[:200])
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cconf = make_conf(args.config, device="cpu")
        sec, kind, cores, sample = time_reference_cpu_full(cconf, args.cpu_threads, steps=2)
        line["cpu_baseline"] = dict(value=1.0 / sec, unit="steps/s", cores=cores, kind=kind, sample=sample)
    if rank == 0:
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)

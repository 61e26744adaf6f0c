"""Time the five per-timestep input-gradient GEMMs of the posterior unroll's BPTT one shape at a time.

Each shape is dX[B*I, in] = dY[B*I, out] . W[out, in] through `ops.gemm(..., b_mn=True)`, as Dreamer._wm_backward calls it
(with the residual where the chain adds one).  A launch reads the whole fp32 weight, so the rate that matters is bytes per
second: weight + dY + residual read, dX written, once each.  Launches are captured in a CUDA graph (the training step
replays one too) and cycle through enough copies of the weight to exceed the 50 MB L2, as the chain does when it moves on
to the next weight.  Rates are set against the device-to-device copy bandwidth measured here (read + write bytes of a 1 GB
copy) and against MEASURED_PEAKS.json if present, otherwise the H100 SXM data sheet's 3.35 TB/s.

    python tools/bench_skinny_gemm.py [--config atari] [--iters 200] [--out FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

L2_BYTES = 50 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["", ""])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "")
    return dict(name=name, power_limit=power)


def reference_bandwidth():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return json.load(f)["hbm_gbs"], "measured (MEASURED_PEAKS.json)"
    return 3350.0, "H100 SXM data sheet (not measured)"


def graph_time_ms(fn, iters):
    """Milliseconds per call of fn, captured `iters` times in one CUDA graph and replayed (after one warm replay)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(3):
            fn(i)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / iters)
    return best


def copy_gbs():
    src = torch.empty(256 << 20, device="cuda")                    # 1 GB
    dst = torch.empty_like(src)
    ms = graph_time_ms(lambda i: dst.copy_(src), 10)
    return 2 * src.numel() * 4 / (ms / 1e3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="atari")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    from pydreamer_b200.config import make_conf
    from pydreamer_b200.ops import NativeOps

    conf = make_conf(a.config)
    D, Hd, Z, M = conf.deter_dim, conf.hidden_dim, conf.stoch_dim * conf.stoch_discrete, conf.batch_size * conf.iwae_samples
    # (name, N = in, K = out, residual): the order of one timestep of the chain
    shapes = [("post_mlp", Hd, Z, False), ("post_mlp_h", D, Hd, True), ("gru.weight_hh", D, 3 * D, True),
              ("gru.weight_ih", Hd, 3 * D, False), ("z_mlp", Z, Hd, False)]
    ops = NativeOps("cuda:0")
    gen = torch.Generator(device="cuda").manual_seed(0)
    ref_gbs, ref_src = reference_bandwidth()
    cp = copy_gbs()
    rows = []
    print(f"{'weight':14s} {'M':>3s} {'N':>5s} {'K':>5s} {'MB':>6s} {'us':>8s} {'GB/s':>7s} {'of copy':>8s} {'of ref':>7s}")
    for name, N, K, res in shapes:
        wbytes = K * N * 4
        copies = max(1, math.ceil(2 * L2_BYTES / wbytes))
        Ws = [torch.randn(K, N, device="cuda", generator=gen) / math.sqrt(K) for _ in range(copies)]
        A = torch.randn(M, K, device="cuda", generator=gen)
        R = torch.randn(M, N, device="cuda", generator=gen) if res else None
        C = torch.empty(M, N, device="cuda")
        ms = graph_time_ms(lambda i: ops.gemm(A, Ws[i % copies], C, b_mn=True, res=R), a.iters)
        nbytes = wbytes + 4 * (M * K + M * N * (2 if res else 1))
        gbs = nbytes / (ms / 1e3) / 1e9
        rows.append(dict(weight=name, M=M, N=N, K=K, bytes=nbytes, us=ms * 1e3, gbs=gbs, of_copy=gbs / cp, of_ref=gbs / ref_gbs))
        print(f"{name:14s} {M:3d} {N:5d} {K:5d} {nbytes / 1e6:6.1f} {ms * 1e3:8.2f} {gbs:7.0f} {gbs / cp:8.2f} {gbs / ref_gbs:7.2f}")
        del Ws
    step_us = sum(r["us"] for r in rows)
    print(f"one timestep of the chain: {step_us:.1f} us; x T = {conf.batch_length}: {step_us * conf.batch_length / 1e3:.2f} ms")
    out = dict(card=card(), config=a.config, copy_gbs=cp, reference_gbs=ref_gbs, reference_source=ref_src, shapes=rows,
               chain_us_per_timestep=step_us)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

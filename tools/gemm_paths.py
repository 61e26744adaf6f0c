"""Per-path GEMM time of one training step, before and after a change.

Reads the tables that `bench.py --dump-gemm-profile FILE` writes (one CUDA-event-timed eager step: per shape key
(M, N, K, a_mn | "f16" | "convN", b_mn | o_mn, accumulate) the launches, milliseconds and FLOPs), groups the rows by the
operand layouts the tensor-core kernel sees, and prints milliseconds and TFLOP/s per group.  Several files per side
(repeated runs) are reduced to the median milliseconds of each group.

    python tools/gemm_paths.py --before a1.json a2.json --after b1.json b2.json
"""
import argparse
import json
import statistics

GROUPS = [
    "fp16, both K-major",
    "tf32, both K-major",
    "dense weight gradients (A and B MN-major, accumulate)",
    "conv weight gradients (im2col modes 2 and 3)",
    "input gradients (B MN-major), M > 64",
    "conv form 1 with MN-major weights (o_mn)",
    "BPTT chain input gradients (B MN-major), M <= 64",
    "other MN-major",
]


def group(key):
    M, _, _, kind, mn2, acc = key
    if kind == "f16":
        return GROUPS[0]
    if kind in ("conv2", "conv3"):
        return GROUPS[3]
    if kind == "conv1":
        return GROUPS[5] if mn2 else GROUPS[1]
    a_mn, b_mn = int(kind), int(mn2)
    if not a_mn and not b_mn:
        return GROUPS[1]
    if a_mn and b_mn and acc:
        return GROUPS[2]
    if b_mn and not a_mn:
        return GROUPS[6] if M <= 64 else GROUPS[4]
    return GROUPS[7]


def load(path):
    """group -> [launches, ms, flops] of one profile file."""
    out = {}
    with open(path) as f:
        rows = json.load(f)["rows"]
    for key, launches, ms, flops, _ in rows:
        a = out.setdefault(group(key), [0, 0.0, 0.0])
        a[0] += launches; a[1] += ms; a[2] += flops
    return out


def reduce(paths):
    runs = [load(p) for p in paths]
    out = {}
    for gname in GROUPS:
        have = [r[gname] for r in runs if gname in r]
        if have:
            out[gname] = [have[0][0], statistics.median(h[1] for h in have), have[0][2]]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--before", nargs="+", required=True)
    ap.add_argument("--after", nargs="+", required=True)
    ap.add_argument("--json", default="", help="also write the table here")
    a = ap.parse_args()
    before, after = reduce(a.before), reduce(a.after)
    table = []
    print(f"{'group':54s} {'launches':>8s} {'GFLOP':>8s} {'ms before':>10s} {'ms after':>9s} {'TF/s before':>11s} "
          f"{'TF/s after':>10s} {'after/before':>12s}")
    tot = [0.0, 0.0]
    for gname in GROUPS:
        if gname not in before and gname not in after:
            continue
        n, mb, fl = before.get(gname, after.get(gname))
        ma = after.get(gname, [0, 0.0, 0.0])[1]
        mb = before.get(gname, [0, 0.0, 0.0])[1]
        tot[0] += mb; tot[1] += ma
        row = dict(group=gname, launches=n, gflop=fl / 1e9, ms_before=mb, ms_after=ma,
                   tflops_before=fl / mb / 1e9 if mb else None, tflops_after=fl / ma / 1e9 if ma else None,
                   ratio=ma / mb if mb else None)
        table.append(row)
        print(f"{gname:54s} {n:8d} {fl / 1e9:8.0f} {mb:10.2f} {ma:9.2f} {row['tflops_before'] or 0:11.1f} "
              f"{row['tflops_after'] or 0:10.1f} {row['ratio'] or 0:12.3f}")
    print(f"{'all GEMM launches':54s} {'':8s} {'':8s} {tot[0]:10.2f} {tot[1]:9.2f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(groups=table, ms_before=tot[0], ms_after=tot[1]), f, indent=1)


if __name__ == "__main__":
    main()

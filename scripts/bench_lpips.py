"""LPIPS (viewformer_b200.lpips.LPIPS) throughput at 128 x 128: one pair per call (the README's ``--batch-size 1`` evaluation) and 64
pairs per call, timed with CUDA events over whole calls (the result's finiteness check included, as an evaluator pays it).  Seeded
random weights in the two files' layouts (oracle/lpips_oracle.py): the timing does not depend on the weights' values.

    python scripts/bench_lpips.py [--steps 20] [--warmup 5]

Algorithmic work: 10.02 GFLOP of VGG16 convs per 128 x 128 image (2 x MACs of the 13 convs), 20.0 per pair; exact mode runs each
tensor-core product as 3 fp16 MMAs (the 3 -> 64 first conv, 0.11 GFLOP per image, is fp32 on the CUDA cores).  Prints the card's name and
power limit next to the numbers, and one JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

SIZE = 128


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "nvidia-smi: no output"
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e!r})"


def conv_gflop_per_image(h, w):
    from viewformer_b200.lpips import CONVS, POOL_BEFORE
    flop = 0
    for idx, cin, cout in CONVS:
        if idx in POOL_BEFORE:
            h, w = h // 2, w // 2
        flop += 2 * h * w * 9 * cin * cout
    return flop / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lpips.py measures on a GPU; there is no CPU timing"
    from oracle import lpips_oracle as lo
    from viewformer_b200.lpips import LPIPS
    with tempfile.TemporaryDirectory() as d:
        metric = LPIPS(*lo.make_lpips_weights(0, d))
    g = torch.Generator().manual_seed(0)
    gflop_pair = 2 * conv_gflop_per_image(SIZE, SIZE)
    results = {"card": card(), "size": SIZE, "gflop_per_pair": round(gflop_pair, 2), "runs": {}}
    print(f"[card] {torch.cuda.get_device_name()} | nvidia-smi: {results['card']}")
    for pairs in (1, 64):
        x = torch.randint(0, 256, (2, pairs, SIZE, SIZE, 3), generator=g, dtype=torch.uint8).cuda()
        for _ in range(a.warmup):
            metric(x[0], x[1])
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.steps):
            metric(x[0], x[1])
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / a.steps
        r = {"ms_per_call": round(ms, 3), "pairs_per_s": round(pairs / ms * 1e3, 1),
             "conv_tflops": round(pairs * gflop_pair / ms, 2)}          # GFLOP / ms = TFLOP/s
        results["runs"][f"pairs{pairs}"] = r
        print(f"[lpips] {pairs:3d} pairs/call: {ms:8.3f} ms/call  {r['pairs_per_s']:9.1f} pairs/s  {r['conv_tflops']:6.2f} TFLOP/s "
              "(algorithmic VGG16 conv work, each tensor-core product as 3 fp16 MMAs)")
    print(json.dumps(results))


if __name__ == "__main__":
    main()

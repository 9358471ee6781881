"""What the fourth image channel costs: BASELINE configs[1] generate (32 scenes, 9 context views, mixed codebook + bf16 transformer,
device-resident inputs, eager launches) with a 3-channel and a 4-channel (RGBA, the CO3Dv2 layout) codebook, alternated in one process,
three timed runs of each.  Only conv_in (C -> 128) and conv_out (128 -> C) change between the two.

    python scripts/bench_rgba.py [--scenes 32] [--steps 20] [--warmup 5] [--runs 3]

Prints the card's name and power limit next to the numbers, and one JSON line at the end.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

T_VIEWS = 10


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "nvidia-smi: no output"
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e!r})"


def inputs(scenes, channels, seed=1234):
    g = torch.Generator().manual_seed(seed)
    x = torch.nn.functional.interpolate(torch.rand((scenes * T_VIEWS, channels, 16, 16), generator=g), size=(128, 128), mode="bilinear",
                                        align_corners=False)
    u8 = (x.clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1).reshape(scenes, T_VIEWS, 128, 128, channels).contiguous()
    q = torch.randn((scenes, T_VIEWS, 4), generator=g)
    q = q / q.norm(dim=-1, keepdim=True)
    cams = torch.cat([torch.randn((scenes, T_VIEWS, 3), generator=g), q * torch.where(q[..., :1] >= 0, 1.0, -1.0)], -1).contiguous()
    return u8.cuda(), cams.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rgba.py measures on a GPU; there is no CPU timing"
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions
    from viewformer_b200.config import VQGANConfig, MIGTConfig
    tcfg = MIGTConfig(localization_weight="0")
    tr = MIGT(tcfg, precision="bf16").init_weights(0)
    arms = {}
    for c in (3, 4):
        cb = VQGAN(VQGANConfig(in_channels=c, out_ch=c), precision="mixed").init_weights(0)
        images, cams = inputs(a.scenes, c)
        arms[c] = (lambda x, p, cb=cb: generate_batch_predictions(tr, cb, x, p), images, cams)
    for c, (gp, images, cams) in arms.items():
        for _ in range(a.warmup):
            gp(images, cams)
    torch.cuda.synchronize()
    times = {3: [], 4: []}
    for _ in range(a.runs):
        for c, (gp, images, cams) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                gp(images, cams)
            e1.record()
            torch.cuda.synchronize()
            times[c].append(e0.elapsed_time(e1) / a.steps)
    gpu = card()
    print(f"[bench_rgba] {gpu}; generate, {a.scenes} scenes x {T_VIEWS} views, mixed codebook + bf16 transformer, eager")
    for c in (3, 4):
        ms = times[c]
        print(f"[bench_rgba] {c} channels: ms/step {', '.join(f'{t:.3f}' for t in ms)} (median {statistics.median(ms):.3f}); "
              f"views/s {a.scenes / (statistics.median(ms) / 1e3):.1f}")
    ratio = statistics.median(times[4]) / statistics.median(times[3])
    print(f"[bench_rgba] 4-channel / 3-channel step time: {ratio:.4f}")
    print(json.dumps(dict(gpu=gpu, scenes=a.scenes, steps=a.steps, runs=a.runs, ms_3ch=times[3], ms_4ch=times[4], ratio_4_over_3=ratio)))


if __name__ == "__main__":
    main()

"""fp32-faithful vs bf16 codebook training step on one GPU: BASELINE configs[3] per-GPU shape (VQGANConfig defaults, 32 images = 256 / 8,
perceptual_weight 0).  The two trainers run alternately in one process, `--runs` timed runs each; prints median ms/step and images/s with
the card's name and power limit, read in the same process.  ``--accumulate N``: every optimizer step accumulates N micro-batches of
``--images`` images (``accumulate_grad_batches``); the rates are then per update of N x images.

    python scripts/bench_vqgan_train.py [--images 32] [--accumulate 1] [--steps 10] [--warmup 3] [--runs 3] [--json OUT]

bench.py --workload train times the fp32 step only.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32, help="images per micro-batch")
    ap.add_argument("--accumulate", type=int, default=1, help="micro-batches per optimizer step")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result here")
    a = ap.parse_args()
    from viewformer_b200 import VQGAN
    from viewformer_b200.config import VQGANConfig
    from viewformer_b200.train import VQGANTrainer
    torch.cuda.set_device(0)
    cfg = VQGANConfig(perceptual_weight=0.0)
    trainers = {p: VQGANTrainer(VQGAN(cfg, precision="fp32", device="cuda:0").init_weights(0), precision=p,
                                 accumulate_grad_batches=a.accumulate) for p in ("fp32", "bf16")}
    x = (torch.rand((a.images, 3, cfg.image_size, cfg.image_size), generator=torch.Generator().manual_seed(7)) * 2 - 1).pin_memory()
    for tr in trainers.values():
        for _ in range(a.warmup * a.accumulate):
            tr.training_step(x)
    torch.cuda.synchronize()
    ms = {p: [] for p in trainers}
    loss = {}
    for _ in range(a.runs):
        for p, tr in trainers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps * a.accumulate):
                loss[p] = tr.training_step(x)
            e1.record()
            torch.cuda.synchronize()
            ms[p].append(e0.elapsed_time(e1) / a.steps)
    name, power = card()
    res = {"gpu": name, "power_limit": power, "images_per_step": a.images * a.accumulate, "micro_batches_per_step": a.accumulate,
           "steps_per_run": a.steps, "runs": a.runs}
    for p in trainers:
        med = statistics.median(ms[p])
        res[p] = {"median_ms_per_step": med, "images_per_s": a.images * a.accumulate * 1e3 / med, "ms_per_step_runs": ms[p], "last_loss": float(loss[p])}
    res["bf16_speedup"] = res["fp32"]["median_ms_per_step"] / res["bf16"]["median_ms_per_step"]
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

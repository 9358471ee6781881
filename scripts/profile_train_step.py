"""Per-kernel breakdown of one full-size codebook training step (BASELINE configs[3] per-GPU shape: 32 images), from torch.profiler.

    python scripts/profile_train_step.py --out DIR [--images 32] [--precision fp32|bf16]

Writes DIR/kernels.md (kernel, launches, ms, share of the step's kernel time) and DIR/trace.pt.trace.json, and prints the table.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from profile_step import kernel_table  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (kernels.md, trace.pt.trace.json)")
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    a = ap.parse_args()
    from viewformer_b200 import VQGAN
    from viewformer_b200.config import VQGANConfig
    from viewformer_b200.train import VQGANTrainer
    tr = VQGANTrainer(VQGAN(VQGANConfig(perceptual_weight=0.0), precision="fp32", device="cuda:0").init_weights(0), precision=a.precision)
    x = torch.rand((a.images, 3, 128, 128), generator=torch.Generator().manual_seed(0)) * 2 - 1
    for _ in range(2):
        tr.training_step(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        tr.training_step(x)
        torch.cuda.synchronize()
    os.makedirs(a.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(a.out, "trace.pt.trace.json"))
    table = f"{torch.cuda.get_device_name(0)}, training step {a.precision}, {a.images} images\n\n" + kernel_table(prof.events())
    with open(os.path.join(a.out, "kernels.md"), "w") as f:
        f.write(table)
    print(table)


if __name__ == "__main__":
    main()

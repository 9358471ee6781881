"""Full-size transformer training step timing (MIGTConfig defaults: 12 layers, d = 768; B scenes x T views x 64 tokens), the fp32-faithful and
the bf16 trainer alternated in one process (three timed runs each, after a warm-up), with each trainer's peak allocated memory.  The default
B = 5, T = 20 is the InteriorNet recipe's batch of 40 scenes over 8 GPUs.  VF_B / VF_T / VF_STEPS change the shape and the steps per run.
``--accumulate N``: every update accumulates N micro-batches of B scenes (``accumulate_steps``); N = 8 is the InteriorNet update of 8
replicas on one GPU.  Times and rates are then per update of N x B scenes.  ``--random-pose-multiplier C``: alternate the bf16 trainer
without the pose-scale augmentation and with random_pose_multiplier C instead of the two precisions (the augmentation's cost)."""
import argparse, dataclasses, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle import synth, migt_oracle as mo
from viewformer_b200 import MIGT
from viewformer_b200.config import MIGTConfig
from viewformer_b200.train_migt import MIGTTrainer

B, T, n = int(os.environ.get("VF_B", "5")), int(os.environ.get("VF_T", "20")), int(os.environ.get("VF_STEPS", "3"))
ap = argparse.ArgumentParser()
ap.add_argument("--accumulate", type=int, default=1, help="micro-batches of B scenes per update")
ap.add_argument("--random-pose-multiplier", type=float, default=None, help="compare bf16 at c = 1 and at this c")
args = ap.parse_args()
N = args.accumulate
cfg = MIGTConfig()
model = MIGT(cfg, precision="fp32").init_weights(0)
if args.random_pose_multiplier is None:
    arms = {"fp32": ("fp32", model), "bf16": ("bf16", model)}
else:
    c = args.random_pose_multiplier
    scaled = MIGT(dataclasses.replace(cfg, random_pose_multiplier=c), precision="fp32").load_state_dict(model.state_dict())
    arms = {"bf16 c=1": ("bf16", model), f"bf16 c={c:g}": ("bf16", scaled)}
codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=1)
cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=2))[0])
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
except OSError:
    card = "unknown"
print(f"[card] {torch.cuda.get_device_name()} | nvidia-smi: {card}")


def run(tr, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        for _ in range(N):
            loss = tr.forward_backward(cams, codes)
        tr.optimizer_step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, float(loss)


trainers, times, peaks, losses = {}, {}, {}, {}
for prec, (precision, m) in arms.items():
    trainers[prec] = MIGTTrainer(m, precision=precision, accumulate_steps=N)
    times[prec] = []
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()                       # the trainers' weights, gradients and moments
    run(trainers[prec], 2)                                     # warm-up: module loads, operand buffers
    peaks[prec] = torch.cuda.max_memory_allocated() - base
for _ in range(3):
    for prec in arms:
        ms, losses[prec] = run(trainers[prec], n)
        times[prec].append(ms)
for prec in arms:
    t = np.array(times[prec])
    med = float(np.median(t))
    print(f"[migt train step, full size, {prec}] {N} x B={B} T={T}: median {med:.1f} ms/update (runs {', '.join(f'{x:.1f}' for x in t)}; "
          f"spread {t.max() - t.min():.1f} ms) -> {N * B * T * 64 / med * 1e3:.0f} tokens/s; step peak {peaks[prec] / 2**30:.2f} GiB above the trainers' state; "
          f"loss {losses[prec]:.4f}")
a, b = arms
print(f"[{b} vs {a}] {np.median(times[a]) / np.median(times[b]):.2f}x")

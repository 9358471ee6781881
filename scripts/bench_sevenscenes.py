"""What 7-Scenes localisation costs per query: the three generation procedures of evaluate_sevenscenes.py at B = 1 (the reference's
loop: standard, pose_refinement, generated_images) and pose_refinement at B = 32, on synthetic 20-view scenes (19 context frames and
the query, 128 x 128) with a 7 000-camera scene database; mixed codebook, bf16 transformer with localisation, eager launches.  Also the
nearest-camera kernel alone (7 000 cameras, k = 9, one and 32 queries) timed with CUDA events.

    python scripts/bench_sevenscenes.py [--queries 8] [--runs 3] [--out results.json]

Each number is the median of ``--runs`` timed runs of ``--queries`` queries after a warm-up, in ms per query.  Prints the card's name
and power limit next to the numbers, read in the same process, and one JSON line at the end.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

DB = 7000


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "nvidia-smi: no output"
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from oracle import synth
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions, _lib as L
    from viewformer_b200.cameras import camera_knn
    from viewformer_b200.config import VQGANConfig, MIGTConfig
    from viewformer_b200.sevenscenes import (SceneLookup, generate_batch_predictions_using_generated_images,
                                             generate_batch_predictions_using_pose_refinement)
    if not torch.cuda.is_available():
        raise SystemExit("bench_sevenscenes: no CUDA device")
    L.load(require_device=True)
    vcfg, tcfg = VQGANConfig(), MIGTConfig()
    vq = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, 0))
    tr = MIGT(tcfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(tcfg, 0))
    g = torch.Generator().manual_seed(7)
    q = torch.nn.functional.normalize(torch.randn(DB, 4, generator=g), dim=-1)
    db = torch.cat([torch.randn(DB, 3, generator=g), q * torch.where(q[:, :1] >= 0, 1.0, -1.0)], -1).numpy()
    frame_pool = synth.make_images_uint8(1, 64, size=128, seed=8)[0].numpy()                  # 7 000 frames would be 344 MB
    lookup = SceneLookup([f"frame-{i:06d}.color.png" for i in range(DB)], db, [frame_pool[i % 64] for i in range(DB)])
    B = 32
    images = synth.make_images_uint8(B, 20, size=128, seed=9)
    cams = synth.make_cameras(B, 20, seed=10)
    rng = random.Random(0)

    procs = {
        "standard_b1": (1, lambda b: generate_batch_predictions(tr, vq, images[b:b + 1], cams[b:b + 1])),
        "pose_refinement_b1": (1, lambda b: generate_batch_predictions_using_pose_refinement(lookup, db, tr, vq, images[b:b + 1],
                                                                                             cams[b:b + 1], num_gen_ctx=9, rng=rng)),
        "generated_images_b1": (1, lambda b: generate_batch_predictions_using_generated_images(
            tr, vq, images[b:b + 1], cams[b:b + 1], num_gen_ctx=5, generator=torch.Generator().manual_seed(b))),
        "pose_refinement_b32": (B, lambda b: generate_batch_predictions_using_pose_refinement(lookup, db, tr, vq, images, cams,
                                                                                              num_gen_ctx=9, rng=rng)),
    }
    res = {"card": card(), "device": torch.cuda.get_device_name()}
    print(f"[card] {res['device']} | nvidia-smi: {res['card']}")
    for name, (per_call, fn) in procs.items():
        calls = 1 if per_call > 1 else a.queries
        fn(0)
        torch.cuda.synchronize()
        runs = []
        for _ in range(a.runs):
            t0 = time.perf_counter()
            for b in range(calls):
                fn(b % B)
            torch.cuda.synchronize()
            runs.append((time.perf_counter() - t0) * 1e3 / (calls * per_call))
        res[name + "_ms_per_query"] = statistics.median(runs)
        print(f"[{name}] ms per query: median {statistics.median(runs):.3f} of {[round(r, 3) for r in runs]}")
    dbd = torch.from_numpy(db).cuda()
    for nq in (1, 32):
        qs = torch.from_numpy(db[:nq] + 0.01).cuda()
        for _ in range(10):
            camera_knn(dbd, qs, 9)
        runs = []
        for _ in range(a.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                camera_knn(dbd, qs, 9)
            e1.record()
            torch.cuda.synchronize()
            runs.append(e0.elapsed_time(e1) * 1e3 / 200)
        res[f"camera_knn_q{nq}_us"] = statistics.median(runs)
        print(f"[camera_knn N {DB} k 9 Q {nq}] us per launch: median {statistics.median(runs):.2f} of {[round(r, 2) for r in runs]}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

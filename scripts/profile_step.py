"""Per-kernel breakdown of one bench generate() step, from torch.profiler with CUDA activities.

    python scripts/profile_step.py --out DIR [--scenes 32] [--precision mixed] [--part all|encode|migt|decode]

`--part all` profiles one replay of the captured CUDA graph the bench times (GraphedPredictions); the other parts launch eagerly.
Writes DIR/kernels.md (kernel, launches, ms, share of the step's kernel time) and DIR/trace.pt.trace.json, and prints the table.
"""
import argparse
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.autograd import DeviceType  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402


def kernel_name(name):
    """Drop the return type, the anonymous namespace and the argument list; keep template arguments (they tell the exact, bf16
    and TF32 instances of one kernel apart)."""
    name = name.replace("(anonymous namespace)::", "")
    if name.startswith("void "):
        name = name[5:]
    if name.endswith(")"):
        depth = 0
        for i in range(len(name) - 1, -1, -1):
            depth += {")": 1, "(": -1}.get(name[i], 0)
            if depth == 0:
                name = name[:i]
                break
    return name


def kernel_table(events):
    agg = defaultdict(lambda: [0, 0.0])
    for e in events:
        if e.device_type != DeviceType.CUDA:
            continue
        a = agg[kernel_name(e.name)]
        a[0] += 1
        a[1] += e.device_time_total / 1e3              # us -> ms
    total = sum(t for _, t in agg.values())
    lines = [f"total kernel time {total:.2f} ms over {sum(c for c, _ in agg.values())} launches", "",
             "| kernel | launches | ms | share |", "|---|---:|---:|---:|"]
    for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"| `{n}` | {c} | {t:.3f} | {100 * t / total:.1f}% |")
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (kernels.md, trace.pt.trace.json)")
    ap.add_argument("--scenes", type=int, default=32)
    ap.add_argument("--precision", default="mixed")
    ap.add_argument("--part", default="all", choices=["all", "encode", "migt", "decode"])
    a = ap.parse_args()

    from bench import synth_inputs, model_pair, T_VIEWS
    from viewformer_b200 import GraphedPredictions
    from viewformer_b200.config import VQGANConfig, MIGTConfig

    assert torch.cuda.is_available(), "profile_step.py needs a GPU"
    dev = torch.device("cuda", 0)
    cb, tr = model_pair(a.precision, VQGANConfig(), MIGTConfig(localization_weight="0"), dev)
    images, cams = synth_inputs(a.scenes, 1234)
    images, cams = images.to(dev), cams.to(dev)

    if a.part == "all":
        graphed = GraphedPredictions(tr, cb, a.scenes, T_VIEWS)
        step = lambda: graphed(images, cams)  # noqa: E731
    elif a.part == "encode":
        step = lambda: cb.encode_u8(images[:, :9].reshape(-1, 128, 128, 3).contiguous())  # noqa: E731
    elif a.part == "migt":
        codes = torch.randint(0, 1024, (a.scenes, 9, 8, 8), device=dev)
        step = lambda: tr.generate_codes(codes, cams)  # noqa: E731
    else:
        codes = torch.randint(0, 1024, (a.scenes, 8, 8), device=dev)
        step = lambda: cb.decode_code_u8(codes)  # noqa: E731

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    os.makedirs(a.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(a.out, "trace.pt.trace.json"))
    table = f"{torch.cuda.get_device_name(0)}, {a.precision}, {a.scenes} scenes, part={a.part}\n\n" + kernel_table(prof.events())
    with open(os.path.join(a.out, "kernels.md"), "w") as f:
        f.write(table)
    print(table)


if __name__ == "__main__":
    main()

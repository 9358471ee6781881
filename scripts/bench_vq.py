"""Codebook-lookup micro-benchmark (SURVEY §8d): z ~ N(0,1) [M,256] fp32 -> int64 indices, K = 1024.
Algorithmic bytes per row: 1024 (z) + 8 (index) = 1032; roofline = measured HBM copy bandwidth."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewformer_b200 import _lib as L

L.load(True)
dev = "cuda"
peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) if os.path.exists("MEASURED_PEAKS.json") else {"hbm_gbs": 6573.8}
E = (torch.rand(256, 1024, device=dev) * 2 - 1) * 3 ** 0.5
et, esq = L.vq_prepare_codebook(E)
eh = L.vq_prepare_codebook_f16(et)


def timeit(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


only = sys.argv[1] if len(sys.argv) > 1 else ""
for M in ([1 << 20] if only == "fused" else [18432, 1 << 17, 1 << 20]):
    z = torch.randn((M, 256), device=dev)
    rows = [("fused wgmma (1 pass, fp16 pairs)", lambda: L.vq_lookup_fused(z, et, esq, eh, emb_dk=E, want_quant=False, want_diff=False))]
    if only != "fused" and M <= 1 << 17:
        rows += [("fp32 CUDA-core", lambda: L.vq_lookup(z, et, esq, want_quant=False, want_diff=False))]
    for name, fn in rows:
        ms = timeit(fn)
        gbs = M * 1032 / ms / 1e6
        extra = ""
        if name.startswith("fused"):
            _, _, _, cnt = L.vq_lookup_fused(z, et, esq, eh, emb_dk=E, want_quant=False, want_diff=False, return_counts=True)
            extra = f"  settled exactly: pair {int(cnt[0])} all-codes {int(cnt[1])}"
        print(f"VQ lookup M={M:8d} {name:36s} {ms:8.3f} ms  {gbs:8.1f} GB/s algorithmic = {100 * gbs / peaks['hbm_gbs']:5.1f}% of {peaks['hbm_gbs']:.0f} GB/s  ({2.0 * M * 1024 * 256 / ms / 1e9:7.1f} TFLOP/s){extra}")

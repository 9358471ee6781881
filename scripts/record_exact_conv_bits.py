"""Records the bits of exact (split-fp16) tc_conv / tc_gemm results on seeded inputs: tests/golden/exact_conv_bits.json.

    python scripts/record_exact_conv_bits.py [--out PATH]

Each case draws its inputs from a seeded CPU torch.Generator, splits them on the GPU (groupnorm(..., float16, normalize=False) for
activations, split_f16x2 for weights) and stores the sha256 of the fp32 output.  Fused GroupNorm statistics come from fp64
atomics whose order depends on the tile schedule, so they are stored as values and compared with a tolerance.
tests/test_exact_conv_bits_gpu.py recomputes every case with the library under test.
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "exact_conv_bits.json")

# convs: (n, h, w, cin, cout, residual) — small batches of the encoder's exact 3x3 shapes, then ragged maps (odd tile counts,
# border tiles).  gemms: the exact attention GEMMs of the 8x8 mid-block (QK^T with alpha, P.V).
CONVS = [(n, s, s, ci, co, r) for (n, s, ci, co) in [(1, 128, 128, 128), (2, 64, 128, 128), (2, 32, 128, 256), (2, 32, 256, 256),
                                                     (2, 16, 256, 256), (2, 8, 256, 512), (2, 8, 512, 512)] for r in (False, True)]
CONVS += [(1, 40, 20, 64, 256, False), (1, 40, 20, 64, 256, True), (2, 33, 9, 128, 128, False), (2, 33, 9, 128, 128, True)]
GEMMS = ["scores", "pv"]


def _sha(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def run_conv(n, h, w, cin, cout, residual):
    from viewformer_b200 import _lib as L
    g = torch.Generator().manual_seed(n * 1000003 + h * 1009 + w * 101 + cin + cout)
    x = torch.randn((n, h, w, cin), generator=g)
    wt = torch.randn((cout * 9, cin), generator=g) / (3.0 * cin ** 0.5)
    b = torch.randn(cout, generator=g)
    res = torch.randn((n, h, w, cout), generator=g) if residual else None
    xs = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False)
    ws = L.split_f16x2(wt.cuda()).reshape(cout, 18 * cin)
    out = L.tc_conv(xs, ws, b.cuda(), residual=None if res is None else res.cuda(), gn_groups=32)
    torch.cuda.synchronize()
    rec = {"sha256": _sha(out)}
    if hasattr(out, "_gn_sums"):
        rec["gn_sums"] = out._gn_sums[0].cpu().flatten().tolist()
    return rec


def run_gemm(kind):
    from viewformer_b200 import _lib as L
    n, hw, c = 2, 64, 512
    g = torch.Generator().manual_seed({"scores": 7, "pv": 8}[kind])
    out = torch.empty((n, hw, c if kind == "pv" else hw), dtype=torch.float32, device="cuda")
    if kind == "scores":                                   # scores = alpha * q k^T, q | k interleaved in one [hw, 2c] row
        qks = L.split_f16x2((torch.randn((n * hw, 2 * c), generator=g) * 0.5).cuda())          # [n*hw, 4c] = hi(q|k) | lo(q|k)
        L.tc_gemm(qks, qks, out, M=hw, N=hw, K=c, lda=4 * c, ldb=4 * c, ldc=hw, batch=(n, 1), a_bs=(hw * 4 * c, 0),
                  b_bs=(hw * 4 * c, 0), c_bs=(hw * hw, 0), b_off=c, alpha=float(c ** -0.5), lo_a=2 * c, lo_b=2 * c)
    else:                                                  # o = P V
        ps = L.split_f16x2(torch.softmax(torch.randn((n * hw, hw), generator=g), -1).cuda())
        vts = L.split_f16x2(torch.randn((n * c, hw), generator=g).cuda())
        L.tc_gemm(ps, vts, out, M=hw, N=c, K=hw, lda=2 * hw, ldb=2 * hw, ldc=c, batch=(n, 1), a_bs=(hw * 2 * hw, 0),
                  b_bs=(c * 2 * hw, 0), c_bs=(hw * c, 0))
    torch.cuda.synchronize()
    return {"sha256": _sha(out)}


def conv_id(case):
    n, h, w, cin, cout, residual = case
    return f"conv_{n}x{h}x{w}_{cin}-{cout}" + ("_res" if residual else "")


def record():
    rec = {conv_id(c): run_conv(*c) for c in CONVS}
    rec.update({f"gemm_{k}": run_gemm(k) for k in GEMMS})
    return rec


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=GOLDEN)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "record_exact_conv_bits.py needs a GPU"
    rec = {"device": torch.cuda.get_device_name(0), "cases": record()}
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(f"wrote {len(rec['cases'])} cases to {a.out}")

"""CUDA-event micro-benchmarks of the hot kernels at the shapes the 32-scene generate() step launches."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewformer_b200 import _lib as L

L.load(True)
dev = "cuda"
PEAK_TF, PEAK_HBM = 1691.2, 6573.8


def timeit(fn, reps=10, warm=3):
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


rows = []


def conv_case(n, hw, cin, cout, residual):
    x = torch.randn((n, hw, hw, cin), device=dev).bfloat16()
    w = (torch.randn((cout, 9 * cin), device=dev) / 30).bfloat16()
    b = torch.zeros(cout, device=dev)
    res = torch.randn((n, hw, hw, cout), device=dev) if residual else None
    out = torch.empty((n, hw, hw, cout), device=dev)
    ms = timeit(lambda: L.tc_conv(x, w, b, out=out, residual=res))
    fl = 2.0 * n * hw * hw * cin * 9 * cout
    rows.append((f"conv3x3 {cin}->{cout} @{hw}^2 n={n} res={int(residual)}", ms, fl / ms / 1e9, None))


def gemm_case(name, M, N, K, batch=(1, 1), out_dtype=torch.float32, residual=False, act=0):
    A = torch.randn((batch[0] * batch[1] * M, K), device=dev).bfloat16()
    B = torch.randn((N, K), device=dev).bfloat16()
    out = torch.empty((batch[0] * batch[1] * M, N), device=dev, dtype=out_dtype)
    bias = torch.zeros(N, device=dev)
    res = torch.randn((batch[0] * batch[1] * M, N), device=dev) if residual else None
    ms = timeit(lambda: L.tc_gemm(A, B, out, M=M * batch[0] * batch[1], N=N, K=K, lda=K, ldb=K, ldc=N, bias=bias, bias_mode=1,
                                  residual=res, act=act))
    rows.append((name, ms, 2.0 * M * batch[0] * batch[1] * N * K / ms / 1e9, None))


def gn_case(n, hw, c):
    x = torch.randn((n, hw, hw, c), device=dev)
    ga, be = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    ms = timeit(lambda: L.groupnorm(x, ga, be, swish=True, out_dtype=torch.bfloat16))
    gb = n * hw * hw * c * (4 + 4 + 2) / 1e9
    rows.append((f"groupnorm+swish n={n} {hw}^2x{c} (stats+apply)", ms, None, gb / ms * 1e3))


conv_case(288, 128, 128, 128, False)
conv_case(288, 128, 128, 128, True)
conv_case(288, 64, 128, 128, True)
conv_case(288, 32, 256, 256, True)
conv_case(288, 16, 256, 256, True)
conv_case(288, 8, 512, 512, True)
conv_case(32, 128, 128, 128, True)
conv_case(32, 64, 256, 256, True)
conv_case(32, 8, 512, 512, True)
gemm_case("migt c_fc  20480x3072x768 gelu->bf16", 20480, 3072, 768, out_dtype=torch.bfloat16, act=1)
gemm_case("migt fc2   20480x768x3072 +res", 20480, 768, 3072, residual=True)
gemm_case("migt cproj 20480x768x768 +res", 20480, 768, 768, residual=True)
gemm_case("migt qk    20480x1536x768 ->bf16", 20480, 1536, 768, out_dtype=torch.bfloat16)
gemm_case("lm head    2048x1024x768", 2048, 1024, 768)
gn_case(288, 128, 128)
gn_case(288, 64, 128)
gn_case(32, 128, 128)
# the two tiny-channel exact convolutions
xin = torch.randn((288, 128, 128, 3), device=dev)
win = torch.randn((27, 128), device=dev) / 5
bin_ = torch.zeros(128, device=dev)
ms = timeit(lambda: L.conv3x3_small_cin(xin, win, bin_, gn_groups=32))
rows.append(("conv_in 3->128 @128^2 n=288 (+GN sums), fp32", ms, 2.0 * 288 * 128 * 128 * 27 * 128 / ms / 1e9, 288 * 128 * 128 * (12 + 512) / 1e9 / ms * 1e3))
xo = torch.randn((32, 128, 128, 128), device=dev)
wo = torch.randn((1152, 3), device=dev) / 30
bo = torch.zeros(3, device=dev)
ms = timeit(lambda: L.conv3x3_small_cout(xo, wo, bo))
rows.append(("conv_out 128->3 @128^2 n=32, fp32", ms, 2.0 * 32 * 128 * 128 * 1152 * 3 / ms / 1e9, 32 * 128 * 128 * (512 + 12) / 1e9 / ms * 1e3))
del xin, xo
# attention pieces at B=32,H=12,S=640
B, H, S, d = 32, 12, 640, 768
qk = torch.randn((B, S, 2 * d), device=dev).bfloat16()
sc = torch.empty((B, H, S, S), device=dev)
p = torch.empty((B, H, S, S), device=dev, dtype=torch.bfloat16)
vt = torch.randn((B, d, S), device=dev).bfloat16()
o = torch.empty((B * S, d), device=dev, dtype=torch.bfloat16)
ms = timeit(lambda: L.tc_gemm(qk, qk, sc, M=S, N=S, K=64, lda=2 * d, ldb=2 * d, ldc=S, batch=(B, H), a_bs=(S * 2 * d, 64), b_bs=(S * 2 * d, 64),
                              c_bs=(H * S * S, S * S), b_off=d, causal_block=64, causal_skip_n=True))
rows.append(("attn QK^T (causal skip) B32 H12 S640", ms, 2.0 * B * H * S * S * 64 * 0.55 / ms / 1e9, None))
ms = timeit(lambda: L.softmax_rows(sc, p, rows_total=B * H * S, rows_per_batch=S, cols=S, ld_in=S, ld_out=S, mask_mode=1, block=64))
rows.append(("attn softmax", ms, None, B * H * S * (S * 0.55 * 4 + S * 2) / 1e6 / ms))
ms = timeit(lambda: L.tc_gemm(p, vt, o, M=S, N=64, K=S, lda=S, ldb=S, ldc=d, batch=(B, H), a_bs=(H * S * S, S * S), b_bs=(d * S, 64 * S),
                              c_bs=(S * d, 64), causal_block=64))
rows.append(("attn P.V (causal k-limit)", ms, 2.0 * B * H * S * S * 64 * 0.55 / ms / 1e9, None))

for (Bq, Sq) in ((32, 640), (32, 1280)):
    qk2 = torch.randn((Bq, Sq, 2 * d), device=dev).bfloat16()
    vt2 = torch.randn((Bq, d, Sq), device=dev).bfloat16()
    ms = timeit(lambda: L.attn_block_causal(qk2, vt2, Bq, Sq, H, d, 64))
    Tn = Sq // 64
    useful = 4.0 * Bq * H * 64 * 64 * 64 * Tn * (Tn + 1) / 2          # 4*dh*L^2*T(T+1)/2 per (b,h): QK^T + PV, visible blocks only
    rows.append((f"FUSED block-causal attention B{Bq} H12 S{Sq} (useful FLOPs)", ms, useful / ms / 1e9, None))

# VQ lookup: exact fp32 kernel (the fused tensor-core lookup: scripts/bench_vq.py)
from oracle import synth
E, _ = synth.make_lookup_inputs(11)
et, esq = L.vq_prepare_codebook(E.cuda())
for Mq in (18432, 1 << 20):
    zq = torch.randn((Mq, 256), device=dev)
    ms = timeit(lambda: L.vq_lookup(zq, et, esq, want_quant=False, want_diff=False), reps=3, warm=1)
    rows.append((f"VQ lookup fp32 CUDA-core  M={Mq}", ms, 2.0 * Mq * 256 * 1024 / ms / 1e9, Mq * 1032 / ms / 1e6))

print(f"{'kernel':58s} {'ms':>8s} {'TFLOP/s':>9s} {'%peak':>6s} {'GB/s':>8s} {'%hbm':>6s}")
for name, ms, tf, gbs in rows:
    a = f"{tf:9.1f} {100*tf/PEAK_TF:6.1f}" if tf else " " * 16
    b = f"{gbs:8.0f} {100*gbs/PEAK_HBM:6.1f}" if gbs else ""
    print(f"{name:58s} {ms:8.3f} {a} {b}")

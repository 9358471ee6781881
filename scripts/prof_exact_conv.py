"""Every exact (split-fp16) 3x3 stride-1 conv shape the bench's encoder launches (288 images), timed alone with CUDA events.

    python scripts/prof_exact_conv.py [n_images]

One line per shape and residual: launch time, executed fp16 MMA rate (three passes per product), the path the shape takes and the
operand bytes that path moves from L2 into shared memory per launch: tap-box (a shifted A box per tap and k-block) or halo (Cin <=
128: one halo tile per channel block and half, resident for the whole tile).  Weight boxes are counted on both paths.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from viewformer_b200 import _lib as L  # noqa: E402

# (map side, Cin, Cout): the encoder's 3x3 stride-1 convs of the exact (mixed) path
SHAPES = [(128, 128, 128), (64, 128, 128), (32, 128, 256), (32, 256, 256), (16, 256, 256), (8, 256, 512), (8, 512, 512)]


def operand_bytes(n, side, cin, cout):
    """(path, L2 -> SM bytes per launch) of the schedule tc_gemm_kernel runs (128-pixel tiles, 64-channel k-blocks of 128 bytes per
    row, 3 product passes)."""
    block_n = 128 if cout > 64 else 64
    cbs = cin // 64
    tiles = n * side * side // 128 * (cout // block_n)
    b = 3 * 9 * cbs * block_n * 128                              # weight boxes per tile
    if cin <= 128 and side >= 16:                              # 16 x 8-pixel tiles, one (8+2) x (16+2) halo tile per (half, block)
        return "halo", tiles * (2 * cbs * 10 * 18 * 128 + b)
    return "tap-box", tiles * (3 * 9 * cbs * 128 * 128 + b)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 288
    assert torch.cuda.is_available(), "prof_exact_conv.py needs a GPU"
    L.load(True)
    dev = "cuda"
    print(f"{torch.cuda.get_device_name(0)}, {n} images per launch")
    print("| map | Cin->Cout | residual | ms | executed fp16 MMA TFLOP/s | path | L2->SM GB |")
    print("|---|---|---|---:|---:|---|---:|")
    g = torch.Generator(device=dev).manual_seed(0)
    for side, cin, cout in SHAPES:
        x = torch.randn((n, side, side, cin), device=dev, generator=g)
        xs = L.groupnorm(x, None, None, swish=False, out_dtype=torch.float16, normalize=False)
        del x
        w = torch.randn((cout * 9, cin), device=dev, generator=g) / (3.0 * cin ** 0.5)
        ws = L.split_f16x2(w).reshape(cout, 18 * cin)
        b = torch.zeros(cout, device=dev)
        o = torch.empty((n, side, side, cout), device=dev)
        res = torch.randn((n, side, side, cout), device=dev, generator=g)
        reps = max(5, int(2e10 / (n * side * side * cin * cout * 9)))
        path, nbytes = operand_bytes(n, side, cin, cout)
        for r in (None, res):
            for _ in range(3):
                L.tc_conv(xs, ws, b, out=o, residual=r, gn_groups=32)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                L.tc_conv(xs, ws, b, out=o, residual=r, gn_groups=32)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            fl = 3 * 2.0 * n * side * side * cin * 9 * cout
            print(f"| {side}x{side} | {cin}->{cout} | {'yes' if r is not None else 'no'} | {ms:.3f} | {fl / ms / 1e9:.1f} | {path} | {nbytes / 1e9:.1f} |")
        del xs, ws, o, res
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""SSIM and the pair-sum image metrics (GPU) against fp64: every ``ssim_u8`` call goes through ``launch_checks.check_ssim_u8`` (exact int64
window sums, S in fp64, the bar derived in its docstring) on the content where E[x^2] - E[x]^2 cancels (flat images at every level against
a level a few steps away), where the covariance is negative (inverted images), at the extremes (0 / 255 checkerboards), and on smooth and
noisy images, at the shapes where the window walk has edges (one window, one row or column of windows, C = 1, 3, 4, many windows per
thread under the 64-chunk cap, N = 1 and N = 1000) and at both constants of the reference (K1 = 0.01 of ssim(), 1 of SSIMMetric)."""
import math
import random

import pytest
import torch

import launch_checks as lc
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def check(L, a, b, k1=None, k2=None):
    """The kernel's per-image SSIM and its worst ratio to the bar of check_ssim_u8."""
    a, b = a.cuda().contiguous(), b.cuda().contiguous()
    got, r = lc.run_check("ssim_u8", L.ssim_u8, (a, b), dict(k1=k1, k2=k2), random.Random(0))
    return got, r


def flat(levels, h, w, c):
    return torch.as_tensor(levels).to(torch.uint8)[:, None, None, None].expand(-1, h, w, c).contiguous()


def noisy(a, amp, seed):
    g = torch.Generator().manual_seed(seed)
    return (a.int() + torch.randint(-amp, amp + 1, a.shape, generator=g)).clamp(0, 255).to(torch.uint8)


CONSTANTS = [(0.01, 0.03), (1.0, 0.03), (0.01, 0.1), (1.0, 0.1)]


@pytest.mark.parametrize("k1,k2", CONSTANTS)
@pytest.mark.parametrize("d", [0, 1, 2, 3, 5, 40])
def test_flat_level_pairs(L, d, k1, k2):
    """One flat 16 x 16 x 3 image per level a in [0, 255] against the flat level min(a + d, 255): the variances vanish, C2 dominates B2,
    and an fp32 E[x^2] - E[x]^2 is off by up to ~1.3e-4 of S in every window alike.  Equal levels give exactly 1."""
    lv = torch.arange(256)
    a, b = flat(lv, 16, 16, 3), flat((lv + d).clamp(max=255), 16, 16, 3)
    got, r = check(L, a, b, k1, k2)
    want = lc.ssim64(a.cuda(), b.cuda(), k1, k2)[1]
    err = (got - want).abs()
    print(f"[ssim flat d={d} K1={k1} K2={k2}] worst |err| {float(err.max()):.3g} (level {int(err.argmax())}), ratio {r:.3g}")
    assert r <= 1.0
    if d == 0:
        assert bool((got == 1.0).all())


@pytest.mark.parametrize("kind", ["random", "flat", "smooth"])
def test_identical_images_give_exactly_one(L, kind):
    """S = 1 in every window when a == b, so the mean is exactly 1.0 (sums of ones are exact, one division by the window count), here at
    512 x 512 x 3 where each thread walks 47 windows, next to the 13 x 29 x 4 and single-window cases."""
    for n, h, w, c in ((2, 512, 512, 3), (3, 13, 29, 4), (4, 7, 7, 1)):
        if kind == "random":
            a = torch.randint(0, 256, (n, h, w, c), generator=torch.Generator().manual_seed(h), dtype=torch.uint8)
        elif kind == "flat":
            a = flat(torch.arange(n) * 73 % 256, h, w, c)
        else:
            a = gradient(n, h, w, c)
        for k1, k2 in CONSTANTS:
            got, r = check(L, a, a, k1, k2)
            assert r <= 1.0 and bool((got == 1.0).all()), (n, h, w, c, k1, k2, got.tolist())


def gradient(n, h, w, c):
    """Smooth ramps, different per image and channel: slowly varying windows with small variances."""
    y = torch.arange(h, dtype=torch.float64)[:, None, None]
    x = torch.arange(w, dtype=torch.float64)[None, :, None]
    ch = torch.arange(c, dtype=torch.float64)[None, None, :]
    imgs = [(40 + 3 * i + 0.5 * (i + 1) * y + 0.3 * x + 17 * ch) % 256 for i in range(n)]
    return torch.stack(imgs).floor().to(torch.uint8).contiguous()


def checkerboard(n, h, w, c, phase=0):
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    board = ((yy + xx + phase) % 2 * 255).to(torch.uint8)
    return board[None, :, :, None].expand(n, h, w, c).contiguous()


def content(kind, n, h, w, c, seed):
    """(a, b) pairs of the named content."""
    g = torch.Generator().manual_seed(seed)
    rand = torch.randint(0, 256, (n, h, w, c), generator=g, dtype=torch.uint8)
    if kind == "inverted":                        # covariance -var: A2 = 2 vxy + C2 cancels
        return rand, 255 - rand
    if kind == "inverted-smooth":
        a = gradient(n, h, w, c)
        return a, 255 - a
    if kind == "checkerboard":                    # the extremes: 0 / 255 windows, against the same board shifted by one pixel and itself
        return checkerboard(n, h, w, c), torch.cat([checkerboard(n - n // 2, h, w, c, 1), checkerboard(n // 2, h, w, c)])
    if kind == "checkerboard-flat":
        return checkerboard(n, h, w, c), flat(torch.arange(n) * 37 % 256, h, w, c)
    if kind == "gradient":
        a = gradient(n, h, w, c)
        return a, noisy(a, 2, seed)
    if kind == "synth":                           # the synthetic dataset's images with noise
        a = synth.make_images_uint8(1, n, size=max(h, w, 16), seed=seed)[0][:, :h, :w, :c].contiguous()
        return a, noisy(a, 20, seed + 1)
    if kind == "half-flat":                       # a flat band next to noise: flat windows and the windows that straddle the edge
        a, b = rand.clone(), noisy(rand, 10, seed)
        a[:, :, : w // 2] = 77
        b[:, :, : w // 2] = 79
        return a, b
    raise ValueError(kind)


@pytest.mark.parametrize("k1,k2", CONSTANTS)
@pytest.mark.parametrize("kind", ["inverted", "inverted-smooth", "checkerboard", "checkerboard-flat", "gradient", "synth", "half-flat"])
def test_content(L, kind, k1, k2):
    a, b = content(kind, 4, 40, 56, 3, 500)
    got, r = check(L, a, b, k1, k2)
    print(f"[ssim {kind} K1={k1} K2={k2}] {[round(v, 6) for v in got.tolist()]} ratio {r:.3g}")
    assert r <= 1.0


SHAPES = [(3, 7, 7, 3), (2, 7, 300, 3), (2, 300, 7, 3), (4, 13, 29, 1), (4, 13, 29, 3), (4, 13, 29, 4), (16, 128, 128, 3), (2, 512, 512, 3),
          (1, 64, 64, 3), (1000, 32, 32, 3)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", ["half-flat", "synth", "inverted"])
def test_shapes(L, shape, kind):
    """Windows at every edge of the walk: a single 7 x 7 window, one row or one column of windows, C = 1 / 3 / 4, the Evaluator's
    128 x 128 x 3, 512 x 512 x 3 (64 chunks, 47 windows per thread), one image, a thousand images."""
    n, h, w, c = shape
    if kind == "synth" and c > 3:
        kind = "half-flat"
    a, b = content(kind, n, h, w, c, 600 + h + w)
    for k1 in (None, 1.0):
        got, r = check(L, a, b, k1)
        print(f"[ssim {kind} {shape} K1={k1}] mean {float(got.mean()):.6f} ratio {r:.3g}")
        assert r <= 1.0


def test_image_metrics_edges(L):
    """A 6-pixel side has no 7 x 7 window: SSIM is NaN and the Evaluator leaves it out of the mean while the other metrics count.  Identical
    images: MSE 0 and PSNR +inf, as tf.image.psnr gives.  512 x 512 x 3 of 0 against 255: sum d^2 = 786432 * 65025 = 5.1e10 > 2^32."""
    from viewformer_b200.metrics import image_metrics, Evaluator
    a7, b7 = content("synth", 2, 7, 7, 3, 700)
    for shape in ((2, 6, 20, 3), (2, 20, 6, 3), (2, 6, 6, 3)):
        a, b = content("half-flat", *shape, 701)
        m = image_metrics(a, b)
        assert bool(torch.isnan(m["ssim"]).all()) and bool(torch.isfinite(m["psnr"]).all()), shape
        ev = Evaluator()
        ev.update_with_image(a, b)
        ev.update_with_image(a7, b7)
        r = ev.result()
        want = float(image_metrics(a7, b7, ssim_k1=1.0)["ssim"].mean())
        assert r["ssim"] == want, (shape, r["ssim"], want)
        assert abs(r["psnr"] - float(torch.cat([m["psnr"], image_metrics(a7, b7)["psnr"]]).mean())) < 1e-9
    a = content("synth", 3, 32, 32, 3, 702)[0]
    m = image_metrics(a, a)
    assert bool((m["mse"] == 0).all()) and bool((m["mae"] == 0).all()) and bool((m["rmse"] == 0).all())
    assert bool((m["psnr"] == math.inf).all()) and bool((m["ssim"] == 1.0).all())
    ev = Evaluator()
    ev.update_with_image(a, a)
    assert ev.result()["psnr"] == math.inf and ev.result()["ssim"] == 1.0
    z, f = torch.zeros(2, 512, 512, 3, dtype=torch.uint8).cuda(), torch.full((2, 512, 512, 3), 255, dtype=torch.uint8).cuda()
    sums, r = lc.run_check("image_pair_sums", L.image_pair_sums, (z, f), {}, random.Random(0))
    assert r == 0.0 and int(sums[0, 1]) == 512 * 512 * 3 * 255 * 255 > 2 ** 32
    m = image_metrics(z, f)
    assert bool((m["mse"] == 1.0).all()) and bool((m["psnr"] == 0.0).all()) and bool((m["rmse"] == 255.0).all())

"""Pure checkers of the float-image wrappers in ``viewformer_b200.float_images``, in the form of tests/launch_checks.py (a check returns
the worst ratio of error to its bar, <= 1 passes; bit-for-bit conditions return inf when they fail), with its helpers and bars:

  f01_to_unit:  x 2 - 1 in fp32, bit for bit (torch's ``x * 2 - 1`` on the same tensor).
  resize_f32:   launch_checks.check_resize_u8's fp64 restatement on the f32 values themselves, clamped to [0, 1], not quantised: nearest
                bit for bit, bilinear within 8 u of the same interpolation of |x| (per row a weight 1 - l, two products and a sum, then the
                same per column, each rounded once: 6 u; the source indices and weights are formed in fp32 as the kernel forms them).
"""
import math

import numpy as np
import torch

from launch_checks import U, before_none, bind, bits_equal, f32, ratio


def check_f01_to_unit(ba, result, st):
    x, fv = ba["x"], ba["first_views"]
    if fv is not None:
        x = x[:, :fv].reshape((-1,) + tuple(x.shape[2:]))
    return bits_equal(result, x * 2 - 1)


def resize64(xv, size, method):
    """fp64 nearest / bilinear (align_corners=False) resize of NHWC ``xv`` to size x size, with the source indices and interpolation
    weights formed in fp32 as vf_resize_u8 / vf_resize_f32 form them."""
    n, h, w, c = xv.shape
    sh, sw = f32(np.float32(h) / np.float32(size)), f32(np.float32(w) / np.float32(size))
    o = torch.arange(size, device=xv.device, dtype=torch.float32)
    if method == "nearest":
        sy = torch.floor(o * sh).long().clamp(max=h - 1)
        sx = torch.floor(o * sw).long().clamp(max=w - 1)
        return xv[:, sy][:, :, sx]
    fy, fx = ((o + 0.5) * sh - 0.5).clamp_min(0), ((o + 0.5) * sw - 0.5).clamp_min(0)
    y0, x0 = fy.long(), fx.long()
    y1, x1 = (y0 + 1).clamp(max=h - 1), (x0 + 1).clamp(max=w - 1)
    ly, lx = (fy - y0).double()[None, :, None, None], (fx - x0).double()[None, None, :, None]
    g = lambda yy, xx: xv[:, yy][:, :, xx]                    # noqa: E731
    return (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))


def check_resize_f32(ba, result, st):
    x, size = ba["x"], int(ba["size"])
    n, h, w, c = x.shape
    if size in (w, h):                                         # resize_u8's pass-through rule
        return 0.0 if result is x else math.inf
    method = ba["method"] or ("nearest" if size > h else "bilinear")
    ref = resize64(x.double(), size, method).clamp(0, 1)
    if method == "nearest":
        return bits_equal(result, ref.float())
    return ratio((result.double() - ref).abs(), 8 * U * resize64(x.double().abs(), size, method))


CHECKERS = {
    "f01_to_unit": (before_none, check_f01_to_unit),
    "resize_f32": (before_none, check_resize_f32),
}


def run_check(name, fn, a, k, rng):
    """launch_checks.run_check for the wrappers above: (result, worst ratio)."""
    before, check = CHECKERS[name]
    ba = bind(fn, *a, **k)
    st = before(ba, rng)
    result = fn(*a, **k)
    return result, check(ba, result, st)

"""Device conversions of float32 images in [0, 1], the input ``tf.image.convert_image_dtype`` keeps as it is: the ``x * 2 - 1`` the
encoder takes, and the dataset resize rule in float.  Thin wrappers of ``vf_f01_to_unit_f32`` / ``vf_resize_f32`` (include/vf_b200.h),
the float counterparts of ``_lib.u8_to_unit`` / ``_lib.resize_u8``; like every launching wrapper they are checked against fp64 on their
own operands (tests/launch_checks_float.py) in the tests and in a launch audit of the four-channel workloads.
"""
import torch

from . import _lib as L


def f01_to_unit(x, first_views=None):
    """f32 images in [0, 1] -> x * 2 - 1 (tf.image.convert_image_dtype is the identity for float32 input), op by op in fp32.
    ``first_views=n`` on a [B,T,H,W,C] tensor: views 0..n-1 of every scene, as ``u8_to_unit``."""
    lib = L.load(True)
    L._dev(x, torch.float32)
    if first_views is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
        L._check(lib.vf_f01_to_unit_f32(x, out, 1, x.numel(), 0, L._stream()))
        return out
    b, t = x.shape[:2]
    per_view = x[0, 0].numel()
    out = torch.empty((b * first_views,) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
    L._check(lib.vf_f01_to_unit_f32(x, out, b, first_views * per_view, t * per_view, L._stream()))
    return out


def resize_f32(x, size, method=None):
    """``resize_u8``'s rule (the same sizes pass through unchanged, the same methods) for f32 NHWC images in [0, 1] -> [N,size,size,C]
    f32, clamped to [0, 1] as resize_th clamps.  Not quantised: resize_th would also round a float image to 1/255 steps, which the
    float path exists to avoid."""
    lib = L.load(True)
    L._dev(x, torch.float32)
    n, h, w, c = x.shape
    if w == size or h == size:
        return x
    if method is None:
        method = "nearest" if size > h else "bilinear"
    assert method in ("nearest", "bilinear")
    out = torch.empty((n, size, size, c), dtype=torch.float32, device=x.device)
    L._check(lib.vf_resize_f32(x, n, h, w, c, size, size, int(method == "bilinear"), out, L._stream()))
    return out

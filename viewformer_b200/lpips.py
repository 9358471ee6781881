"""LPIPS, the perceptual image metric every evaluator of the reference reports (utils/metrics.py:199-214 LPIPSMetric through
models/utils.py:297-307: ``lpips.LPIPS(net='vgg', version='0.1')``, lpips 0.1.3), on the GPU.

The reference converts both uint8 batches with ``tf.image.convert_image_dtype`` (x * fp32(1/255)) and hands them to LPIPS.forward with
``normalize=False``, so the scaling layer sees images in [0, 1], not the [-1, 1] it was designed for; the numbers here include that.
Per pair of images: the scaling layer (x - shift) / scale, VGG16 ``features`` up to relu5_3 (13 3x3 convs with bias and ReLU, 2x2
max-pools), at relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3 the channel-normalised features' squared difference weighted by the
``lin`` layer and averaged over the map, and the sum of the five.

Weights are read from the two files the reference's stack uses, never downloaded: torchvision's ImageNet VGG16 checkpoint
(``vgg16-397923af.pth``; ``classifier.*`` is ignored) and lpips' ``weights/v0.1/vgg.pth``.

Kernels (include/vf_b200_lpips.h, bound by ``PROTOTYPES`` as ``_lib.PROTOTYPES`` binds include/vf_b200.h; tests/test_lpips_host.py holds
the table to the header): the first conv reads the uint8 images through the conversion and the scaling layer (fp32 CUDA cores); the other
twelve are exact split-fp16 tensor-core convolutions (``vf_tc_gemm``) with a ReLU epilogue, fp32-faithful while activations stay below
65520; each pool writes the next conv's split operand; a fused head adds each tap's term per pair in a fixed order.  The two images of
every pair run as one batch, so each layer is one launch.
"""
import ctypes as C
import os

import torch

from . import _lib as L

SHIFT = (-0.030, -0.088, -0.188)           # lpips ScalingLayer
SCALE = (0.458, 0.448, 0.450)
# VGG16 ``features`` convolutions: (index in ``features``, Cin, Cout); a 2x2 max-pool precedes the first conv of stages 2 to 5
CONVS = [(0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256),
         (17, 256, 512), (19, 512, 512), (21, 512, 512), (24, 512, 512), (26, 512, 512), (28, 512, 512)]
POOL_BEFORE = {5, 10, 17, 24}              # features[4], [9], [16], [23]
TAPS = {2: 0, 7: 1, 14: 2, 21: 3, 28: 4}   # conv index -> lin layer: relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
TAP_CHANNELS = (64, 128, 256, 512, 512)
MIN_SIZE = 16                              # four 2x2 pools leave at least one pixel


def _prototypes():
    """Parameter types of every function include/vf_b200_lpips.h declares, in order (p: a device pointer, s: vf_stream_t)."""
    i, p, s = C.c_int, L.DevPtr, C.c_void_p
    return {
        "vf_lpips_conv_in": [p, p, p, p, p, i, i, i, i, p, s],
        "vf_maxpool2x2_split": [p, i, i, i, i, p, s],
        "vf_lpips_tap": [p, i, i, i, i, p, p, p, s],
    }


PROTOTYPES = _prototypes()          # every entry point returns int
_declared = []


def load():
    """libvf_b200.so (``_lib.load``, which checks the device) with these entry points' types declared."""
    lib = L.load(True)
    if not _declared:
        for name, argtypes in PROTOTYPES.items():
            if not hasattr(lib, name):
                raise L.LibraryError(f"{L.LIB_PATH} does not export {name}")
            fn = getattr(lib, name)
            fn.argtypes, fn.restype = argtypes, C.c_int
        _declared.append(True)
    return lib


# ----------------------------------------------------------------------------------------------- weights
VGG16_FILE = "VGG16 weights (torchvision's vgg16-397923af.pth)"
LIN_FILE = "LPIPS lin weights (lpips' weights/v0.1/vgg.pth)"


def vgg16_shapes():
    """{key: shape} a torchvision VGG16 checkpoint must hold for the 13 convs (``classifier.*`` is not used)."""
    out = {}
    for idx, cin, cout in CONVS:
        out[f"features.{idx}.weight"] = (cout, cin, 3, 3)
        out[f"features.{idx}.bias"] = (cout,)
    return out


def lin_shapes():
    return {f"lin{k}.model.1.weight": (1, c, 1, 1) for k, c in enumerate(TAP_CHANNELS)}


def _read(path, what):
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{what} not found at {path!r}")
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise ValueError(f"{what} at {path!r}: expected a state dict, got {type(sd).__name__}")
    return sd


def check_state(sd, shapes, what, ignore=()):
    """fp32 copies of the tensors of ``shapes`` from state dict ``sd``: every key present with its exact shape and a floating dtype; keys
    starting with one of ``ignore`` are skipped, any other key raises ValueError."""
    missing = sorted(set(shapes) - set(sd))
    extra = sorted(k for k in sd if k not in shapes and not k.startswith(tuple(ignore)))
    if missing or extra:
        raise ValueError(f"{what}: missing keys {missing}, unexpected keys {extra}")
    out = {}
    for k, shape in shapes.items():
        t = sd[k]
        if not isinstance(t, torch.Tensor) or not t.is_floating_point() or tuple(t.shape) != shape:
            got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{what}: {k} must be a floating-point tensor of shape {shape}, got {got}")
        out[k] = t.detach().to(torch.float32)
    return out


def load_weights(vgg16_path, lin_path):
    """(VGG16 conv state dict, lin state dict) read on the CPU from the two files and checked strictly, fp32."""
    vgg = check_state(_read(vgg16_path, VGG16_FILE), vgg16_shapes(), VGG16_FILE, ignore=("classifier.",))
    lin = check_state(_read(lin_path, LIN_FILE), lin_shapes(), LIN_FILE)
    return vgg, lin


# ----------------------------------------------------------------------------------------------- kernel wrappers
def conv_in(x_u8, shift, scale, w_kn, bias):
    """relu(conv3x3(scaling layer(x / 255)) + bias): uint8 [N,H,W,3] -> fp32 [N,H,W,Cout]; w_kn [27, Cout]."""
    lib = load()
    L._dev(x_u8, torch.uint8)
    n, h, w, _ = x_u8.shape
    cout = w_kn.shape[1]
    y = torch.empty((n, h, w, cout), dtype=torch.float32, device=x_u8.device)
    L._check(lib.vf_lpips_conv_in(x_u8, shift, scale, w_kn, bias, n, h, w, cout, y, L._stream()))
    return y


def maxpool2x2_split(x):
    """fp32 [N,H,W,C] -> split fp16 [N,H//2,W//2,2C]: the 2x2 max, as the next exact conv's [hi | lo] operand."""
    lib = load()
    L._dev(x, torch.float32)
    n, h, w, c = x.shape
    out = torch.empty((n, h // 2, w // 2, 2 * c), dtype=torch.float16, device=x.device)
    L._check(lib.vf_maxpool2x2_split(x, n, h, w, c, out, L._stream()))
    return out


def lpips_tap(f, lin, out):
    """out [N] fp64 += one tap's LPIPS term of the N pairs in f [2N,H,W,C] (pair n: images n and n + N)."""
    lib = load()
    L._dev(f, torch.float32)
    n2, h, w, c = f.shape
    n = n2 // 2
    partial = torch.empty((n * -(-(h * w) // 64),), dtype=torch.float64, device=f.device)
    L._check(lib.vf_lpips_tap(f, n, h, w, c, lin, partial, out, L._stream()))
    return out


# ----------------------------------------------------------------------------------------------- metric
class LPIPS:
    """``LPIPS(vgg16_path, lin_path)(images0, images1)``: per-pair LPIPS (VGG, v0.1) of uint8 NHWC RGB images, as the reference's
    LPIPSMetric computes it.  Weights are loaded once, checked (a missing file raises FileNotFoundError naming it; a missing,
    misshapen or unexpected key ValueError) and prepared for the kernels: [27, 64] fp32 for the first conv, K-major split fp16 for
    the others.  One precision: fp32-faithful throughout."""

    def __init__(self, vgg16_path, lin_path, device="cuda"):
        from .ops import Precision
        from .vqgan import _Conv3
        vgg, lin = load_weights(vgg16_path, lin_path)
        self.device = torch.device(device)
        exact = Precision("x3")
        self._convs = [_Conv3(vgg[f"features.{i}.weight"], vgg[f"features.{i}.bias"], exact, self.device) for i, _, _ in CONVS]
        self._lin = [lin[f"lin{k}.model.1.weight"].reshape(-1).to(self.device).contiguous() for k in range(len(TAP_CHANNELS))]
        self._shift = torch.tensor(SHIFT, dtype=torch.float32, device=self.device)
        self._scale = torch.tensor(SCALE, dtype=torch.float32, device=self.device)

    @staticmethod
    def check_images(images0, images1):
        """The two batches as uint8 [N,H,W,3] tensors of equal shape; ValueError / TypeError otherwise (before any launch)."""
        a, b = torch.as_tensor(images0), torch.as_tensor(images1)
        if a.dtype != torch.uint8 or b.dtype != torch.uint8:
            raise TypeError(f"LPIPS takes uint8 images, got {a.dtype} and {b.dtype}")
        if a.dim() != 4 or a.shape != b.shape:
            raise ValueError(f"LPIPS takes two uint8 [N,H,W,3] batches of equal shape, got {tuple(a.shape)} and {tuple(b.shape)}")
        if a.shape[3] != 3:
            raise ValueError(f"LPIPS (VGG16) takes RGB images, got {a.shape[3]} channels")
        if min(a.shape[1], a.shape[2]) < MIN_SIZE:
            raise ValueError(f"LPIPS needs images of at least {MIN_SIZE}x{MIN_SIZE} pixels (four 2x2 pools), got {a.shape[1]}x{a.shape[2]}")
        return a, b

    @L.on_model_device
    def __call__(self, images0_u8, images1_u8):
        """float64 [N] on the device: LPIPS of pair n = (images0[n], images1[n]).  A non-finite value raises FloatingPointError (an
        activation beyond the split-fp16 range, 65520, turns into NaN)."""
        a, b = self.check_images(images0_u8, images1_u8)
        n = a.shape[0]
        out = torch.zeros((n,), dtype=torch.float64, device=self.device)
        if n == 0:
            return out
        x = torch.cat([a.to(self.device), b.to(self.device)]).contiguous()     # first images, then second: one batch of 2N
        c0 = self._convs[0]
        y = conv_in(x, self._shift, self._scale, c0.w_kn, c0.bias)
        for (idx, _, _), cw in zip(CONVS[1:], self._convs[1:]):
            if idx in POOL_BEFORE:
                opd = maxpool2x2_split(y)
            else:
                opd = L.split_f16x2(y.reshape(-1, y.shape[-1])).reshape(*y.shape[:3], 2 * y.shape[-1])
            y = L.tc_conv(opd, cw.w_nk, cw.bias, act=L.ACT_RELU)
            if idx in TAPS:
                lpips_tap(y, self._lin[TAPS[idx]], out)
        if not bool(torch.isfinite(out).all()):
            raise FloatingPointError("LPIPS is not finite: a VGG16 activation left the range of the exact split-fp16 convolutions "
                                     "(|x| < 65520)")
        return out

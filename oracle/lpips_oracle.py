"""TEST INFRASTRUCTURE — fp64 restatement of ``lpips.LPIPS(net='vgg', version='0.1').forward(in0, in1)`` (lpips 0.1.3, normalize=False)
from the two state dicts it loads: torchvision's VGG16 ``features`` and lpips' ``lin0..lin4``.  Written from the published definition of
the network (no lpips source is on this path); tests/test_lpips_host.py pins the five taps to ``torchvision.models.vgg16().features``.

    scaling layer   (x - shift) / scale per channel
    VGG16 taps      features[0:4], [4:9], [9:16], [16:23], [23:30]: relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
    per tap         f / (sqrt(sum_c f^2) + 1e-10) on both sides, squared difference, 1x1 conv lin{k} (no bias), mean over H x W
    result          sum of the five taps, one value per image

Device-agnostic torch: NCHW in (any float dtype; computed in fp64 on the inputs' device), [N] fp64 out.
``lpips_state_dicts`` / ``make_lpips_weights`` give seeded random weights in both files' key layouts.
"""
import math
import os

import torch
import torch.nn.functional as F

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
# torchvision vgg16().features up to index 29: 'C' = Conv2d(3x3, pad 1) + ReLU at index i, i + 1; 'M' = MaxPool2d(2, 2) at index i
_LAYOUT = [(0, "C", 3, 64), (2, "C", 64, 64), (4, "M"), (5, "C", 64, 128), (7, "C", 128, 128), (9, "M"),
           (10, "C", 128, 256), (12, "C", 256, 256), (14, "C", 256, 256), (16, "M"),
           (17, "C", 256, 512), (19, "C", 512, 512), (21, "C", 512, 512), (23, "M"),
           (24, "C", 512, 512), (26, "C", 512, 512), (28, "C", 512, 512)]
TAP_ENDS = (4, 9, 16, 23, 30)              # the slices' ends: a tap is the activation after the layers below this index
TAP_CHANNELS = (64, 128, 256, 512, 512)
CONVS = [(e[0], e[2], e[3]) for e in _LAYOUT if e[1] == "C"]

VGG16_NAME = "vgg16-397923af.pth"          # torchvision's file name
LIN_NAME = "vgg.pth"                       # lpips: weights/v0.1/vgg.pth


def scaling_layer(x):
    sh = torch.tensor(SHIFT, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    sc = torch.tensor(SCALE, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    return (x.double() - sh) / sc


def taps(x, vgg):
    """The five VGG16 taps of x (NCHW, already through the scaling layer), fp64."""
    h, out = x.double(), []
    for e in _LAYOUT:
        if e[1] == "C":
            w, b = vgg[f"features.{e[0]}.weight"], vgg[f"features.{e[0]}.bias"]
            h = F.relu(F.conv2d(h, w.to(h), b.to(h), padding=1))
        else:
            h = F.max_pool2d(h, 2, 2)
        end = e[0] + (2 if e[1] == "C" else 1)
        if end in TAP_ENDS:
            out.append(h)
    return out


def normalize_tensor(f, eps=1e-10):
    return f / (torch.sqrt((f * f).sum(1, keepdim=True)) + eps)


def tap_terms(f0, f1, lin_w):
    """[N] fp64: mean over H x W of the lin-weighted squared difference of the channel-normalised features of one tap."""
    d = (normalize_tensor(f0) - normalize_tensor(f1)) ** 2
    return (d * lin_w.to(d).reshape(1, -1, 1, 1)).sum(1).mean((1, 2))


def forward(in0, in1, vgg, lin):
    """LPIPS of each pair (in0[n], in1[n]), NCHW images as LPIPS.forward receives them: [N] fp64."""
    t0, t1 = taps(scaling_layer(in0), vgg), taps(scaling_layer(in1), vgg)
    val = 0.0
    for k, (a, b) in enumerate(zip(t0, t1)):
        val = val + tap_terms(a, b, lin[f"lin{k}.model.1.weight"])
    return val


def forward_u8(images0_u8, images1_u8, vgg, lin):
    """forward() of uint8 NHWC batches converted as LPIPSMetric does (tf.image.convert_image_dtype: x * fp32(1/255) in fp32)."""
    conv = lambda x: (torch.as_tensor(x).to(torch.float32) * torch.tensor(1.0 / 255, dtype=torch.float32)).permute(0, 3, 1, 2)
    return forward(conv(images0_u8), conv(images1_u8), vgg, lin)


def lpips_state_dicts(seed):
    """(VGG16 features state dict, lpips lin state dict), fp32, seeded: the convs as torchvision initialises VGG16 (Kaiming normal,
    fan_out, ReLU gain) plus small random biases so that the bias path is exercised; non-negative lin weights, as lpips' released ones."""
    g = torch.Generator().manual_seed(int(seed))
    vgg = {}
    for idx, cin, cout in CONVS:
        vgg[f"features.{idx}.weight"] = torch.randn((cout, cin, 3, 3), generator=g) * math.sqrt(2.0 / (cout * 9))
        vgg[f"features.{idx}.bias"] = 0.02 * torch.randn((cout,), generator=g)
    lin = {f"lin{k}.model.1.weight": torch.rand((1, c, 1, 1), generator=g) for k, c in enumerate(TAP_CHANNELS)}
    return vgg, lin


def make_lpips_weights(seed, directory):
    """Writes lpips_state_dicts(seed) as ``vgg16-397923af.pth`` and ``vgg.pth`` under ``directory``; returns the two paths."""
    vgg, lin = lpips_state_dicts(seed)
    os.makedirs(directory, exist_ok=True)
    paths = os.path.join(directory, VGG16_NAME), os.path.join(directory, LIN_NAME)
    torch.save(vgg, paths[0])
    torch.save(lin, paths[1])
    return paths


def weight_sums(vgg, lin):
    """fp64 sums of every tensor in key order: guards the regeneration of the seeded weights."""
    return [float(t.double().sum()) for sd in (vgg, lin) for _, t in sorted(sd.items())]

"""Evaluation-side pieces around the hot path (GPU): dataset resize rule, image / camera metrics, transformer_predict,
test_step / predict_step, generate() on images that need resizing — against plain torch restatements of the reference code."""
import math
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import launch_checks as lc
from oracle import synth, vqgan_oracle as vo, migt_oracle as mo
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu


def resize_th_ref(x_u8_nhwc, size, method=None):
    """data/_common.py:19-62 restated (torch CPU): resize() keeps NHWC images whose width is ``size``, resize_th() keeps NCHW images whose
    height is ``size`` and picks the method from the height."""
    if x_u8_nhwc.shape[2] == size:                                      # resize(): images.shape[-2] of NHWC
        return x_u8_nhwc
    x = x_u8_nhwc.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    if x.shape[-2] == size:                                             # resize_th(): th_images.shape[-2] of NCHW
        return x_u8_nhwc
    if method is None:
        method = "nearest" if size > x.shape[-2] else "bilinear"
    y = F.interpolate(x, (size, size), mode="nearest") if method == "nearest" else F.interpolate(x, (size, size), mode="bilinear", align_corners=False)
    return (y.clamp_(0, 1) * 255.0).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("h,size,method", [(96, 128, None), (200, 128, None), (256, 128, None), (128, 64, "nearest"), (50, 128, "bilinear"), (128, 128, None)]
                         + [pytest.param(hw, 128, None, id=f"{hw[0]}x{hw[1]}-128-None") for hw in ((96, 160), (160, 96), (128, 200), (200, 128), (480, 640))])
def test_resize_matches_torch(h, size, method):
    """Square frames, and non-square ones where the reference's rule (method from the height, unchanged when either side is the size)
    differs from one that looks at the width: 96 x 160 grows with nearest, 160 x 96 shrinks bilinearly, 128 x 200 and 200 x 128 come back
    unchanged (and non-square).  Every output is also held to launch_checks.check_resize_u8 (fp64, bit-exact but within 64 u of an integer).
    The non-square bilinear cases scale by 1.25 / 0.75 and 3.75 / 5: their interpolation weights are multiples of 1/8 or 1/64, so many
    pixels land exactly on an integer before truncation, where fp32 rounding in torch's CPU kernel and in ours may fall on either side
    (0.2 to 0.7 % of pixels, 1 LSB); there the checker, not the share of exact pixels, is the bar."""
    from viewformer_b200 import _lib as L
    hh, ww = h if isinstance(h, tuple) else (h, h)
    x = torch.randint(0, 256, (3, hh, ww, 3), generator=torch.Generator().manual_seed(hh if hh == ww else hh * 1000 + ww), dtype=torch.uint8)
    want = resize_th_ref(x, size, method)
    xc = x.cuda()
    got_dev, r = lc.run_check("resize_u8", L.resize_u8, (xc, size, method), {}, random.Random(0))
    assert r == 0.0
    assert (got_dev is xc) == (want is x)
    got = got_dev.cpu()
    assert got.shape == want.shape
    d = (got.int() - want.int()).abs()
    print(f"[resize {hh}x{ww}->{size} {method}] exact {float((d == 0).float().mean()):.5f}, max diff {int(d.max())}")
    assert int(d.max()) <= 1
    if hh == ww:
        assert float((d == 0).float().mean()) > 0.999


def ssim_ref(X, Y):
    """utils/metrics.py:17-73 restated with a depthwise 7x7 box filter (NHWC float in [0,1])."""
    X, Y = X.permute(0, 3, 1, 2).double(), Y.permute(0, 3, 1, 2).double()
    c = X.shape[1]
    k = torch.full((c, 1, 7, 7), 1 / 49.0, dtype=torch.float64)
    f = lambda t: F.conv2d(t, k, groups=c)
    ux, uy, uxx, uyy, uxy = f(X), f(Y), f(X * X), f(Y * Y), f(X * Y)
    cn = 49 / 48
    vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
    return S.mean((1, 2, 3))


def test_image_and_camera_metrics():
    from viewformer_b200.metrics import image_metrics, Evaluator, camera_orientation_error
    g = torch.Generator().manual_seed(4)
    a = synth.make_images_uint8(1, 5, size=64, seed=1)[0]
    b = (a.int() + torch.randint(-20, 21, a.shape, generator=g)).clamp(0, 255).to(torch.uint8)
    m = image_metrics(a, b)
    A, B = a.double() / 255, b.double() / 255
    mse = ((A - B) ** 2).mean((1, 2, 3))
    assert torch.allclose(m["mse"].cpu(), mse, rtol=1e-12) and torch.allclose(m["mae"].cpu(), (A - B).abs().mean((1, 2, 3)), rtol=1e-12)
    assert torch.allclose(m["psnr"].cpu(), 10 * torch.log10(1 / mse), rtol=1e-12)
    assert torch.allclose(m["rmse"].cpu(), torch.sqrt(((a.double() - b.double()) ** 2).mean((1, 2, 3))), rtol=1e-12)
    s = ssim_ref(A.float(), B.float())
    print(f"[ssim] got {m['ssim'].cpu().tolist()} want {s.tolist()}")
    assert torch.allclose(m["ssim"].cpu(), s, atol=2e-5)
    ev = Evaluator()
    ev.update_with_image(a, b)
    cams = synth.make_cameras(1, 5, seed=3)[0]
    rot = cams.clone()
    rot[:, :3] += 0.5
    ev.update_with_camera(cams, rot)
    r = ev.result()
    assert abs(r["psnr"] - float(m["psnr"].mean())) < 1e-9 and abs(r["loc-dist"] - math.sqrt(0.75)) < 1e-5 and r["loc-angle"] < 1e-3
    half = torch.tensor([[0, 0, 0, math.cos(0.25), math.sin(0.25), 0, 0]], dtype=torch.float32)
    ident = torch.tensor([[0, 0, 0, 1.0, 0, 0, 0]])
    assert abs(float(camera_orientation_error(half, ident)) - 0.5) < 1e-6


def _small_models(precision="fp32", loc="1"):
    from viewformer_b200 import VQGAN, MIGT
    vcfg = VQGANConfig(ch=64, ch_mult=[1, 2, 2, 2], attn_resolutions=[8], image_size=32, embed_dim=64, z_channels=64, n_embed=256, num_res_blocks=1)
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=4, n_loss_skip=1,
                      localization_weight=loc)
    vsd, tsd = synth.make_vqgan_state_dict(vcfg, 31), synth.make_migt_state_dict(tcfg, 32)
    return vcfg, tcfg, vsd, tsd, VQGAN(vcfg, precision=precision).load_state_dict(vsd), MIGT(tcfg, precision=precision).load_state_dict(tsd)


def test_transformer_predict_and_steps_match_oracle():
    from viewformer_b200 import transformer_predict, run_with_batchsize, encode_images, decode_code
    vcfg, tcfg, vsd, tsd, cb, tr = _small_models()
    images = synth.make_images_uint8(3, 4, size=32, seed=41)
    cams = synth.make_cameras(3, 4, seed=42)
    codes = encode_images(images, codebook_model=cb)
    with torch.no_grad():
        want_codes = vo.encode(vsd, vcfg, mo.images_to_float(images.reshape(-1, 32, 32, 3)).permute(0, 3, 1, 2).contiguous())[2].reshape(3, 4, 4, 4)
        want = mo.generate_batch_predictions_multictx(lambda d: mo.forward(tsd, tcfg, d), lambda x: vo.encode(vsd, vcfg, x)[2],
                                                      lambda c: vo.decode_code(vsd, vcfg, c), tcfg, images, cams)
    assert torch.equal(codes.cpu(), want_codes)
    gen_cams, gen_codes = run_with_batchsize(transformer_predict, 2, cams, codes.cpu(), transformer_model=tr)
    assert torch.equal(gen_codes.cpu(), want["generated_codes"])
    assert torch.allclose(gen_cams.cpu(), want["generated_cameras"], atol=1e-3)
    imgs = decode_code(gen_codes, codebook_model=cb)
    assert int((imgs.cpu().int() - want["generated_images"].int()).abs().max()) <= 1
    # Keras evaluation steps
    tr.codebook_model = cb
    rel = mo.normalize_cameras(mo.to_relative_cameras(cams)[0])
    with torch.no_grad():
        o = mo.forward(tsd, tcfg, dict(input_ids=codes.cpu(), poses=rel), compute_losses=True)
    res = tr.test_step((rel, codes))
    assert abs(res["loss"] - float(o["loss"].mean())) < 1e-4 * max(1.0, abs(float(o["loss"].mean())))
    acc = float((o["logits"].argmax(-1)[:, 1:] == codes.cpu()[:, 1:]).float().mean())
    assert abs(res["acc"] - acc) < 1e-6 and res["psnr"] > 0
    ps = tr.predict_step((rel, codes))
    assert torch.equal(ps["latent_code"].cpu(), o["logits"].argmax(-1)) and list(ps["decoded_image"].shape) == [12, 32, 32, 3]


def test_generate_resizes_inputs_like_the_reference():
    """48x48 inputs for a 32x32 codebook: generate() applies resize_tf (bilinear, align_corners=False) before encoding."""
    from viewformer_b200 import generate_batch_predictions
    vcfg, tcfg, vsd, tsd, cb, tr = _small_models(loc="0")
    images = synth.make_images_uint8(2, 3, size=48, seed=51)
    cams = synth.make_cameras(2, 3, seed=52)
    small = resize_th_ref(images.reshape(-1, 48, 48, 3), 32).reshape(2, 3, 32, 32, 3)
    with torch.no_grad():
        want = mo.generate_batch_predictions(lambda d: mo.forward(tsd, tcfg, d, use_localization=False), lambda x: vo.encode(vsd, vcfg, x)[2],
                                             lambda c: vo.decode_code(vsd, vcfg, c), tcfg, small, cams, use_localization=False)
    got = generate_batch_predictions(tr, cb, images, cams)
    agree = float((got["generated_codes"].cpu() == want["generated_codes"]).float().mean())
    print(f"[generate + resize] generated-code agreement {agree:.3f}")
    assert agree >= 0.95            # a 1-LSB difference in a resized pixel may flip a near-tied code
    assert got["ground_truth_images"].shape[-3:] == (48, 48, 3)

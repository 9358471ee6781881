"""Four-channel (RGBA) codebooks on the GPU: the CO3Dv2 codebook layout (in_channels = out_ch = 4: masked RGB + mask), end to end.

  * the exact conv_in / conv_out kernels at 4 channels against fp64 (tests/launch_checks.py, the bars of conv3x3_small_cin / _cout,
    fused GroupNorm sums included), next to the 3-channel instances; the float-image conversions against theirs
    (tests/launch_checks_float.py);
  * codes bit-identical to the real reference's 4-channel VQGAN (tests/golden/vqgan_rgba_small.npz) in fp32 and mixed, pixels within
    DESIGN.md section 7's bars;
  * generate_batch_predictions on uint8 RGBA frames and on float32 RGBA frames in [0, 1] (evaluate_co3dv2_challenge.py:72-77);
  * both codebook training steps against two steps of the reference (tests/golden/vqgan_rgba_train_small.npz), and the commit
    quantizer's bf16 step against its fp32 step;
  * one fp64 launch audit of a 4-channel generate and of both 4-channel training steps.
"""
import os
import random

import numpy as np
import pytest
import torch

import launch_checks as lc
import launch_checks_float as lcf
from oracle import synth, migt_oracle as mo
from oracle.make_golden_rgba import RGBA_VQ, RGBA_TC_VQ, rgba_images
from viewformer_b200 import float_images
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu

# ch 128: conv_in 4 -> 128 and conv_out 128 -> 4 take the dedicated kernels (the small fixture config's ch 32 takes the generic ones)
RGBA_TC = dict(RGBA_TC_VQ, perceptual_weight=0.0)


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def _nchw(u8):
    return mo.images_to_float(u8).permute(0, 3, 1, 2).contiguous()


def _stats(name, got, want):
    err = (got.double().cpu() - want.double().cpu()).abs()
    print(f"[{name}] max_abs_err={err.max():.3e} mean_abs_err={err.mean():.3e}")
    return float(err.max()), float(err.mean())


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("cin", [3, 4])
@pytest.mark.parametrize("shape", [(2, 128, 128), (1, 37, 45)])
def test_conv_in_small_kernels_vs_fp64(L, cin, shape):
    """conv_in C -> 128 with the fused GroupNorm(32) sums, and C -> 32 (the generic small-Cin kernel), against fp64 on the same operands."""
    n, h, w = shape
    g = torch.Generator().manual_seed(10 * cin + h)
    x = (torch.rand((n, h, w, cin), generator=g) * 2 - 1).cuda()
    worst = {}
    for cout in (128, 32):
        wk = ((torch.rand((9 * cin, cout), generator=g) * 2 - 1) / (9 * cin) ** 0.5).cuda()
        b = (torch.rand(cout, generator=g) * 0.2 - 0.1).cuda()
        y, r = lc.run_check("conv3x3_small_cin", L.conv3x3_small_cin, (x, wk, b), dict(gn_groups=32), random.Random(0))
        assert hasattr(y, "_gn_sums") == (cout == 128)
        worst[cout] = r
    print(f"[conv_in {cin} ch {shape}] worst ratio to the bar: {worst}")
    assert max(worst.values()) <= 1.0


@pytest.mark.parametrize("cout", [3, 4])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 128, 128), (1, 37, 45)])
def test_conv_out_small_kernel_vs_fp64(L, cout, dtype, shape):
    """conv_out 128 -> C on fp32 and bf16 activations against fp64 on the same (bf16-stored) operands; odd widths end runs mid-window."""
    n, h, w = shape
    g = torch.Generator().manual_seed(100 * cout + w)
    x = torch.randn((n, h, w, 128), generator=g).to(dtype).cuda()
    wk = ((torch.rand((1152, cout), generator=g) * 2 - 1) / 34.0).cuda()
    b = (torch.rand(cout, generator=g) * 0.2 - 0.1).cuda()
    y, r = lc.run_check("conv3x3_small_cout", L.conv3x3_small_cout, (x, wk, b), {}, random.Random(0))
    print(f"[conv_out {cout} ch {dtype} {shape}] worst ratio to the bar: {r:.3g}")
    assert y.shape == (n, h, w, cout) and r <= 1.0


def test_small_kernels_reject_other_channel_counts(L):
    x5 = torch.zeros((1, 8, 8, 5), device="cuda")
    with pytest.raises(L.LibraryError, match="Cin = 3 or 4"):
        L.conv3x3_small_cin(x5, torch.zeros((45, 128), device="cuda"), None)
    with pytest.raises(L.LibraryError, match="128->3 and 128->4"):
        L.conv3x3_small_cout(torch.zeros((1, 8, 8, 128), device="cuda"), torch.zeros((1152, 5), device="cuda"), None)


# ----------------------------------------------------------------------------------------------- the codebook against the reference
@pytest.mark.parametrize("prefix,precision,pix_max,pix_mean", [("", "fp32", 2e-4, 2e-5), ("tc.", "fp32", 2e-4, 2e-5),
                                                               ("tc.", "mixed", 1.5e-1, 2e-2)])
def test_rgba_codebook_matches_reference(golden_dir, prefix, precision, pix_max, pix_mean):
    """Codes bit-identical to the reference's 4-channel VQGAN in both precisions whose encoder is fp32-faithful; decode_code and forward
    pixels within the fp32 bar (2e-4) or, for mixed (bf16 decoder), the bf16 bars of tests/test_models_gpu.py.  mixed runs at ch 128
    (``tc.``): its exact tensor-core GEMMs need 64-channel multiples, which the small config's ch 32 is not, at any channel count."""
    from viewformer_b200 import VQGAN
    f = np.load(os.path.join(golden_dir, "vqgan_rgba_small.npz"))
    g = {k[len(prefix):]: f[k] for k in f.files if k.startswith(prefix) and (prefix or not k.startswith("tc."))}
    cfg = VQGANConfig(**(RGBA_TC_VQ if prefix else RGBA_VQ))
    model = VQGAN(cfg, precision=precision).load_state_dict(synth.make_vqgan_state_dict(cfg, 0))
    u8 = torch.from_numpy(g["images"])
    x = _nchw(u8)
    q, d, c = model.encode(x)
    assert torch.equal(c.cpu(), torch.from_numpy(g["codes"])), f"codes differ at {int((c.cpu() != torch.from_numpy(g['codes'])).sum())} positions"
    assert abs(float(d) - float(g["diff"])) < 1e-5 * max(1.0, float(g["diff"]))
    dec = model.decode_code(torch.from_numpy(g["codes"]))
    assert dec.shape == (2, 4, 32, 32)
    mx, mean = _stats(f"decode_code {precision}", dec, torch.from_numpy(g["dec"]))
    assert mx < pix_max and mean < pix_mean
    rec, _, _, c2 = model(x)
    mx, mean = _stats(f"forward {precision}", rec, torch.from_numpy(g["rec"]))
    assert mx < pix_max and mean < pix_mean and torch.equal(c2, c)
    # the uint8 NHWC entry point converts as the reference does: the same codes
    assert torch.equal(model.encode_u8(u8.cuda()).cpu(), c.cpu())


def _generate_models(precision="fp32"):
    from viewformer_b200 import VQGAN, MIGT
    vcfg = VQGANConfig(**RGBA_VQ)
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=8,
                      localization_weight="0")
    vq = VQGAN(vcfg, precision=precision).load_state_dict(synth.make_vqgan_state_dict(vcfg, 0))
    tr = MIGT(tcfg, precision=precision).load_state_dict(synth.make_migt_state_dict(tcfg, 12))
    return tr, vq


def test_generate_rgba_uint8_and_float(L):
    """generate_batch_predictions on uint8 RGBA frames and on float32 frames equal to them / 255 (the challenge's input), formed as
    tf.image.convert_image_dtype forms it (x * fp32(1/255); x / 255 rounds differently for 111 of the 256 byte values): the float
    conversion is torch's x * 2 - 1 bit for bit, the context codes are those of ``encode`` on the converted tensor, the uint8 and float
    inputs give the same codes and views, 4-channel uint8.  Float frames of another size go through the float resize; float64 frames are refused."""
    from viewformer_b200 import generate_batch_predictions, generate_batch_predictions_multictx
    from viewformer_b200.evaluate import encode_images
    tr, vq = _generate_models()
    B, T = 2, 4
    u8 = rgba_images(B * T, 32, 4200).reshape(B, T, 32, 32, 4)
    f = u8.float() * torch.tensor(1.0 / 255.0, dtype=torch.float32)
    cams = synth.make_cameras(B, T, seed=14)
    fd = f.cuda()
    conv, r = lcf.run_check("f01_to_unit", float_images.f01_to_unit, (fd,), dict(first_views=T - 1), random.Random(0))
    assert r == 0.0
    assert torch.equal(conv.view(torch.int32), (fd[:, :T - 1].reshape(-1, 32, 32, 4) * 2 - 1).view(torch.int32))
    codes_f = vq.encode_images(fd, first_views=T - 1)
    assert torch.equal(codes_f, vq.encode(conv.permute(0, 3, 1, 2).contiguous())[2])
    codes_u = vq.encode_images(u8.cuda(), first_views=T - 1)
    assert torch.equal(codes_u, vq.encode(_nchw(u8[:, :T - 1].reshape(-1, 32, 32, 4)).cuda())[2])
    out_u = generate_batch_predictions(tr, vq, u8, cams)
    out_f = generate_batch_predictions(tr, vq, f, cams)
    assert out_u["generated_images"].shape == (B, 32, 32, 4) and out_u["generated_images"].dtype == torch.uint8
    print(f"[generate rgba] context codes equal between uint8 and float input: {float((codes_u == codes_f).float().mean()):.4f}")
    assert torch.equal(codes_u, codes_f)
    assert torch.equal(out_u["generated_codes"], out_f["generated_codes"])
    assert torch.equal(out_u["generated_images"], out_f["generated_images"])
    assert torch.equal(out_f["ground_truth_images"], f[:, -1])
    # a float frame at 48 x 48 shrinks bilinearly in float (no 1/255 quantisation) before the encoder
    big = torch.nn.functional.interpolate(f.reshape(-1, 32, 32, 4).permute(0, 3, 1, 2), size=(48, 48), mode="nearest")
    big = big.permute(0, 2, 3, 1).reshape(B, T, 48, 48, 4).contiguous()
    small, r = lcf.run_check("resize_f32", float_images.resize_f32, (big[:, :T - 1].reshape(-1, 48, 48, 4).cuda(), 32), {}, random.Random(0))
    assert r <= 1.0 and small.dtype == torch.float32
    out_big = generate_batch_predictions(tr, vq, big, cams)
    assert out_big["generated_images"].shape == (B, 32, 32, 4)
    assert torch.equal(encode_images(big[:, :T - 1], codebook_model=vq).reshape(-1, 8, 8), vq.encode_images(small))
    from viewformer_b200 import MIGT
    loc = MIGT(MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=64, token_image_size=8),
               precision="fp32").load_state_dict(synth.make_migt_state_dict(MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4,
                                                                                       n_embeddings=64, token_image_size=8), 12))
    m = generate_batch_predictions_multictx(loc, vq, f, cams)
    assert m["generated_images"].shape == (B, T, 32, 32, 4)
    for bad in (f.double(), u8.to(torch.int32)):
        with pytest.raises(TypeError):
            generate_batch_predictions(tr, vq, bad, cams)
    with pytest.raises(ValueError, match="4-channel"):
        vq.encode_images(u8[..., :3].contiguous().cuda(), first_views=T - 1)


# ----------------------------------------------------------------------------------------------- training
def _rgba_step_model(train_precision, quantizer="ema", overrides=None, seed=5):
    from viewformer_b200 import VQGAN
    cfg = VQGANConfig(**(overrides or dict(RGBA_VQ, perceptual_weight=0.0)))
    sd = synth.make_vqgan_state_dict(cfg, seed)
    if quantizer == "commit":
        sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
    model = VQGAN(cfg, precision="fp32", quantizer=quantizer, train_precision=train_precision).load_state_dict(sd)
    return cfg, model, model.configure_optimizers()


def test_rgba_training_step_fp32_matches_reference(golden_dir):
    """Two fp32 steps against the reference's, at tests/test_train_gpu.py's bars: codes equal, loss 2e-5, gradient norm / projection
    3e-3 relative over all tensors, element-wise gradients 2e-3 (conv_in and conv_out among them), post-step weights, EMA codebook."""
    g = np.load(os.path.join(golden_dir, "vqgan_rgba_train_small.npz"))
    cfg, model, tr = _rgba_step_model("fp32")
    assert tr.convs["encoder.conv_in"].cw.small_cin and (tr.convs["encoder.conv_in"].fw, tr.convs["decoder.conv_out"].fw) == ("cuda", "cuda")
    names = [str(n) for n in g["names"]]
    gen = torch.Generator().manual_seed(99)
    probe = None
    for step in range(2):
        x = _nchw(torch.from_numpy(g[f"images{step}"]))
        loss = tr.forward_backward(x)
        torch.cuda.synchronize()
        assert np.array_equal(tr.last["codes"].cpu().numpy(), g[f"codes{step}"])
        assert abs(float(loss) - float(g[f"loss{step}"])) < 2e-5 * max(1.0, abs(float(g[f"loss{step}"])))
        grads = tr.export_gradients()
        assert set(grads) == set(names)
        if probe is None:
            probe = {n: torch.randn(grads[n].shape, generator=gen) for n in names}
        worst = 0.0
        for i, n in enumerate(names):
            gn, gd = float(grads[n].norm()), float((grads[n] * probe[n]).sum())
            rn, rd = float(g[f"gnorm{step}"][i]), float(g[f"gdot{step}"][i])
            e = max(abs(gn - rn), abs(gd - rd)) / max(rn, 1e-4)
            worst = max(worst, e)
            assert e < 3e-3, f"step {step} {n}: |g| {gn:.6e} vs {rn:.6e}, <g,probe> {gd:.6e} vs {rd:.6e}"
        full = [k[len(f"g{step}."):] for k in g.files if k.startswith(f"g{step}.")]
        for n in full:
            ref = torch.from_numpy(g[f"g{step}.{n}"])
            err = float((grads[n] - ref).abs().max() / ref.abs().max().clamp_min(1e-4))
            assert err < 2e-3, f"step {step} grad {n}: max rel err {err:.3e}"
        print(f"[rgba fp32 step {step}] loss {float(loss):.6f} (ref {float(g[f'loss{step}']):.6f}); worst gradient norm/projection {worst:.2e}")
        tr.optimizer_step()
        sd = tr.export_state_dict()
        for n in full:
            d = (sd[n] - torch.from_numpy(g[f"p{step}.{n}"])).abs()
            assert float((d > 0.05 * cfg.learning_rate).float().mean()) < 0.02, f"step {step} weight {n}"
        np.testing.assert_allclose(model._w["q"]["emb"].cpu().numpy(), g[f"emb{step}"], rtol=2e-4 if step == 0 else 5e-3,
                                   atol=2e-5 if step == 0 else 2e-4)


def test_rgba_training_step_bf16_matches_reference(golden_dir):
    """The bf16 step against the reference's first step: loss within 5e-3 relative (tests/test_train_bf16_gpu.py's bar) and >= 97 % of the
    codes equal.  Its gradients are held by test_rgba_bf16_step_matches_fp32_step_medium (cosine >= 0.99 to the fp32 step, which this
    file pins to the reference tensor by tensor): at this config's ch 32 the bf16 gradients of the small-norm tensors are further from the
    reference than the full-size bars (measured on an H100: median 1.3e-1, worst 7.9e-1 at decoder.mid.attn_1.q.bias)."""
    g = np.load(os.path.join(golden_dir, "vqgan_rgba_train_small.npz"))
    cfg, model, tr = _rgba_step_model("bf16")
    names = [str(n) for n in g["names"]]
    loss = float(tr.forward_backward(_nchw(torch.from_numpy(g["images0"]))))
    torch.cuda.synchronize()
    grads = tr.export_gradients()
    gen = torch.Generator().manual_seed(99)
    probe = {n: torch.randn(grads[n].shape, generator=gen) for n in names}
    errs = []
    for i, n in enumerate(names):
        gn, gd = float(grads[n].norm()), float((grads[n] * probe[n]).sum())
        rn, rd = float(g["gnorm0"][i]), float(g["gdot0"][i])
        errs.append((max(abs(gn - rn), abs(gd - rd)) / max(rn, 1e-4), n))
    worst, med = max(errs), float(np.median([e for e, _ in errs]))
    same = float((tr.last["codes"].cpu() == torch.from_numpy(g["codes0"])).float().mean())
    print(f"[rgba bf16 step] loss {loss:.6f} vs ref {float(g['loss0']):.6f}; codes equal {same:.3f}; worst {worst[0]:.2e} ({worst[1]}), median {med:.2e}")
    assert abs(loss - float(g["loss0"])) <= 5e-3 * abs(float(g["loss0"]))
    assert same >= 0.97


@pytest.mark.parametrize("quantizer", ["ema", "commit"])
def test_rgba_bf16_step_matches_fp32_step_medium(quantizer):
    """ch 128 (conv_in 4 -> 128 and conv_out 128 -> 4 on the dedicated kernels): one bf16 step next to the fp32 step from the same
    weights, at tests/test_train_bf16_gpu.py's medium bars (loss 5e-3 relative, gradient cosine >= 0.99); both quantizers.  The ends
    take the same routes as in a 3-channel model."""
    from viewformer_b200.train import conv_routes
    cfg, _, t32 = _rgba_step_model("fp32", quantizer, RGBA_TC)
    _, _, t16 = _rgba_step_model("bf16", quantizer, RGBA_TC)
    for t in (t32, t16):
        for name, (cin3, cout3) in (("encoder.conv_in", (3, 128)), ("decoder.conv_out", (128, 3))):
            c = t.convs[name]
            assert (c.fw, c.dgrad, c.wgrad) == conv_routes(t.precision, t.use_tc, 3, cin3, cout3, out=c.out)
    assert t32.convs["encoder.conv_in"].cw.small_cin and t32.convs["decoder.conv_out"].cw.small_cout
    x = _nchw(rgba_images(4, 32, 4300))
    l32, l16 = float(t32.forward_backward(x)), float(t16.forward_backward(x))
    torch.cuda.synchronize()
    g32, g16 = t32.export_gradients(), t16.export_gradients()
    top = max(float(v.norm()) for v in g32.values())
    cos = {k: float((v.double() * g16[k].double()).sum() / (v.double().norm() * g16[k].double().norm()))
           for k, v in g32.items() if float(v.norm()) > 1e-4 * top}
    worst = min(cos, key=cos.get)
    print(f"[rgba bf16 vs fp32, {quantizer}] loss {l16:.6f} vs {l32:.6f}; min cosine {cos[worst]:.5f} ({worst}) over {len(cos)} tensors")
    assert abs(l16 - l32) <= 5e-3 * abs(l32)
    assert cos[worst] >= 0.99
    for t in (t32, t16):
        t.optimizer_step()


# ----------------------------------------------------------------------------------------------- launch audit
def test_rgba_launch_audit(L, monkeypatch):
    """Every checked launch of a 4-channel generate (mixed codebook at ch 128, float frames resized from 48 x 48) and of one fp32 and
    one bf16 4-channel training step, against fp64 on its own operands (tests/launch_checks.py and, for the float-image conversions,
    tests/launch_checks_float.py), through the same wrapper hooks as tests/test_launch_audit_gpu.py."""
    from test_launch_audit_gpu import Audit
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions
    audit = Audit(L, monkeypatch)

    def wrap(name, fn):
        def call(*a, **k):
            with torch.no_grad():
                result, r = lcf.run_check(name, fn, a, k, audit.rng)
            audit.rec[(name, str(a[0].dtype).replace("torch.", "")) + audit._site()].append(r)
            return result
        return call
    for name in lcf.CHECKERS:
        monkeypatch.setattr(float_images, name, wrap(name, getattr(float_images, name)))
    vcfg = VQGANConfig(**RGBA_TC)
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=16,
                      localization_weight="0")
    cb = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, 0))
    tr = MIGT(tcfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(tcfg, 0))
    B, T = 2, 4
    f = rgba_images(B * T, 48, 4400).reshape(B, T, 48, 48, 4).float() / 255
    out = generate_batch_predictions(tr, cb, f, synth.make_cameras(B, T, seed=15))
    assert out["generated_images"].shape == (B, 32, 32, 4)
    for prec in ("fp32", "bf16"):
        _, _, t = _rgba_step_model(prec, "ema", RGBA_TC)
        t.training_step(_nchw(rgba_images(2, 32, 4500)))
    torch.cuda.synchronize()
    bad = audit.report("rgba")
    reached = audit.reached()
    for want in (("conv3x3_small_cin", "float32"), ("conv3x3_small_cout", "float32"), ("f01_to_unit", "float32"), ("resize_f32", "float32"),
                 ("conv_wgrad", "float32"), ("tc_conv", "bfloat16")):
        assert want in reached, f"{want} not reached"
    assert not bad, bad

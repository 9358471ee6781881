"""Model-level parity (GPU): the CUDA VQGAN / MIGT / generate() against the CPU oracle on the same seeded
weights and inputs, and against the golden vectors produced by the real reference.

Tolerances (stated per precision):
  fp32  (exact CUDA-core path): codes bit-exact; pixels / logits atol 2e-4 (reference's own th<->tf harness: 1e-5 on
        single layers, viewformer/utils/testing.py:98; a 60-conv network accumulates ~1e-5..1e-4).
  tf32  (wgmma .tf32): pixels atol 2e-2, >= 97% codes identical.
  bf16  (wgmma .bf16, the benchmarked mode): pixels atol 1.5e-1 / mean err <= 2e-2, >= 85% codes identical,
        logits: top-1 agreement >= 90% with |dlogit| small relative to the logit spread.
"""
import os

import numpy as np
import pytest
import torch

from oracle import synth, vqgan_oracle as vo, migt_oracle as mo
from oracle.make_golden import SMALL_VQ, SMALL_MIGT, vq_images
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu

TC_VQ = dict(ch=128, ch_mult=[1, 2], attn_resolutions=[16], image_size=32, embed_dim=64, z_channels=64, n_embed=256,
             num_res_blocks=1)


def _stats(name, got, want):
    err = (got.double().cpu() - want.double().cpu()).abs()
    print(f"[{name}] max_abs_err={err.max():.3e} mean_abs_err={err.mean():.3e} ref_std={want.double().std():.3e}")
    return float(err.max()), float(err.mean())


def _vq(cfg, seed, precision):
    from viewformer_b200 import VQGAN
    sd = synth.make_vqgan_state_dict(cfg, seed)
    return sd, VQGAN(cfg, precision=precision).load_state_dict(sd)


@pytest.mark.parametrize("name,overrides", [("small", SMALL_VQ), ("tc_small", TC_VQ)])
def test_vqgan_fp32_exact_path(name, overrides):
    cfg = VQGANConfig(**overrides)
    sd, model = _vq(cfg, 0, "fp32")
    x = vq_images(3, cfg.image_size, 77)
    with torch.no_grad():
        qo, do, co, zo = vo.encode(sd, cfg, x, return_pre_quant=True)
        deco = vo.decode_code(sd, cfg, co)
        reco, _, _, _ = vo.forward(sd, cfg, x)
    q, d, c = model.encode(x)
    assert torch.equal(c.cpu(), co), f"codes differ at {(c.cpu() != co).sum()} positions"
    assert _stats("quant", q, qo)[0] < 2e-4
    assert abs(float(d) - float(do)) < 1e-5 * max(1.0, float(do))
    assert _stats("decode_code", model.decode_code(co), deco)[0] < 2e-4
    dec, d2, q2, c2 = model(x)
    assert _stats("forward", dec, reco)[0] < 2e-4 and torch.equal(c2.cpu(), co)
    # NHWC (TF-twin) entry points agree with the NCHW ones
    qn, dn, cn = model.encode_nhwc(x.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(cn.cpu(), co) and torch.equal(qn.permute(0, 3, 1, 2).contiguous(), q)
    assert torch.equal(model.embed_code(co).cpu(), vo.embed_code(sd["quantize.embeddings"], co))


def test_vqgan_fp32_full_size_vs_reference_golden(golden_dir):
    """BASELINE config 1 shape: 4 images 128x128, weights from oracle/synth, golden from the REAL reference."""
    g = np.load(os.path.join(golden_dir, "vqgan_full.npz"))
    cfg = VQGANConfig()
    sd, model = _vq(cfg, int(g["seed"]), "fp32")
    x = vq_images(int(g["n_images"]), cfg.image_size, 1000 + int(g["seed"]))
    q, d, c = model.encode(x)
    mism = int((c.cpu().numpy() != g["codes"]).sum())
    print(f"[full fp32] code mismatches vs reference: {mism}/256")
    assert mism == 0
    assert abs(float(d) - float(g["diff"])) < 1e-4
    dec = model.decode_code(torch.from_numpy(g["codes"]))
    assert _stats("dec0", dec[0], torch.from_numpy(g["dec0"]))[0] < 3e-4
    assert _stats("dec sub", dec[:, :, ::4, ::4], torch.from_numpy(g["dec"]))[0] < 3e-4


@pytest.mark.parametrize("precision,pix_tol,mean_tol,code_frac", [("tf32", 2e-2, 2e-3, 0.99), ("bf16", 1e-1, 1e-2, 0.97)])
def test_vqgan_tensor_core_path_full_size(golden_dir, precision, pix_tol, mean_tol, code_frac):
    g = np.load(os.path.join(golden_dir, "vqgan_full.npz"))
    cfg = VQGANConfig()
    sd, model = _vq(cfg, int(g["seed"]), precision)
    x = vq_images(int(g["n_images"]), cfg.image_size, 1000 + int(g["seed"]))
    q, d, c = model.encode(x)
    agree = float((c.cpu().numpy() == g["codes"]).mean())
    print(f"[full {precision}] code agreement with reference: {agree:.4f}")
    assert agree >= code_frac
    dec = model.decode_code(torch.from_numpy(g["codes"]))
    mx, mean = _stats(f"dec0 {precision}", dec[0], torch.from_numpy(g["dec0"]))
    assert mx < pix_tol and mean < mean_tol


def test_vqgan_tc_small_all_precisions_agree():
    cfg = VQGANConfig(**TC_VQ)
    x = vq_images(5, cfg.image_size, 5)           # odd image count: exercises the TN=2 image-pair tiles at 8x8
    sd = synth.make_vqgan_state_dict(cfg, 3)
    with torch.no_grad():
        qo, do, co, zo = vo.encode(sd, cfg, x, return_pre_quant=True)
        deco = vo.decode_code(sd, cfg, co)
    from viewformer_b200 import VQGAN
    for prec, tol in (("tf32", 2e-2), ("bf16", 1.5e-1)):
        m = VQGAN(cfg, precision=prec).load_state_dict(sd)
        _, _, c = m.encode(x)
        print(f"[tc_small {prec}] code agreement {float((c.cpu() == co).float().mean()):.3f}")
        assert _stats(f"dec {prec}", m.decode_code(co), deco)[0] < tol


def test_vqgan_train_mode_ema_side_effect():
    """The reference updates the codebook inside forward when module.training (utils_th.py:46-64)."""
    cfg = VQGANConfig(**SMALL_VQ)
    sd, model = _vq(cfg, 1, "fp32")
    x = vq_images(2, cfg.image_size, 9)
    with torch.no_grad():
        z = vo._conv(sd, "quant_conv", vo.encoder(sd, cfg, x))
        _, _, ids, new = vo.quantize_ema(sd, z, training=True)
    model.train()
    _, _, c = model.encode(x)
    model.eval()
    assert torch.equal(c.cpu(), ids)
    got = model.state_dict()
    assert int(got["quantize.counter"]) == 1
    np.testing.assert_allclose(got["quantize.embeddings"].numpy(), new["quantize.embeddings"].numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got["quantize.ema_cluster_size_hidden"].numpy(), new["quantize.ema_cluster_size_hidden"].numpy(), rtol=1e-5, atol=1e-7)


# ----------------------------------------------------------------------------------------- MIGT
def _migt(cfg, seed, precision):
    from viewformer_b200 import MIGT
    sd = synth.make_migt_state_dict(cfg, seed)
    return sd, MIGT(cfg, precision=precision).load_state_dict(sd)


def _migt_inputs(cfg, B, T, seed=5):
    codes = synth.make_codes(B, T, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0])
    ids = torch.cat([codes[:, :-1], torch.full_like(codes[:, :1], cfg.n_embeddings)], 1)
    return codes, cams, ids


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-4), ("tf32", 1e-2), ("bf16", 6e-2)])
def test_migt_single_stream_small(precision, tol):
    cfg = MIGTConfig(**SMALL_MIGT)
    sd, model = _migt(cfg, 3, precision)
    codes, cams, ids = _migt_inputs(cfg, 3, 4)
    with torch.no_grad():
        o = mo.forward(sd, cfg, dict(input_ids=ids, poses=cams))
        o_loc = mo.forward(sd, cfg, dict(input_ids=codes, poses=cams[:, :-1]))
    got = model(dict(input_ids=ids, poses=cams))
    assert list(got["logits"].shape) == [3, 4, 8, 8, 1024]
    assert _stats(f"logits {precision}", got["logits"], o["logits"])[0] < tol
    assert _stats(f"pose {precision}", got["pose_prediction"], o["pose_prediction"])[0] < max(tol, 1e-3) * 5
    last = model(dict(input_ids=ids, poses=cams), last_only=True)["logits"]
    assert torch.allclose(last[:, 0], got["logits"][:, -1], atol=1e-5)
    got_loc = model(dict(input_ids=codes, poses=cams[:, :-1]))              # T-1 poses: LOC token in the last slot
    assert _stats(f"loc pose {precision}", got_loc["pose_prediction"][:, -1], o_loc["pose_prediction"][:, -1])[0] < max(tol, 1e-3) * 5
    gc = model.generate_codes(codes[:, :-1], cams)
    if precision == "fp32":
        assert torch.equal(gc.cpu(), o["logits"][:, -1].argmax(-1))


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-4), ("bf16", 6e-2)])
def test_migt_three_streams_small(precision, tol):
    """multi-context call (evaluate_transformer_multictx.py:61-73): output_poses + localization_tokens."""
    cfg = MIGTConfig(**SMALL_MIGT)
    sd, model = _migt(cfg, 4, precision)
    codes, cams, ids = _migt_inputs(cfg, 2, 4, seed=8)
    ctx_c = torch.cat([cams[:, :-1], torch.zeros_like(cams[:, :1])], 1)
    inp = dict(input_ids=ids, poses=ctx_c, output_poses=cams[:, -1:].repeat(1, 4, 1), localization_tokens=codes[:, -1:].repeat(1, 4, 1, 1))
    with torch.no_grad():
        o = mo.forward(sd, cfg, inp)
    got = model(inp)
    assert _stats(f"3-stream logits {precision}", got["logits"], o["logits"])[0] < tol
    assert _stats(f"3-stream pose {precision}", got["pose_prediction"], o["pose_prediction"])[0] < max(tol, 1e-3) * 5


@pytest.mark.parametrize("precision,tol,smoothing", [("fp32", 1e-4, 0.0), ("fp32", 1e-4, 0.1), ("bf16", 3e-2, 0.0)])
def test_migt_compute_losses_small(precision, tol, smoothing):
    """MIGT.call(compute_losses=True) (migt.py:364-373, 417-448): teacher-forced CE + pose regression losses."""
    import dataclasses
    cfg = dataclasses.replace(MIGTConfig(**SMALL_MIGT), n_loss_skip=2, label_smoothing=smoothing, image_generation_weight=0.7,
                              localization_weight="0.5")
    sd, model = _migt(cfg, 6, precision)
    codes, cams, _ = _migt_inputs(cfg, 3, 5, seed=12)
    with torch.no_grad():
        o = mo.forward(sd, cfg, dict(input_ids=codes, poses=cams), compute_losses=True, localization_weight=0.5)
        if smoothing > 0:       # restate the smoothed CE of migt.py:99-104 on the oracle logits
            lg = o["logits"].reshape(-1, cfg.n_embeddings)
            y = torch.nn.functional.one_hot(codes.reshape(-1), cfg.n_embeddings).float() * (1 - smoothing) + smoothing / cfg.n_embeddings
            ce = -(y * torch.log_softmax(lg, -1)).sum(-1).reshape(3, 5, 64)[:, cfg.n_loss_skip:].mean((1, 2))
            o["loss"] = o["loss"] - o["ce_loss"] * cfg.image_generation_weight + ce * cfg.image_generation_weight
            o["ce_loss"] = ce
    got = model(dict(input_ids=codes, poses=cams), compute_losses=True)
    for k in ("ce_loss", "pose_pos_loss", "pose_ori_loss", "pose_loss", "loss"):
        assert list(got[k].shape) == [3]
        rel = ((got[k].cpu() - o[k]).abs() / o[k].abs().clamp_min(1e-6)).max().item()
        print(f"[losses {precision}] {k}: got {got[k].cpu().tolist()} want {o[k].tolist()} rel {rel:.2e}")
        assert rel < tol, k
    assert got["localization_weight"] == 0.5
    assert _stats(f"losses logits {precision}", got["logits"], o["logits"])[0] < max(tol, 2e-4) * 2
    with pytest.raises(NotImplementedError):
        model(dict(input_ids=codes, poses=cams), training=True)


def test_migt_full_size_vs_oracle_golden(golden_dir):
    """Full-size MIGT (12 layers, d=768), B=1,T=10: golden from the restatement, reproduced by the reference's own MIGT.call over
    oracle/tf_shim.py (tests/test_reference_on_shim.py)."""
    g = np.load(os.path.join(golden_dir, "migt_full.npz"))
    cfg = MIGTConfig()
    B, T = int(g["B"]), int(g["T"])
    codes, cams, ids = _migt_inputs(cfg, B, T, seed=5)
    want = torch.from_numpy(g["logits_last"])
    for precision, tol, agree_min in (("fp32", 5e-4, 1.0), ("bf16", 5e-2, 0.93)):
        sd, model = _migt(cfg, 3, precision)
        last = model(dict(input_ids=ids, poses=cams), last_only=True)["logits"][:, 0]
        mx, mean = _stats(f"full logits {precision}", last[:1], want)
        agree = float((last.argmax(-1).cpu().numpy() == g["argmax_last"]).mean())
        print(f"[full migt {precision}] argmax agreement {agree:.3f}")
        assert mx < tol and agree >= agree_min
        del model
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------- generate()
def test_generate_end_to_end_matches_oracle():
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions
    vcfg = VQGANConfig(ch=64, ch_mult=[1, 2, 2, 2], attn_resolutions=[8], image_size=32, embed_dim=64, z_channels=64,
                       n_embed=256, num_res_blocks=1)                       # stride 8 -> 4x4 tokens per view
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=4)
    vsd, tsd = synth.make_vqgan_state_dict(vcfg, 11), synth.make_migt_state_dict(tcfg, 12)
    images = synth.make_images_uint8(2, 3, size=32, seed=13)
    cams = synth.make_cameras(2, 3, seed=14)
    with torch.no_grad():
        want = mo.generate_batch_predictions(lambda d: mo.forward(tsd, tcfg, d), lambda x: vo.encode(vsd, vcfg, x)[2],
                                             lambda c: vo.decode_code(vsd, vcfg, c), tcfg, images, cams)
    cb = VQGAN(vcfg, precision="fp32").load_state_dict(vsd)
    tr = MIGT(tcfg, precision="fp32").load_state_dict(tsd)
    got = generate_batch_predictions(tr, cb, images, cams)
    assert torch.equal(got["generated_codes"].cpu(), want["generated_codes"])
    diff = (got["generated_images"].cpu().int() - want["generated_images"].int()).abs()
    print(f"[generate] u8 pixel diffs: max {int(diff.max())}, nonzero {int((diff > 0).sum())}/{diff.numel()}")
    assert int(diff.max()) <= 1
    assert torch.allclose(got["generated_cameras"].cpu(), want["generated_cameras"], atol=1e-3)
    assert torch.equal(got["ground_truth_images"], images[:, -1])
    # fast path (bf16) runs and produces images of the right shape/dtype
    cb16, tr16 = VQGAN(vcfg, precision="bf16").load_state_dict(vsd), MIGT(tcfg, precision="bf16").load_state_dict(tsd)
    g16 = generate_batch_predictions(tr16, cb16, images, cams)
    assert g16["generated_images"].dtype == torch.uint8 and list(g16["generated_images"].shape) == [2, 32, 32, 3]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_graphed_predictions_equal_eager(precision):
    """CUDA-graph replay of generate() == the eager call, bit for bit, for successive different inputs (host and device)."""
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions, GraphedPredictions
    vcfg = VQGANConfig(ch=64, ch_mult=[1, 2, 2, 2], attn_resolutions=[8], image_size=32, embed_dim=64, z_channels=64,
                       n_embed=256, num_res_blocks=1)                       # stride 8 -> 4x4 tokens per view
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=4,
                      localization_weight="0")
    vsd, tsd = synth.make_vqgan_state_dict(vcfg, 11), synth.make_migt_state_dict(tcfg, 12)
    cb = VQGAN(vcfg, precision=precision).load_state_dict(vsd)
    tr = MIGT(tcfg, precision=precision).load_state_dict(tsd)
    gp = GraphedPredictions(tr, cb, 2, 3)
    assert gp.launches_per_replay > 10
    for seed, on_dev in ((13, False), (17, True), (19, False)):
        images = synth.make_images_uint8(2, 3, size=32, seed=seed)
        cams = synth.make_cameras(2, 3, seed=seed + 1)
        want = generate_batch_predictions(tr, cb, images, cams)
        got = gp(images.cuda() if on_dev else images.pin_memory(), cams.cuda() if on_dev else cams.pin_memory())
        assert torch.equal(got["generated_codes"], want["generated_codes"])
        assert torch.equal(got["generated_images"], want["generated_images"])
        assert torch.allclose(got["generated_cameras"], want["generated_cameras"])
    with pytest.raises(NotImplementedError):
        GraphedPredictions(MIGT(MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=256, token_image_size=4),
                                precision=precision).load_state_dict(synth.make_migt_state_dict(
                                    MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=256, token_image_size=4), 12)),
                           cb, 2, 3)


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-4), ("bf16", 6e-2)])
def test_migt_kv_cache_query_equals_full_forward(precision, tol):
    """BASELINE config 5 path: prefill the context once, then query-only passes reproduce the full forward's last view."""
    cfg = MIGTConfig(**SMALL_MIGT)
    sd, model = _migt(cfg, 7, precision)
    B, T = 3, 4
    codes, cams, ids = _migt_inputs(cfg, B, T, seed=21)
    with torch.no_grad():
        want = mo.forward(sd, cfg, dict(input_ids=ids, poses=cams))["logits"][:, -1]
    cache = model.prefill_context(codes[:, :-1], cams[:, :-1].contiguous())
    got_codes, got_logits = model.query(cache, cams[:, -1].contiguous(), return_logits=True)
    assert _stats(f"kv-cache logits {precision}", got_logits, want)[0] < tol
    if precision == "fp32":
        assert torch.equal(got_codes.cpu(), want.argmax(-1))
    # one scene shared by many queries (stride-0 cache batch): scene 0's context, the three different query poses
    cache1 = model.prefill_context(codes[:1, :-1], cams[:1, :-1].contiguous())
    _, l_shared = model.query(cache1, cams[:, -1].contiguous(), return_logits=True)
    with torch.no_grad():
        for j in range(B):
            cj = torch.cat([cams[:1, :-1], cams[j:j + 1, -1:]], 1)
            wj = mo.forward(sd, cfg, dict(input_ids=ids[:1], poses=cj))["logits"][:, -1]
            assert _stats(f"shared-cache query {j} {precision}", l_shared[j:j + 1], wj)[0] < tol


def test_generate_multictx_matches_oracle():
    """evaluate_transformer_multictx.py:37-95 through the 3-stream branching attention path."""
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions_multictx
    vcfg = VQGANConfig(ch=64, ch_mult=[1, 2, 2, 2], attn_resolutions=[8], image_size=32, embed_dim=64, z_channels=64,
                       n_embed=256, num_res_blocks=1)
    tcfg = MIGTConfig(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_embeddings=vcfg.n_embed, token_image_size=4)
    vsd, tsd = synth.make_vqgan_state_dict(vcfg, 21), synth.make_migt_state_dict(tcfg, 22)
    images = synth.make_images_uint8(2, 3, size=32, seed=23)
    cams = synth.make_cameras(2, 3, seed=24)
    with torch.no_grad():
        want = mo.generate_batch_predictions_multictx(lambda d: mo.forward(tsd, tcfg, d), lambda x: vo.encode(vsd, vcfg, x)[2],
                                                      lambda c: vo.decode_code(vsd, vcfg, c), tcfg, images, cams)
    cb = VQGAN(vcfg, precision="fp32").load_state_dict(vsd)
    tr = MIGT(tcfg, precision="fp32").load_state_dict(tsd)
    got = generate_batch_predictions_multictx(tr, cb, images, cams)
    assert list(got["generated_images"].shape) == [2, 3, 32, 32, 3]
    diff = (got["generated_images"].cpu().int() - want["generated_images"].int()).abs()
    print(f"[generate multictx] u8 pixel diffs: max {int(diff.max())}, nonzero {int((diff > 0).sum())}/{diff.numel()}")
    assert int(diff.max()) <= 1
    assert torch.allclose(got["generated_cameras"].cpu(), want["generated_cameras"], atol=1e-3)


def test_load_model_from_checkpoint_dir(tmp_path):
    """registry.load_model: config.json + Lightning-style .ckpt ('state_dict') -> working model (utils/torch.py:9-17)."""
    import json
    from viewformer_b200 import load_model, VQGAN
    cfg = VQGANConfig(**SMALL_VQ)
    sd = synth.make_vqgan_state_dict(cfg, 2)
    (tmp_path / "config.json").write_text(json.dumps(cfg.asdict()))
    torch.save({"state_dict": dict(sd, **{"perceptual_loss.net.x": torch.zeros(1)})}, tmp_path / "last.ckpt")
    model = load_model(str(tmp_path), precision="fp32")
    assert isinstance(model, VQGAN)
    x = vq_images(2, cfg.image_size, 3)
    with torch.no_grad():
        co = vo.encode(sd, cfg, x)[2]
    assert torch.equal(model.encode(x)[2].cpu(), co)

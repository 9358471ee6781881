"""TEST INFRASTRUCTURE — regenerate the four-channel (RGBA) codebook fixtures tests/golden/vqgan_rgba_*.npz from the REAL reference
(container only), as oracle/make_golden.py does for the 3-channel ones: weights from oracle/synth.py, the RGBA frames stored in the files.

    python -m oracle.make_golden_rgba
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth, ref_loader, migt_oracle  # noqa: E402
from oracle.make_golden import OUT, SMALL_VQ  # noqa: E402
from viewformer_b200.config import VQGANConfig  # noqa: E402


RGBA_VQ = dict(SMALL_VQ, in_channels=4, out_ch=4)
# ch 128: conv_in 4 -> 128 and conv_out 128 -> 4 on the dedicated kernels, every 3x3 conv tensor-core sized (the mixed encoder's)
RGBA_TC_VQ = dict(ch=128, ch_mult=[1, 2], attn_resolutions=[16], image_size=32, embed_dim=64, z_channels=64, n_embed=256, num_res_blocks=1,
                  in_channels=4, out_ch=4)


def rgba_images(n, size, seed):
    """uint8 [n,H,W,4] frames shaped like CO3Dv2's (data/loaders/co3dv2.py:149-153): the RGB masked by a smooth blob mask, then the
    mask as the fourth channel."""
    rgb = synth.make_images_uint8(1, n, size=size, seed=seed)[0]
    g = torch.Generator().manual_seed(seed + 1)
    lo = torch.rand((n, 1, 4, 4), generator=g)
    soft = torch.nn.functional.interpolate(lo, size=(size, size), mode="bilinear", align_corners=False)[:, 0]
    mask = (soft > 0.45).to(torch.uint8) * 255
    return torch.cat([rgb * (mask[..., None] > 0), mask[..., None]], -1).contiguous()


def golden_vqgan_rgba():
    """The small codebook with 4 input and output channels (the co3dv2-all-codebook-th layout): encode codes, decode_code pixels and
    forward, from the reference module itself, on seeded RGBA frames (stored, uint8); the same under ``tc.`` for RGBA_TC_VQ."""
    out = {}
    for prefix, overrides in (("", RGBA_VQ), ("tc.", RGBA_TC_VQ)):
        cfg = VQGANConfig(**overrides)
        sd = synth.make_vqgan_state_dict(cfg, 0)
        ref = ref_loader.build_reference_vqgan(sd, **overrides)
        u8 = rgba_images(2, cfg.image_size, 1100)
        x = migt_oracle.images_to_float(u8).permute(0, 3, 1, 2).contiguous()
        with torch.no_grad():
            quant, diff, codes = ref.encode(x)
            dec = ref.decode_code(codes)
            rec, _, _, _ = ref(x)
        out.update({prefix + k: v for k, v in dict(images=u8.numpy(), codes=codes.numpy(), diff=diff.numpy(), dec=dec.numpy(),
                                                    rec=rec.numpy()).items()})
        print(f"rgba {prefix or 'small'} codes", codes.shape, "diff", float(diff), "dec std", float(dec.std()))
    np.savez_compressed(os.path.join(OUT, "vqgan_rgba_small.npz"), **out)


def golden_vqgan_rgba_train():
    """Two optimisation steps of that 4-channel reference codebook (QuantizeEMA, perceptual_weight = 0), as golden_vqgan_train records
    them; the RGBA frames of each step are stored."""
    overrides = dict(RGBA_VQ, perceptual_weight=0.0)
    cfg = VQGANConfig(**overrides)
    sd = synth.make_vqgan_state_dict(cfg, 5)
    ref = ref_loader.build_reference_vqgan(sd, **overrides)
    ref.train()
    opt = torch.optim.Adam(ref.parameters(), lr=cfg.learning_rate, betas=(0.5, 0.9))
    g = torch.Generator().manual_seed(99)
    names = [n for n, _ in ref.named_parameters()]
    probe = {n: torch.randn(p.shape, generator=g) for n, p in ref.named_parameters()}
    keep = ["encoder.conv_in.weight", "encoder.conv_in.bias", "quant_conv.weight", "decoder.conv_out.weight", "decoder.conv_out.bias",
            "decoder.norm_out.bias"]
    out = dict(names=np.array(names))
    for step in range(2):
        u8 = rgba_images(3, cfg.image_size, 2100 + step)
        x = migt_oracle.images_to_float(u8).permute(0, 3, 1, 2).contiguous()
        out[f"images{step}"] = u8.numpy()
        opt.zero_grad()
        xrec, qloss, _, codes = ref(x)
        loss, log = ref._compute_loss(qloss, x, xrec, split="train")
        loss.backward()
        out[f"loss{step}"] = loss.detach().numpy()
        out[f"rec{step}"] = log["train/rec_loss"].numpy()
        out[f"quant{step}"] = log["train/quant_loss"].numpy()
        out[f"codes{step}"] = codes.numpy()
        out[f"gnorm{step}"] = np.array([float(p.grad.norm()) for _, p in ref.named_parameters()])
        out[f"gdot{step}"] = np.array([float((p.grad * probe[n]).sum()) for n, p in ref.named_parameters()])
        for k in keep:
            out[f"g{step}.{k}"] = dict(ref.named_parameters())[k].grad.numpy().copy()
        opt.step()
        out[f"pdot{step}"] = np.array([float((p.detach() * probe[n]).sum()) for n, p in ref.named_parameters()])
        for k in keep:
            out[f"p{step}.{k}"] = dict(ref.named_parameters())[k].detach().numpy().copy()
        out[f"emb{step}"] = ref.quantize.embeddings.numpy().copy()
    np.savez_compressed(os.path.join(OUT, "vqgan_rgba_train_small.npz"), **out)
    print("rgba train golden: losses", float(out["loss0"]), float(out["loss1"]))



if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    golden_vqgan_rgba()
    golden_vqgan_rgba_train()

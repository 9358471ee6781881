"""The codebook model's encoder / decoder layout (vqgan.layout) and the two orders derived from it, on the CPU: the reference
state_dict order of ``VQGAN.param_shapes`` (which is also the order ``init_weights`` draws its random numbers in) and the codebook
trainer's parameter order (which fixes the flat-buffer layout, the bucket boundaries and the order of the clipping norm's sum)."""
import json
import os

import pytest
import torch

from oracle import synth
from oracle.make_golden import SMALL_VQ
from viewformer_b200 import _lib as L
from viewformer_b200.config import VQGANConfig
from viewformer_b200.train import VQGANTrainer
from viewformer_b200.vqgan import VQGAN, layout

CONFIGS = {
    "default": {},
    "small_vq": SMALL_VQ,
    "host_logic": dict(ch=32, ch_mult=[1, 2], image_size=16, attn_resolutions=[8], embed_dim=16, z_channels=16, n_embed=32),
    "four_levels": dict(ch=32, ch_mult=[1, 1, 2, 4], image_size=32, attn_resolutions=[8], embed_dim=16, z_channels=16, n_embed=32),
    "one_res_block": dict(SMALL_VQ, num_res_blocks=1),
    "three_res_blocks": dict(SMALL_VQ, num_res_blocks=3),
    "no_attention": dict(SMALL_VQ, attn_resolutions=[]),
    "attention_at_two_levels": dict(SMALL_VQ, attn_resolutions=[16, 8]),
}


@pytest.mark.parametrize("quantizer", ["ema", "commit"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_param_shapes_order_equals_the_oracle(name, quantizer):
    cfg = VQGANConfig(**CONFIGS[name])
    want = [(k, tuple(s)) for k, s in synth.vqgan_param_shapes(cfg).items()
            if quantizer == "ema" or k not in ("quantize.ema_cluster_size_hidden", "quantize.ema_dw_hidden", "quantize.counter")]
    got = [(k, tuple(s)) for k, s in VQGAN(cfg, quantizer=quantizer).param_shapes().items()]
    assert got == want


@pytest.mark.parametrize("name", list(CONFIGS))
def test_layout_chains_channels_and_names_each_stage_once(name):
    cfg = VQGANConfig(**CONFIGS[name])
    enc, dec = layout(cfg)
    for half, stages, cin, cout in (("encoder", enc, cfg.in_channels, cfg.z_channels), ("decoder", dec, cfg.z_channels, cfg.out_ch)):
        assert stages[0].kind == "conv_in" and stages[0].cin == cin and stages[-1].kind == "out" and stages[-1].cout == cout
        assert all(a.cout == b.cin for a, b in zip(stages, stages[1:]))
        assert all(st.name.startswith(half) for st in stages)
        assert [st.exact for st in stages] == [half == "encoder"] + [False] * (len(stages) - 2) + [half == "decoder"]
    assert len({st.name for st in enc + dec}) == len(enc) + len(dec)
    assert sum(st.kind == "down" for st in enc) == sum(st.kind == "up" for st in dec) == len(cfg.ch_mult) - 1
    assert all(st.stride == (2 if st.kind == "down" else 1) and st.upsample == (st.kind == "up") for st in enc + dec)


@pytest.mark.parametrize("quantizer", ["ema", "commit"])
@pytest.mark.parametrize("name", ["small_vq", "default"])
def test_trainer_parameter_order_is_pinned(name, quantizer, golden_dir, monkeypatch):
    """The trainer's registry (encoder, quant_conv, [quantize.embeddings], post_quant_conv, decoder) against its recorded order.  An fp32
    model lays its weights out with torch alone, so the device steps of loading (library load, codebook tables) are stubbed out."""
    monkeypatch.setattr(L, "load", lambda require_device=False: None)
    monkeypatch.setattr(VQGAN, "_refresh_codebook", lambda self: None)
    cfg = VQGANConfig(**CONFIGS[name])
    model = VQGAN(cfg, precision="fp32", device="cpu", quantizer=quantizer)
    sd = synth.make_vqgan_state_dict(cfg, 0)
    model.load_state_dict({k: v for k, v in sd.items() if k in model.param_shapes()})
    tr = VQGANTrainer.__new__(VQGANTrainer)
    tr.model, tr.cfg = model, model.config
    tr._collect_params()
    want = json.load(open(os.path.join(golden_dir, "vqgan_trainer_order.json")))[f"{name}/{quantizer}"]
    assert [p.name for p in tr.params] == want
    assert all(torch.equal(p.tensor, sd[p.name].reshape(p.tensor.shape)) for p in tr.params if p.kind == "vec" and not p.part)

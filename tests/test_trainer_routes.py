"""The kernel route of every trainable layer of both training steps, on the CPU, against its recorded table: forward, data gradient and
weight gradient of every codebook conv ("bf16" single-pass bf16 wgmma, "split" the exact split-fp16 tensor-core kernels, "cuda" the fp32
CUDA-core kernels), and the route of every transformer dense layer and of the tied LM head ("wte").  The routes are decided when a layer
is registered, from the step's precision, VF_TRAIN_TC and the layer's shape; the trainers' registries are built without the library."""
import json
import os

import pytest
import torch

from oracle import synth
from oracle.make_golden import SMALL_VQ, MIGT_TRAIN
from test_launch_audit_gpu import FULL_MIGT_TRAIN, MEDIUM_VQ
from viewformer_b200 import _lib as L
from viewformer_b200.config import MIGTConfig, VQGANConfig
from viewformer_b200.migt import MIGT
from viewformer_b200.train import VQGANTrainer
from viewformer_b200.train_migt import MIGTTrainer
from viewformer_b200.vqgan import VQGAN

VQ_CONFIGS = {"small": dict(SMALL_VQ, perceptual_weight=0.0), "medium": MEDIUM_VQ, "default": dict(perceptual_weight=0.0)}
MIGT_CONFIGS = {"MIGT_TRAIN": MIGT_TRAIN, "FULL_MIGT_TRAIN": FULL_MIGT_TRAIN}
SETTINGS = {"fp32": ("fp32", True), "fp32 VF_TRAIN_TC=0": ("fp32", False), "bf16": ("bf16", True)}


def vq_routes(name, quantizer):
    """{setting: {conv: [forward, data gradient, weight gradient]}} of the codebook trainer's registry.  An fp32 model lays its weights out
    with torch alone, so the device steps of loading (library load, codebook tables) are stubbed out."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(L, "load", lambda require_device=False: None)
        mp.setattr(VQGAN, "_refresh_codebook", lambda self: None)
        cfg = VQGANConfig(**VQ_CONFIGS[name])
        model = VQGAN(cfg, precision="fp32", device="cpu", quantizer=quantizer)
        model.load_state_dict({k: v for k, v in synth.make_vqgan_state_dict(cfg, 0).items() if k in model.param_shapes()})
    out = {}
    for setting, (precision, use_tc) in SETTINGS.items():
        tr = VQGANTrainer.__new__(VQGANTrainer)
        tr.model, tr.cfg, tr.precision, tr.use_tc = model, model.config, precision, use_tc
        tr._collect_params()
        tr._route_convs()
        out[setting] = {n: [c.fw, c.dgrad, c.wgrad] for n, c in tr.convs.items()}
    return out


def migt_routes(name):
    """{setting: {layer: route}} of the transformer trainer's dense-layer records, built over buffers on the meta device (no memory)."""
    cfg = MIGTConfig(**MIGT_CONFIGS[name])
    model = MIGT(cfg, precision="fp32", device="cpu")
    out = {}
    for setting, (precision, use_tc) in SETTINGS.items():
        if precision == "bf16" and cfg.d_model // cfg.n_head != 64:
            with pytest.raises(NotImplementedError):                 # the fused attention kernels need head dimension 64
                MIGTTrainer(model, precision="bf16")
            continue
        tr = MIGTTrainer.__new__(MIGTTrainer)
        tr.model, tr.cfg, tr.device, tr.bucket_bytes, tr.group = model, cfg, torch.device("meta"), 64 << 20, None
        tr.precision, tr.use_tc = precision, use_tc or precision == "bf16"
        tr._build({k: torch.empty(s, device="meta") for k, s in model.param_shapes().items()})
        tr._build_dense()
        out[setting] = {n: r.route for n, r in tr.dense.items()}
    return out


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "trainer_routes.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("quantizer", ["ema", "commit"])
@pytest.mark.parametrize("name", list(VQ_CONFIGS))
def test_codebook_conv_routes_are_pinned(name, quantizer, golden):
    assert vq_routes(name, quantizer) == golden["codebook"][f"{name}/{quantizer}"]


@pytest.mark.parametrize("name", list(MIGT_CONFIGS))
def test_transformer_dense_routes_are_pinned(name, golden):
    assert migt_routes(name) == golden["transformer"][name]

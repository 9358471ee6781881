"""Host-side logic that needs no GPU: config parsing, registry, strict state-dict checks, camera maths."""
import json
import os

import pytest
import torch

from oracle import synth, migt_oracle as mo
from viewformer_b200 import config as C
from viewformer_b200 import generate as G


def test_config_defaults_match_reference():
    v, m = C.VQGANConfig(), C.MIGTConfig()
    assert (v.model, v.stride, v.n_embed, v.embed_dim, v.ch_mult, v.attn_resolutions) == ("vqgan", 16, 1024, 256, [1, 1, 2, 2, 4], [16])
    assert (m.model, m.n_layer, m.n_head, m.d_model, m.sequence_size, m.n_loss_skip) == ("migt", 12, 12, 768, 20, 4)
    assert m.use_localization and m.model_type == "transformer" and v.model_type == "codebook"


def test_load_config_roundtrip(tmp_path):
    d = C.MIGTConfig(n_layer=3, localization_weight="0").asdict()
    p = tmp_path / "config.json"
    p.write_text(json.dumps(d))
    cfg = C.load_config(str(p))
    assert isinstance(cfg, C.MIGTConfig) and cfg.n_layer == 3 and not cfg.use_localization
    with pytest.raises(C.ModelNotFoundError):
        C.load_config({"model": "nope"})


def test_strict_state_dict_errors_before_touching_the_device():
    from viewformer_b200 import VQGAN, MIGT
    m = VQGAN(ch=32, ch_mult=[1, 2], image_size=16, attn_resolutions=[8], embed_dim=16, z_channels=16, n_embed=32)
    sd = synth.make_vqgan_state_dict(m.config, 0)
    bad = dict(sd); bad.pop("quant_conv.bias")
    with pytest.raises(RuntimeError, match="Missing keys"):
        m.load_state_dict(bad)
    bad = dict(sd); bad["foo.bar"] = torch.zeros(1)
    with pytest.raises(RuntimeError, match="Unexpected keys"):
        m.load_state_dict(bad)
    ok = dict(sd); ok["perceptual_loss.net.weight"] = torch.zeros(1)   # ignored like the reference (vqgan_th.py:322)
    assert set(k for k in ok if not k.startswith("perceptual_loss")) == set(m.expected_keys())
    t = MIGT(n_layer=1, d_model=64, n_head=2)
    with pytest.raises(RuntimeError, match="Missing keys"):
        t.load_state_dict({})


def test_registry_picks_b200_classes():
    from viewformer_b200 import AutoModel, AutoModelTH, VQGAN, MIGT
    assert isinstance(AutoModelTH.from_config({"model": "vqgan"}), VQGAN)
    assert isinstance(AutoModel.from_config({"model": "migt", "n_layer": 2}), MIGT)


def test_camera_helpers_equal_oracle():
    cams = synth.make_cameras(4, 6, seed=9)
    r1, t1 = G.to_relative_cameras(cams)
    r2, t2 = mo.to_relative_cameras(cams)
    assert torch.allclose(r1, r2, atol=1e-6) and torch.equal(t1, t2)
    assert torch.allclose(G.normalize_cameras(r1), mo.normalize_cameras(r2), atol=1e-7)
    assert torch.allclose(G.from_relative_cameras(r1, t1), mo.from_relative_cameras(r2, t2), atol=1e-6)
    x = torch.randn(2, 3, 64, 7)
    assert torch.allclose(G.reduce_cameras(x, -2), mo.reduce_cameras(x, -2), atol=1e-6)


def test_schedule_strings():
    """viewformer_b200/schedules.py: the string forms of utils/schedules.py:72-247 (linear / cosine / warmup / constant)."""
    import math
    from viewformer_b200.schedules import parse
    assert parse("0.5")(123) == 0.5 and parse(2)(0) == 2.0 and parse("0").is_zero() and not parse("1").is_zero()
    lin = parse("linear(1,3,10)")
    assert lin(0) == 1.0 and lin(5) == 2.0 and lin(10) == 3.0 and lin(50) == 3.0
    cos = parse("cosine(2,0)").with_total_steps(8)
    assert abs(cos(0) - 2.0) < 1e-12 and abs(cos(4) - 1.0) < 1e-12 and abs(cos(8)) < 1e-12 and abs(cos(80)) < 1e-12
    assert abs(cos(2) - (0 + (2 - 0) * 0.5 * (math.cos(math.pi * 0.25) + 1))) < 1e-12
    wu = parse("warmup(cosine(1,0.5,100),4)")
    assert wu(0) == 0.0 and abs(wu(2) - 0.5 * 1.0) < 1e-12 and abs(wu(4) - 1.0) < 1e-12
    assert abs(wu(54) - (0.5 + 0.5 * 0.5 * (math.cos(math.pi * 0.5) + 1))) < 1e-12
    assert str(parse("warmup(1,2000)")) == "warmup(1.0,2000)" and not parse("warmup(1,2000)").is_zero()
    assert parse("linear(0,0,5)").is_zero() and parse("warmup(0,7)").is_zero()
    with pytest.raises(ValueError):
        parse("cosine(1,0)")(3)                      # no horizon yet
    with pytest.raises(ValueError):
        parse("step(1,2)")
    from viewformer_b200.config import MIGTConfig
    assert MIGTConfig(localization_weight="0").use_localization is False
    assert MIGTConfig(localization_weight="warmup(1,2000)").use_localization is True


def test_bench_roofline_traffic_is_algorithmic():
    """bench.py's `roofline.traffic` is the DRAM traffic the conv needs at least, computed from its shapes (not a literal)."""
    import importlib.util, os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("vf_bench", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    conv, src = bench.algorithmic_traffic(288, True)
    assert 4.5e9 < conv < 5.2e9 and "algorithmic" in src                        # 288 x 16384 x 128 x 8 B = 4.83 GB
    bf16, _ = bench.algorithmic_traffic(288, False)
    assert 3.3e9 < bf16 < 3.9e9                                                  # 288 x 16384 x 128 x 6 B = 3.62 GB


def test_camera_metrics_match_the_reference_evaluator_fixture(golden_dir):
    """The host-side half of viewformer_b200.metrics.Evaluator (camera errors, running means, medians) against numbers produced by the
    reference's own Evaluator (evaluate_transformer.py:22-67, utils/metrics.py:91-170) over oracle/tf_shim.py
    (tests/golden/evaluator_reference_shim.npz, oracle/make_golden.py).  The image half runs on the GPU (tests/test_vs_reference_evaluator_gpu.py)."""
    import numpy as np
    from oracle import make_golden as G
    from viewformer_b200.metrics import Evaluator
    g = np.load(os.path.join(golden_dir, "evaluator_reference_shim.npz"))
    gt, gen = G.evaluator_cameras()
    ev = Evaluator()                                    # no device is touched until an image arrives
    ev.update_with_camera(gt[:4], gen[:4])              # two updates: the running state must accumulate
    ev.update_with_camera(gt[4:], gen[4:])
    r = ev.result()
    for k in ("loc-angle", "loc-dist", "loc-angle-med", "loc-dist-med"):
        assert abs(r[k] - float(g["cam." + k])) < 2e-6 * max(1.0, abs(r[k])), k
    info = ev.get_progress_bar_info()
    assert set(info) == {"img_psnr", "cam_loc", "cam_ang"} and abs(info["cam_loc"] - r["loc-dist"]) < 1e-12


def test_bench_json_contract_of_both_arms():
    """The keys of the JSON line: (a) a committed line of the CUDA arm (tests/golden/bench_line_h100.json, produced on an H100 by this
    bench.py), (b) the reference arm run live on the host cores with a tiny wall budget (`bench.py --impl reference`: the CPU oracle, bounded)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    line = json.load(open(os.path.join(root, "tests", "golden", "bench_line_h100.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
              "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline", "parity"):
        assert k in line, k
    assert line["higher_is_better"] is True and line["scaling"] == "weak" and line["vs_baseline"] is None and line["data"] == "synthetic"
    assert "workload" in line["config"] and not any(k in line["config"] for k in ("model", "global_batch", "seq_len"))
    assert set(line["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and line["e2e"]["h2d_bytes_per_step"] > 0
    assert set(line["roofline"]) >= {"bound", "achieved", "peak", "unit", "frac", "traffic"} and line["roofline"]["bound"] in ("hbm", "tensor")
    assert set(line["cpu_baseline"]) >= {"value", "unit", "cores", "kind", "sample"} and line["cpu_baseline"]["kind"] in ("port", "reference")
    assert set(line["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"} and line["gpu_launches"] > 0 and line["parity"]["code_mismatches"] == 0
    assert abs(line["value"] - line["config"]["scenes_per_gpu"] * line["n_gpus"] / (line["ms_per_step"] / 1e3)) < 1e-6 * line["value"]
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--cpu-budget-s", "5"],
                       capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    ref = json.loads(r.stdout.strip().splitlines()[-1])
    assert ref["impl"] == "reference" and ref["metric"] == line["metric"] and ref["unit"] == line["unit"] and ref["higher_is_better"] is True
    assert ref["config"]["workload"] == __import__("importlib").import_module("bench").WORKLOAD
    assert ref["e2e"] == {"value": ref["value"], "unit": ref["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert ref["cpu_baseline"]["value"] == ref["value"] and ref["cpu_baseline"]["kind"] == "port" and ref["cpu_baseline"]["cores"] >= 1
    assert ref["steps"] == 1 and ref["value"] > 0

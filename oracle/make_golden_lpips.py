"""TEST INFRASTRUCTURE — writes tests/golden/lpips_reference_shim.npz: the ``lpips`` the reference's own evaluators report.

The reference's Evaluator (evaluate/evaluate_transformer.py:22-67) and codebook Evaluator (evaluate/evaluate_codebook.py:18-49) run
unmodified over oracle/tf_shim.py on make_golden.EVALUATOR_CASES.  Only ``viewformer.models.utils.load_lpips_model`` (the ONNX export of
lpips.LPIPS, models/utils.py:267-294) is replaced, by the fp64 oracle/lpips_oracle.py over seeded random weights
(lpips_oracle.lpips_state_dicts(SEED)); LPIPSMetric.update_state (utils/metrics.py:210-214) and the ``lpips`` call (models/utils.py:297-307)
run as shipped: convert_image_dtype to [0, 1], NHWC -> NCHW, the model, reshape, the running mean.

Stored per case: ``{tag}.lpips`` (Evaluator.result()['lpips']), ``{tag}.codebook_lpips`` (the codebook Evaluator's), ``{tag}.per_image``
(the model's per-pair values), ``{tag}.input_sums``; and ``weight_sums`` of the seeded weights.

    python -m oracle.make_golden_lpips          (needs the reference sources)
"""
import os
import sys

import numpy as np
import torch

from oracle import lpips_oracle as lo, ref_loader, synth

SEED = 5
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


class OracleLPIPSModel:
    """What ``load_lpips_model`` returns (a saved ONNX graph called as ``model(**{'0': image_0, '1': image_1})``): here the fp64 oracle.
    Keeps the per-pair values of its last call and the range of every input it was given."""

    def __init__(self, vgg, lin):
        self.vgg, self.lin, self.last, self.input_range = vgg, lin, None, (float("inf"), -float("inf"))

    def __call__(self, **inputs):
        a = torch.as_tensor(inputs["0"]).as_subclass(torch.Tensor)
        b = torch.as_tensor(inputs["1"]).as_subclass(torch.Tensor)
        lo_, hi_ = self.input_range
        self.input_range = (min(lo_, float(a.min()), float(b.min())), max(hi_, float(a.max()), float(b.max())))
        self.last = lo.forward(a, b, self.vgg, self.lin)
        return self.last.reshape(-1, 1, 1, 1)


def reference_lpips_evaluators():
    """(transformer Evaluator class, codebook Evaluator class, the oracle model) of the reference, with LPIPSMetric bound to the oracle."""
    ev, _ = ref_loader.load_reference_evaluate()                      # installs oracle/tf_shim.py as `tensorflow`
    path = os.path.join(ref_loader.REFERENCE_ROOT, "viewformer", "evaluate", "evaluate_codebook.py")
    ec = sys.modules.get("viewformer.evaluate.evaluate_codebook") or ref_loader._load("viewformer.evaluate.evaluate_codebook", path)
    model = OracleLPIPSModel(*lo.lpips_state_dicts(SEED))
    sys.modules["viewformer.models.utils"].load_lpips_model = lambda net="alex", version="0.1", overwrite=False: model
    metrics = sys.modules["viewformer.utils.metrics"]
    metrics.LPIPSMetric._lpips_pool.pop("vgg", None)                  # built anew by the next LPIPSMetric through models/utils.lpips
    return ev.Evaluator, ec.Evaluator, model


def compute():
    from oracle import make_golden as G
    Ev, Ec, model = reference_lpips_evaluators()
    import tensorflow as tf
    out = {}
    for tag, n, gs, ns, image_size, seed in G.EVALUATOR_CASES:
        gt, gen = synth.make_metric_pair(n, gs, ns, seed)
        E = Ev(image_size)
        E.update_with_image(tf.convert_to_tensor(gt.numpy()), tf.convert_to_tensor(gen.numpy()))
        r = E.result()
        assert [k for k in r if k in ("mse", "rmse", "mae", "psnr", "lpips", "ssim")] == ["mse", "rmse", "mae", "psnr", "lpips", "ssim"]
        out[f"{tag}.lpips"] = np.float64(r["lpips"])
        out[f"{tag}.per_image"] = model.last.numpy().astype(np.float64)
        E = Ec(image_size)
        E.update_state(tf.convert_to_tensor(gt.numpy()), tf.convert_to_tensor(gen.numpy()))
        out[f"{tag}.codebook_lpips"] = np.float64(E.result()["lpips"])
        out[f"{tag}.input_sums"] = np.asarray([int(gt.sum()), int(gen.sum())], np.int64)
    out["weight_sums"] = np.asarray(lo.weight_sums(model.vgg, model.lin), np.float64)
    return out


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    out = compute()
    np.savez_compressed(os.path.join(OUT, "lpips_reference_shim.npz"), **out)
    print("lpips golden:", {k: float(v) for k, v in out.items() if k.endswith("lpips")})

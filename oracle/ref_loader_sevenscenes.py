"""TEST INFRASTRUCTURE — the reference's 7-Scenes evaluation callers on oracle/tf_shim.py (container only), on top of oracle/ref_loader.py's
recipe for the other evaluation scripts: evaluate/evaluate_sevenscenes.py and evaluate_sevenscenes_baseline.py are executed UNMODIFIED
from the reference's tree; nothing is copied.
"""
import os
import sys
import types

import torch

from oracle import ref_loader
from oracle.ref_loader import REFERENCE_ROOT, _load

_cache = {}


def load_reference_sevenscenes():
    """(evaluate_sevenscenes module, evaluate_sevenscenes_baseline module): generate_other_viewpoints, compute_camera_distances,
    generate_batch_predictions_using_{generated_images,pose_refinement}; generate_batch_predictions_baseline, Evaluator.  The raw-dataset
    loader they import (SevenScenesLoader, ALL_SCENES) is stubbed: it is not on the path and these functions do not call it.  The three
    TensorFlow ops they use beyond the shim's set are given here: tf.argsort (stable, as torch.argsort(stable=True)), tf.argmin (first
    minimum) and tf.math.l2_normalize (tf.linalg's)."""
    if "sevenscenes" in _cache:
        return _cache["sevenscenes"]
    ref_loader.load_reference_evaluate()
    tf = sys.modules["tensorflow"]
    if not hasattr(tf, "argsort"):
        tf.argsort = lambda values, axis=-1, direction="ASCENDING", stable=False, name=None: torch.argsort(
            values, dim=axis, descending=direction != "ASCENDING", stable=True).to(torch.int32)
    if not hasattr(tf, "argmin"):
        tf.argmin = lambda x, axis=None, output_type=torch.int64, name=None: torch.argmin(x, dim=axis)
    if not hasattr(tf.math, "l2_normalize"):
        tf.math.l2_normalize = tf.linalg.l2_normalize
    R = os.path.join(REFERENCE_ROOT, "viewformer")
    loaders = sys.modules["viewformer.data.loaders"]
    if not hasattr(loaders, "SevenScenesLoader"):
        def _no_loader(*a, **k):
            raise RuntimeError("SevenScenesLoader (raw 7-Scenes parsing) is not available; build a SceneLookup from arrays")
        loaders.SevenScenesLoader = _no_loader
    ss = types.ModuleType("viewformer.data.loaders.sevenscenes")
    ss.ALL_SCENES = ["chess", "fire", "heads", "office", "pumpkin", "redkitchen", "stairs"]
    sys.modules["viewformer.data.loaders.sevenscenes"] = ss
    _load("viewformer.utils.geometry", os.path.join(R, "utils", "geometry.py"))
    sys.modules["viewformer.utils"].geometry = sys.modules["viewformer.utils.geometry"]
    s7 = _load("viewformer.evaluate.evaluate_sevenscenes", os.path.join(R, "evaluate", "evaluate_sevenscenes.py"))
    bl = _load("viewformer.evaluate.evaluate_sevenscenes_baseline", os.path.join(R, "evaluate", "evaluate_sevenscenes_baseline.py"))
    _cache["sevenscenes"] = (s7, bl)
    return _cache["sevenscenes"]

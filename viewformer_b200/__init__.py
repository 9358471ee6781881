"""viewformer_b200 — H100-native (sm_90a) implementation of ViewFormer's novel-view-synthesis hot path:
VQGAN codebook encode/decode + MIGT context-view transformer, behind the reference's model surface."""
from .config import VQGANConfig, MIGTConfig, load_config, ModelNotFoundError  # noqa: F401


def __getattr__(name):   # lazy: importing the package must not require the built library
    if name in ("VQGAN",):
        from .vqgan import VQGAN
        return VQGAN
    if name in ("MIGT",):
        from .migt import MIGT
        return MIGT
    if name in ("AutoModel", "AutoModelTH", "load_model"):
        from . import registry
        return getattr(registry, name)
    if name in ("generate_batch_predictions", "generate_batch_predictions_multictx", "GraphedPredictions"):
        from . import generate
        return getattr(generate, name)
    if name in ("generate_other_viewpoints", "compute_camera_distances", "SceneLookup", "generate_batch_predictions_using_generated_images",
                "generate_batch_predictions_using_pose_refinement", "generate_batch_predictions_baseline", "BaselineEvaluator"):
        from . import sevenscenes
        return getattr(sevenscenes, name)
    if name in ("transformer_predict", "run_with_batchsize", "encode_images", "decode_code", "generate_codebook_predictions"):
        from . import evaluate
        return getattr(evaluate, name)
    if name in ("Evaluator", "CodebookEvaluator", "MultiContextEvaluator", "image_metrics"):
        from . import metrics
        return getattr(metrics, name)
    if name in ("VQGANTrainer",):
        from .train import VQGANTrainer
        return VQGANTrainer
    if name in ("MIGTTrainer",):
        from .train_migt import MIGTTrainer
        return MIGTTrainer
    if name in ("LatentCodeTransformer", "write_token_dataset", "load_token_dataset", "read_tfrecords", "TFRecordWriter", "process_batch"):
        from . import data
        return getattr(data, name)
    if name in ("compat", "schedules", "tf_checkpoint", "cabi", "metrics", "data", "evaluate", "generate", "registry", "train", "train_migt",
                "sevenscenes"):
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)

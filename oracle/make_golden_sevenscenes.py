"""TEST INFRASTRUCTURE — regenerate tests/golden/sevenscenes_reference_shim.npz from the REAL reference (container only): the 7-Scenes
procedures of evaluate/evaluate_sevenscenes.py and evaluate_sevenscenes_baseline.py executed unmodified over oracle/tf_shim.py, with the
reference's torch codebook and its MIGT (weights from oracle/synth.py), on a synthetic scene database.

    python -m oracle.make_golden_sevenscenes

Everything the procedures read is regenerated from the seeds stored here (scene(), query_batch()); the file records what they drew and
picked (the raw uniform draws, the sampled file names, the selected database indices, the gap after the k-th nearest camera) and what
they returned, with the top-2 logit margin of every generated code.
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth, ref_loader, ref_loader_sevenscenes  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402
from viewformer_b200.config import VQGANConfig, MIGTConfig  # noqa: E402

# ch 128: the mixed codebook's tensor-core convs need 64-channel multiples; 32 x 32 frames, 8 x 8 tokens
SEVENSCENES_VQ = dict(ch=128, ch_mult=[1, 2, 2], attn_resolutions=[8], image_size=32, embed_dim=64, z_channels=64, n_embed=256,
                      num_res_blocks=1)
SEVENSCENES_MIGT = dict(n_layer=2, n_head=4, d_model=128, sequence_size=20, n_embeddings=256, token_image_size=8, n_loss_skip=1,
                        localization_weight="1")
VQ_SEED, MIGT_SEED = 0, 21
DB_FRAMES = 300
QUERY_SEED = 7300
NUM_GEN_CTX = {"pose_refinement": 9, "generated_images": 5}
# the nearest-camera selection must not turn on a near tie: the sorted distances of the first k + 1 database cameras stay this far
# apart, far above what a camera error of 1e-3 per component (the bar the GPU tests hold the first-stage camera to) can move them
SELECTION_GAP = 2e-2
MARGIN_BAR = 1e-3                       # top-2 logit margin above which an fp32 transformer must pick the reference's code


def scene(seed):
    """files, cameras f32 [N,7], frames uint8 [N,32,32,3] of a synthetic scene database (the training split of one 7-Scenes scene)."""
    files = [f"seq-{1 + i // 100:02d}/frame-{i % 100:06d}.color.png" for i in range(DB_FRAMES)]
    cams = synth.make_cameras(1, DB_FRAMES, seed=seed)[0].numpy()
    frames = synth.make_images_uint8(1, DB_FRAMES, size=32, seed=seed + 1)[0].numpy()
    return files, cams, frames


def query_batch(seed, B=1, T=20):
    """images uint8 [B,T,32,32,3] and cameras f32 [B,T,7]: 19 context frames and the query."""
    return synth.make_images_uint8(B, T, size=32, seed=seed), synth.make_cameras(B, T, seed=seed + 1)


class RecordingLookup:
    """The reference's SceneLookup duck type over arrays, recording every name it is asked for."""

    def __init__(self, files, cams, frames):
        self.files, self.cameras, self.frames = files, cams, frames
        self._lookup = {x: i for i, x in enumerate(files)}
        self.asked = []

    def __getitem__(self, name):
        self.asked.append(name)
        i = self._lookup[name]
        return self.cameras[i], self.frames[i]


def models():
    vcfg, tcfg = VQGANConfig(**SEVENSCENES_VQ), MIGTConfig(**SEVENSCENES_MIGT)
    vq = ref_loader.build_reference_vqgan(synth.make_vqgan_state_dict(vcfg, VQ_SEED), **SEVENSCENES_VQ)
    model = ref_loader.build_reference_migt(synth.make_migt_state_dict(tcfg, MIGT_SEED), **SEVENSCENES_MIGT)
    return model, ref_loader.ReferenceCodebookNHWC(vq)


def _recorder(model):
    """Wrap model.call: keep (codes, top-2 margin) of the last view of every generation forward (mask token in the last view)."""
    gens, orig = [], model.call

    def call(inputs, *a, **k):
        out = orig(inputs, *a, **k)
        ids = torch.as_tensor(inputs["input_ids"])
        if bool((ids[:, -1] == model.mask_token).all()):
            top = torch.topk(torch.as_tensor(out["logits"]).as_subclass(torch.Tensor)[:, -1].float(), 2, dim=-1).values
            gens.append((torch.as_tensor(out["logits"]).as_subclass(torch.Tensor)[:, -1].argmax(-1), top[..., 0] - top[..., 1]))
        return out
    model.call = call
    return gens


def _sorted_gaps(d, k):
    s = torch.sort(torch.as_tensor(d).as_subclass(torch.Tensor).double()).values
    return (s[1:k + 1] - s[:k]).numpy()


def golden_sevenscenes():
    s7, bl = ref_loader_sevenscenes.load_reference_sevenscenes()
    model, codebook = models()
    gens = _recorder(model)
    out = {}
    images, cams = query_batch(QUERY_SEED)
    out["query_seed"] = np.int64(QUERY_SEED)

    # ---- pose refinement: find a database seed whose nearest cameras to the first-stage estimate are well separated
    seen = {}
    orig_dist = s7.compute_camera_distances

    def rec_dist(db, camera):
        seen["camera"] = torch.as_tensor(camera).as_subclass(torch.Tensor).clone()
        return orig_dist(db, camera)
    s7.compute_camera_distances = rec_dist
    k = NUM_GEN_CTX["pose_refinement"]
    db_seed = 7400
    files, dbc, frames = scene(db_seed)
    with torch.no_grad():
        for _ in range(200):
            files, dbc, frames = scene(db_seed)
            d = orig_dist(torch.as_tensor(dbc), seen["camera"]) if "camera" in seen else None
            if d is not None and _sorted_gaps(d, k).min() > SELECTION_GAP:
                break
            if d is None:                                           # first pass: one run to get the estimate
                random.seed(1)
                s7.generate_batch_predictions_using_pose_refinement(RecordingLookup(files, dbc, frames), torch.as_tensor(dbc), model,
                                                                    codebook, images.clone(), cams.clone(), num_gen_ctx=k)
                continue
            db_seed += 2
        else:
            raise RuntimeError("no database seed separates the nearest cameras")
        lookup = RecordingLookup(files, dbc, frames)
        gens.clear()
        rng_seed = 7500
        random.seed(rng_seed)
        r = s7.generate_batch_predictions_using_pose_refinement(lookup, torch.as_tensor(dbc), model, codebook, images.clone(),
                                                                cams.clone(), num_gen_ctx=k)
    d = orig_dist(torch.as_tensor(dbc), seen["camera"])
    order = torch.argsort(torch.as_tensor(d).as_subclass(torch.Tensor), stable=True)
    gaps = _sorted_gaps(d, k)
    out.update({"pr.db_seed": np.int64(db_seed), "pr.rng_seed": np.int64(rng_seed), "pr.num_gen_ctx": np.int64(k),
                "pr.estimate": seen["camera"].numpy(), "pr.distances": torch.as_tensor(d).as_subclass(torch.Tensor).numpy(),
                "pr.selected": order[:k].numpy().astype(np.int64), "pr.gaps": gaps, "pr.files": np.array(lookup.asked),
                "pr.generated_images": torch.as_tensor(r["generated_images"]).as_subclass(torch.Tensor).numpy(),
                "pr.generated_cameras": torch.as_tensor(r["generated_cameras"]).as_subclass(torch.Tensor).float().numpy(),
                "pr.ground_truth_cameras": torch.as_tensor(r["ground_truth_cameras"]).as_subclass(torch.Tensor).float().numpy(),
                "pr.codes": gens[-1][0].numpy(), "pr.margins": gens[-1][1].numpy()})
    print(f"pose refinement: database seed {db_seed}, selected {order[:k].tolist()}, min gap {gaps.min():.4f}, "
          f"min code margin {float(gens[-1][1].min()):.2e}")

    # ---- generated images: the draws of generate_other_viewpoints under torch.manual_seed, stage-2 margins above the bar
    n = NUM_GEN_CTX["generated_images"]
    draws = []
    tf = sys.modules["tensorflow"]
    orig_uniform = tf.random.uniform

    def rec_uniform(*a, **kw):
        u = orig_uniform(*a, **kw)
        draws.append(torch.as_tensor(u).as_subclass(torch.Tensor).clone())
        return u
    tf.random.uniform = rec_uniform
    seed = 7600
    with torch.no_grad():
        for _ in range(100):
            gens.clear()
            draws.clear()
            torch.manual_seed(seed)
            r = s7.generate_batch_predictions_using_generated_images(model, codebook, images.clone(), cams.clone(), num_gen_ctx=n)
            if float(gens[0][1].min()) > MARGIN_BAR:
                break
            seed += 1
        else:
            raise RuntimeError("no draw seed keeps the generated context views' codes off near ties")
    tf.random.uniform = orig_uniform
    s7.compute_camera_distances = orig_dist
    out.update({"gi.seed": np.int64(seed), "gi.num_gen_ctx": np.int64(n)})
    out.update({f"gi.draw{i}": u.numpy() for i, u in enumerate(draws)})
    out.update({"gi.generated_images": torch.as_tensor(r["generated_images"]).as_subclass(torch.Tensor).numpy(),
                "gi.generated_cameras": torch.as_tensor(r["generated_cameras"]).as_subclass(torch.Tensor).float().numpy(),
                "gi.context_codes": gens[0][0].numpy(), "gi.context_margins": gens[0][1].numpy(),
                "gi.codes": gens[1][0].numpy(), "gi.margins": gens[1][1].numpy()})
    print(f"generated images: draw seed {seed}, context-code min margin {float(gens[0][1].min()):.2e}")

    # ---- baselines: four rows, each through the reference's one-row function
    bc = synth.make_cameras(4, 20, seed=7700)
    out["bl.cameras"] = bc.numpy()
    for name in ("position_oracle", "orientation_oracle"):
        rows = [bl.generate_batch_predictions_baseline(bc[b:b + 1].clone(), name) for b in range(4)]
        out[f"bl.{name}"] = torch.cat([torch.as_tensor(x["generated_cameras"]).as_subclass(torch.Tensor) for x in rows]).numpy()
    np.savez_compressed(os.path.join(OUT, "sevenscenes_reference_shim.npz"), **out)
    print("sevenscenes golden:", len(out), "arrays")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    golden_sevenscenes()

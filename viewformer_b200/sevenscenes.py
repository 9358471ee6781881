"""7-Scenes camera localisation, H100-native: the procedures of viewformer/evaluate/evaluate_sevenscenes.py and
evaluate_sevenscenes_baseline.py with the reference's names and argument meaning.

    generate_other_viewpoints                          evaluate_sevenscenes.py:20-33
    compute_camera_distances                           :36-45 (mode "combined"), evaluate_sevenscenes_baseline.py:43-51 (the other two)
    SceneLookup                                        the ``.files`` / ``.cameras`` / ``[name] -> (camera, frame)`` object both read
    generate_batch_predictions_using_generated_images  evaluate_sevenscenes.py:80-154
    generate_batch_predictions_using_pose_refinement   evaluate_sevenscenes.py:157-197
    generate_batch_predictions_baseline                evaluate_sevenscenes_baseline.py:84-97 (position_oracle, orientation_oracle)
    BaselineEvaluator                                  evaluate_sevenscenes_baseline.py:18-40

The database scans (argsort over a scene's training cameras, argmin over a row's context) run in the ``vf_camera_knn`` kernel, whose
order is the stable one: ascending distance, ties to the lower index.  Camera arithmetic of a few floats stays host-side torch, as in
generate.py; random draws are made on the CPU so that they do not depend on the device.
"""
import random as _random

import numpy as np
import torch

from . import _lib as L
from .cameras import camera_knn
from .evaluate import encode_images
from .generate import (generate_batch_predictions, localize_last_view, normalize_cameras, quaternion_multiply, quaternion_normalize)
from .metrics import Evaluator
from .vqgan import image_tensor

CONTEXT_VIEWS = 19                     # evaluate_sevenscenes.py:191, 240: 19 context frames and the query


def _l2_normalize_all(x, epsilon=1e-12):
    """tf.math.l2_normalize without an axis: ONE norm over the whole tensor."""
    return x * torch.rsqrt(torch.clamp((x * x).sum(dim=None, keepdim=True), min=epsilon))


def generate_other_viewpoints(camera, generator=None):
    """evaluate_sevenscenes.py:20-33: random poses up to 1 m and 0.3 rad away from ``camera`` [..., 7].

    The four tf.random.uniform draws are made in the reference's order and shapes, on the CPU generator ``generator`` (torch's default
    one when None), each as ``u * (hi - lo) + lo``.  As in the reference, the position offset and the rotation axis are L2-normalised
    over the WHOLE tensor, not per camera: the cameras of one call share one norm, and an axis is not a unit vector unless the call has
    one camera.  The result is computed on the CPU in ``camera``'s dtype and returned on ``camera``'s device."""
    camera = torch.as_tensor(camera)
    dev, c = camera.device, camera.detach().cpu()

    def uniform(shape, lo, hi):
        return torch.rand(shape, generator=generator, dtype=c.dtype) * (hi - lo) + lo
    pos_offset = _l2_normalize_all(uniform(c[..., :3].shape, -1, 1))
    axis = _l2_normalize_all(uniform(c[..., :3].shape, -1, 1))
    pos_offset = pos_offset * uniform(c[..., :1].shape, 0, 1.)
    angle = uniform(c[..., :1].shape, 0, 0.3)
    rot = torch.cat((torch.cos(angle / 2), torch.sin(angle / 2) * axis), -1)
    new_pose = torch.cat((pos_offset + c[..., :3], quaternion_normalize(quaternion_multiply(rot, c[..., 3:]))), -1)
    return new_pose.to(dev)


def compute_camera_distances(db_cameras, camera, mode="combined"):
    """Distances [N] from every database camera [N,7] to ``camera`` [1,7] (or [7]): mode "combined" is evaluate_sevenscenes.py:36-45,
    "position" and "orientation" the two terms evaluate_sevenscenes_baseline.py:43-51 uses alone.  fp32, on the GPU (vf_camera_knn with
    slices of 64, one query per slice); the argument of asin is clamped to 1 (see include/vf_b200.h).  Returned in database order."""
    db = torch.as_tensor(np.asarray(db_cameras) if not torch.is_tensor(db_cameras) else db_cameras, dtype=torch.float32).cuda()
    q = torch.as_tensor(camera, dtype=torch.float32).reshape(1, 7).to(db.device)
    n = db.shape[0]
    s = (n + 63) // 64                                          # k <= 64: slices of 64 cameras, the last padded with the query itself
    pad = torch.cat((db, q.expand(s * 64 - n, 7)), 0).reshape(s, 64, 7).contiguous()
    idx, dist = camera_knn(pad, q.expand(s, 7).contiguous(), 64, mode)
    pos = (idx.long() + 64 * torch.arange(s, device=db.device)[:, None]).reshape(-1)
    keep = pos < n
    out = torch.empty(n, dtype=torch.float32, device=db.device)
    out[pos[keep]] = dist.reshape(-1)[keep]
    return out


class SceneLookup:
    """The scene database the 7-Scenes procedures read (evaluate_sevenscenes.py:48-68): ``.files`` (frame names), ``.cameras`` [N,7]
    and ``lookup[name] -> (camera [7], frame [H,W,C])``.  Built here from arrays; the reference builds its own from the raw dataset
    (SevenScenesLoader), and the procedures accept that object as it is."""

    def __init__(self, files, cameras, frames):
        self.files = list(files)
        self.cameras = np.asarray(cameras, dtype=np.float32)
        self.frames = frames
        if len(self.files) != len(self.cameras) or len(self.files) != len(frames):
            raise ValueError(f"SceneLookup: {len(self.files)} files, {len(self.cameras)} cameras, {len(frames)} frames")
        self._lookup = {x: i for i, x in enumerate(self.files)}

    def __getitem__(self, name):
        i = self._lookup[name]
        return self.cameras[i], self.frames[i]

    def __len__(self):
        return len(self.files)


def _prepare(transformer_model, codebook_model, images, cameras):
    """Shared head of both procedures (:81-100, :158-177): cameras in the model's pose frame and the codes of all T views."""
    dev = transformer_model.device
    images = image_tensor(images, "7-Scenes procedure")
    cameras = torch.as_tensor(cameras).to(torch.float32)
    relative = transformer_model.config.augment_poses == "relative"
    cams, transform = L.cameras_prepare(cameras.to(dev).contiguous(), relative)
    codes = encode_images(images, codebook_model=codebook_model).to(dev)
    return images, cameras, cams, transform, relative, codes


def generate_batch_predictions_using_generated_images(transformer_model, codebook_model, images, cameras, num_gen_ctx=5, generator=None):
    """evaluate_sevenscenes.py:80-154 as written, for one scene (B = 1).  ``images`` [1,T,H,W,C] uint8 (or float32 in [0, 1]),
    ``cameras`` [1,T,7]; ``generator`` is the CPU generator of generate_other_viewpoints' draws.

    1. Localise the query (view T-1) from all T views' codes; the estimate stays in the model's pose frame.
    2. Draw ``num_gen_ctx`` poses around it (generate_other_viewpoints) and render one view at each from context views 0..T-2.
    3. The sequence becomes context views 0..T-1-num_gen_ctx plus the generated views.  This drops the query's own codes and, with
       num_gen_ctx > 1, real context views too; this is what the reference computes.
    4. Render the last view of that sequence again (``generated_images``) and localise it (``generated_cameras``).  Both refer to
       the last GENERATED view, not the query, although they are scored against the query's image and camera.

    The reference puts the generated views on the view axis with a reshape that only works for one scene, so B != 1 raises
    ValueError, as does num_gen_ctx < 1 (at the reference's command-line default of 0 its slice ``[:-0]`` is empty)."""
    B, T = torch.as_tensor(cameras).shape[:2]
    if B != 1:
        raise ValueError(f"generate_batch_predictions_using_generated_images: one scene per call (the reference's reshape), got {B}")
    if not 1 <= num_gen_ctx < T:
        raise ValueError(f"generate_batch_predictions_using_generated_images: num_gen_ctx must be in [1, {T - 1}], got {num_gen_ctx}")
    images, cameras, cams, transform, relative, codes = _prepare(transformer_model, codebook_model, images, cameras)
    est = localize_last_view(transformer_model, codes, cams)                                      # :103-104
    new_cams = normalize_cameras(generate_other_viewpoints(est[:, -1:].repeat(num_gen_ctx, 1, 1), generator))   # :107-108
    new_cams = new_cams.to(cams.device)
    poses = torch.cat((cams[:, :-1].repeat(num_gen_ctx, 1, 1), new_cams), 1).contiguous()
    new_codes = transformer_model.generate_codes(codes[:, :-1].repeat(num_gen_ctx, 1, 1, 1), poses)           # :109-119
    codes = torch.cat((codes[:, :-num_gen_ctx], new_codes[None].to(codes.dtype)), 1)                           # :120-123
    cams = torch.cat((cams[:, :-num_gen_ctx], new_cams.reshape(1, num_gen_ctx, 7)), 1).contiguous()            # :124-127
    gen_codes = transformer_model.generate_codes(codes[:, :-1], cams)                                          # :130-134
    gen_images = codebook_model.decode_code_u8(gen_codes)                                                      # :137-140
    gen_cam = localize_last_view(transformer_model, codes, cams)                                               # :143-144
    if relative:
        gen_cam = L.cameras_from_relative(gen_cam.to(cams.device).contiguous(), transform)
    return dict(ground_truth_images=images[:, -1], generated_images=gen_images, ground_truth_cameras=cameras[:, -1],
                generated_cameras=gen_cam[:, -1], generated_codes=gen_codes)


def generate_batch_predictions_using_pose_refinement(scene_lookup, db_cameras, transformer_model, codebook_model, images, cameras,
                                                     num_gen_ctx=9, rng=_random):
    """evaluate_sevenscenes.py:157-197: localise the query (view T-1) from the given context, bring the estimate to world coordinates,
    take the ``num_gen_ctx`` database frames nearest to it (``db_cameras`` [N,7], combined distance, ascending, ties to the lower
    index) and ``19 - num_gen_ctx`` frames from ``rng.sample(scene_lookup.files, ...)``, and run generate_batch_predictions on those 19
    frames plus the query.  ``scene_lookup`` is a SceneLookup or the reference's own object; ``rng`` anything with ``sample`` (the
    module ``random`` by default, as in the reference).

    The reference takes one scene per call.  Here row b of a batch of B is what a one-scene call gives, with the lookups and the
    rng draws made row after row, in row order."""
    gt_cameras, gt_frames = torch.as_tensor(cameras)[:, -1], image_tensor(images, "pose refinement")[:, -1]
    images, cameras, cams, transform, relative, codes = _prepare(transformer_model, codebook_model, images, cameras)
    est = localize_last_view(transformer_model, codes, cams)                                   # :180-181
    if relative:
        est = L.cameras_from_relative(est.contiguous(), transform)                            # :184-185
    B = est.shape[0]
    top = [[] for _ in range(B)]
    if num_gen_ctx > 0:                                                                        # :188-189
        db = torch.as_tensor(np.asarray(db_cameras), dtype=torch.float32).to(est.device).contiguous()
        idx, _ = camera_knn(db, est[:, 0].contiguous(), num_gen_ctx, "combined")
        top = idx.cpu().tolist()
    ctx_cams, ctx_frames = [], []
    for b in range(B):
        files = [scene_lookup.files[x] for x in top[b]]                                        # :190-191
        files += rng.sample(scene_lookup.files, CONTEXT_VIEWS - len(files))
        c, f = tuple(np.stack(y, 0) for y in zip(*(scene_lookup[x] for x in files)))          # :192
        ctx_cams.append(torch.as_tensor(c))
        ctx_frames.append(torch.as_tensor(f))
    new_cams = torch.cat((torch.stack(ctx_cams).to(torch.float32), gt_cameras.to(torch.float32).cpu()[:, None]), 1)    # :195-196
    frames = torch.cat((torch.stack(ctx_frames).to(gt_frames.device), gt_frames[:, None].to(ctx_frames[0].dtype)), 1)
    return generate_batch_predictions(transformer_model, codebook_model, frames, new_cams)                             # :197


def generate_batch_predictions_baseline(cameras, baseline):
    """evaluate_sevenscenes_baseline.py:84-97 for ``position_oracle`` and ``orientation_oracle``: each row's context camera (views
    0..T-2 of ``cameras`` [B,T,7]) nearest to its query (view T-1) by position or by orientation, the first one on a tie.  The
    reference takes one row; every row here is that row's one-row result.  Returns dict(ground_truth_cameras [B,7],
    generated_cameras [B,7]) on the cameras' device.

    The ``mean`` baseline is not provided: it takes a ROW of np.linalg.eig's eigenvector matrix (utils/geometry.py:274-281), so its
    value depends on the per-column signs the LAPACK build picks."""
    if baseline not in ("position_oracle", "orientation_oracle"):
        raise ValueError(f"generate_batch_predictions_baseline: baseline {baseline!r}; 'position_oracle' or 'orientation_oracle'"
                         " ('mean' depends on LAPACK's eigenvector signs and is not reproducible)")
    cameras = torch.as_tensor(cameras, dtype=torch.float32)
    dev = cameras.device
    cams = cameras.cuda()
    ctx = cams[:, :-1].contiguous()                                                            # db_stride (T-1) * 7
    idx, _ = camera_knn(ctx, cams[:, -1].contiguous(), 1, "position" if baseline == "position_oracle" else "orientation")
    pred = ctx.gather(1, idx.long()[:, :, None].expand(-1, -1, 7))[:, 0]
    return dict(ground_truth_cameras=cameras[:, -1], generated_cameras=pred.to(dev))


class BaselineEvaluator(Evaluator):
    """evaluate_sevenscenes_baseline.py:18-40: the localisation metrics only (loc-angle, loc-dist and their medians) and a progress
    bar of cam_loc and cam_ang."""

    def update_state(self, ground_truth_cameras, generated_cameras):
        self.update_with_camera(ground_truth_cameras, generated_cameras)

    def get_progress_bar_info(self):
        return dict(cam_loc=self._loc["dist"].result(), cam_ang=self._loc["angle"].result())

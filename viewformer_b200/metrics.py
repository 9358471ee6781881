"""Evaluation metrics of the reference (viewformer/utils/metrics.py:17-230, evaluate/evaluate_transformer.py:22-67) on the GPU.

Image metrics take uint8 NHWC images (what ``generate_batch_predictions`` returns) and reduce them with libvf_b200 kernels: exact
integer sums for MSE / MAE / RMSE / PSNR, the 7x7 uniform-window SSIM of ``ssim()``.  Camera metrics are a handful of floats per
scene and stay host-side torch (same formulas as CameraPositionError / CameraOrientationError, NaN-tolerant means, medians).
LPIPS (utils/metrics.py:199-214) is ``viewformer_b200.lpips.LPIPS``, computed from VGG16 / lpips weight files the caller passes in; the
evaluators report it when given one (``lpips=``).
"""

import torch

from . import _lib as L
from .generate import quaternion_multiply, quaternion_conjugate, quaternion_normalize


def _u8(x, device):
    t = torch.as_tensor(x)
    if t.dtype != torch.uint8:
        raise TypeError("image metrics take uint8 images (the reference converts with tf.image.convert_image_dtype)")
    if t.dim() == 3:
        t = t[None]
    return t.to(device).contiguous()


def image_metrics(gt_images, images, device="cuda", ssim_k1=None):
    """uint8 [N,H,W,C] x2 -> dict of per-image float64 tensors: mse, mae (range [0,1]), rmse (range [0,255]), psnr (dB), ssim.
    ``ssim_k1``: K1 of ``ssim()`` (metrics.py:17; default 0.01).  The reference's SSIMMetric passes 1 (metrics.py:183)."""
    a, b = _u8(gt_images, device), _u8(images, device)
    n = a.shape[0]
    sums = L.image_pair_sums(a, b).to(torch.float64)
    cnt = float(a[0].numel())
    mse = sums[:, 1] / (cnt * 255.0 * 255.0)
    return dict(mse=mse, mae=sums[:, 0] / (cnt * 255.0), rmse=torch.sqrt(sums[:, 1] / cnt),
                psnr=10.0 * torch.log10(1.0 / mse),                      # tf.image.psnr(max_val = 1)
                ssim=(L.ssim_u8(a, b, k1=ssim_k1) if min(a.shape[1], a.shape[2]) >= 7
                      else torch.full((n,), float("nan"), dtype=torch.float64)))


def camera_position_error(x1, x2):
    return torch.linalg.norm(torch.as_tensor(x1)[..., :3] - torch.as_tensor(x2)[..., :3], dim=-1)


def camera_orientation_error(x1, x2):
    """2 asin |vec(q1 * conj(q2))| (metrics.py:103-115)."""
    q1 = quaternion_normalize(torch.as_tensor(x1)[..., 3:])
    q2 = quaternion_normalize(torch.as_tensor(x2)[..., 3:])
    diff = quaternion_multiply(q1, quaternion_conjugate(q2))
    return 2 * torch.asin(torch.linalg.norm(diff[..., 1:], dim=-1))


class Mean:
    """Running mean.  ``nan="skip"``: NaN samples carry no weight (image metrics of images too small for a 7x7 window).
    ``nan="zero"``: what the reference's AllowNanMean (metrics.py:76-88) actually computes for the camera errors — it replaces NaN
    by 0 and THEN derives the weight from is_nan of the cleaned values, so a NaN sample counts as an error of 0 with full weight."""

    def __init__(self, name, nan="skip"):
        assert nan in ("skip", "zero")
        self.name, self.total, self.count, self.nan = name, 0.0, 0.0, nan

    def update_state(self, values):
        v = torch.as_tensor(values, dtype=torch.float64).reshape(-1).cpu()
        ok = ~torch.isnan(v)
        self.total += float(v[ok].sum())
        self.count += float(ok.sum()) if self.nan == "skip" else float(v.numel())

    def result(self):
        return self.total / self.count if self.count else 0.0


class Median:
    """metrics.py:118-144."""

    def __init__(self, name):
        self.name, self.store = name, []

    def update_state(self, values):
        self.store.append(torch.as_tensor(values, dtype=torch.float64).reshape(-1).cpu())

    def result(self):
        if not self.store:
            return 0.0
        v = torch.sort(torch.cat(self.store)).values
        n = len(v)
        return float(v[(n - 1) // 2]) if n % 2 == 1 else 0.5 * float(v[n // 2 - 1] + v[n // 2])


class Evaluator:
    """evaluate/evaluate_transformer.py:22-67: image-generation metrics (mse, rmse, mae, psnr, ssim) and localisation metrics
    (loc-angle, loc-dist and their medians); images are brought to a common size with the dataset resize rule first.

    The numbers are the ones the reference's Evaluator reports, including what follows from HOW it calls its metric classes
    (pinned by running the reference's Evaluator itself, tests/test_reference_on_shim.py and tests/golden/evaluator_reference_shim.npz):
    ``mse`` / ``mae`` are Keras MeanSquaredError / MeanAbsoluteError on the uint8 images CAST to float (0..255 scale, not [0,1]);
    ``ssim`` is ``SSIMMetric``, which passes 1 as the third positional argument of ``ssim()`` — K1 = 1, not the data range
    (metrics.py:183); ground truth is resized with the default rule, the generated image bilinearly (evaluate_transformer.py:42-45).

    ``lpips``: an ``viewformer_b200.lpips.LPIPS`` (may be shared between evaluators).  With it, ``lpips`` of the resized pair is reported
    between ``psnr`` and ``ssim``, as the reference's LPIPSMetric is; without it the results have no ``lpips`` key."""

    def __init__(self, image_size=None, device="cuda", lpips=None):
        self.image_size, self.device, self.lpips = image_size, device, lpips
        self._loc = dict(angle=Mean("loc-angle", nan="zero"), dist=Mean("loc-dist", nan="zero"), angle_med=Median("loc-angle-med"),
                         dist_med=Median("loc-dist-med"))
        names = ("mse", "rmse", "mae", "psnr") + (("lpips",) if lpips is not None else ()) + ("ssim",)
        self._img = {k: Mean(k) for k in names}

    def update_with_image(self, ground_truth_images, generated_images):
        gt, gen = _u8(ground_truth_images, self.device), _u8(generated_images, self.device)
        size = self.image_size or max(gt.shape[-2], gen.shape[-2])
        gt, gen = L.resize_u8(gt, size), L.resize_u8(gen, size, method="bilinear")
        m = image_metrics(gt, gen, self.device, ssim_k1=1.0)
        m["mse"], m["mae"] = m["mse"] * (255.0 * 255.0), m["mae"] * 255.0
        if self.lpips is not None:
            m["lpips"] = self.lpips(gt, gen)
        for k, v in m.items():
            self._img[k].update_state(v)

    def update_with_camera(self, ground_truth_cameras, generated_cameras):
        gt, gen = torch.as_tensor(ground_truth_cameras).cpu(), torch.as_tensor(generated_cameras).cpu()
        ang, dist = camera_orientation_error(gt, gen), camera_position_error(gt, gen)
        self._loc["angle"].update_state(ang); self._loc["angle_med"].update_state(ang)
        self._loc["dist"].update_state(dist); self._loc["dist_med"].update_state(dist)

    def update_state(self, ground_truth_cameras=None, generated_cameras=None, ground_truth_images=None, generated_images=None):
        if ground_truth_images is not None and generated_images is not None:
            self.update_with_image(ground_truth_images, generated_images)
        if ground_truth_cameras is not None and generated_cameras is not None:
            self.update_with_camera(ground_truth_cameras, generated_cameras)

    def get_progress_bar_info(self):
        """evaluate_transformer.py:56-61 (img_lpips only with an LPIPS)."""
        info = dict(img_psnr=self._img["psnr"].result())
        if "lpips" in self._img:
            info["img_lpips"] = self._img["lpips"].result()
        info.update(cam_loc=self._loc["dist"].result(), cam_ang=self._loc["angle"].result())
        return info

    def result(self):
        out = {m.name: float(m.result()) for m in self._img.values() if m.count}
        out.update({m.name: float(m.result()) for m in self._loc.values() if (getattr(m, "count", 0) or getattr(m, "store", None))})
        return out


class CodebookEvaluator(Evaluator):
    """evaluate/evaluate_codebook.py:18-49: the image half only, ``update_state(ground_truth_images, generated_images)``."""

    def update_state(self, ground_truth_images, generated_images):
        self.update_with_image(ground_truth_images, generated_images)

    def get_progress_bar_info(self):
        info = dict(img_rgbl1=self._img["mae"].result())
        if "lpips" in self._img:
            info["img_lpips"] = self._img["lpips"].result()
        return info

    def result(self):
        return {m.name: float(m.result()) for m in self._img.values() if m.count}


class MultiContextEvaluator:
    """evaluate/evaluate_transformer_multictx.py:13-34: one Evaluator per context size.  ``generated_images`` [B,T,H,W,3] /
    ``generated_cameras`` [B,T,7] hold the prediction made from the first i views at index i; index 0 (no context) is skipped and
    the result is keyed ``ctx01`` ... ``ctx{T-1}``.  ``lpips``: shared by every context size's Evaluator."""

    def __init__(self, sequence_size, image_size=None, device="cuda", lpips=None):
        self.sequence_size = sequence_size
        self._evaluators = [Evaluator(image_size=image_size, device=device, lpips=lpips) for _ in range(sequence_size - 1)]

    def update_state(self, ground_truth_cameras=None, generated_cameras=None, ground_truth_images=None, generated_images=None):
        n = generated_images.shape[1] if generated_images is not None else generated_cameras.shape[1]
        for i in range(1, n):
            self._evaluators[i - 1].update_state(ground_truth_cameras, None if generated_cameras is None else generated_cameras[:, i],
                                                 ground_truth_images, None if generated_images is None else generated_images[:, i])

    def get_progress_bar_info(self):
        return self._evaluators[-1].get_progress_bar_info()

    def result(self):
        from collections import OrderedDict
        return OrderedDict((f"ctx{i + 1:02d}", x.result()) for i, x in enumerate(self._evaluators))


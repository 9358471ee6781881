"""Pure checkers of the pose-scale wrappers in ``viewformer_b200.pose_scale`` (include/vf_b200_pose.h), in the form of
tests/launch_checks.py: each restates the wrapper's result in fp64 from the operands the kernel read and returns the worst ratio of error
to its bar (<= 1 passes; conditions that must hold exactly return inf when they fail).  The bars are those of the unscaled pose kernels'
checkers, 8 u of the magnitudes involved (u = 2^-24), with the predicted xyz r replaced by r / c, c the row's scene multiplier.
"""
import math
import random

import torch

from launch_checks import U, _pose_target, before_none, bind, f32, ratio


def _scene_mult(ba, rows):
    """The multiplier c of each row's scene, fp64 [rows, 1] (rows // tokens_per_view is the view, view // views_per_scene the scene)."""
    c = ba["scene_mult"].double()
    return c[rows // int(ba["tokens_per_view"]) // int(ba["views_per_scene"])][:, None]


def check_pose_loss_rows_scaled(ba, result, st):
    """pos = mean_3 (y m - r / c)^2, ori = mean_4 (y - r)^2 per row: 8 u mean (|y m| + |r / c|)^2 and 8 u mean (|y| + |r|)^2."""
    raw = ba["raw_rows"]
    rows = torch.arange(raw.shape[0], device=raw.device)
    y, r, c = _pose_target(ba, rows), raw.double(), _scene_mult(ba, rows)
    m = f32(ba["mult"])
    pos, ori = result
    ym, rc = y[:, :3] * m, r[:, :3] / c
    return max(ratio((pos.double() - ((ym - rc) ** 2).mean(1)).abs(), 8 * U * ((ym.abs() + rc.abs()) ** 2).mean(1) + 1e-38),
               ratio((ori.double() - ((y[:, 3:] - r[:, 3:]) ** 2).mean(1)).abs(), 8 * U * ((y[:, 3:].abs() + r[:, 3:].abs()) ** 2).mean(1) + 1e-38))


def check_pose_loss_grad_scaled(ba, result, st):
    """d/draw of sum w (ps mean_3 (y m - r / c)^2 + os mean_4 (y - r)^2): the position part is -w ps 2/3 (y m - r / c) / c; bar
    8 u w scale (|y m| + |r / c|) / c."""
    raw, w = ba["raw_rows"], ba["row_weight"].double()[:, None]
    rows = torch.arange(raw.shape[0], device=raw.device)
    y, r, c = _pose_target(ba, rows), raw.double(), _scene_mult(ba, rows)
    mv = torch.tensor([f32(ba["mult"])] * 3 + [1.0] * 4, dtype=torch.float64, device=raw.device)
    scl = torch.tensor([f32(ba["pos_scale"]) * 2 / 3] * 3 + [f32(ba["ori_scale"]) * 2 / 4] * 4, dtype=torch.float64, device=raw.device)
    div = torch.cat([c.expand(-1, 3), torch.ones_like(c).expand(-1, 4)], 1)               # r / c and the outer 1 / c: xyz columns only
    want = -w * scl * (y * mv - r / div) / div
    return ratio((result.double() - want).abs(), 8 * U * w.abs() * scl * ((y * mv).abs() + (r / div).abs()) / div + 1e-38)


def check_pose_model_input(ba, result, st):
    """[(xyz m) c | quaternion] of each pose, c its scene's multiplier (1 without scene_mult): two fp32 roundings of the xyz, 2 u |x m c|;
    the quaternion copied bit for bit."""
    p = ba["poses_bt7"]
    rows = torch.arange(p.shape[0], device=p.device)
    c = torch.ones((p.shape[0], 1), dtype=torch.float64, device=p.device)
    if ba["scene_mult"] is not None:
        c = ba["scene_mult"].double()[rows // int(ba["views_per_scene"])][:, None]
    want = p[:, :3].double() * f32(ba["mult"]) * c
    if not torch.equal(result[:, 3:], p[:, 3:]):
        return math.inf
    return ratio((result[:, :3].double() - want).abs(), 2 * U * want.abs() + 1e-38)


CHECKERS = {
    "pose_model_input": (before_none, check_pose_model_input),
    "pose_loss_rows_scaled": (before_none, check_pose_loss_rows_scaled),
    "pose_loss_grad_scaled": (before_none, check_pose_loss_grad_scaled),
}


def run_check(name, fn, a, k, rng=None):
    """Call wrapper ``fn`` with its snapshot taken first; return (result, worst ratio)."""
    before, check = CHECKERS[name]
    ba = bind(fn, *a, **k)
    st = before(ba, rng or random.Random(0))
    result = fn(*a, **k)
    return result, check(ba, result, st)

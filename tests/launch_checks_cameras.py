"""Pure checker of the nearest-camera wrapper ``viewformer_b200.cameras.camera_knn`` (vf_camera_knn), in the form of tests/launch_checks.py
(a check returns the worst ratio of error to its bar, <= 1 passes; conditions that must hold exactly return inf when they fail), with its
helpers and unit roundoff u = 2^-24.  The distances are restated in fp64 from the cameras the kernel read (``camera_distances64``); the
picks are held to fp64's stable order wherever the distances are separated by more than their bars.
"""
import math

import numpy as np
import torch

from launch_checks import U, _conj, _qmul, before_none, bind, f32, ratio

KNN_MODES = {"combined": 0, "position": 1, "orientation": 2}


def camera_distances64(db, queries, mode):
    """fp64 distances [Q, N] of vf_camera_knn (x1 = database camera, x2 = query) and their bars.  Position: the fp32 differences, three
    squares, two sums and sqrt, 8 u |xyz|.  Orientation: s = |vec(n(q1) n(q2)*)| carries about 16 u absolute (two normalisations and a
    product of unit quaternions, each component a sum of four products bounded by 1) and the norm 3 u more; 2 asin is steep near s = 1,
    so the bar is the width of 2 asin over [s - 32 u, s + 32 u] (clamped to [0, 1]) plus 4 u of the angle.  Combined: fp32(0.3) times
    the position (one rounding), plus the orientation (one rounding)."""
    db, q = db.double(), queries.double()
    if db.dim() == 2:
        db = db[None].expand(q.shape[0], -1, -1)
    m = KNN_MODES[mode] if isinstance(mode, str) else int(mode)
    pos = (db[..., :3] - q[:, None, :3]).norm(dim=-1)
    pbar = 8 * U * pos

    def unit(x):
        return x / torch.sqrt((x * x).sum(-1, keepdim=True).clamp_min(1e-12))
    s = _qmul(unit(db[..., 3:]), _conj(unit(q[:, None, 3:])).expand_as(db[..., 3:]))[..., 1:].norm(dim=-1).clamp(max=1.0)
    ang = 2 * torch.asin(s)
    abar = 2 * (torch.asin((s + 32 * U).clamp(max=1.0)) - torch.asin((s - 32 * U).clamp(min=0.0))) + 4 * U * ang
    if m == 1:
        return pos, pbar
    if m == 2:
        return ang, abar
    c = f32(np.float32(0.3))
    d = c * pos + ang
    return d, c * pbar + U * c * pos + abar + 2 * U * d


def check_camera_knn(ba, result, st):
    """The k nearest database cameras of each query against the fp64 distances of ``camera_distances64``: indices in range and distinct;
    each returned distance within its bar of the fp64 distance of its index, and within both bars of the fp64 j-th smallest (so a pick
    may differ from fp64's only inside a near tie); the same index as fp64's stable order wherever the sorted fp64 distances leave a gap
    of more than twice the bars on both sides, and the same set wherever the k-th and (k+1)-th do; fp32 distances ascending, an exact
    tie in lower-index-first order."""
    idx, dist = result
    k = int(ba["k"])
    d64, bar = camera_distances64(ba["db"], ba["queries"], ba["mode"])
    n = d64.shape[1]
    gi = idx.long()
    if gi.shape != (d64.shape[0], k) or bool(((gi < 0) | (gi >= n)).any()):
        return math.inf
    if k > 1 and bool((gi.sort(1).values.diff(dim=1) == 0).any()):
        return math.inf
    if k > 1 and bool(((dist[:, 1:] < dist[:, :-1]) | ((dist[:, 1:] == dist[:, :-1]) & (gi[:, 1:] <= gi[:, :-1]))).any()):
        return math.inf
    d_at, b_at = d64.gather(1, gi), bar.gather(1, gi)
    sd, si = torch.sort(d64, dim=1, stable=True)
    sb = bar.gather(1, si)
    worst = max(ratio((dist.double() - d_at).abs(), b_at), ratio((d_at - sd[:, :k]).abs(), b_at + sb[:, :k]))
    inf = torch.full_like(sd[:, :1], math.inf)
    gap = torch.cat([inf, sd.diff(dim=1) - 2 * (sb[:, 1:] + sb[:, :-1]), inf], 1)          # gap[:, j]: between sorted j - 1 and j
    sep = (gap[:, :k] > 0) & (gap[:, 1:k + 1] > 0)
    if bool((sep & (gi != si[:, :k])).any()):
        return math.inf
    cut = gap[:, k] > 0
    if bool((cut & (gi.sort(1).values != si[:, :k].sort(1).values).any(1)).any()):
        return math.inf
    return worst


CHECKERS = {
    "camera_knn": (before_none, check_camera_knn),
}


def run_check(name, fn, a, k, rng):
    """launch_checks.run_check for the wrapper above: (result, worst ratio)."""
    before, check = CHECKERS[name]
    ba = bind(fn, *a, **k)
    st = before(ba, rng)
    result = fn(*a, **k)
    return result, check(ba, result, st)

"""The nearest-camera search of 7-Scenes localisation on the device: a thin wrapper of ``vf_camera_knn`` (include/vf_b200.h), which
scans a scene's camera database with the reference's distances (evaluate_sevenscenes.py:36-45, evaluate_sevenscenes_baseline.py:43-51)
in a stable order.  Like every launching wrapper it is checked against fp64 on its own operands in the tests
(tests/launch_checks_cameras.py).
"""
import torch

from . import _lib as L

DISTANCE_MODES = {"combined": 0, "position": 1, "orientation": 2}


def camera_knn(db, queries, k, mode="combined"):
    """The ``k`` nearest database cameras of each query, ascending, ties to the lower index.  ``db`` f32 [N,7] (one database for all
    queries) or [Q,N,7] (one per query); ``queries`` f32 [Q,7]; ``mode`` "combined", "position" or "orientation".
    -> (indices int32 [Q,k], distances f32 [Q,k])."""
    lib = L.load(True)
    L._dev(db, torch.float32)
    L._dev(queries, torch.float32)
    q = queries.shape[0]
    if queries.dim() != 2 or queries.shape[1] != 7 or db.dim() not in (2, 3) or db.shape[-1] != 7 or (db.dim() == 3 and db.shape[0] != q):
        raise ValueError(f"camera_knn: database {tuple(db.shape)} and queries {tuple(queries.shape)}, expected [N,7] or [Q,N,7] and [Q,7]")
    n, stride = db.shape[-2], (db.shape[1] * 7 if db.dim() == 3 else 0)
    idx = torch.empty((q, max(int(k), 0)), dtype=torch.int32, device=queries.device)
    dist = torch.empty((q, max(int(k), 0)), dtype=torch.float32, device=queries.device)
    L._check(lib.vf_camera_knn(db, n, stride, queries, q, DISTANCE_MODES[mode], int(k), idx, dist, L._stream()))
    return idx, dist

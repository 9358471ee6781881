"""The pose-scale augmentation of transformer training (MIGTConfig.random_pose_multiplier = c, models/migt.py:349-354): in training each
scene b takes r_b = c ** u_b, u_b ~ U[-1, 1); its poses' xyz enter the pose MLP scaled by r_b and the pose head's xyz is divided by r_b
before the position loss.

The three kernels are declared in include/vf_b200_pose.h and built into libvf_b200.so; ``PROTOTYPES`` binds them as ``_lib.PROTOTYPES``
binds include/vf_b200.h (tests/test_pose_scale_host.py holds the table to that header).  ``pose_scale_exponents`` is the trainer's
stateless draw of u."""
import ctypes as C

import torch

from . import _lib as L


def _prototypes():
    """Parameter types of every function include/vf_b200_pose.h declares, in order (p: a device pointer, s: vf_stream_t)."""
    i, i64, f32, p, s = C.c_int, C.c_int64, C.c_float, L.DevPtr, C.c_void_p
    return {
        "vf_pose_model_input": [p, i64, i, f32, p, p, s],
        "vf_pose_loss_rows_scaled": [p, p, i64, i, f32, i, p, p, p, s],
        "vf_pose_loss_grad_scaled": [p, p, p, i64, i, f32, i, p, f32, f32, p, s],
    }


PROTOTYPES = _prototypes()          # every entry point returns int
_declared = []


def load():
    """libvf_b200.so (``_lib.load``, which checks the device) with these entry points' types declared."""
    lib = L.load(True)
    if not _declared:
        for name, argtypes in PROTOTYPES.items():
            if not hasattr(lib, name):
                raise L.LibraryError(f"{L.LIB_PATH} does not export {name}")
            fn = getattr(lib, name)
            fn.argtypes, fn.restype = argtypes, C.c_int
        _declared.append(True)
    return lib


def pose_model_input(poses_bt7, mult, views_per_scene, scene_mult=None):
    """get_model_input (models/migt.py:139-145): [(xyz * mult) * scene_mult[b] | quaternion] of poses [B*T, 7] fp32 (scene_mult None:
    [xyz * mult | quaternion])."""
    lib = load()
    L._dev(poses_bt7, torch.float32)
    out = torch.empty_like(poses_bt7)
    L._check(lib.vf_pose_model_input(poses_bt7, poses_bt7.shape[0], views_per_scene, mult, scene_mult, out, L._stream()))
    return out


def pose_loss_rows_scaled(raw_rows, poses_bt7, tokens_per_view, mult, views_per_scene, scene_mult):
    """_lib.pose_loss_rows with the predicted xyz of scene b divided by scene_mult[b] (fp32 [B]; None: no division)."""
    lib = load()
    rows = raw_rows.shape[0]
    pos = torch.empty((rows,), dtype=torch.float32, device=raw_rows.device)
    ori = torch.empty((rows,), dtype=torch.float32, device=raw_rows.device)
    L._check(lib.vf_pose_loss_rows_scaled(raw_rows, poses_bt7, rows, tokens_per_view, mult, views_per_scene, scene_mult, pos, ori, L._stream()))
    return pos, ori


def pose_loss_grad_scaled(raw_rows, poses_bt7, row_weight, tokens_per_view, mult, views_per_scene, scene_mult, pos_scale=1.0, ori_scale=1.0):
    """_lib.pose_loss_grad of pose_loss_rows_scaled."""
    lib = load()
    out = torch.empty_like(raw_rows)
    L._check(lib.vf_pose_loss_grad_scaled(raw_rows, poses_bt7, row_weight, raw_rows.shape[0], tokens_per_view, mult, views_per_scene, scene_mult,
                                          pos_scale, ori_scale, out, L._stream()))
    return out


def _mix64(k):
    """The 64-bit finaliser of vf_common.cuh's mix32 (MurmurHash3 fmix64)."""
    M = (1 << 64) - 1
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M
    return k ^ (k >> 33)


def pose_scale_exponents(seed, iterations, rank, micro_batch, n_scenes):
    """The exponents u ~ U[-1, 1) for the scenes of one micro-batch: fp32 [n_scenes] on a 2^-23 grid, a hash of (seed, iterations, rank,
    micro-batch, scene) built as the dropout seeds are, so every scene of the global batch draws its own value and a resumed run draws
    what the uninterrupted run would have."""
    base = ((int(seed) * 1000003 + int(iterations)) * 4096 + int(rank)) * 4096 + int(micro_batch)
    M = (1 << 64) - 1
    h = [_mix64(((base * 65536 + b) * 0x9E3779B97F4A7C15) & M) >> 40 for b in range(n_scenes)]
    return torch.tensor(h, dtype=torch.float64).mul_(2.0 ** -23).sub_(1.0).to(torch.float32)

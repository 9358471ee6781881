"""The data formats either side of the hot path (SURVEY.md §8 f2 / f4), without TensorFlow:

  * TFRecord container + ``tf.train.Example`` codec for the three feature kinds the reference writes
    (viewformer/data/tfrecord_dataset.py: ``codes`` int64_list, ``cameras`` float_list, ``frames`` bytes_list of JPEG/PNG);
  * ``LatentCodeTransformer`` — the ``generate-codes`` transform (viewformer/commands/generate_codes.py:20-78): scenes of frames +
    cameras in, scenes of codes + cameras out, encoding in fixed-size image batches across scene boundaries;
  * ``write_token_dataset`` / ``load_token_dataset`` — the transformer-training loader (data/tfrecord_dataset.py:134-197): per
    scene shuffle, windows of ``sequence_size`` views (drop remainder), up to ``max_samples_per_environment`` windows per scene,
    shuffle buffer, batches; rank / world sharding over files as ``dataset.shard`` does.
"""
import io
import json
import os
import random
import struct

import numpy as np
import torch

from .tf_checkpoint import masked_crc, _varint, _put_varint, _fields, _f_bytes


# ----------------------------------------------------------------------------------------------- TFRecord container
class TFRecordWriter:
    def __init__(self, path):
        self.f = open(path, "wb")

    def write(self, record):
        hdr = struct.pack("<Q", len(record))
        self.f.write(hdr + struct.pack("<I", masked_crc(hdr)) + record + struct.pack("<I", masked_crc(record)))

    def close(self):
        self.f.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def read_tfrecords(path, verify=False):
    with open(path, "rb") as f:
        while True:
            hdr = f.read(12)
            if len(hdr) < 12:
                return
            (n,) = struct.unpack("<Q", hdr[:8])
            if verify and struct.unpack("<I", hdr[8:])[0] != masked_crc(hdr[:8]):
                raise ValueError(f"{path}: corrupt record length")
            data = f.read(n)
            crc = f.read(4)
            if verify and struct.unpack("<I", crc)[0] != masked_crc(data):
                raise ValueError(f"{path}: corrupt record")
            yield data


# ----------------------------------------------------------------------------------------------- tf.train.Example
def encode_example(features):
    """{name: np.int64 array | np.float32 array | list of bytes} -> serialized tf.train.Example."""
    feats = b""
    for name, val in features.items():
        if isinstance(val, (list, tuple)) and val and isinstance(val[0], (bytes, bytearray)):
            inner = _f_bytes(1, b"".join(_f_bytes(1, bytes(v)) for v in val))                    # Feature.bytes_list
        else:
            arr = np.asarray(val)
            if arr.dtype.kind == "f":
                inner = _f_bytes(2, _f_bytes(1, arr.astype("<f4").reshape(-1).tobytes()))          # Feature.float_list (packed)
            else:
                inner = _f_bytes(3, _f_bytes(1, b"".join(_put_varint(int(v)) for v in arr.reshape(-1))))   # Feature.int64_list (packed)
        feats += _f_bytes(1, _f_bytes(1, name.encode()) + _f_bytes(2, inner))                    # map entry: key, value
    return _f_bytes(1, feats)                                                                   # Example.features


def decode_example(buf):
    out = {}
    for fn, _, features in _fields(buf):
        if fn != 1:
            continue
        for f2, _, entry in _fields(features):
            if f2 != 1:
                continue
            name, feat = None, b""
            for f3, _, v in _fields(entry):
                if f3 == 1:
                    name = v.decode()
                elif f3 == 2:
                    feat = v
            for kind, _, lst in _fields(feat):
                if kind == 1:
                    out[name] = [v for f4, _, v in _fields(lst) if f4 == 1]
                elif kind == 2:
                    vals = []
                    for f4, wt, v in _fields(lst):
                        if f4 == 1 and wt == 2:
                            vals.append(np.frombuffer(v, dtype="<f4"))
                        elif f4 == 1:
                            vals.append(np.asarray([struct.unpack("<f", struct.pack("<I", v))[0]], dtype=np.float32))
                    out[name] = np.concatenate(vals) if vals else np.zeros((0,), np.float32)
                elif kind == 3:
                    vals = []
                    for f4, wt, v in _fields(lst):
                        if f4 == 1 and wt == 2:
                            pos = 0
                            while pos < len(v):
                                x, pos = _varint(v, pos)
                                vals.append(x if x < (1 << 63) else x - (1 << 64))
                        elif f4 == 1:
                            vals.append(v if v < (1 << 63) else v - (1 << 64))
                    out[name] = np.asarray(vals, dtype=np.int64)
    return out


def decode_frames(frame_bytes):
    """bytes_list of encoded images -> uint8 [T,H,W,C] with the channels that are stored, as tf.io.decode_image returns them (PIL):
    C = 4 for the RGBA PNG frames of 4-channel datasets (data/tfrecord_dataset.py:318-321, CO3Dv2's masked RGB + mask), C = 3 for
    everything else (RGB JPEG; other modes are converted to RGB)."""
    from PIL import Image

    def decode(b):
        im = Image.open(io.BytesIO(b))
        return np.asarray(im if im.mode == "RGBA" else im.convert("RGB"))
    return np.stack([decode(b) for b in frame_bytes])


# ----------------------------------------------------------------------------------------------- generate-codes
class LatentCodeTransformer:
    """commands/generate_codes.py:20-78 with a viewformer_b200 codebook: ``transformer(split, scenes)`` yields one dict(cameras, codes)
    per input scene; images are encoded ``batch_size`` at a time irrespective of scene boundaries (the reference's
    unbatched_ / batched_ / update_cummulative_variable dance)."""

    def __init__(self, model, batch_size=None, device=None):
        self.model = model if device is None else model.to(device)
        self.image_size = model.config.image_size
        self.in_channels = getattr(model.config, "in_channels", 3)      # a config without the field is an RGB codebook's
        self.batch_size = batch_size if batch_size is not None else model.config.batch_size
        self.dataset_info = None

    def update_dataset_info(self, dataset_info):
        dataset_info["token_image_size"] = self.image_size // self.model.config.stride
        self.dataset_info = dataset_info
        return dataset_info

    def output_features(self, features):
        return ["codes", "cameras-gqn"] if features is not None and "cameras-gqn" in features else ["codes", "cameras"]

    def __call__(self, split, dataset):
        from . import _lib as L
        pending = []                                   # (cameras, n_frames) of scenes whose codes are not complete yet
        frames_buf, codes_buf = [], []

        def flush(final=False):
            nonlocal frames_buf, codes_buf
            while frames_buf and (final or sum(len(f) for f in frames_buf) >= self.batch_size):
                allf = np.concatenate(frames_buf)
                take = len(allf) if final else self.batch_size
                x = torch.from_numpy(np.ascontiguousarray(allf[:take])).to(self.model.device)
                x = L.resize_u8(x, self.image_size)
                codes_buf.append(self.model.encode_u8(x).cpu())
                frames_buf = [allf[take:]] if take < len(allf) else []

        def emit():
            nonlocal codes_buf
            have = torch.cat(codes_buf) if codes_buf else None
            while pending and have is not None and len(have) >= pending[0][1]:
                cams, n = pending.pop(0)
                yield dict(cameras=cams, codes=have[:n].numpy())
                have = have[n:]
            codes_buf = [have] if have is not None and len(have) else []

        for scene in dataset:
            frames = np.asarray(scene["frames"])
            if frames.dtype != np.uint8:
                raise TypeError("LatentCodeTransformer takes uint8 frames (NHWC)")
            if frames.ndim != 4 or frames.shape[-1] != self.in_channels:
                raise ValueError(f"LatentCodeTransformer: the codebook takes {self.in_channels}-channel frames, got frames of shape "
                                 f"{frames.shape}")
            pending.append((np.asarray(scene["cameras"], dtype=np.float32), len(frames)))
            frames_buf.append(frames)
            flush()
            yield from emit()
        flush(final=True)
        yield from emit()


# ----------------------------------------------------------------------------------------------- pose augmentation of the training loader
def _axis_quaternion(axis, angle):
    """utils/geometry_tf.py:16-33 (make_quaternion_x / _y): (cos(a/2), sin(a/2) * axis)."""
    angle = torch.as_tensor(angle)
    return torch.cat([torch.cos(angle / 2)[..., None], torch.sin(angle / 2)[..., None] * torch.tensor(axis, dtype=angle.dtype)], -1)


def process_batch(cameras, tokens, augment, split, generator=None):
    """train/train_transformer.py:31-64 — what the reference maps over every training sample (``transform=partial(process_batch,
    augment=config.augment_poses)``): 'relative' re-expresses the poses in the frame of the first view; 'simple' / 'advanced' (train split
    only) add one random translation ~ N(0, I) and one random rotation (y(U[0,2pi)) * x(U[0,pi/8)) * y(U[0,2pi)), resp. y(U[0,2pi))) to
    the whole window; 'no' leaves them; every branch ends with quaternion normalisation and the w >= 0 sign convention.  Host-side torch
    on the loader's tensors (a few floats per sample; the reference runs it inside tf.data on the CPU as well).  Random numbers are
    drawn in the reference's order — translation first, then the angles as Python evaluates the nested calls — from ``generator`` (or
    torch's global generator)."""
    import math
    from .generate import quaternion_multiply, quaternion_conjugate, quaternion_rotate, quaternion_normalize, quaternion_remove_sign
    cameras = torch.as_tensor(cameras)
    xyz, quaternion = cameras[..., :3], cameras[..., 3:]
    dt = xyz.dtype

    def normal():
        return torch.randn((1, 3), dtype=dt, generator=generator)

    def uniform(hi):
        return torch.rand((1,), dtype=dt, generator=generator) * hi

    if augment == "relative":
        rotation_inverse = quaternion_conjugate(quaternion[..., :1, :])
        xyz = quaternion_rotate(xyz - xyz[..., :1, :], rotation_inverse.expand_as(quaternion))
        quaternion = quaternion_multiply(rotation_inverse.expand_as(quaternion), quaternion)
    elif augment == "no" or split != "train":
        pass
    elif augment == "simple":
        xyz = xyz + normal()
        qy1 = _axis_quaternion([0.0, 1.0, 0.0], uniform(2 * math.pi))
        qx = _axis_quaternion([1.0, 0.0, 0.0], uniform(math.pi / 8))
        qy2 = _axis_quaternion([0.0, 1.0, 0.0], uniform(2 * math.pi))
        rotation = quaternion_multiply(qy1, quaternion_multiply(qx, qy2))
        xyz = quaternion_rotate(xyz, rotation.expand(*xyz.shape[:-1], 4))
        quaternion = quaternion_multiply(quaternion, rotation.expand_as(quaternion))
    elif augment == "advanced":
        xyz = xyz + normal()
        rotation = _axis_quaternion([0.0, 1.0, 0.0], uniform(2 * math.pi))
        xyz = quaternion_rotate(xyz, rotation.expand(*xyz.shape[:-1], 4))
        quaternion = quaternion_multiply(quaternion, rotation.expand_as(quaternion))
    else:
        raise ValueError(f"Augment {augment} is not supported")
    quaternion = quaternion_remove_sign(quaternion_normalize(quaternion))
    return torch.cat([xyz, quaternion], -1), tokens


# ----------------------------------------------------------------------------------------------- token dataset
def write_token_dataset(path, split, scenes, token_image_size, scenes_per_shard=64, name="b200-codes"):
    """Scenes of dict(cameras [T,7], codes [T,h,w]) -> ``<path>/<name>-<split>-<shard>-of-<n>.tfrecord`` + info.json."""
    os.makedirs(path, exist_ok=True)
    scenes = list(scenes)
    n_shards = max(1, (len(scenes) + scenes_per_shard - 1) // scenes_per_shard)
    for s in range(n_shards):
        with TFRecordWriter(os.path.join(path, f"{name}-{split}-{s:06d}-of-{n_shards:06d}.tfrecord")) as w:
            for sc in scenes[s * scenes_per_shard:(s + 1) * scenes_per_shard]:
                w.write(encode_example(dict(cameras=np.asarray(sc["cameras"], np.float32), codes=np.asarray(sc["codes"], np.int64))))
    info_path = os.path.join(path, "info.json")
    info = json.load(open(info_path)) if os.path.exists(info_path) else dict(name=name, token_image_size=token_image_size, features=["codes", "cameras"], splits=[])
    info[f"{split}_size"] = len(scenes)
    info["splits"] = sorted(set(info.get("splits", [])) | {split})
    with open(info_path, "w") as f:
        json.dump(info, f)
    return info


def load_token_dataset(path, batch_size, sequence_size, token_image_size, split="train", repeat=None, max_samples_per_environment=-1,
                       seed=0, rank=0, world=1, shuffle_buffer=1000, drop_last=True, max_windows_per_environment=None, transform=None):
    """Generator of (poses f32 [B,sequence_size,7], tokens int64 [B,sequence_size,h,w]) torch batches (data/tfrecord_dataset.py:134-197).
    ``batch_size`` is the GLOBAL batch; every rank yields batch_size // world samples from its own shard of the files.

    ``max_samples_per_environment`` does what the reference's does: ``.take(k)`` is applied to the dataset built from ONE window of
    ``sequence_size`` views (tfrecord_dataset.py:177-181), which holds exactly one sample — so k < 0 and every k >= 1 keep all windows of
    every scene and k == 0 yields nothing.  ``max_windows_per_environment`` is the limit the name suggests (at most that many windows per
    scene); it has no counterpart in the reference.  ``transform(cameras [S,7], tokens [S,h,w], split=...)`` is applied to every window,
    like the reference's ``env_d.map(partial(transform, split=...))`` — e.g. ``functools.partial(process_batch, augment=cfg.augment_poses)``."""
    files = []
    for p in path.split(","):
        files += sorted(os.path.join(p, f) for f in os.listdir(p) if f.endswith(".tfrecord") and f"-{split}-" in f)
    files = files[rank::world]
    local_bs = max(1, batch_size // world)
    rng = random.Random(seed * 1000003 + rank)
    epoch = 0
    while repeat is None or epoch < repeat or (repeat == 0 and epoch == 0):
        order = list(files)
        if split == "train":
            rng.shuffle(order)
        buf, batch = [], []

        def drain(final):
            while buf and (final or len(buf) >= shuffle_buffer):
                i = rng.randrange(len(buf)) if split == "train" else 0
                batch.append(buf.pop(i))
                if len(batch) == local_bs:
                    yield (torch.from_numpy(np.stack([b[0] for b in batch])), torch.from_numpy(np.stack([b[1] for b in batch])))
                    batch.clear()

        for fpath in order:
            for rec in read_tfrecords(fpath):
                ex = decode_example(rec)
                poses = ex["cameras"].reshape(-1, 7)
                tokens = ex["codes"].reshape(-1, token_image_size, token_image_size)
                idx = list(range(len(poses)))
                rng.shuffle(idx)                                   # "Shuffle train environments" (applied to every split, as in the reference)
                n_win = len(idx) // sequence_size
                if max_samples_per_environment == 0:
                    n_win = 0
                if max_windows_per_environment is not None:
                    n_win = min(n_win, max(0, int(max_windows_per_environment)))
                for wi in range(n_win):
                    sel = idx[wi * sequence_size:(wi + 1) * sequence_size]
                    sample = (poses[sel], tokens[sel])
                    if transform is not None:
                        p_t, t_t = transform(torch.from_numpy(sample[0]), torch.from_numpy(sample[1]), split="train" if split == "train" else "test")
                        sample = (np.asarray(p_t, dtype=np.float32), np.asarray(t_t))
                    buf.append(sample)
                yield from drain(False)
        yield from drain(True)
        if batch and not drop_last:
            yield (torch.from_numpy(np.stack([b[0] for b in batch])), torch.from_numpy(np.stack([b[1] for b in batch])))
        epoch += 1
        if repeat is None and not files:
            return
        if repeat is not None and epoch >= repeat:
            return

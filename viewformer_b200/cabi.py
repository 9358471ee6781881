"""Python half of the MODEL-LEVEL C-ABI (include/vf_b200_model.h -> viewformer_b200/libvf_b200_model.so).

SURVEY.md §8(b) lists the entry points a non-Python host would want (vf_vq_create / encode / decode_code, vf_migt_create / forward /
prefill_context / query, generate).  The layer sequencing of the two models is host logic written once, in Python (vqgan.py, migt.py);
instead of restating it in C++, libvf_b200_model.so is a thin C shim that embeds (or, inside a Python process, re-uses) the CPython
interpreter and calls the functions below with raw device pointers, sizes and a cudaStream_t.  Every function here takes plain ints /
floats / str and returns an int or None; device memory is wrapped zero-copy through ``__cuda_array_interface__``; work is issued on the
caller's stream (``torch.cuda.ExternalStream``).  The kernels underneath are the same libvf_b200.so entry points.

Reference surface served: vqgan_th.py:379-393 (encode / decode_code), migt.py:338-455 (call), evaluate_transformer.py:97-146
(generate_batch_predictions), evaluate_transformer_multictx_allimg.py:141-173 (context prefill + queries).
"""
import json

import torch

_models = {}
_next = [1]

_DT = {"u8": (torch.uint8, "|u1", 1), "i32": (torch.int32, "<i4", 4), "i64": (torch.int64, "<i8", 8), "f32": (torch.float32, "<f4", 4)}


class _Ext:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def _wrap(ptr, shape, dt, device):
    """Device pointer -> torch tensor view (no copy, no ownership)."""
    if not ptr:
        raise ValueError("null device pointer")
    tdt, ts, _ = _DT[dt]
    n = 1
    for s in shape:
        n *= int(s)
    if n == 0:
        return torch.empty(tuple(shape), dtype=tdt, device=device)
    return torch.as_tensor(_Ext(ptr, shape, ts), device=device)


def _put(model):
    h = _next[0]
    _next[0] += 1
    _models[h] = model
    return h


def _stream(model, stream_ptr):
    dev = model["device"] if isinstance(model, dict) else model.device
    return torch.cuda.stream(torch.cuda.ExternalStream(int(stream_ptr), device=dev)) if stream_ptr else torch.cuda.stream(torch.cuda.current_stream(dev))


def _build(kind, config_json, checkpoint, precision, device, seed):
    from . import VQGAN, MIGT, load_model
    dev = torch.device("cuda", int(device))
    with torch.cuda.device(dev):
        if checkpoint:
            m = load_model(checkpoint, precision=precision)      # built on the current device (= dev inside this block)
            if m.device.index is None:
                m.device = dev
        else:
            cfg = json.loads(config_json) if config_json else {}
            cfg.pop("model", None)
            cls = VQGAN if kind == "vqgan" else MIGT
            m = cls(precision=precision, device=dev, **cfg).init_weights(int(seed))
        want = "codebook" if kind == "vqgan" else "transformer"
        if m.config.model_type != want:
            raise ValueError(f"checkpoint holds a {m.config.model_type} model, a {want} was asked for")
    return _put(m)


# ------------------------------------------------------------------------------------------------ codebook
def vq_create(config_json, checkpoint, precision, device, seed):
    """-> handle.  ``checkpoint``: directory with config.json + Lightning .ckpt (utils/torch.py:9-17), or "" for reference initialisers
    under ``seed`` with the config given as JSON (models/config.py keys)."""
    return _build("vqgan", config_json, checkpoint, precision or "mixed", device, seed)


def vq_info(h):
    """-> (image_size, tokens_per_side, n_embed, in_channels)"""
    c = _models[h].config
    return int(c.image_size), int(c.image_size // c.stride), int(c.n_embed), int(c.in_channels)


def vq_encode(h, images_ptr, layout, n, codes_ptr, stream):
    """images with C = the model's in_channels: layout 0 = uint8 NHWC [n,S,S,C] (evaluate_transformer.py:105-110), 1 = f32 NCHW in
    [-1,1] (generate_codes.py:21-26), 2 = f32 NHWC.  codes: int64 [n,s,s] (vqgan_th.py:379-383 ``[-1]``)."""
    m = _models[h]
    S, s, _, C = vq_info(h)
    with torch.cuda.device(m.device), _stream(m, stream):
        if layout == 0:
            codes = m.encode_u8(_wrap(images_ptr, (n, S, S, C), "u8", m.device))
        elif layout == 1:
            codes = m.encode(_wrap(images_ptr, (n, C, S, S), "f32", m.device))[2]
        elif layout == 2:
            codes = m.encode_nhwc(_wrap(images_ptr, (n, S, S, C), "f32", m.device))[2]
        else:
            raise ValueError("layout must be 0 (u8 NHWC), 1 (f32 NCHW) or 2 (f32 NHWC)")
        _wrap(codes_ptr, (n, s, s), "i64", m.device).copy_(codes.reshape(n, s, s))
    return 0


def vq_decode_code(h, codes_ptr, n, images_ptr, layout, stream):
    """codes int64 [n,s,s] -> images with C = the model's out_ch in the given layout (vqgan_th.py:390-393; layout 0 applies
    evaluate_transformer.py:127-129)."""
    m = _models[h]
    S, s, _, _ = vq_info(h)
    C = int(m.config.out_ch)
    with torch.cuda.device(m.device), _stream(m, stream):
        codes = _wrap(codes_ptr, (n, s, s), "i64", m.device)
        if layout == 0:
            _wrap(images_ptr, (n, S, S, C), "u8", m.device).copy_(m.decode_code_u8(codes))
        elif layout == 1:
            _wrap(images_ptr, (n, C, S, S), "f32", m.device).copy_(m.decode_code(codes))
        elif layout == 2:
            _wrap(images_ptr, (n, S, S, C), "f32", m.device).copy_(m.decode_code_nhwc(codes))
        else:
            raise ValueError("layout must be 0 (u8 NHWC), 1 (f32 NCHW) or 2 (f32 NHWC)")
    return 0


# ------------------------------------------------------------------------------------------------ transformer
def migt_create(config_json, checkpoint, precision, device, seed):
    return _build("migt", config_json, checkpoint, precision or "bf16", device, seed)


def migt_info(h):
    """-> (tokens_per_side, n_embeddings, mask_token, use_localization)"""
    m = _models[h]
    return int(m.token_image_size), int(m.config.n_embeddings), int(m.mask_token), int(bool(m.use_localization))


def migt_forward(h, ids_ptr, poses_ptr, B, T, codes_last_ptr, logits_last_ptr, stream):
    """MIGT.call (migt.py:338-455), single stream: input_ids int32 [B,T,s,s] (the caller puts mask tokens where views are to be
    generated), poses f32 [B,T,7] (relative / normalised).  Outputs for the LAST view (what evaluate_transformer.py:122-123 consumes):
    argmax codes int64 [B,s,s] and, if the pointer is non-null, logits f32 [B,s,s,n_embeddings]."""
    m = _models[h]
    s, V, _, _ = migt_info(h)
    with torch.cuda.device(m.device), _stream(m, stream):
        ids = _wrap(ids_ptr, (B, T, s, s), "i32", m.device)
        poses = _wrap(poses_ptr, (B, T, 7), "f32", m.device)
        from . import _lib as L
        logits = m({"input_ids": ids, "poses": poses}, last_only=True)["logits"].reshape(B * s * s, V)
        _wrap(codes_last_ptr, (B, s, s), "i64", m.device).copy_(L.argmax_rows(logits).reshape(B, s, s))
        if logits_last_ptr:
            _wrap(logits_last_ptr, (B, s, s, V), "f32", m.device).copy_(logits.reshape(B, s, s, V))
    return 0


def migt_prefill_context(h, ids_ptr, poses_ptr, B, Tc, stream):
    """Context pass kept as a KV cache (BASELINE configs[4]); -> cache handle."""
    m = _models[h]
    s = m.token_image_size
    with torch.cuda.device(m.device), _stream(m, stream):
        cache = m.prefill_context(_wrap(ids_ptr, (B, Tc, s, s), "i32", m.device), _wrap(poses_ptr, (B, Tc, 7), "f32", m.device))
    return _put(dict(cache=cache, model=h, device=m.device))


def migt_query(h, cache_h, poses_ptr, Nq, codes_ptr, stream):
    """One query view per pose against the cached context: codes int64 [Nq,s,s]."""
    m = _models[h]
    c = _models[cache_h]
    if c["model"] != h:
        raise ValueError("the cache was built by another model")
    s = m.token_image_size
    with torch.cuda.device(m.device), _stream(m, stream):
        codes = m.query(c["cache"], _wrap(poses_ptr, (Nq, 7), "f32", m.device))
        _wrap(codes_ptr, (Nq, s, s), "i64", m.device).copy_(codes)
    return 0


def generate(h_migt, h_vq, images_ptr, cameras_ptr, B, T, out_images_ptr, out_cameras_ptr, stream):
    """generate_batch_predictions (evaluate_transformer.py:97-146): images uint8 [B,T,S,S,in_channels], cameras f32 [B,T,7] ->
    generated_images uint8 [B,S,S,out_ch] (+ generated_cameras f32 [B,7] if the pointer is non-null and the model localises)."""
    tr, vq = _models[h_migt], _models[h_vq]
    S, _, _, C = vq_info(h_vq)
    C_out = int(vq.config.out_ch)
    from .generate import generate_batch_predictions
    with torch.cuda.device(vq.device), _stream(vq, stream):
        out = generate_batch_predictions(tr, vq, _wrap(images_ptr, (B, T, S, S, C), "u8", vq.device), _wrap(cameras_ptr, (B, T, 7), "f32", vq.device))
        _wrap(out_images_ptr, (B, S, S, C_out), "u8", vq.device).copy_(torch.as_tensor(out["generated_images"]).to(vq.device))
        if out_cameras_ptr:
            _wrap(out_cameras_ptr, (B, 7), "f32", vq.device).copy_(torch.as_tensor(out["generated_cameras"], dtype=torch.float32).to(vq.device))
    return 0


def destroy(h):
    _models.pop(int(h), None)
    return 0

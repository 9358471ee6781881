"""Callers of the hot path that the reference keeps under viewformer/evaluate/ — same names, argument meaning and results:

    transformer_predict   evaluate_transformer_multictx_allimg.py:15-48   3-stream call: per context size, the query view and its pose
    run_with_batchsize    evaluate_transformer_multictx_allimg.py:51-62
    encode_images / decode_code   :65-80  uint8 frames -> codes (with the dataset resize rule), codes -> uint8 images
    generate_codebook_predictions   evaluate_codebook.py:66-76 (its ``generate_batch_predictions``): the codebook's encode -> decode round trip
                                    (BASELINE.json configs[0])
"""
import torch

from . import _lib as L
from .generate import reduce_cameras, resize_images
from .vqgan import image_tensor


def transformer_predict(cameras, codes, *, transformer_model):
    """cameras f32 [B,T,7], codes int [B,T,h,w] -> (generated_cameras [B,T,7] | None, generated_codes int64 [B,T,h,w])."""
    dev = transformer_model.device
    cameras = torch.as_tensor(cameras, dtype=torch.float32).to(dev).contiguous()
    codes = torch.as_tensor(codes).to(dev)
    relative = transformer_model.config.augment_poses == "relative"
    cams, transform = L.cameras_prepare(cameras, relative)                             # to_relative_cameras + normalize_cameras
    B, T = codes.shape[:2]
    mask = torch.full_like(codes[:, :1], transformer_model.mask_token)
    input_ids = torch.cat([codes[:, :-1], mask], 1)
    context_cameras = torch.cat([cams[:, :-1], torch.zeros_like(cams[:, :1])], 1)
    inputs = dict(input_ids=input_ids, poses=context_cameras, output_poses=cams[:, -1:].repeat(1, T, 1).contiguous())
    if transformer_model.use_localization:
        inputs["localization_tokens"] = codes[:, -1:].repeat(1, T, 1, 1).contiguous()
    out = transformer_model(inputs, training=False)
    logits = out["logits"]
    gen_codes = L.argmax_rows(logits.reshape(-1, logits.shape[-1])).reshape(codes.shape)
    gen_cams = None
    if "pose_prediction" in out:
        gen_cams = reduce_cameras(out["pose_prediction"], -2)
        if relative:
            gen_cams = L.cameras_from_relative(gen_cams.to(dev).contiguous(), transform)
    return gen_cams, gen_codes


def run_with_batchsize(fn, batch_size, *args, **kwargs):
    total = len(args[0])
    outs = [fn(*[x[i:i + batch_size] for x in args], **kwargs) for i in range(0, total, batch_size)]
    if torch.is_tensor(outs[0]):
        return torch.cat(outs, 0)
    return tuple(torch.cat([o[i] for o in outs], 0) if outs[0][i] is not None else None for i in range(len(outs[0])))


def encode_images(frames, *, codebook_model):
    """frames [..., H, W, C], uint8 or float32 in [0, 1] -> codes int64 [..., h, w]; frames are resized with the dataset rule
    (data/_common.py:19-44).  Any other dtype raises TypeError."""
    frames = image_tensor(frames, "encode_images")
    lead = frames.shape[:-3]
    x = frames.reshape((-1,) + tuple(frames.shape[-3:])).to(codebook_model.device).contiguous()
    x = resize_images(x, codebook_model.config.image_size)
    codes = codebook_model.encode_images(x)
    return codes.reshape(tuple(lead) + tuple(codes.shape[-2:]))


def decode_code(codes, *, codebook_model):
    """codes [..., h, w] -> uint8 images [..., H, W, out_ch] (clip, /2 + 0.5, saturate-cast; evaluate_transformer.py:127-129)."""
    codes = torch.as_tensor(codes)
    lead = codes.shape[:-2]
    img = codebook_model.decode_code_u8(codes.reshape((-1,) + tuple(codes.shape[-2:])))
    return img.reshape(tuple(lead) + tuple(img.shape[-3:]))


def generate_codebook_predictions(codebook_model, images):
    """evaluate/evaluate_codebook.py:66-76: uint8 images [N,H,W,3] -> resize to the codebook's size -> encode -> decode_code -> clip ->
    uint8; returns dict(ground_truth_images = the inputs as given, generated_images uint8 [N,S,S,3], codes int64 [N,h,w])."""
    images = torch.as_tensor(images)
    codes = encode_images(images, codebook_model=codebook_model)
    return dict(ground_truth_images=images, generated_images=decode_code(codes, codebook_model=codebook_model), codes=codes)


"""Four-channel frames on the host: decode_frames keeps the stored channels (tf.io.decode_image does), LatentCodeTransformer checks them
against the codebook, and images of any dtype other than uint8 / float32 are refused instead of cast."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from viewformer_b200 import data as D
from viewformer_b200.config import VQGANConfig


def _encoded(arr, fmt):
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, format=fmt)
    return buf.getvalue()


def test_decode_frames_keeps_stored_channels():
    g = np.random.default_rng(0)
    rgba = g.integers(0, 256, (2, 16, 12, 4), dtype=np.uint8)
    rgb = g.integers(0, 256, (2, 16, 12, 3), dtype=np.uint8)
    for frames, fmt in ((rgba, "PNG"), (rgb, "JPEG"), (rgb, "PNG")):
        blobs = [_encoded(f, fmt) for f in frames]
        got = D.decode_frames(blobs)
        want = np.stack([np.array(Image.open(io.BytesIO(b))) for b in blobs])
        assert got.dtype == np.uint8 and got.shape == want.shape == frames.shape[:3] + (frames.shape[-1],)
        assert np.array_equal(got, want)
    assert np.array_equal(D.decode_frames([_encoded(f, "PNG") for f in rgba]), rgba)        # PNG is lossless: the alpha channel survives


class _Codebook:
    """Stands in for a 4-channel VQGAN: "codes" are the top-left pixels of the first and the last channel."""
    config = VQGANConfig(image_size=8, ch_mult=[1, 1, 2], in_channels=4, out_ch=4, batch_size=3)
    device = "cpu"

    def __init__(self):
        self.seen = []

    def encode_u8(self, x):
        self.seen.append(tuple(x.shape))
        return torch.stack([x[:, :2, :2, 0], x[:, :2, :2, 3]], 1).to(torch.int64)


@pytest.fixture
def no_resize(monkeypatch):
    import viewformer_b200._lib as L
    monkeypatch.setattr(L, "resize_u8", lambda x, size, method=None: x)          # frames already have the codebook's size


def test_latent_code_transformer_keeps_four_channels(no_resize):
    cb = _Codebook()
    tr = D.LatentCodeTransformer(cb, batch_size=3)
    scenes = []
    for i, t in enumerate([2, 3]):
        fr = np.zeros((t, 8, 8, 4), np.uint8)
        fr[..., 3] = 100 + i
        scenes.append(dict(frames=fr, cameras=np.zeros((t, 7), np.float32)))
    out = list(tr("train", iter(scenes)))
    assert [len(o["codes"]) for o in out] == [2, 3]
    assert all(s[-1] == 4 for s in cb.seen)
    assert (out[0]["codes"][:, 1] == 100).all() and (out[1]["codes"][:, 1] == 101).all()


def test_latent_code_transformer_rejects_channel_mismatch(no_resize):
    tr = D.LatentCodeTransformer(_Codebook(), batch_size=3)
    scene = dict(frames=np.zeros((2, 8, 8, 3), np.uint8), cameras=np.zeros((2, 7), np.float32))
    with pytest.raises(ValueError, match="4-channel"):
        list(tr("train", iter([scene])))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.int32])
def test_encode_u8_refuses_to_cast(dtype):
    """A float image in [0, 1] cast to uint8 would be encoded as 0 / 1 bytes: encode_u8 raises before touching the device."""
    from viewformer_b200 import VQGAN
    model = VQGAN(VQGANConfig(in_channels=4, out_ch=4), precision="fp32")
    with pytest.raises(TypeError, match="not cast"):
        model.encode_u8(torch.full((1, 128, 128, 4), 0.5, dtype=dtype))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float16, torch.int64])
def test_float_entry_points_refuse_other_dtypes(dtype):
    from viewformer_b200 import VQGAN, generate_batch_predictions
    from viewformer_b200.evaluate import encode_images
    model = VQGAN(VQGANConfig(in_channels=4, out_ch=4), precision="fp32")
    images = torch.zeros((1, 2, 128, 128, 4), dtype=dtype)
    with pytest.raises(TypeError, match="uint8 or float32"):
        model.encode_images(images[0])
    with pytest.raises(TypeError, match="uint8 or float32"):
        encode_images(images, codebook_model=model)

    class _Transformer:
        device = torch.device("cpu")

        class config:
            augment_poses = "none"
    with pytest.raises(TypeError, match="uint8 or float32"):
        generate_batch_predictions(_Transformer(), model, images, torch.zeros((1, 2, 7)))

"""The evaluation paths are batch-invariant, bit for bit: every scene's result does not depend on which other scenes share its batch.

The launch audit (tests/test_launch_audit_gpu.py) holds these paths to fp64 bars on three sampled batch entries per launch; the checks
here cover every entry.  Bit-identity is the right bar, because no kernel on these paths changes its reduction order with the batch:
  - tc_gemm / simt_gemm: no split-K; an output element is one K-chain fixed by K and the tile width, and the tile width depends on N
    only (vf_tc_gemm: block_n from Ncols); the persistent walk only changes which CTA computes a tile.
  - attn_block_causal / attn_block_multiend: one work item per (query tile, batch, head), keys never split across CTAs (attn_launch).
  - layernorm, softmax_rows, argmax_rows, migt_embed, pose_postprocess, cameras_prepare / cameras_from_relative: one row, token or
    scene per warp or thread.
The one exception is reduce_cameras (generate.py), the reference's camera reduction restated as torch ops on the device: torch's
reduction kernels pick their launch configuration (threads per output, values per thread, vectorisation) from the number of outputs, so
the per-view quaternion norm and mean over 64 tokens can round differently when the batch holds more scenes (1 ulp on an H100).  There
the test holds the pose predictions that feed it bit for bit, and each batch size's reduced cameras to the fp64 bar of that reduction.
"""
import pytest
import torch

from oracle import synth, migt_oracle as mo
from viewformer_b200.config import MIGTConfig

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


@pytest.fixture(scope="module")
def scenes(lib):
    return synth.make_cameras(5, 10, seed=7100), synth.make_codes(5, 10, seed=7101)


U = 2.0 ** -24


def _reduce_bar(pp, got):
    """|got - reduce_cameras in fp64| / bar for pose predictions pp [B, T, 64, 7]: xyz a mean of n fp32 values, 2 (n + 1) u mean|x|; the
    quaternion normalised per token (a 4-term sum and rsqrt, 8 u), averaged (2 (n + 1) u mean|q|) and normalised again, which divides the
    error by the mean's norm: (2 (n + 8) u mean|q| / |mean q| + 8 u) per component."""
    from viewformer_b200.generate import reduce_cameras
    n = pp.shape[-2]
    x = pp.double()
    ref = reduce_cameras(x, -2)
    qn = x[..., 3:] / x[..., 3:].norm(dim=-1, keepdim=True)
    qn = qn * torch.where(qn[..., :1] >= 0, 1.0, -1.0)
    qm = qn.mean(-2).norm(dim=-1, keepdim=True)
    bar = torch.cat([2 * (n + 1) * U * x[..., :3].abs().mean(-2),
                     2 * (n + 8) * U * qn.abs().mean(-2) / qm + 8 * U], -1)
    return float(((got.double() - ref).abs() / bar).max())


@pytest.mark.parametrize("localization_weight", ["1", "0"])
def test_transformer_predict_batch_invariant(scenes, monkeypatch, localization_weight):
    """run_with_batchsize(transformer_predict, b, ...) over 5 scenes x 10 views at b = 1, 2 and 5 (batches 5; 2, 2, 1; 1 x 5): the codes
    and, with localisation, the pose predictions are bit-identical; the cameras reduced from them are within the fp64 bar of the
    reduction, and bit-identical wherever the reduction rounded alike.  3 streams with localisation, 2 without (attn_block_multiend)."""
    from viewformer_b200 import MIGT
    from viewformer_b200 import evaluate
    from viewformer_b200.evaluate import run_with_batchsize, transformer_predict
    cfg = MIGTConfig(localization_weight=localization_weight)
    tr = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 15))
    cams, codes = scenes
    seen = []
    reduce = evaluate.reduce_cameras

    def recording(x, axis=-2):
        y = reduce(x, axis)
        seen.append((x.clone(), y.clone()))
        return y
    monkeypatch.setattr(evaluate, "reduce_cameras", recording)
    out, pp, red = {}, {}, {}
    for b in (5, 2, 1):
        seen.clear()
        out[b] = run_with_batchsize(transformer_predict, b, cams, codes, transformer_model=tr)
        if seen:
            pp[b], red[b] = torch.cat([x for x, _ in seen]), torch.cat([y for _, y in seen])
    torch.cuda.synchronize()
    cams5, codes5 = out[5]
    assert codes5.shape == codes.shape and (cams5 is None) == (localization_weight == "0") and bool(pp) == (cams5 is not None)
    for b in (2, 1):
        cb, kb = out[b]
        diff = (kb != codes5).sum().item()
        print(f"[allimg loc={localization_weight}] batch {b} vs 5: {diff} of {codes5.numel()} codes differ")
        assert diff == 0, f"batch size {b}: {diff} codes differ from the batch of 5"
        if cams5 is None:
            continue
        assert torch.equal(_bits(pp[b]), _bits(pp[5])), f"batch size {b}: pose predictions differ from the batch of 5"
        r = _reduce_bar(pp[5], red[b])
        alike = (_bits(red[b]) == _bits(red[5])).flatten(1).all(1)
        print(f"[allimg loc={localization_weight}] batch {b} vs 5: reduce_cameras within {r:.3g} of its fp64 bar, "
              f"{int(alike.sum())} of {alike.numel()} scenes bit-identical; cameras max |diff| {(cb - cams5).abs().max().item():.3g}")
        assert r <= 1.0, f"batch size {b}: reduced cameras at {r:.3g} of the fp64 bar"
        assert torch.equal(_bits(cb[alike]), _bits(cams5[alike])), f"batch size {b}: cameras differ where the reduction agrees"
    if cams5 is not None:
        assert _reduce_bar(pp[5], red[5]) <= 1.0


def test_shared_scene_query_subsets(lib):
    """MIGT.query on a one-scene cache (stride-0 cache batch, _query_block) with 8 poses, and with 3 and 5 of them: every query's logits
    are bit-identical across the three calls."""
    from viewformer_b200 import MIGT
    cfg = MIGTConfig(localization_weight="0")
    model = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 16))
    codes = synth.make_codes(1, 19, seed=7200)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(1, 27, seed=7201))[0])
    cache = model.prefill_context(codes, cams[:, :19].contiguous())
    poses = cams[0, 19:].contiguous()
    codes8, logits8 = model.query(cache, poses, return_logits=True)
    for idx in ([0, 3, 7], [1, 2, 4, 5, 6]):
        codes_s, logits_s = model.query(cache, poses[idx].contiguous(), return_logits=True)
        torch.cuda.synchronize()
        want = logits8[idx]
        print(f"[shared query] subset {idx}: max |logit diff| {(logits_s - want).abs().max().item():.3g}")
        assert torch.equal(_bits(logits_s), _bits(want)), f"queries {idx}: logits depend on the other queries of the call"
        assert torch.equal(codes_s, codes8[idx])

"""7-Scenes localisation on the GPU: the nearest-camera kernel (vf_camera_knn) against fp64, and the procedures of viewformer_b200.sevenscenes
against the reference's, recorded in tests/golden/sevenscenes_reference_shim.npz (tests/test_sevenscenes_host.py reproduces that file
with the reference's own code).  Transformer fp32, codebook mixed (fp32-faithful encoder, bf16 decoder)."""
import os
import random

import numpy as np
import pytest
import torch

import launch_checks_cameras as lc
from oracle import synth
from oracle import make_golden_sevenscenes as mg
from viewformer_b200.cameras import camera_knn
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu

CAMERA_ATOL = 1e-3                    # generated cameras against the reference's (tests/test_models_gpu.py's bar)


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sevenscenes_reference_shim.npz"))


@pytest.fixture(scope="module")
def models(L):
    from viewformer_b200 import VQGAN, MIGT
    vcfg, tcfg = VQGANConfig(**mg.SEVENSCENES_VQ), MIGTConfig(**mg.SEVENSCENES_MIGT)
    vq = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, mg.VQ_SEED))
    tr = MIGT(tcfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(tcfg, mg.MIGT_SEED))
    return tr, vq


def _cams(n, g, lead=()):
    q = torch.nn.functional.normalize(torch.randn(lead + (n, 4), generator=g), dim=-1)
    return torch.cat([torch.randn(lead + (n, 3), generator=g) * 2, q], -1).contiguous()


# ----------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("mode", ["combined", "position", "orientation"])
@pytest.mark.parametrize("n,q,k,shared", [(1000, 5, 9, True), (7000, 3, 64, True), (300, 4, 1, False), (777, 6, 9, False),
                                          (9001, 2, 64, True), (64, 3, 64, False)])
def test_camera_knn_vs_fp64(L, mode, n, q, k, shared):
    """Shared and per-query databases, N not a multiple of the 256-thread block, N above the 8192 keys kept in shared memory (9001: the
    rest are recomputed each round), k = 1, 9, 64 and k = N."""
    g = torch.Generator().manual_seed(n + q + k)
    db = _cams(n, g, () if shared else (q,))
    qs = _cams(q, g)
    (idx, dist), r = lc.run_check("camera_knn", camera_knn, (db.cuda(), qs.cuda(), k, mode), {}, random.Random(0))
    print(f"[camera_knn {mode} N {n} Q {q} k {k} shared {shared}] worst ratio to the fp64 bar {r:.3g}")
    assert r <= 1.0 and idx.shape == (q, k) and dist.shape == (q, k)


def test_camera_knn_duplicates_own_pose_and_half_turn(L):
    """Exact duplicates come lower index first; the query's own pose is nearest (distance 0 up to rounding); a pose a half turn away
    has the finite distance pi, where the reference's unclamped asin can give NaN."""
    g = torch.Generator().manual_seed(5)
    db = _cams(500, g)
    db[300] = db[40]
    db[41] = db[40]
    qs = torch.stack([db[40], _cams(1, g)[0]])
    w, x, y, z = qs[1, 3:].tolist()
    db[7] = torch.cat([qs[1, :3], torch.tensor([-x, w, -z, y]) * 1.7])          # orthogonal and not unit: |vec| rounds near 1
    for mode in ("combined", "position", "orientation"):
        (idx, dist), r = lc.run_check("camera_knn", camera_knn, (db.cuda(), qs.cuda(), 64, mode), {}, random.Random(0))
        assert r <= 1.0
        assert idx[0, :3].tolist() == [40, 41, 300] and float(dist[0, 0]) < 1e-6, mode
        assert bool(torch.isfinite(dist).all())
    idx, dist = camera_knn(db[7:8].contiguous().cuda(), qs[1:].contiguous().cuda(), 1, "orientation")
    assert abs(float(dist[0, 0]) - np.pi) < 1e-5


def test_camera_knn_rejects_bad_arguments(L):
    db, qs = torch.zeros(10, 7, device="cuda"), torch.zeros(2, 7, device="cuda")
    db[:, 3] = 1
    for k in (0, 11, 65):
        with pytest.raises(L.LibraryError, match="k"):
            camera_knn(db, qs, k)
    with pytest.raises(L.LibraryError, match="mode"):
        L._check(L.load().vf_camera_knn(db, 10, 0, qs, 2, 3, 1, torch.empty(2, dtype=torch.int32, device="cuda"), torch.empty(2, device="cuda"),
                                        L._stream()))
    with pytest.raises(L.LibraryError, match="db_stride"):
        L._check(L.load().vf_camera_knn(db, 10, 35, qs, 2, 0, 1, torch.empty(2, dtype=torch.int32, device="cuda"), torch.empty(2, device="cuda"),
                                        L._stream()))
    with pytest.raises(ValueError):
        camera_knn(torch.zeros(3, 10, 7, device="cuda"), qs, 1)


def test_compute_camera_distances_in_database_order(L):
    from viewformer_b200.sevenscenes import compute_camera_distances
    g = torch.Generator().manual_seed(6)
    db, q = _cams(1000, g), _cams(1, g)
    for mode in ("combined", "position", "orientation"):
        d64, bar = lc.camera_distances64(db, q, mode)
        got = compute_camera_distances(db, q, mode).cpu().double()
        assert got.shape == (1000,) and bool(((got - d64[0]).abs() <= bar[0]).all()), mode


# ----------------------------------------------------------------------------------------------- the procedures against the reference
def _compare(tag, got, g, prefix):
    codes = got["generated_codes"].cpu().reshape(-1)
    want, margin = torch.from_numpy(g[f"{prefix}.codes"]).reshape(-1), torch.from_numpy(g[f"{prefix}.margins"]).reshape(-1)
    sure = margin > mg.MARGIN_BAR
    print(f"[{tag}] codes equal {int((codes == want).sum())}/{codes.numel()}, above the margin bar {int(sure.sum())}; "
          f"camera max |diff| {float((got['generated_cameras'].cpu() - torch.from_numpy(g[f'{prefix}.generated_cameras'])).abs().max()):.3g}")
    assert torch.equal(codes[sure], want[sure])
    assert torch.allclose(got["generated_cameras"].cpu().float(), torch.from_numpy(g[f"{prefix}.generated_cameras"]), atol=CAMERA_ATOL)
    img, ref = got["generated_images"].cpu().int(), torch.from_numpy(g[f"{prefix}.generated_images"]).int()
    assert img.shape == ref.shape and img.dtype == torch.int32
    if torch.equal(codes, want):                     # the same codes through the bf16 decoder: test_rgba_gpu.py's mixed pixel bars
        d = (img - ref).abs().float()
        print(f"[{tag}] u8 pixel diff max {int(d.max())} mean {float(d.mean()):.3f}")
        assert float(d.max()) <= 0.15 * 127.5 and float(d.mean()) <= 0.02 * 127.5


def test_pose_refinement_matches_the_reference(models, golden):
    from viewformer_b200 import generate_batch_predictions_using_pose_refinement
    tr, vq = models
    images, cams = mg.query_batch(int(golden["query_seed"]))
    lookup = mg.RecordingLookup(*mg.scene(int(golden["pr.db_seed"])))
    got = generate_batch_predictions_using_pose_refinement(lookup, lookup.cameras, tr, vq, images, cams,
                                                           num_gen_ctx=int(golden["pr.num_gen_ctx"]),
                                                           rng=random.Random(int(golden["pr.rng_seed"])))
    assert lookup.asked == [str(x) for x in golden["pr.files"]]               # the selected database frames, then the sampled ones
    assert torch.equal(got["ground_truth_cameras"].cpu(), torch.from_numpy(golden["pr.ground_truth_cameras"]))
    _compare("pose_refinement", got, golden, "pr")


def test_generated_images_matches_the_reference(models, golden):
    from viewformer_b200 import generate_batch_predictions_using_generated_images
    tr, vq = models
    images, cams = mg.query_batch(int(golden["query_seed"]))
    got = generate_batch_predictions_using_generated_images(tr, vq, images, cams, num_gen_ctx=int(golden["gi.num_gen_ctx"]),
                                                            generator=torch.Generator().manual_seed(int(golden["gi.seed"])))
    assert torch.equal(got["ground_truth_images"], images[:, -1])
    _compare("generated_images", got, golden, "gi")


def test_pose_refinement_batch_equals_single_rows(models, golden):
    """B = 4 against four B = 1 calls, the rng drawn row after row in both: the same database frames asked in the same order, the same
    codes and views; cameras within 1e-6 (reduce_cameras' torch reductions may round 1 ulp apart between batch sizes, see
    tests/test_eval_paths_gpu.py)."""
    from viewformer_b200 import generate_batch_predictions_using_pose_refinement as pr
    tr, vq = models
    images, cams = mg.query_batch(8100, B=4)
    files, dbc, frames = mg.scene(int(golden["pr.db_seed"]))
    lb = mg.RecordingLookup(files, dbc, frames)
    batch = pr(lb, dbc, tr, vq, images, cams, num_gen_ctx=9, rng=random.Random(3))
    ls = mg.RecordingLookup(files, dbc, frames)
    rng = random.Random(3)
    rows = [pr(ls, dbc, tr, vq, images[b:b + 1], cams[b:b + 1], num_gen_ctx=9, rng=rng) for b in range(4)]
    assert lb.asked == ls.asked and len(lb.asked) == 4 * 19
    for k in ("generated_codes", "generated_images", "ground_truth_images", "ground_truth_cameras"):
        assert torch.equal(batch[k].cpu(), torch.cat([r[k].cpu() for r in rows])), k
    assert torch.allclose(batch["generated_cameras"].cpu(), torch.cat([r["generated_cameras"].cpu() for r in rows]), atol=1e-6, rtol=0)


def test_baselines_match_the_reference(L, golden):
    from viewformer_b200 import generate_batch_predictions_baseline, BaselineEvaluator
    cams = torch.from_numpy(golden["bl.cameras"])
    for name in ("position_oracle", "orientation_oracle"):
        out = generate_batch_predictions_baseline(cams, name)
        assert torch.equal(out["generated_cameras"].cpu(), torch.from_numpy(golden[f"bl.{name}"])), name
        assert torch.equal(out["ground_truth_cameras"], cams[:, -1])
        ev = BaselineEvaluator()
        ev.update_state(**out)
        assert set(ev.result()) == {"loc-angle", "loc-dist", "loc-angle-med", "loc-dist-med"}
        assert list(ev.get_progress_bar_info()) == ["cam_loc", "cam_ang"]

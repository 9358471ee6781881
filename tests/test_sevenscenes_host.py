"""7-Scenes localisation on the CPU: the reference's procedures over oracle/tf_shim.py reproduce tests/golden/sevenscenes_reference_shim.npz
(what tests/test_sevenscenes_gpu.py holds the GPU procedures to), the random draws and the database call order the GPU procedures make are
the reference's, and the nearest-camera checker of tests/launch_checks_cameras.py accepts the fp64 answer and rejects wrong ones."""
import os
import random

import numpy as np
import pytest
import torch

import launch_checks_cameras as lc
from oracle import ref_loader, ref_loader_sevenscenes
from oracle import make_golden_sevenscenes as mg
from viewformer_b200 import sevenscenes as S


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sevenscenes_reference_shim.npz"))


@pytest.fixture(scope="module")
def ref():
    if not ref_loader.migt_available():
        pytest.skip("reference sources not present")
    from oracle import tf_shim
    tf_shim.install()
    s7, bl = ref_loader_sevenscenes.load_reference_sevenscenes()
    yield s7, bl
    tf_shim.uninstall()


def _np(x):
    return torch.as_tensor(x).as_subclass(torch.Tensor).numpy()


# ----------------------------------------------------------------------------------------------- the reference reproduces the fixture
def test_reference_reproduces_the_fixture(ref, golden):
    """The three procedures run again from the recorded seeds: the same database files, the same picks, the same outputs bit for bit."""
    s7, bl = ref
    model, codebook = mg.models()
    images, cams = mg.query_batch(int(golden["query_seed"]))
    lookup = mg.RecordingLookup(*mg.scene(int(golden["pr.db_seed"])))
    random.seed(int(golden["pr.rng_seed"]))
    with torch.no_grad():
        r = s7.generate_batch_predictions_using_pose_refinement(lookup, torch.as_tensor(lookup.cameras), model, codebook, images.clone(),
                                                                cams.clone(), num_gen_ctx=int(golden["pr.num_gen_ctx"]))
    assert lookup.asked == [str(x) for x in golden["pr.files"]]
    assert lookup.asked[:9] == [lookup.files[i] for i in golden["pr.selected"]]
    assert np.array_equal(_np(r["generated_images"]), golden["pr.generated_images"])
    assert np.array_equal(_np(r["generated_cameras"]), golden["pr.generated_cameras"])
    d = _np(s7.compute_camera_distances(torch.as_tensor(lookup.cameras), torch.as_tensor(golden["pr.estimate"])))
    assert np.array_equal(d, golden["pr.distances"])
    torch.manual_seed(int(golden["gi.seed"]))
    with torch.no_grad():
        r = s7.generate_batch_predictions_using_generated_images(model, codebook, images.clone(), cams.clone(),
                                                                 num_gen_ctx=int(golden["gi.num_gen_ctx"]))
    assert np.array_equal(_np(r["generated_images"]), golden["gi.generated_images"])
    assert np.array_equal(_np(r["generated_cameras"]), golden["gi.generated_cameras"])
    bc = torch.from_numpy(golden["bl.cameras"])
    for name in ("position_oracle", "orientation_oracle"):
        got = np.concatenate([_np(bl.generate_batch_predictions_baseline(bc[b:b + 1].clone(), name)["generated_cameras"]) for b in range(4)])
        assert np.array_equal(got, golden[f"bl.{name}"])


def test_fixture_selection_is_separated(golden):
    """The nearest-camera picks of the fixture do not hang on near ties: every gap among the first k + 1 sorted distances is above
    SELECTION_GAP, and the picks are the stable argsort of the recorded distances."""
    k = int(golden["pr.num_gen_ctx"])
    assert golden["pr.gaps"].shape == (k,) and float(golden["pr.gaps"].min()) > mg.SELECTION_GAP
    assert np.array_equal(np.argsort(golden["pr.distances"], kind="stable")[:k], golden["pr.selected"])
    assert float(golden["gi.context_margins"].min()) > mg.MARGIN_BAR


# ----------------------------------------------------------------------------------------------- draws and call order
def test_recorded_draws_are_torch_rand_under_the_seed(golden):
    """The four tf.random.uniform draws of generate_other_viewpoints, recorded from the reference under torch.manual_seed(seed), are
    torch.rand on a CPU generator seeded alike, as u (hi - lo) + lo, bit for bit; generate_other_viewpoints(generator=...) consumes them
    in that order: its result is the reference's formula over the recorded draws."""
    n = int(golden["gi.num_gen_ctx"])
    draws = [torch.from_numpy(golden[f"gi.draw{i}"]) for i in range(4)]
    assert [tuple(d.shape) for d in draws] == [(n, 1, 3), (n, 1, 3), (n, 1, 1), (n, 1, 1)]
    g = torch.Generator().manual_seed(int(golden["gi.seed"]))
    for d, (lo, hi) in zip(draws, ((-1, 1), (-1, 1), (0, 1.), (0, 0.3))):
        assert torch.equal(torch.rand(d.shape, generator=g) * (hi - lo) + lo, d)
    cam = torch.tensor([[0.3, -1.2, 2.0, 0.8, -0.1, 0.5, 0.3]]).repeat(n, 1)[:, None]
    got = S.generate_other_viewpoints(cam, torch.Generator().manual_seed(int(golden["gi.seed"])))
    off = S._l2_normalize_all(draws[0]) * draws[2]
    axis = S._l2_normalize_all(draws[1])
    rot = torch.cat((torch.cos(draws[3] / 2), torch.sin(draws[3] / 2) * axis), -1)
    want = torch.cat((off + cam[..., :3], S.quaternion_normalize(S.quaternion_multiply(rot, cam[..., 3:]))), -1)
    assert torch.equal(got, want)
    assert abs(float(axis.norm()) - 1.0) < 1e-6 and n > 1 and float(axis[0].norm()) < 0.9    # one norm for all n axes: not unit each


def test_generate_other_viewpoints_equals_the_reference(ref):
    s7, _ = ref
    cam = torch.tensor([[[0.3, -1.2, 2.0, 0.8, -0.1, 0.5, 0.3]], [[1.0, 0.0, -0.5, 0.1, 0.9, -0.2, 0.4]]]).repeat(3, 1, 1)
    for seed in (0, 5, 123):
        torch.manual_seed(seed)
        want = _np(s7.generate_other_viewpoints(cam.clone()))
        got = S.generate_other_viewpoints(cam, torch.Generator().manual_seed(seed)).numpy()
        assert np.array_equal(got, want), seed


def test_pose_refinement_lookup_and_rng_call_order(golden, monkeypatch):
    """With the device steps replaced by stand-ins that return the fixture's picks, the procedure asks the lookup for the reference's
    names in the reference's order, draws the rest with rng.sample(files, 19 - k) after the picks, and row by row for B > 1."""
    k = int(golden["pr.num_gen_ctx"])
    sel = torch.from_numpy(golden["pr.selected"]).to(torch.int32)
    images, cams = mg.query_batch(int(golden["query_seed"]))
    calls = []

    class Model:
        device = torch.device("cpu")
        config = type("C", (), {"augment_poses": "no"})

    monkeypatch.setattr(S, "_prepare", lambda tm, cm, im, ca: (im, ca, ca, None, False, None))
    monkeypatch.setattr(S, "localize_last_view", lambda tm, codes, c: c[:, -1:])
    monkeypatch.setattr(S, "camera_knn", lambda db, q, kk, mode: (sel[None, :kk].repeat(q.shape[0], 1), None))
    monkeypatch.setattr(S, "generate_batch_predictions", lambda tm, cm, frames, cameras: calls.append((frames, cameras)) or {})

    class Rng:
        def __init__(self, seed):
            self.r, self.log = random.Random(seed), []

        def sample(self, pop, n):
            self.log.append(n)
            return self.r.sample(pop, n)
    lookup = mg.RecordingLookup(*mg.scene(int(golden["pr.db_seed"])))
    rng = Rng(int(golden["pr.rng_seed"]))
    S.generate_batch_predictions_using_pose_refinement(lookup, lookup.cameras, Model(), None, images, cams, num_gen_ctx=k, rng=rng)
    assert lookup.asked == [str(x) for x in golden["pr.files"]] and rng.log == [19 - k]
    frames, cameras = calls[0]
    assert frames.shape == (1, 20, 32, 32, 3) and torch.equal(cameras[0, -1], cams[0, -1])
    assert torch.equal(cameras[0, :k], torch.from_numpy(lookup.cameras[golden["pr.selected"]]))
    # B = 3: three rows, each its picks then its draws, in row order
    lookup3 = mg.RecordingLookup(*mg.scene(int(golden["pr.db_seed"])))
    rng3 = Rng(int(golden["pr.rng_seed"]))
    S.generate_batch_predictions_using_pose_refinement(lookup3, lookup3.cameras, Model(), None, images.repeat(3, 1, 1, 1, 1),
                                                       cams.repeat(3, 1, 1), num_gen_ctx=k, rng=rng3)
    r1 = random.Random(int(golden["pr.rng_seed"]))
    want = []
    for _ in range(3):
        want += [lookup3.files[i] for i in golden["pr.selected"]] + r1.sample(lookup3.files, 19 - k)
    assert lookup3.asked == want and rng3.log == [19 - k] * 3 and calls[1][0].shape[0] == 3


def test_scene_lookup_and_argument_checks():
    files, cams, frames = mg.scene(1)
    sl = S.SceneLookup(files, cams, frames)
    c, f = sl[files[7]]
    assert len(sl) == 300 and np.array_equal(c, cams[7]) and np.array_equal(f, frames[7]) and sl.cameras.dtype == np.float32
    with pytest.raises(ValueError):
        S.SceneLookup(files[:-1], cams, frames)
    cams2 = torch.zeros(2, 20, 7)
    with pytest.raises(ValueError, match="one scene"):
        S.generate_batch_predictions_using_generated_images(None, None, None, cams2)
    with pytest.raises(ValueError, match="num_gen_ctx"):
        S.generate_batch_predictions_using_generated_images(None, None, None, cams2[:1], num_gen_ctx=0)
    with pytest.raises(ValueError, match="mean"):
        S.generate_batch_predictions_baseline(cams2, "mean")


def test_baseline_evaluator_reports_the_reference_keys(ref):
    """BaselineEvaluator == the reference's baseline Evaluator: the same result keys and values, the same progress-bar keys."""
    _, bl = ref
    g = torch.Generator().manual_seed(3)
    gt, gen = torch.randn(6, 7, generator=g), torch.randn(6, 7, generator=g)
    mine, theirs = S.BaselineEvaluator(), bl.Evaluator()
    for i in range(0, 6, 2):
        mine.update_state(gt[i:i + 2], gen[i:i + 2])
        theirs.update_state(gt[i:i + 2].clone(), gen[i:i + 2].clone())
    a, b = mine.result(), theirs.result()
    assert list(a) == list(b) and all(abs(a[k] - b[k]) < 1e-5 * max(1.0, abs(b[k])) for k in a)
    pa, pb = mine.get_progress_bar_info(), theirs.get_progress_bar_info()
    assert list(pa) == list(pb) and all(abs(pa[k] - pb[k]) < 1e-5 for k in pa)


# ----------------------------------------------------------------------------------------------- the launch checker
def _knn64(db, q, k, mode):
    d, _ = lc.camera_distances64(db, q, mode)
    s, i = torch.sort(d, dim=1, stable=True)
    return i[:, :k].to(torch.int32), s[:, :k].float()


def _run(db, q, k, mode, result):
    return lc.check_camera_knn(dict(db=db, queries=q, k=k, mode=mode), result, None)


@pytest.mark.parametrize("mode", ["combined", "position", "orientation"])
def test_camera_knn_checker_passes_fp64_and_catches_faults(mode):
    g = torch.Generator().manual_seed(40)
    db = torch.cat([torch.randn(500, 3, generator=g), torch.nn.functional.normalize(torch.randn(500, 4, generator=g), dim=-1)], -1)
    q = torch.cat([torch.randn(3, 3, generator=g), torch.nn.functional.normalize(torch.randn(3, 4, generator=g), dim=-1)], -1)
    db[77] = db[12]                                      # an exact duplicate
    q[1] = db[12]                                        # the query's own pose: distance 0, index 12 before 77
    idx, dist = _knn64(db, q, 9, mode)
    assert _run(db, q, 9, mode, (idx, dist)) <= 1.0
    assert idx[1, 0] == 12 and idx[1, 1] == 77 and float(dist[1, 0]) < 1e-6
    bad = idx.clone()
    bad[0, [2, 3]] = bad[0, [3, 2]]                      # two picks swapped
    assert _run(db, q, 9, mode, (bad, dist)) > 1.0
    bad = idx.clone()
    bad[2, 8] = (bad[2, 8] + 1) % 500                    # the last pick off by one
    assert _run(db, q, 9, mode, (bad, dist)) > 1.0
    bad = idx.clone()
    bad[1, [0, 1]] = bad[1, [1, 0]]                      # the tie in higher-index-first order
    assert _run(db, q, 9, mode, (bad, dist)) > 1.0
    off = dist.clone()
    off[0, 4] *= 1 + 1e-4                                # a distance off by 1e-4 relative
    assert _run(db, q, 9, mode, (idx, off)) > 1.0
    assert _run(db, q, 9, mode, (idx[:, :8].contiguous(), dist[:, :8].contiguous())) > 1.0


def test_camera_knn_checker_per_query_database_and_half_turn():
    """Per-query databases [Q, N, 7]; a database camera a half turn from the query (asin's argument at 1) has distance pi."""
    g = torch.Generator().manual_seed(41)
    db = torch.cat([torch.randn(2, 70, 3, generator=g), torch.nn.functional.normalize(torch.randn(2, 70, 4, generator=g), dim=-1)], -1)
    q = db[:, 5].clone()
    w, x, y, z = q[1, 3:].tolist()
    db[1, 9, 3:] = torch.tensor([-x, w, -z, y])          # orthogonal to the query's quaternion: a half turn
    d, _ = lc.camera_distances64(db, q, "orientation")
    assert abs(float(d[1, 9]) - np.pi) < 1e-6 and bool(torch.isfinite(d).all())
    s, i = torch.sort(d, dim=1, stable=True)
    assert _run(db, q, 64, "orientation", (i[:, :64].to(torch.int32), s[:, :64].float())) <= 1.0
    assert int(i[0, 0]) == 5 and int(i[1, -1]) == 9

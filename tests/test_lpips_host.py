"""LPIPS on the host: the fp64 oracle against torchvision's VGG16, the strict weight loader, the input checks, the binding of
include/vf_b200_lpips.h, and tests/golden/lpips_reference_shim.npz reproduced by the reference's own evaluators over oracle/tf_shim.py
(skipped where the reference is absent)."""
import ast
import glob
import os
import re
import sys

import numpy as np
import pytest
import torch

from oracle import lpips_oracle as lo, ref_loader, synth
from test_abi import expected_argtype
from viewformer_b200 import lpips as LP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def lpips_header_prototypes():
    """{name: (return type, [(type, is pointer, parameter name)])} of every function include/vf_b200_lpips.h declares."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vf_b200_lpips.h")).read(), flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^(int|const char\*)\s+(vf_\w+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        parsed = []
        for prm in params.split(","):
            m = re.fullmatch(r"\s*(?:const\s+)?(\w+)\s*(\*?)\s*(\w+)\s*", prm)
            assert m, f"{name}: cannot parse parameter {prm!r}"
            parsed.append((m.group(1), bool(m.group(2)), m.group(3)))
        out[name] = (ret, parsed)
    assert len(out) == len(set(re.findall(r"\b(vf_[a-z0-9_]+)\s*\(", src))), "a declaration the prototype parser does not read"
    return out


def test_prototype_table_matches_header():
    from viewformer_b200 import _lib
    declared = lpips_header_prototypes()
    assert sorted(declared) == sorted(LP.PROTOTYPES) == ["vf_lpips_conv_in", "vf_lpips_tap", "vf_maxpool2x2_split"]
    assert not set(declared) & set(_lib.PROTOTYPES)
    for name, (ret, params) in declared.items():
        assert ret == "int", name
        got = LP.PROTOTYPES[name]
        assert len(got) == len(params), f"{name}: {len(got)} argtypes, the header declares {len(params)} parameters"
        for k, (have, prm) in enumerate(zip(got, params)):
            want = expected_argtype(name, *prm)
            assert have is want, f"{name} parameter {k} {prm}: the table has {have.__name__}, the header wants {want.__name__}"


def test_library_exports_the_entry_points(lib):
    for name in LP.PROTOTYPES:
        assert hasattr(lib, name), f"libvf_b200.so does not export {name}"


def test_call_sites_pass_each_prototypes_argument_count():
    files = (glob.glob(os.path.join(ROOT, "viewformer_b200", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "tests", "*.py"))
             + glob.glob(os.path.join(ROOT, "scripts", "*.py")))
    seen = set()
    for path in files:
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in LP.PROTOTYPES:
                name, where = node.func.attr, f"{os.path.relpath(path, ROOT)}:{node.lineno}"
                assert not node.keywords and not any(isinstance(a, ast.Starred) for a in node.args), f"{where}: {name} with keywords or *args"
                assert len(node.args) == len(LP.PROTOTYPES[name]), f"{where}: {name} takes {len(LP.PROTOTYPES[name])} arguments"
                seen.add(name)
    assert seen == set(LP.PROTOTYPES)


def test_layer_tables_agree():
    """The host's layer table, the oracle's and the loader's expected shapes describe the same 13 convs and 5 taps."""
    assert LP.CONVS == lo.CONVS and LP.TAP_CHANNELS == lo.TAP_CHANNELS and (LP.SHIFT, LP.SCALE) == (lo.SHIFT, lo.SCALE)
    vgg, lin = lo.lpips_state_dicts(0)
    assert {k: tuple(v.shape) for k, v in vgg.items()} == LP.vgg16_shapes()
    assert {k: tuple(v.shape) for k, v in lin.items()} == LP.lin_shapes()
    assert all(bool((t >= 0).all()) for t in lin.values())


# ----------------------------------------------------------------------------------------------- oracle vs torchvision
def test_oracle_taps_equal_torchvision_vgg16_slices():
    """relu1_2 ... relu5_3 of the oracle equal torchvision.models.vgg16(weights=None).features[0:4], [4:9], [9:16], [16:23], [23:30]
    loaded with the same random weights, in fp64 (an odd-sized image exercises the floor of the pools)."""
    tv = pytest.importorskip("torchvision")
    vgg, _ = lo.lpips_state_dicts(3)
    feats = tv.models.vgg16(weights=None).features.double().eval()
    feats.load_state_dict({k[len("features."):]: v for k, v in vgg.items()}, strict=True)
    with torch.no_grad():
        x = lo.scaling_layer(torch.rand((2, 3, 36, 44), generator=torch.Generator().manual_seed(1), dtype=torch.float64))
        got = lo.taps(x, vgg)
        h = x
        for k, (a, b) in enumerate(((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))):
            h = feats[a:b](h)
            assert got[k].shape == h.shape
            assert float((got[k] - h).abs().max()) <= 1e-12 * max(1.0, float(h.abs().max())), k


def test_oracle_terms_follow_the_definition():
    """Identical inputs give 0; one tap's term is the lin-weighted mean of the squared difference of unit-normalised features."""
    vgg, lin = lo.lpips_state_dicts(2)
    x = torch.rand((2, 3, 16, 16), generator=torch.Generator().manual_seed(4))
    assert torch.equal(lo.forward(x, x, vgg, lin), torch.zeros(2, dtype=torch.float64))
    f0, f1 = torch.randn((1, 4, 2, 3), dtype=torch.float64), torch.randn((1, 4, 2, 3), dtype=torch.float64)
    w = torch.rand(4, dtype=torch.float64)
    want = 0.0
    for y in range(2):
        for xx in range(3):
            a, b = f0[0, :, y, xx], f1[0, :, y, xx]
            want += float((w * (a / (a.norm() + 1e-10) - b / (b.norm() + 1e-10)) ** 2).sum()) / 6
    assert abs(float(lo.tap_terms(f0, f1, w)[0]) - want) < 1e-14


# ----------------------------------------------------------------------------------------------- loader and input checks
@pytest.fixture()
def weight_files(tmp_path):
    return lo.make_lpips_weights(0, str(tmp_path))


def test_loader_reads_both_files(weight_files):
    vgg, lin = LP.load_weights(*weight_files)
    ref_vgg, ref_lin = lo.lpips_state_dicts(0)
    assert all(torch.equal(vgg[k], ref_vgg[k]) for k in ref_vgg) and all(torch.equal(lin[k], ref_lin[k]) for k in ref_lin)


def test_loader_names_the_missing_file(tmp_path, weight_files):
    vgg_path, lin_path = weight_files
    with pytest.raises(FileNotFoundError, match="VGG16"):
        LP.load_weights(str(tmp_path / "absent.pth"), lin_path)
    with pytest.raises(FileNotFoundError, match="lin"):
        LP.load_weights(vgg_path, str(tmp_path / "absent.pth"))


@pytest.mark.parametrize("which", ["vgg", "lin"])
@pytest.mark.parametrize("fault", ["missing", "extra", "shape"])
def test_loader_rejects_malformed_state_dicts(tmp_path, which, fault):
    vgg, lin = lo.lpips_state_dicts(0)
    sd = vgg if which == "vgg" else lin
    key = sorted(sd)[3 % len(sd)]
    if fault == "missing":
        del sd[key]
    elif fault == "extra":
        sd["features.99.weight" if which == "vgg" else "lin5.model.1.weight"] = torch.zeros(3)
    else:
        sd[key] = sd[key][:, :-1] if sd[key].dim() > 1 else sd[key][:-1]
    paths = str(tmp_path / "v.pth"), str(tmp_path / "l.pth")
    torch.save(vgg, paths[0])
    torch.save(lin, paths[1])
    with pytest.raises(ValueError, match="VGG16" if which == "vgg" else "lin"):
        LP.load_weights(*paths)


def test_loader_accepts_torchvisions_full_state_dict(tmp_path, weight_files):
    """A torchvision VGG16 state dict as saved (features and classifier) loads; the classifier is ignored."""
    tv = pytest.importorskip("torchvision")
    sd = tv.models.vgg16(weights=None).state_dict()
    assert any(k.startswith("classifier.") for k in sd)
    path = str(tmp_path / lo.VGG16_NAME)
    torch.save(sd, path)
    vgg, _ = LP.load_weights(path, weight_files[1])
    assert sorted(vgg) == sorted(LP.vgg16_shapes()) and torch.equal(vgg["features.28.bias"], sd["features.28.bias"])


def test_input_checks_reject_before_any_launch():
    rgb = torch.zeros((2, 32, 32, 3), dtype=torch.uint8)
    a, b = LP.LPIPS.check_images(rgb, rgb.clone())
    assert a.shape == (2, 32, 32, 3)
    with pytest.raises(ValueError, match="RGB"):
        LP.LPIPS.check_images(torch.zeros((2, 32, 32, 4), dtype=torch.uint8), torch.zeros((2, 32, 32, 4), dtype=torch.uint8))
    with pytest.raises(ValueError, match="16"):
        LP.LPIPS.check_images(torch.zeros((1, 15, 32, 3), dtype=torch.uint8), torch.zeros((1, 15, 32, 3), dtype=torch.uint8))
    with pytest.raises(ValueError, match="equal shape"):
        LP.LPIPS.check_images(rgb, torch.zeros((2, 32, 40, 3), dtype=torch.uint8))
    with pytest.raises(TypeError, match="uint8"):
        LP.LPIPS.check_images(rgb.float(), rgb.float())


# ----------------------------------------------------------------------------------------------- the reference's evaluators
@pytest.mark.skipif(not ref_loader.migt_available(), reason="reference sources not present (container-only test)")
def test_fixture_is_what_the_reference_evaluators_report():
    """tests/golden/lpips_reference_shim.npz is reproduced by the reference's own Evaluator and codebook Evaluator, with LPIPSMetric and
    models/utils.lpips as shipped around the fp64 oracle: the model receives images in [0, 1] (normalize=False), and the per-image values
    are the oracle's on the resized pair."""
    from oracle import make_golden as G, make_golden_lpips as MG, tf_shim
    tf_shim.install()
    try:
        got = MG.compute()
        model = sys.modules["viewformer.models.utils"].load_lpips_model()
        sys.modules["viewformer.utils.metrics"].LPIPSMetric._lpips_pool.pop("vgg", None)
    finally:
        tf_shim.uninstall()
    lo_, hi_ = model.input_range
    assert 0.0 <= lo_ and hi_ <= 1.0 and hi_ > 0.9, model.input_range            # the [0, 1] quirk, from the reference's own code
    g = np.load(os.path.join(GOLDEN, "lpips_reference_shim.npz"))
    assert sorted(got) == sorted(g.files)
    np.testing.assert_array_equal(got["weight_sums"], g["weight_sums"])
    for tag, n, gs, ns, image_size, seed in G.EVALUATOR_CASES:
        np.testing.assert_array_equal(got[f"{tag}.input_sums"], g[f"{tag}.input_sums"])
        for k in ("lpips", "codebook_lpips"):
            assert abs(float(got[f"{tag}.{k}"]) - float(g[f"{tag}.{k}"])) <= 1e-6 * abs(float(g[f"{tag}.{k}"])), (tag, k)
        np.testing.assert_allclose(got[f"{tag}.per_image"], g[f"{tag}.per_image"], rtol=1e-6)
        assert abs(float(g[f"{tag}.per_image"].mean()) - float(g[f"{tag}.lpips"])) <= 1e-6 * float(g[f"{tag}.lpips"])


def test_fixture_per_image_values_are_the_oracle_on_the_unresized_case():
    """Everywhere (no reference needed): the 'same' case (no resize) per-image values are lpips_oracle.forward_u8 of the synthetic pair."""
    from oracle import make_golden_lpips as MG
    g = np.load(os.path.join(GOLDEN, "lpips_reference_shim.npz"))
    vgg, lin = lo.lpips_state_dicts(MG.SEED)
    np.testing.assert_array_equal(np.asarray(lo.weight_sums(vgg, lin)), g["weight_sums"])
    gt, gen = synth.make_metric_pair(5, 64, 64, 21)
    assert [int(gt.sum()), int(gen.sum())] == g["same.input_sums"].tolist()
    np.testing.assert_allclose(lo.forward_u8(gt, gen, vgg, lin).numpy(), g["same.per_image"], rtol=1e-9)

"""The pose-scale augmentation of the transformer training step (MIGTConfig.random_pose_multiplier, migt.py:349-354) on the host: the
binding of its three entry points (include/vf_b200_pose.h, viewformer_b200.pose_scale) and their checkers, the hashed per-scene draw, and
tests/golden/migt_train_rpm_small.npz reproduced by the reference's own MIGT.train_step over oracle/tf_shim.py (skipped where the
reference is absent) and by the oracle's training forward with a per-scene multiplier."""
import ast
import glob
import inspect
import os
import re
import sys

import numpy as np
import pytest
import scipy.stats
import torch

import launch_checks as lc
import launch_checks_pose as lcp
from oracle import ref_loader, migt_oracle as mo, migt_oracle_rpm as mor
from test_abi import expected_argtype
from viewformer_b200 import pose_scale as PS
from viewformer_b200.config import MIGTConfig
from viewformer_b200.pose_scale import pose_scale_exponents

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pose_header_prototypes():
    """{name: (return type, [(type, is pointer, parameter name)])} of every function include/vf_b200_pose.h declares."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vf_b200_pose.h")).read(), flags=re.S)
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


def run(name, fn, write, *a, **k):
    """Bind ``fn``'s arguments, snapshot as the audit does, let ``write`` play the kernel, return the checker's ratio."""
    before, check = lcp.CHECKERS[name]
    ba = lc.bind(fn, *a, **k)
    st = before(ba, None)
    return check(ba, write(ba), st)


def assert_pass_and_catch(name, fn, good, bad, *a, **k):
    r_good, r_bad = run(name, fn, good, *a, **k), run(name, fn, bad, *a, **k)
    print(f"[{name}] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0, f"{name}: the fp64 restatement fails its own check ({r_good:.3g})"
    assert r_bad > 1.0, f"{name}: the mutation was not caught ({r_bad:.3g})"


def test_prototype_table_matches_header():
    """pose_scale.PROTOTYPES against include/vf_b200_pose.h: the same three functions, int returns, per function the header's parameter
    count and, position by position, the ctypes type _lib's mapping gives each C type (tests/test_abi.py does this for vf_b200.h)."""
    from viewformer_b200 import _lib
    declared = pose_header_prototypes()
    assert sorted(declared) == sorted(PS.PROTOTYPES) == ["vf_pose_loss_grad_scaled", "vf_pose_loss_rows_scaled", "vf_pose_model_input"]
    assert not set(declared) & set(_lib.PROTOTYPES)
    for name, (ret, params) in declared.items():
        assert ret == "int", name
        got = PS.PROTOTYPES[name]
        assert len(got) == len(params), f"{name}: {len(got)} argtypes, the header declares {len(params)} parameters"
        for k, (have, prm) in enumerate(zip(got, params)):
            want = expected_argtype(name, *prm)
            assert have is want, f"{name} parameter {k} {prm}: the table has {have.__name__}, the header wants {want.__name__}"


def test_library_exports_and_load_declares(lib):
    for name in PS.PROTOTYPES:
        assert hasattr(lib, name), f"libvf_b200.so does not export {name}"


def test_call_sites_pass_each_prototypes_argument_count():
    """Every `*.vf_pose_...(...)` call of the package, tests and scripts passes the prototype's argument count, positionally."""
    files = (glob.glob(os.path.join(ROOT, "viewformer_b200", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "tests", "*.py"))
             + glob.glob(os.path.join(ROOT, "scripts", "*.py")))
    seen = set()
    for path in files:
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in PS.PROTOTYPES:
                name, where = node.func.attr, f"{os.path.relpath(path, ROOT)}:{node.lineno}"
                assert not node.keywords and not any(isinstance(a, ast.Starred) for a in node.args), f"{where}: {name} with keywords or *args"
                assert len(node.args) == len(PS.PROTOTYPES[name]), f"{where}: {name} takes {len(PS.PROTOTYPES[name])} arguments"
                seen.add(name)
    assert seen == set(PS.PROTOTYPES)


def test_every_launching_wrapper_has_a_checker():
    """Every public pose_scale function that names one of its entry points has a checker in tests/launch_checks_pose.py."""
    public = {name for name, fn in vars(PS).items() if inspect.isfunction(fn) and fn.__module__ == PS.__name__ and not name.startswith("_")
              and any(n in PS.PROTOTYPES for n in fn.__code__.co_names)}
    assert public == set(lcp.CHECKERS) == {"pose_model_input", "pose_loss_rows_scaled", "pose_loss_grad_scaled"}


def test_launch_checkers_of_the_scaled_pose_wrappers():
    """The fp64 checkers of the three wrappers accept an fp64 restatement rounded to fp32 and reject it with a named fault: the scale of
    the neighbouring scene, the outer 1 / c of the gradient left out, a quaternion scaled with the position."""
    g = torch.Generator().manual_seed(7)
    tpv, T, B = 8, 3, 4
    raw, poses = torch.randn(tpv * T * B, 7, generator=g), torch.randn(T * B, 7, generator=g)
    w, c = torch.rand(tpv * T * B, generator=g), torch.tensor([0.45, 2.2, 1.0, 1.7])
    m = 0.3
    y = poses.double().repeat_interleave(tpv, 0)
    cr = c.double().repeat_interleave(tpv * T)[:, None]
    rc = raw.double()[:, :3] / cr
    pos = ((y[:, :3] * lc.f32(m) - rc) ** 2).mean(1).float()
    ori = ((y[:, 3:] - raw.double()[:, 3:]) ** 2).mean(1).float()
    bad = ((y[:, :3] * lc.f32(m) - raw.double()[:, :3] / cr.roll(1, 0)) ** 2).mean(1).float()        # another row's scene
    assert_pass_and_catch("pose_loss_rows_scaled", PS.pose_loss_rows_scaled, lambda ba: (pos, ori), lambda ba: (bad, ori), raw, poses, tpv, m,
                          T, c)
    scl = torch.tensor([lc.f32(0.6) * 2 / 3] * 3 + [lc.f32(1.7) * 2 / 4] * 4, dtype=torch.float64)
    div = torch.cat([cr.expand(-1, 3), torch.ones_like(cr).expand(-1, 4)], 1)
    mv = torch.tensor([lc.f32(m)] * 3 + [1.0] * 4, dtype=torch.float64)
    gr = (-w.double()[:, None] * scl * (y * mv - raw.double() / div) / div).float()
    bad = (-w.double()[:, None] * scl * (y * mv - raw.double() / div)).float()                      # the outer 1 / c left out
    assert_pass_and_catch("pose_loss_grad_scaled", PS.pose_loss_grad_scaled, lambda ba: gr, lambda ba: bad, raw, poses, w, tpv, m, T, c,
                          0.6, 1.7)
    cv = c.double().repeat_interleave(T)[:, None]
    pin = torch.cat([(poses[:, :3].double() * lc.f32(m) * cv).float(), poses[:, 3:]], 1)
    bad = torch.cat([pin[:, :3], poses[:, 3:] * 1.5], 1)
    assert_pass_and_catch("pose_model_input", PS.pose_model_input, lambda ba: pin, lambda ba: bad, poses, m, T, c)
    plain = torch.cat([poses[:, :3] * np.float32(m), poses[:, 3:]], 1)
    assert_pass_and_catch("pose_model_input", PS.pose_model_input, lambda ba: plain, lambda ba: pin, poses, m, T)


# ------------------------------------------------------------------------------------------------ the hashed draw
def test_draw_is_deterministic_and_differs_in_every_input():
    base = dict(seed=3, iterations=17, rank=1, micro_batch=2, n_scenes=6)
    u = pose_scale_exponents(**base)
    assert u.dtype == torch.float32 and u.shape == (6,)
    assert torch.equal(u, pose_scale_exponents(**base))
    assert len(set(u.tolist())) == 6                                                     # scenes
    for key in ("seed", "iterations", "rank", "micro_batch"):
        other = pose_scale_exponents(**dict(base, **{key: base[key] + 1}))
        assert not torch.equal(other, u), key
        assert not set(other.tolist()) & set(u.tolist()), key
    # more scenes extend the draw: scene b's value does not depend on the batch size
    assert torch.equal(pose_scale_exponents(**dict(base, n_scenes=9))[:6], u)
    # a 2^-23 grid in [-1, 1)
    assert bool(((u + 1) * 2 ** 23 == torch.round((u + 1) * 2 ** 23)).all())


def test_draw_is_uniform_and_r_lies_in_range():
    """10^5 draws over iterations, ranks, micro-batches and scenes: u in [-1, 1) passes a KS test against U[-1, 1), and
    r = c ** u lies in [1/c, c] (fp32, as the trainer computes it)."""
    us = [pose_scale_exponents(5, it, rank, micro, 25) for it in range(500) for rank in range(4) for micro in range(2)]
    u = torch.cat(us)
    assert u.numel() == 100_000
    assert float(u.min()) >= -1.0 and float(u.max()) < 1.0
    ks = scipy.stats.kstest(u.double().numpy(), scipy.stats.uniform(loc=-1.0, scale=2.0).cdf)
    print(f"[pose scale draw] KS statistic {ks.statistic:.2e}, p = {ks.pvalue:.3f}")
    assert ks.pvalue > 1e-3
    for c in (2.5, 1.3, 0.5):
        r = torch.pow(torch.tensor(c, dtype=torch.float32), u)
        lo, hi = min(c, 1 / c), max(c, 1 / c)
        assert float(r.min()) >= np.float32(lo) * (1 - 2 ** -23) and float(r.max()) <= np.float32(hi) * (1 + 2 ** -23)
        assert float((torch.log(r.double()) / np.log(c) - u.double()).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ the fixture against the reference
@pytest.fixture(scope="module")
def tf():
    if not ref_loader.migt_available():
        pytest.skip("reference sources not present")
    from oracle import tf_shim
    tf_shim.install()
    ref_loader.load_reference_migt()
    yield sys.modules["tensorflow"]
    tf_shim.uninstall()                       # later test modules must not see a `tensorflow` in sys.modules


@pytest.mark.parametrize("prefix", ["", "dyn."])
def test_reference_train_step_reproduces_fixture(tf, prefix):
    """Three calls of the reference's MIGT.train_step with random_pose_multiplier 2.5 write the fixture again: the draws, losses,
    gradients and post-step weights."""
    from oracle import make_golden_rpm as mg
    G = np.load(os.path.join(GOLDEN, "migt_train_rpm_small.npz"))
    extra = dict(mg.VARIANTS)[prefix]
    rec = mg.run_reference(dict(mg.MIGT_TRAIN_RPM, **extra), torch_seed=len(prefix))
    assert set(prefix + k for k in rec) == {k for k in G.files if k.startswith(prefix) and (prefix or not k.startswith("dyn."))}
    for k, v in rec.items():
        want = G[prefix + k]
        if k[0] in "ur" and k[1:].isdigit():                         # the draws: the same generator, seeded alike
            assert np.array_equal(v, want), prefix + k
        elif want.dtype.kind == "f":                                  # CPU reductions split across threads: last-bit differences
            np.testing.assert_allclose(v, want, rtol=2e-5, atol=2e-5 * float(np.abs(want).max()), err_msg=prefix + k)
        else:
            assert np.array_equal(v, want), prefix + k
    for step in range(mg.STEPS):
        r = G[f"{prefix}r{step}"]
        assert np.all((r >= 1 / 2.5) & (r <= 2.5))


@pytest.mark.parametrize("prefix", ["", "dyn."])
def test_oracle_with_pose_scale_reproduces_fixture_gradients(prefix):
    """Autograd through oracle/migt_oracle_rpm.forward, fed the fixture's r, gives the reference's first-step losses and gradients; with
    r = None or r = 1 it computes migt_oracle.forward's values bit for bit."""
    from oracle import make_golden_rpm as mg
    G = np.load(os.path.join(GOLDEN, "migt_train_rpm_small.npz"))
    cfg = MIGTConfig(**dict(mg.MIGT_TRAIN_RPM, **dict(mg.VARIANTS)[prefix]))
    sd = mg.state_dict(cfg)
    cams, codes = mg.batch(cfg, 0)
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    r = torch.from_numpy(G[f"{prefix}r0"])
    o = mor.forward(leaves, cfg, dict(input_ids=codes, poses=cams), r, localization_weight=0.5)
    o["loss"].mean().backward()
    assert abs(float(o["loss"].detach().mean()) - float(G[f"{prefix}loss0"])) < 1e-5 * abs(float(G[f"{prefix}loss0"]))
    np.testing.assert_allclose(o["pose_pos_loss"].detach().numpy(), G[f"{prefix}pos0"], rtol=1e-5)
    names = [str(n) for n in G[f"{prefix}names"]]
    for i, k in enumerate(names):
        g = leaves[k].grad if leaves[k].grad is not None else torch.zeros_like(sd[k])
        rn = G[f"{prefix}gnorm0"][i]
        assert abs(float(g.norm()) - rn) <= 1e-4 * rn + 1e-7, k
    with torch.no_grad():
        a = mo.forward(sd, cfg, dict(input_ids=codes, poses=cams), compute_losses=True, localization_weight=0.5)
        for rr in (None, torch.ones(2)):
            b = mor.forward(sd, cfg, dict(input_ids=codes, poses=cams), rr, localization_weight=0.5)
            for k in ("loss", "ce_loss", "pose_pos_loss", "pose_ori_loss", "pose_loss", "pose_prediction", "logits"):
                assert torch.equal(a[k], b[k]), k
        a = mo.forward(sd, cfg, dict(input_ids=codes, poses=cams), compute_losses=True, use_localization=False)
        b = mor.forward(sd, cfg, dict(input_ids=codes, poses=cams), None, use_localization=False)
        assert torch.equal(a["loss"], b["loss"]) and torch.equal(a["logits"], b["logits"])

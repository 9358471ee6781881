"""The pose-scale augmentation of the transformer training step (MIGTConfig.random_pose_multiplier, migt.py:349-354) on the GPU: the
three scaled pose kernels against fp64, their unit-scale bits, both trainers against tests/golden/migt_train_rpm_small.npz (the reference's
own train_step with random_pose_multiplier 2.5, fed the same draws), the full-size fp32 step against fp64 autograd through the oracle, the
hashed draw across a resume and under gradient accumulation, and every launch of a full-size step under its fp64 bar."""
import os

import numpy as np
import pytest
import torch

import launch_checks_pose as lcp
from oracle import synth, migt_oracle as mo, migt_oracle_rpm as mor
from oracle.make_golden import MIGT_TRAIN, MIGT_TRAIN_WARMUP
from oracle.make_golden_rpm import MIGT_TRAIN_RPM, VARIANTS, STEPS, batch, state_dict
from test_faithful_steps_gpu import faithful_report, migt_grads64, step_errors
from test_launch_audit_gpu import Audit, FULL_MIGT_TRAIN, _migt_step
from viewformer_b200 import pose_scale as PS
from viewformer_b200.config import MIGTConfig
from viewformer_b200.pose_scale import pose_scale_exponents

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def _trainer(cfg_kw, sd=None, precision="fp32", **kw):
    from viewformer_b200 import MIGT
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**cfg_kw)
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9) if sd is None else sd)
    return cfg, MIGTTrainer(model, precision=precision, **kw)


def _batch(cfg, B, T, seed):
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0])
    return cams, codes


# ----------------------------------------------------------------------------------------------- kernels
def test_scaled_pose_kernels_vs_fp64(L):
    """vf_pose_model_input, vf_pose_loss_rows_scaled and vf_pose_loss_grad_scaled against fp64 (tests/launch_checks_pose.py) at the bars of the
    unscaled pose kernels, 8 ulps of |y m| + |raw / c|, with pose_multiplier, pos_scale, ori_scale and every scene's c != 1."""
    import random
    g = torch.Generator().manual_seed(31)
    tpv, T, B = 64, 5, 3
    raw = (torch.randn(tpv * T * B, 7, generator=g) * 3).cuda()
    poses = torch.randn(T * B, 7, generator=g).cuda()
    w = torch.rand(tpv * T * B, generator=g).cuda()
    c = torch.pow(torch.tensor(2.5), torch.rand(B, generator=g) * 2 - 1).cuda()
    m, rng = 0.3, random.Random(0)
    ratios = {}
    for name, fn, a in (("pose_model_input", PS.pose_model_input, (poses, m, T, c)), ("pose_model_input", PS.pose_model_input, (poses, m, T)),
                        ("pose_loss_rows_scaled", PS.pose_loss_rows_scaled, (raw, poses, tpv, m, T, c)),
                        ("pose_loss_grad_scaled", PS.pose_loss_grad_scaled, (raw, poses, w, tpv, m, T, c, 0.6, 1.7))):
        _, r = lcp.run_check(name, fn, a, {}, rng)
        torch.cuda.synchronize()
        ratios[name] = max(ratios.get(name, 0.0), r)
    print("[scaled pose kernels] worst ratio to the fp64 bar: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    assert all(v <= 1.0 for v in ratios.values()), ratios


def test_unit_scale_is_bit_identical(L):
    """With every scene's c = 1 the scaled entry points return the unscaled ones' bits, the pose input equals torch's poses * [m,m,m,1,1,1,1],
    and a whole fp32 step with random_pose_multiplier 2 and u = 0 (r = 2^0 = 1) equals the step without the augmentation."""
    g = torch.Generator().manual_seed(5)
    tpv, T, B, m = 64, 4, 3, 0.3
    raw, poses = torch.randn(tpv * T * B, 7, generator=g).cuda(), torch.randn(T * B, 7, generator=g).cuda()
    w, ones = torch.rand(tpv * T * B, generator=g).cuda(), torch.ones(B, device="cuda")
    for a, b in zip(PS.pose_loss_rows_scaled(raw, poses, tpv, m, T, ones), L.pose_loss_rows(raw, poses, tpv, m)):
        assert torch.equal(a, b)
    assert torch.equal(PS.pose_loss_grad_scaled(raw, poses, w, tpv, m, T, ones, 0.6, 1.7), L.pose_loss_grad(raw, poses, w, tpv, m, 0.6, 1.7))
    plain = poses * torch.tensor([m] * 3 + [1.0] * 4, dtype=torch.float32, device="cuda")
    assert torch.equal(PS.pose_model_input(poses, m, T, ones), plain) and torch.equal(PS.pose_model_input(poses, m, T), plain)

    kw = dict(MIGT_TRAIN, pose_multiplier=0.3)
    cams, codes = _batch(MIGTConfig(**kw), 2, 4, 90)

    def step(c, u=None):
        _, tr = _trainer(dict(kw, random_pose_multiplier=c))
        loss = float(tr.forward_backward(cams, codes, pose_scale_u=u))
        torch.cuda.synchronize()
        return loss, tr.flat_g.clone(), tr
    base, again, (l2, g2, tr) = step(1.0), step(1.0), step(2.0, [0.0, 0.0])
    assert torch.equal(tr.last["pose_scale"], torch.ones(2))
    if torch.equal(base[1], again[1]) and base[0] == again[0]:
        assert l2 == base[0] and torch.equal(g2, base[1])
    else:                                            # the step itself is not bitwise repeatable: hold the r = 1 step to its spread
        spread = float((base[1] - again[1]).abs().max())
        print(f"[unit scale] two plain steps differ by {spread:.2e}")
        assert float((g2 - base[1]).abs().max()) <= 4 * spread


# ----------------------------------------------------------------------------------------------- against the reference's train_step
def _against_fixture(golden_dir, prefix, precision):
    G = np.load(os.path.join(golden_dir, "migt_train_rpm_small.npz"))
    cfg = MIGTConfig(**dict(MIGT_TRAIN_RPM, **dict(VARIANTS)[prefix]))
    cfg, tr = _trainer(dict(MIGT_TRAIN_RPM, **dict(VARIANTS)[prefix]), sd=state_dict(cfg), precision=precision,
                       warmup_steps=MIGT_TRAIN_WARMUP, bucket_bytes=1 << 18)
    names = [str(n) for n in G[prefix + "names"]]
    gen = torch.Generator().manual_seed(77)
    probe = {k: torch.randn(tuple(tr.p[k].shape), generator=gen) for k in names}
    full = [k[len(prefix) + 3:] for k in G.files if k.startswith(prefix + "g0.")]
    for step in range(STEPS):
        cams, codes = batch(cfg, step)
        assert abs(tr.learning_rate() - float(G[f"{prefix}lr{step}"])) < 1e-9
        loss = float(tr.forward_backward(cams, codes, pose_scale_u=G[f"{prefix}u{step}"]))
        torch.cuda.synchronize()
        assert torch.equal(tr.last["pose_scale"], torch.from_numpy(G[f"{prefix}r{step}"]))          # r = c ** u on the host, as the reference
        grads = {k: v / tr.loss_scale for k, v in tr.gradients().items()}
        errs = []
        for i, n in enumerate(names):
            gn, gd = float(grads[n].norm()), float((grads[n] * probe[n]).sum())
            rn, rd = float(G[f"{prefix}gnorm{step}"][i]), float(G[f"{prefix}gdot{step}"][i])
            errs.append((max(abs(gn - rn), abs(gd - rd)) / max(rn, 1e-4), n))
        want = float(G[f"{prefix}loss{step}"])
        pos = tr.last["pose_pos_loss"].cpu().numpy()
        print(f"[rpm {precision} {prefix or 'plain'} step {step}] loss {loss:.6f} (ref {want:.6f}), r {G[f'{prefix}r{step}']}, gradients: "
              f"median {np.median([e for e, _ in errs]):.2e}, worst {max(errs)[0]:.2e} ({max(errs)[1]})")
        if precision == "fp32":                                                   # tests/test_train_gpu.py's migt_train_small bars
            assert abs(loss - want) < 3e-5 * abs(want)
            np.testing.assert_allclose(tr.last["ce_loss"].cpu().numpy(), G[f"{prefix}ce{step}"], rtol=3e-5)
            np.testing.assert_allclose(pos, G[f"{prefix}pos{step}"], rtol=1e-4)
            assert max(errs)[0] < 3e-3, max(errs)
            for n in full:
                ref = torch.from_numpy(G[f"{prefix}g{step}.{n}"])
                err = float((grads[n] - ref).abs().max() / ref.abs().max().clamp_min(1e-4))
                assert err < 2e-3, f"step {step} grad {n}: max rel err {err:.3e}"
        else:                                                                     # tests/test_train_migt_bf16_gpu.py's bars
            assert abs(loss - want) <= 5e-3 * abs(want)
            np.testing.assert_allclose(tr.last["ce_loss"].cpu().numpy(), G[f"{prefix}ce{step}"], rtol=5e-3)
            assert float(np.median([e for e, _ in errs])) <= 1e-2 and max(errs)[0] <= 1e-1, max(errs)
        assert tr.optimizer_step()
        if precision == "fp32":
            sd, lr = tr.state_dict(), max(float(G[f"{prefix}lr{step}"]), 1e-12)
            for n in full:
                d = (sd[n] - torch.from_numpy(G[f"{prefix}p{step}.{n}"])).abs()
                frac_bad = float((d > 0.05 * lr + 1e-7).float().mean())
                assert frac_bad < 0.02, f"step {step} weight {n}: {frac_bad:.3%} elements differ by more than 5% of lr"


@pytest.mark.parametrize("prefix", ["", "dyn."])
def test_fp32_trainer_matches_reference_fixture(golden_dir, prefix):
    _against_fixture(golden_dir, prefix, "fp32")


@pytest.mark.parametrize("prefix", ["", "dyn."])
def test_bf16_trainer_matches_reference_fixture(golden_dir, prefix):
    _against_fixture(golden_dir, prefix, "bf16")


# ----------------------------------------------------------------------------------------------- full size against fp64
def test_full_size_fp32_step_vs_fp64(L, monkeypatch):
    """Full size (12 layers, d = 768, B = 2, T = 5), random_pose_multiplier 2, pose_multiplier 0.5, the hashed draw: every gradient of the
    fp32 step against fp64 autograd through the oracle fed the same r, at tests/test_faithful_steps_gpu.py's bar (e_tc <= 2 e_cuda +
    STEP_FLOOR, e_cuda from the VF_TRAIN_TC=0 step)."""
    kw = dict(FULL_MIGT_TRAIN, random_pose_multiplier=2.0, pose_multiplier=0.5)
    cfg = MIGTConfig(**kw)
    sd = synth.make_migt_state_dict(cfg, 13)
    cams, codes = _batch(cfg, 2, 5, 170)
    errs, r_seen, ref = {}, [], None
    for tc in ("1", "0"):
        monkeypatch.setenv("VF_TRAIN_TC", tc)
        _, tr = _trainer(kw, sd={k: v.clone() for k, v in sd.items()}, seed=4)
        assert tr.use_tc == (tc == "1")
        tr.forward_backward(cams, codes)
        torch.cuda.synchronize()
        r = tr.last["pose_scale"]
        r_seen.append(r)
        if ref is None:
            leaves = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
            o = mor.forward(leaves, cfg, dict(input_ids=codes, poses=cams.double()), r.double(), localization_weight=tr.loc_weight)
            o["loss"].mean().backward()
            ref = {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaves.items()}
        errs[tc] = step_errors(tr.gradients(), ref)
        del tr
        torch.cuda.empty_cache()
    assert torch.equal(r_seen[0], r_seen[1]) and not torch.equal(r_seen[0], torch.ones(2)) and r_seen[0][0] != r_seen[0][1]
    bad = faithful_report("rpm migt-full", errs)
    assert not bad, "tensor-core gradients less accurate than 2x the CUDA-core trainer's: " + ", ".join(
        f"{k} {errs['1'][k]:.2e} vs {errs['0'][k]:.2e}" for k in bad[:8])
    # the augmentation reaches the pose MLPs: without it the fp64 gradient of the pose embedding differs by far more than the bar
    plain = migt_grads64(sd, cfg, cams, codes, 0.7)
    k = "pose_embedding.c_fc.weight"
    assert float((plain[k] - ref[k]).norm()) > 100 * errs["0"][k] * float(ref[k].norm())


# ----------------------------------------------------------------------------------------------- the draw across resume and accumulation
def test_resume_redraws_the_uninterrupted_run():
    """Four steps in one run, and two steps, optimizer_state + state_dict into a fresh trainer, two more: the last two steps draw the same
    exponents; each step draws pose_scale_exponents(seed, iterations, 0, 0, B)."""
    kw = dict(MIGT_TRAIN, random_pose_multiplier=2.0)
    cfg = MIGTConfig(**kw)
    batches = [_batch(cfg, 2, 4, 200 + i) for i in range(4)]
    _, whole = _trainer(kw, seed=11, warmup_steps=2)
    draws = []
    for b in batches:
        whole.train_step(b)
        draws.append(whole.last["pose_scale_u"])
    for it, u in enumerate(draws):
        assert torch.equal(u, pose_scale_exponents(11, it, 0, 0, 2))
    assert len({tuple(u.tolist()) for u in draws}) == 4
    _, first = _trainer(kw, seed=11, warmup_steps=2)
    for b in batches[:2]:
        first.train_step(b)
    _, resumed = _trainer(kw, seed=0, warmup_steps=2)                       # the seed too comes from the saved state
    resumed.load_state_dict(first.state_dict()).load_optimizer_state(first.optimizer_state())
    for i, b in enumerate(batches[2:]):
        resumed.train_step(b)
        assert torch.equal(resumed.last["pose_scale_u"], draws[2 + i])


def test_accumulation_draws_per_micro_batch():
    """accumulate_steps = 2: each micro-batch of a window draws its own exponents, pose_scale_exponents(seed, iterations, 0, micro, B)."""
    kw = dict(MIGT_TRAIN, random_pose_multiplier=2.0)
    cfg = MIGTConfig(**kw)
    _, tr = _trainer(kw, seed=3, accumulate_steps=2)
    seen = []
    for i in range(4):
        out = tr.train_step(_batch(cfg, 2, 4, 300 + i))
        it, micro = i // 2, i % 2
        assert out["applied"] == (micro == 1)
        assert torch.equal(tr.last["pose_scale_u"], pose_scale_exponents(3, it, 0, micro, 2))
        seen.append(tuple(tr.last["pose_scale_u"].tolist()))
    assert len(set(seen)) == 4


def test_pose_scale_u_needs_the_augmentation():
    _, tr = _trainer(dict(MIGT_TRAIN))
    cams, codes = _batch(tr.cfg, 2, 4, 1)
    with pytest.raises(ValueError, match="random_pose_multiplier is 1"):
        tr.forward_backward(cams, codes, pose_scale_u=[0.5, 0.5])


# ----------------------------------------------------------------------------------------------- launch audit
SCALED = {("pose_model_input", "float32"), ("pose_loss_rows_scaled", "float32"), ("pose_loss_grad_scaled", "float32")}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_launch_audit_full_size_step(L, monkeypatch, precision):
    """A full-size train_step (B = 2, T = 5) with random_pose_multiplier 2: every checked launch within its fp64 bar, the three scaled pose
    wrappers (checked by tests/launch_checks_pose.py) reached and the unscaled pose-loss wrappers not."""
    audit = Audit(L, monkeypatch)
    for name, fn in [(n, getattr(PS, n)) for n in lcp.CHECKERS]:
        def call(*a, _name=name, _fn=fn, **k):
            with torch.no_grad():
                result, r = lcp.run_check(_name, _fn, a, k, audit.rng)
            audit.rec[(_name, str(a[0].dtype).replace("torch.", "")) + audit._site()].append(r)
            return result
        monkeypatch.setattr(PS, name, call)
    _migt_step(dict(FULL_MIGT_TRAIN, random_pose_multiplier=2.0, pose_multiplier=0.5), 2, 5, precision, 6100, full=True)
    torch.cuda.synchronize()
    bad = audit.report(f"rpm-step-{precision}-full")
    reached = audit.reached()
    torch.cuda.empty_cache()
    assert SCALED <= reached, sorted(SCALED - reached)
    assert not {n for n, _ in reached} & {"pose_loss_rows", "pose_loss_grad"}
    assert not bad, "launches outside their bar:\n  " + "\n  ".join(bad)

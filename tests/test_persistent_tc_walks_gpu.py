"""The tensor-core GEMM / conv kernel's persistent walk at sizes where a CTA walks several tiles: against fp64, and against its own
single-tile bits.

tc_gemm_kernel (viewformer_b200/csrc/vf_tc_gemm.cu) is persistent: the launcher sets the grid to min(tiles, SMs) and CTA c walks tiles
c, c + grid, ... (n tile fastest, then the m tile: for a conv the x tile, y tile and image tile, then the batch).  State runs on from
one tile to the next: the parity of the four resident halo buffers of the exact (split-fp16) halo conv, whose next tile's lo halves load
while the previous tile's last passes still read its hi halves; the weight ring's stage / phase; the per-tile reset of the chunk sums;
the residual's L2 prefetch; the staging tile, handed over only after the next tile's K loop; the bf16 halo double buffer, which
alternates across tiles when the channel-block count is odd; the image whose statistics normalise-on-load reads; and the causal GEMMs'
skipped tiles.  Each case here

* restates the launcher's tiling (TW / TH / TN, halo, block_n, tiles) with launch_checks.tc_conv_tiling, requires the launcher's own plan
  (tc_conv / tc_gemm with plan=True, which reads vf_tc_gemm_plan) to equal it, prints how many tiles the busiest CTA walks on this GPU and
  asserts >= 2 (>= 3 where stated), so that a GPU with more SMs cannot pass the test without walking;
* checks every image, batch entry and row against fp64 with check_tc_conv / check_tc_gemm of tests/launch_checks.py (their bars:
  _epilogue, and _gn_ratio for the fused GroupNorm sums), chunk by chunk, and prints the worst ratio;
* requires every image (TN = 1), image pair (TN = 2), batch entry or 128-row block to equal, bit for bit, a launch of that part alone, in
  which no CTA walks a second tile: a tile's arithmetic (chunk order, staging layout, epilogue order) does not depend on the CTA that runs
  it, so this is exact and sees a leak far below the fp64 bar.  Fused GroupNorm sums are added with fp64 atomics in schedule order, so
  they are compared with rtol 1e-12.

The benchmark's roofline launch (the exact halo conv at 288 x 128^2, 128 -> 128, with a residual: 36 864 tiles, up to 280 per CTA) is
checked on every one of its 288 images, against fp64 and against single-image launches.

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); every bit comparison equal; the file runs in about 10 s.  Busiest CTA's
tiles / worst ratio to the fp64 bar:
  exact halo: 3 x 128^2 3 / 0.00063 (also without residual, and with the residual aliased to the output), 2 x 128^2 2 / 0.00062,
      9 x 64^2 3 / 0.0018, 17 x 32^2 128->256 3 / 0.0027, 40x20 64->256 2 / 0.0028; benchmark shape 280 / 0.00078.
  exact tap-box 9 x 32^2 256->256 2 / 0.0028, 67 x 8^2 256->512 (TN = 2) 2 / 0.012; Downsample 34 x 64^2 3 / 0.0032.
  bf16 halo 64->128 3 / 0.0038, 128->128 with a bf16 copy 3 / 0.0025; normalise-on-load 128^2 3 / 0.0032, 40x20 2 / 0.0044; TF32 3 /
      0.0054.
  GEMMs (2 each): split-fp16 0.011, bf16 BIAS_M + GELU 0.0055, TF32 aliased residual 0.022, K offsets 0.012, causal QK^T 0.018, P.V
      0.0018, row blocks 0.0098; conv_wgrad_tc 0.0026, conv_wgrad_bf16 0.0011.
Four kernel mutants fail these tests: chunk sums carried into the next tile and the hi halo halves loaded at the previous tile's
position (every exact halo case), the tap-box pass 0 reading the hi half after a CTA's first tile (the tap-box and Downsample cases),
and normalise-on-load reading the previous tile's image statistics (both normalise-on-load cases).
"""
import random

import pytest
import torch

import launch_checks as lc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


@pytest.fixture(autouse=True)
def gn_hook(L, monkeypatch):
    """The normalise-on-load operand is vf_groupnorm_apply's bf16 output bit for bit (as in the launch audit)."""
    groupnorm = L.groupnorm
    monkeypatch.setitem(lc.HOOKS, "gn_apply_bf16", lambda x, mr, gamma, beta, swish: groupnorm(
        x.contiguous(), gamma, beta, swish=swish, out_dtype=torch.bfloat16, stats=mr.contiguous(), groups=mr.shape[1]))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _walk(tag, plan, want, need=2):
    """plan: the launcher's tiling; want: the restated one.  Asserts they agree and that the busiest CTA walks >= ``need`` tiles."""
    for k, v in want.items():
        assert plan[k] == v, f"{tag}: the launcher plans {k} = {plan[k]}, the restatement {v} (plan {plan})"
    ctas = min(plan["tiles"], _sms())
    assert plan["ctas"] == ctas, f"{tag}: {plan['ctas']} CTAs for {plan['tiles']} tiles on {_sms()} SMs"
    per_cta = -(-plan["tiles"] // ctas)
    mode = f"TW {plan['TW']} TH {plan['TH']} TN {plan['TN']} halo {plan['halo']} " if plan["TW"] else ""
    print(f"[walk {tag}] {mode}block_n {plan['block_n']}: {plan['tiles']} tiles on {ctas} CTAs, up to {per_cta} per CTA")
    assert per_cta >= need, f"{tag}: the busiest CTA walks {per_cta} tiles, the case needs {need}; make the launch larger for this GPU"


def _same_bits(tag, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    it = {2: torch.int16, 4: torch.int32}[got.element_size()]
    diff = (got.view(it) != want.view(it)).nonzero()
    assert diff.shape[0] == 0, f"{tag}: {diff.shape[0]} elements differ from the single-tile launch, first at {tuple(diff[0].tolist())}"


def _split(x):
    """fp32 [..., C] -> the split-fp16 operand [..., hi(C) | lo(C)]."""
    from viewformer_b200 import _lib
    return _lib.split_f16x2(x.reshape(-1, x.shape[-1]).contiguous()).reshape(*x.shape[:-1], 2 * x.shape[-1])


# ----------------------------------------------------------------------------------------------- a. convolutions
def _conv_operands(kind, n, h, w, cin, cout, seed, ntaps=9, s2d=False):
    """x (the operand tc_conv reads) and w_nk for ``kind`` exact | bf16 | tf32; fp32 values ~ N(0, 1.5^2), weights scaled by 1 / sqrt(K)."""
    from viewformer_b200 import _lib
    x = torch.randn((n, h, w, cin), generator=_gen(seed), device="cuda") * 1.5
    wt = torch.randn((cout, ntaps, cin), generator=_gen(seed + 1), device="cuda") / (ntaps * cin) ** 0.5
    if kind == "exact":
        if s2d:
            x = _lib.groupnorm(x, None, None, swish=False, out_dtype=torch.float16, normalize=False, s2d=True)
        else:
            x = _split(x)
        return x, _split(wt).reshape(cout, ntaps * 2 * cin)
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    return x.to(dt), wt.reshape(cout, ntaps * cin).to(dt)


def _conv_plan(L, tag, x, w_nk, need, **k):
    """The launcher's plan of tc_conv(x, w_nk, **k) against the restatement; returns TN."""
    n, h, wd, ctot = x.shape
    ba = lc.bind(L.tc_conv, x, w_nk, None, **k)
    split = x.dtype == torch.float16
    cin = ctot // (2 if split else 1) if ba["cin"] is None else ba["cin"]
    tw, th, tn, halo = lc.tc_conv_tiling(h, wd, ctot, cin, h, wd, ba["taps"], ba["coffs"], split, x.dtype == torch.float32)
    cout = w_nk.shape[0]
    bn = lc.tc_block_n(cout)
    tiles = -(-wd // tw) * -(-h // th) * -(-n // tn) * -(-cout // bn)
    _walk(tag, L.tc_conv(x, w_nk, None, plan=True, **k), dict(block_n=bn, TW=tw, TH=th, TN=tn, halo=int(halo), exact=int(split),
                                                                tiles=tiles), need)
    return tn


def _conv_case(L, tag, x, w_nk, bias, need=2, residual=None, chunk=16, out2_dtype=None, **k):
    """One many-tile tc_conv launch: the plan, every image against fp64, every image group of one tile against its own launch."""
    n = x.shape[0]
    tn = _conv_plan(L, tag, x, w_nk, need, **k)
    out2 = None if out2_dtype is None else torch.empty(x.shape[:3] + (w_nk.shape[0],), dtype=out2_dtype, device="cuda")
    before, check = lc.CHECKERS["tc_conv"]
    ba = lc.bind(L.tc_conv, x, w_nk, bias, residual=residual, out2=out2, **k)
    st = before(ba, random.Random(0))
    out = L.tc_conv(x, w_nk, bias, residual=residual, out2=out2, **k)
    torch.cuda.synchronize()
    worst, at = -1.0, None
    for i0 in range(0, n, chunk):
        st["images"] = list(range(i0, min(n, i0 + chunk)))
        r = check(ba, out, st)
        if r > worst:
            worst, at = r, st["images"]
    gn = getattr(out, "_gn_sums", None)
    print(f"[fp64 {tag}] every image of {n}: worst ratio {worst:.3g} (images {at[0]}..{at[-1]})"
          f"{', fused GroupNorm sums included' if gn is not None else ''}")
    assert worst <= 1.0, f"{tag}: images {at[0]}..{at[-1]} outside the fp64 bar, ratio {worst:.3g}"
    for i in range(0, n, tn):
        j = min(n, i + tn)
        o2 = None if out2 is None else torch.empty_like(out2[i:j])
        one = L.tc_conv(x[i:j], w_nk, bias, residual=None if residual is None else residual[i:j], out2=o2, **k)
        _same_bits(f"{tag} images {i}..{j - 1}", out[i:j], one)
        if o2 is not None:
            _same_bits(f"{tag} images {i}..{j - 1} second output", out2[i:j], o2)
        if gn is not None:
            torch.testing.assert_close(gn[0][i:j], one._gn_sums[0], rtol=1e-12, atol=0, msg=lambda m: f"{tag} images {i}..{j - 1} gn sums: {m}")
    return worst


def _bias_res(n, h, w, cout, seed, residual):
    b = torch.randn(cout, generator=_gen(seed + 7), device="cuda")
    r = torch.randn((n, h, w, cout), generator=_gen(seed + 8), device="cuda") if residual else None
    return b, r


@pytest.mark.parametrize("n,hw,cin,cout,residual,gn,need", [
    (3, (128, 128), 128, 128, True, 32, 3),       # 384 tiles
    (3, (128, 128), 128, 128, False, 0, 3),
    (2, (128, 128), 128, 128, True, 32, 2),       # 256 tiles: CTAs finish after 1 or 2
    (9, (64, 64), 128, 128, True, 32, 3),         # 288 tiles
    (17, (32, 32), 128, 256, True, 32, 3),        # two n tiles: a CTA's walk mixes them
    (8, (40, 20), 64, 256, True, 32, 2),          # ragged 40 x 20: border tiles, 160 tiles
], ids=["128sq-n3-res-gn", "128sq-n3", "128sq-n2", "64sq-n9", "32sq-n17-cout256", "40x20-n8"])
def test_exact_halo_conv_walk(L, n, hw, cin, cout, residual, gn, need):
    """The exact split-fp16 halo conv (TN = 1, four resident halo buffers whose parity runs on across tiles)."""
    h, w = hw
    seed = n * 1000 + h + cin
    x, w_nk = _conv_operands("exact", n, h, w, cin, cout, seed)
    b, r = _bias_res(n, h, w, cout, seed, residual)
    _conv_case(L, f"exact halo {n} x {h}x{w} {cin}->{cout}{' res' if residual else ''}{' gn' if gn else ''}", x, w_nk, b, need,
               residual=r, gn_groups=gn)


def test_exact_halo_conv_walk_residual_aliased_to_output(L):
    """The residual given as the output buffer itself (out = conv(x) + out), at 3 x 128^2."""
    n, h, w, c = 3, 128, 128, 128
    x, w_nk = _conv_operands("exact", n, h, w, c, c, 77)
    b, r = _bias_res(n, h, w, c, 77, True)
    tag = "exact halo aliased residual"
    _conv_plan(L, tag, x, w_nk, 3)
    before, check = lc.CHECKERS["tc_conv"]
    out = r.clone()
    ba = lc.bind(L.tc_conv, x, w_nk, b, residual=out, out=out, gn_groups=32)
    st = before(ba, random.Random(0))
    st["images"] = list(range(n))
    L.tc_conv(x, w_nk, b, residual=out, out=out, gn_groups=32)
    torch.cuda.synchronize()
    worst = check(ba, out, st)
    print(f"[fp64 {tag}] every image of {n}: worst ratio {worst:.3g}")
    assert worst <= 1.0
    for i in range(n):
        one = r[i:i + 1].clone()
        L.tc_conv(x[i:i + 1], w_nk, b, residual=one, out=one, gn_groups=32)
        _same_bits(f"{tag} image {i}", out[i:i + 1], one)


def test_exact_halo_conv_walk_at_the_benchmark_shape(L):
    """bench.py's roofline launch: the exact halo conv at 288 x 128^2, 128 -> 128, with a residual (36 864 tiles, up to 280 per CTA on 132
    SMs).  Every one of the 288 images is held to the fp64 bar and to a launch of that image alone."""
    n, h, w, c = 288, 128, 128, 128
    x, w_nk = _conv_operands("exact", n, h, w, c, c, 288)
    b, r = _bias_res(n, h, w, c, 288, True)
    _conv_case(L, "benchmark shape 288 x 128x128 128->128 res", x, w_nk, b, 3, residual=r, chunk=8)


@pytest.mark.parametrize("n,hw,cin,cout,gn", [
    (9, (32, 32), 256, 256, 32),                  # 144 tiles
    (67, (8, 8), 256, 512, 32),                   # TN = 2, odd image count: the last tile is half empty
])
def test_exact_tap_box_conv_walk(L, n, hw, cin, cout, gn):
    """The exact tap-box conv (one shifted TMA box per tap, 3 product passes through the weight ring)."""
    h, w = hw
    x, w_nk = _conv_operands("exact", n, h, w, cin, cout, n + cin)
    b, _ = _bias_res(n, h, w, cout, n, False)
    _conv_case(L, f"exact tap-box {n} x {h}x{w} {cin}->{cout}", x, w_nk, b, 2, gn_groups=gn)


def test_exact_downsample_conv_walk(L):
    """The exact stride-2 Downsample: a space-to-depth split operand and the TAPS_S2D tap table, 34 x 64^2 -> 32^2 (272 tiles)."""
    n, c = 34, 128
    x, w_nk = _conv_operands("exact", n, 64, 64, c, c, 342, s2d=True)
    b, _ = _bias_res(n, 32, 32, c, 342, False)
    _conv_case(L, "exact downsample 34 x 64x64 128->128", x, w_nk, b, 3, taps=L.TAPS_S2D, coffs=L.s2d_coffs(c), cin=c, gn_groups=32)


@pytest.mark.parametrize("cin,out_bf16", [(64, False), (128, True)], ids=["cin64-odd-blocks", "cin128-bf16-out"])
def test_bf16_halo_conv_walk(L, cin, out_bf16):
    """The bf16 halo conv at 3 x 128^2 (384 tiles): one channel block (odd, so the halo double buffer alternates across tiles), and two
    channel blocks with an fp32 + bf16 output and the fused GroupNorm sums."""
    n, h, w, cout = 3, 128, 128, 128
    x, w_nk = _conv_operands("bf16", n, h, w, cin, cout, 500 + cin)
    b, r = _bias_res(n, h, w, cout, 500 + cin, True)
    _conv_case(L, f"bf16 halo 3 x 128x128 {cin}->{cout}", x, w_nk, b, 3, residual=r, gn_groups=32,
               out2_dtype=torch.bfloat16 if out_bf16 else None)


@pytest.mark.parametrize("n,hw,cin,cout,need", [(3, (128, 128), 128, 128, 3), (8, (40, 20), 64, 256, 2)], ids=["128sq-n3", "40x20-n8"])
def test_normalise_on_load_walk(L, n, hw, cin, cout, need):
    """GroupNorm + swish applied to each halo tile with the statistics of that tile's image: consecutive tiles of a CTA lie in different
    images, so statistics read for the wrong image fail both checks."""
    h, w = hw
    seed = 600 + n
    xr = (torch.randn((n, h, w, cin), generator=_gen(seed), device="cuda") * 1.3
          + torch.randn((n, 1, 1, cin), generator=_gen(seed + 1), device="cuda"))          # a different mean per image and channel
    x = xr.bfloat16()
    xg = x.double().reshape(n, h * w, 32, cin // 32)
    mean, var = xg.mean((1, 3)), xg.var((1, 3), unbiased=False)
    mr = torch.stack([mean, 1.0 / torch.sqrt(var + 1e-6)], -1).float().contiguous()
    ga = 1 + 0.1 * torch.randn(cin, generator=_gen(seed + 2), device="cuda")
    be = 0.1 * torch.randn(cin, generator=_gen(seed + 3), device="cuda")
    wt = (torch.randn((cout, 9 * cin), generator=_gen(seed + 4), device="cuda") / (9 * cin) ** 0.5).bfloat16()
    b, r = _bias_res(n, h, w, cout, seed, True)
    tag = f"normalise-on-load {n} x {h}x{w} {cin}->{cout}"
    _conv_plan(L, tag, x, wt, need)
    before, check = lc.CHECKERS["tc_conv"]
    norm = (mr, ga, be, 32, True)
    ba = lc.bind(L.tc_conv, x, wt, b, residual=r, gn_groups=32, norm=norm)
    st = before(ba, random.Random(0))
    st["images"] = list(range(n))
    out = L.tc_conv(x, wt, b, residual=r, gn_groups=32, norm=norm)
    torch.cuda.synchronize()
    worst = check(ba, out, st)
    print(f"[fp64 {tag}] every image of {n}: worst ratio {worst:.3g}")
    assert worst <= 1.0, f"{tag}: outside the fp64 bar, ratio {worst:.3g}"
    for i in range(n):
        one = L.tc_conv(x[i:i + 1], wt, b, residual=r[i:i + 1], gn_groups=32, norm=(mr[i:i + 1].contiguous(), ga, be, 32, True))
        _same_bits(f"{tag} image {i}", out[i:i + 1], one)
        torch.testing.assert_close(out._gn_sums[0][i:i + 1], one._gn_sums[0], rtol=1e-12, atol=0)


def test_tf32_halo_conv_walk(L):
    """The TF32 halo conv at 9 x 64^2, 128 -> 128 (288 tiles)."""
    n, h, w, c = 9, 64, 64, 128
    x, w_nk = _conv_operands("tf32", n, h, w, c, c, 700)
    b, r = _bias_res(n, h, w, c, 700, True)
    _conv_case(L, "tf32 halo 9 x 64x64 128->128", x, w_nk, b, 3, residual=r, gn_groups=32)


# ----------------------------------------------------------------------------------------------- b. GEMMs
def _gemm_plan(L, tag, args, k, need):
    M, N = k["M"], k["N"]
    b1, b2 = k.get("batch", (1, 1))
    bn = lc.tc_block_n(N)
    tiles = -(-M // lc.TC_BM) * -(-N // bn) * b1 * b2
    _walk(tag, L.tc_gemm(*args, plan=True, **k), dict(block_n=bn, exact=int(args[0].dtype == torch.float16), tiles=tiles), need)


def _gemm_case(L, tag, A, B, out, need=2, fresh=None, **k):
    """One many-tile tc_gemm launch: the plan, every batch entry and row against fp64, and every batch entry against a launch of it alone
    (``fresh()`` gives the output buffer of a single launch in its state before the call: the residual when it is aliased)."""
    _gemm_plan(L, tag, (A, B, out), k, need)
    before, check = lc.CHECKERS["tc_gemm"]
    ba = lc.bind(L.tc_gemm, A, B, out, **k)
    st = before(ba, random.Random(0))
    b1n, b2n = ba["batch"]
    L.tc_gemm(A, B, out, **k)
    torch.cuda.synchronize()
    st["batches"], st["rows"] = list(range(b1n * b2n)), torch.arange(ba["M"])
    worst = check(ba, out, st)
    print(f"[fp64 {tag}] every batch entry and row of {b1n} x {b2n} x {ba['M']}: worst ratio {worst:.3g}")
    assert worst <= 1.0, f"{tag}: outside the fp64 bar, ratio {worst:.3g}"
    koffs = ba["k_offsets"]
    for bi in range(b1n * b2n):
        i1, i2 = divmod(bi, b2n)
        one = fresh() if fresh is not None else torch.full_like(out, float("nan"))
        kk = dict(k, batch=(1, 1), a_off=ba["a_off"] + i1 * ba["a_bs"][0] + i2 * ba["a_bs"][1],
                  b_off=ba["b_off"] + i1 * ba["b_bs"][0] + i2 * ba["b_bs"][1], c_off=ba["c_off"] + i1 * ba["c_bs"][0] + i2 * ba["c_bs"][1],
                  a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0), k_offsets=None if koffs is None else [koffs[i1]])
        kk.pop("out2", None)                      # a second output is compared by the caller
        if k.get("residual") is not None and fresh is not None:
            kk["residual"] = one
        L.tc_gemm(A, B, one, **kk)
        c0 = kk["c_off"]
        sl = lambda t: lc.view(t, c0, (ba["M"], ba["N"]), (ba["ldc"], 1))
        _same_bits(f"{tag} batch entry {bi}", sl(out), sl(one))
    return worst


def _mat(shape, seed, scale=1.0):
    return torch.randn(shape, generator=_gen(seed), device="cuda") * scale


def test_exact_split_gemm_walk(L):
    """Split-fp16 GEMM (lo_a / lo_b halves) with batch strides on both batch axes and a shared B: 8 x 2 tiles x 9 entries = 144 tiles."""
    M, N, K, b1, b2 = 1024, 256, 192, 3, 3
    A = _split(_mat((b1, b2, M, K), 800) * 1.5)
    B = _split(_mat((b2, N, K), 801) / K ** 0.5)
    out = torch.empty((b1, b2, M, N), device="cuda")
    _gemm_case(L, "exact split gemm 3x3 x 1024x256 K192", A, B, out, M=M, N=N, K=K, lda=2 * K, ldb=2 * K, ldc=N, batch=(b1, b2),
               a_bs=(b2 * M * 2 * K, M * 2 * K), b_bs=(0, N * 2 * K), c_bs=(b2 * M * N, M * N), bias=_mat(N, 802), bias_mode=L.BIAS_N)


def test_bf16_gemm_walk_bias_m_gelu(L):
    """bf16 GEMM, BIAS_M + GELU, fp32 and bf16 outputs, batch (3, 3) with A shared along the second batch axis: 144 tiles."""
    M, N, K, b1, b2 = 1024, 256, 256, 3, 3
    A = _mat((b1, M, K), 810).bfloat16()
    B = (_mat((b1, b2, N, K), 811) / K ** 0.5).bfloat16()
    out, out2 = torch.empty((b1, b2, M, N), device="cuda"), torch.empty((b1, b2, M, N), dtype=torch.bfloat16, device="cuda")
    k = dict(M=M, N=N, K=K, lda=K, ldb=K, ldc=N, batch=(b1, b2), a_bs=(M * K, 0), b_bs=(b2 * N * K, N * K), c_bs=(b2 * M * N, M * N),
             bias=_mat(M, 812), bias_mode=L.BIAS_M, act=L.ACT_GELU)
    _gemm_case(L, "bf16 gemm bias_m gelu", A, B, out, out2=out2, **k)
    L.tc_gemm(A, B, out, out2=out2, **k)
    for bi in range(b1 * b2):                     # the bf16 copy of every entry against a single launch
        i1, i2 = divmod(bi, b2)
        o32, o16 = torch.empty((M, N), device="cuda"), torch.empty((M, N), dtype=torch.bfloat16, device="cuda")
        L.tc_gemm(A[i1], B[i1, i2], o32, out2=o16, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, bias=k["bias"], bias_mode=L.BIAS_M, act=L.ACT_GELU)
        _same_bits(f"bf16 gemm bias_m gelu entry {bi} bf16 output", out2[i1, i2], o16)


def test_tf32_gemm_walk_residual_aliased(L):
    """TF32 GEMM with BIAS_N and the residual aliased to the output, batch (2, 1): 8 x 9 x 2 = 144 tiles, N tail (1100 = 8 x 128 + 76)."""
    M, N, K, b1 = 1024, 1100, 96, 2
    A = _mat((b1, M, K), 820)
    B = _mat((N, K), 821) / K ** 0.5
    R = _mat((b1, M, N), 822)
    out = R.clone()
    _gemm_case(L, "tf32 gemm aliased residual", A, B, out, fresh=lambda: R.clone(), M=M, N=N, K=K, lda=K, ldb=K, ldc=N, batch=(b1, 1),
               a_bs=(M * K, 0), c_bs=(M * N, 0), bias=_mat(N, 823), bias_mode=L.BIAS_N, residual=out)


def test_bf16_gemm_walk_k_offsets(L):
    """K offsets (the weight-gradient layout: batch1 index b reads A shifted by k_offsets[b] along K), batch (3, 4): 12 x 12 = 144 tiles."""
    M, N, K, b2 = 512, 384, 128, 4
    koffs = [0, 72, 144]
    A = _mat((b2, M, K + 144), 830).bfloat16()
    B = (_mat((3, b2, N, K), 831) / K ** 0.5).bfloat16()
    out = torch.empty((3, b2, M, N), device="cuda")
    _gemm_case(L, "bf16 gemm k offsets", A, B, out, M=M, N=N, K=K, lda=K + 144, ldb=K, ldc=N, batch=(3, b2), a_bs=(0, M * (K + 144)),
               b_bs=(b2 * N * K, N * K), c_bs=(b2 * M * N, M * N), k_offsets=koffs)


def test_causal_gemms_walk(L):
    """The attention's causal GEMMs with batch > 1: QK^T with skipped n tiles (8 x 8 tiles per scene, 28 skipped, 3 scenes: 192 tiles, so
    skipped and live tiles interleave in one CTA's walk) and P.V with the k limit (20 scenes x 8 tiles = 160)."""
    S, dh, blk = 1024, 64, 64
    B = 3
    q, kk = _mat((B, S, dh), 840).bfloat16(), _mat((B, S, dh), 841).bfloat16()
    sc = torch.zeros((B, S, S), device="cuda")              # skipped tiles are never written: they stay 0 here and in the single launches
    k = dict(M=S, N=S, K=dh, lda=dh, ldb=dh, ldc=S, batch=(B, 1), a_bs=(S * dh, 0), b_bs=(S * dh, 0), c_bs=(S * S, 0), causal_block=blk,
             causal_skip_n=True)
    _gemm_case(L, "causal qk^T skip", q, kk, sc, fresh=lambda: torch.zeros_like(sc), **k)
    view = torch.arange(S, device="cuda") // blk
    B = 20
    p = (torch.rand((B, S, S), generator=_gen(842), device="cuda") * (view[:, None] >= view[None, :])).bfloat16()
    vt = _mat((B, dh, S), 843).bfloat16()
    o = torch.empty((B, S, dh), device="cuda")
    _gemm_case(L, "causal p.v k limit", p, vt, o, M=S, N=dh, K=S, lda=S, ldb=S, ldc=dh, batch=(B, 1), a_bs=(S * S, 0), b_bs=(dh * S, 0),
               c_bs=(S * dh, 0), causal_block=blk)


def test_gemm_walk_by_row_blocks(L):
    """An unbatched bf16 GEMM of 24 x 8 = 192 tiles against launches of each 128-row block alone."""
    M, N, K = 3000, 1024, 128
    A, B = _mat((M, K), 850).bfloat16(), (_mat((N, K), 851) / K ** 0.5).bfloat16()
    out = torch.empty((M, N), device="cuda")
    k = dict(M=M, N=N, K=K, lda=K, ldb=K, ldc=N, bias=_mat(N, 852), bias_mode=L.BIAS_N)
    _gemm_plan(L, "bf16 gemm row blocks", (A, B, out), k, 2)
    with pytest.raises(L.LibraryError, match="row strides"):     # the plan validates a parameter block as the launch does
        L.tc_gemm(A, B, out, plan=True, **dict(k, lda=K + 1))
    before, check = lc.CHECKERS["tc_gemm"]
    ba = lc.bind(L.tc_gemm, A, B, out, **k)
    st = before(ba, random.Random(0))
    L.tc_gemm(A, B, out, **k)
    torch.cuda.synchronize()
    st["rows"] = torch.arange(M)
    worst = check(ba, out, st)
    print(f"[fp64 bf16 gemm row blocks] every row of {M}: worst ratio {worst:.3g}")
    assert worst <= 1.0
    for m0 in range(0, M, 128):
        m = min(128, M - m0)
        one = torch.empty((m, N), device="cuda")
        L.tc_gemm(A[m0:m0 + m], B, one, **dict(k, M=m))
        _same_bits(f"bf16 gemm rows {m0}..{m0 + m - 1}", out[m0:m0 + m], one)


# ----------------------------------------------------------------------------------------------- c. weight gradients
@pytest.mark.parametrize("bf16,n,hw,cin,cout", [(False, 2, 16, 256, 256), (True, 2, 16, 128, 128)], ids=["split-256", "bf16-128"])
def test_conv_wgrad_walk(L, bf16, n, hw, cin, cout):
    """conv_wgrad_tc / conv_wgrad_bf16 where the split-K plan (splits = ceil(132 / (3 x tiles))) gives more tiles than SMs: 256 -> 256
    makes 144 tiles, 128 -> 128 makes 135, so some CTAs walk 2.  dW against fp64, and every (block, split) partial product of the
    batched GEMM against a launch of that entry alone."""
    name = "conv_wgrad_bf16" if bf16 else "conv_wgrad_tc"
    x = _mat((n, hw, hw, cin), 900 + cin) * 1.5
    dy = _mat((n, hw, hw, cout), 901 + cin)
    dw = _mat((9 * cin, cout), 902)
    before, check = lc.CHECKERS[name]
    fn = getattr(L, name)
    ba = lc.bind(fn, x, dy, dw)
    st = before(ba, random.Random(0))
    fn(x, dy, dw)
    torch.cuda.synchronize()
    worst = check(ba, dw, st)
    # the launch, restated from _wgrad_tc's plan
    pitch = (hw + 2 + 7) // 8 * 8
    klen, margin, M = n * (hw + 2) * pitch, pitch + 8, 3 * cin
    splits = max(1, min(64, -(-132 // (3 * (M // 128) * (cout // 128)))))
    kc = (-(-klen // splits) + 63) // 64 * 64
    la, lb = kc * splits + 2 * margin, kc * splits
    at, bt, partial = L._wgrad_bufs[(bf16, True, x.device, tuple(dy.shape[:-1]), cin, cout)]
    assert partial.shape == (3, splits, M, cout)
    ld = 1 if bf16 else 2
    koffs = [margin - pitch, margin, margin + pitch]
    k = dict(M=M, N=cout, K=kc, lda=ld * la, ldb=ld * lb, ldc=cout, lo_a=la, lo_b=lb)
    tag = f"{name} {n} x {hw}x{hw} {cin}->{cout}, {splits} splits"
    _gemm_plan(L, tag, (at, bt, partial), dict(k, batch=(3, splits), a_bs=(0, kc), b_bs=(0, kc), c_bs=(splits * M * cout, M * cout),
                                                k_offsets=koffs), 2)
    print(f"[fp64 {tag}] dW: worst ratio {worst:.3g}")
    assert worst <= 1.0, f"{tag}: dW outside the fp64 bar, ratio {worst:.3g}"
    one = torch.full_like(partial, float("nan"))
    for b1 in range(3):
        for s in range(splits):
            L.tc_gemm(at, bt, one[b1, s], a_off=s * kc, b_off=s * kc, k_offsets=[koffs[b1]], **k)
    _same_bits(f"{tag} partial products", partial, one)

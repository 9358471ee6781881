"""The fused attention's persistent walk at the sizes the workloads launch it: against fp64, and against its own single-item bits.

attn_block_causal_kernel (viewformer_b200/csrc/vf_attn_fused.cu) is persistent.  The inference instance launches min(items, 2 SMs) CTAs,
the training instance min(items, SMs), items = B H n_qtiles, and CTA c walks items c, c + grid, c + 2 grid, ..., heaviest query tile
first.  What one item leaves behind for the next is where such a kernel goes wrong: the double-buffered Q tile and the producer's
q_empty wait from the third item on, the K (4 slots) and V (3 slots) rings whose counters and parities run on across items of different
n_kt, the per-item reset of O and of the softmax statistics, the multi-end schedule of streams >= 1, and the first-tile / skipped-tile
arithmetic of the KV-cache decode.  Each case here

* computes, from the launcher's formulas and this GPU's SM count, how many items its busiest CTA walks, prints it and asserts >= 2
  (>= 3 at the benchmark's shape), so that a GPU with more SMs cannot pass the test without walking;
* checks every (batch, head) pair against fp64 with the checkers and bars of tests/launch_checks.py, and prints the worst ratio with the
  (query tile, CTA, iteration) of the worst pair's items;
* at rate 0 requires each scene's forward output (and out_f32 and the LSE of the training instance) to equal, bit for bit, a launch of
  that scene alone, in which no CTA walks a second item.  An item's arithmetic depends neither on the CTA that runs it nor on the
  order, so this is exact and sees a leak far below the fp64 bar.  With dropout the mask's element index contains b, so there only the
  fp64 bar applies.

The last test replays the benchmark's CUDA graph at its own size (32 scenes x 10 views) and requires it to equal the eager call.  The
launch audit checks eager calls only; with this equality its `mixed-generate-bench` workload holds every launch of the timed step.

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), worst ratio to the fp64 bar over every (b, h) and the items of the busiest
CTA; every bit comparison equal; the file runs in about 20 s:
  inference, one query tile per scene: resident - 1 0.79 (1 item, the control), resident + 1 0.85 (2), 2 resident + 1 0.82 (3).
  benchmark shape (32 x 12 heads, S = 640, 8 items): 0.86, growing logits 0.95; multi-end streams 1 / 2: T = 10 0.86 / 0.85, T = 9
      0.85 / 0.88.
  KV-cache decode (2 items): Tc = 9 0.75, Tc = 19 0.74 (empty slot), Tc = 10 0.77.
  training forward (5 items), streams 0 / 1 / 2: rate 0 0.89 / 0.91 / 0.84, rate 0.1 0.90 / 0.92 / 0.84; backward 0.86 / 0.87.
  graphed benchmark step: 384 launches per replay, generated codes and pixels equal to the eager call.
Two kernel mutants fail these tests: O, m and l initialised once per CTA instead of once per item (every case with a second item,
fp64 ratios 7e2 .. 3e7), and the third item's Q read from the second item's buffer (the cases with three or more items per CTA).  No
earlier kernel, model, transformer-training, baseline-configuration or launch-audit test failed with either; the end-to-end bar of
test_c2_benchmarked_mode_vs_exact_on_all_scenes (generated-code agreement >= 0.90) passed with both.
"""
import random

import pytest
import torch

import launch_checks as lc
from oracle import synth
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu

BLK, DH = 64, 64


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


@pytest.fixture(autouse=True)
def dropout_hook(L, monkeypatch):
    dropout = L.dropout
    monkeypatch.setitem(lc.HOOKS, "dropout_mask", lambda shape, rate, seed, device: dropout(
        torch.ones(shape, dtype=torch.float32, device=device), rate, seed))


def _resident(train):
    return (1 if train else 2) * torch.cuda.get_device_properties(0).multi_processor_count


def _walk(tag, B, H, S, train, first_query=0, need=2):
    """Items of the launch and of its busiest CTA; asserts that CTA walks at least ``need`` items (need 1: exactly one, the control)."""
    items = lc.attn_items(B, H, S, first_query)
    grid = min(items, _resident(train))
    per_cta = -(-items // grid)
    print(f"[walk {tag}] {items} items on {grid} CTAs ({_resident(train)} resident): up to {per_cta} items per CTA")
    if need == 1:
        assert per_cta == 1, f"{tag}: the control case must give every CTA one item, the busiest walks {per_cta}"
    assert per_cta >= need, f"{tag}: the busiest CTA walks {per_cta} items, the case needs {need}; make the launch larger for this GPU"
    return per_cta


def _single(B, H, S, train, first_query=0):
    """Asserts that a launch of this size gives every CTA at most one item (the per-scene launches the bits are compared with)."""
    items = lc.attn_items(B, H, S, first_query)
    assert items <= _resident(train), f"a single-scene launch has {items} items, more than the {_resident(train)} resident CTAs"


def _items_of(b, h, B, H, S, train, first_query=0, qtiles=None):
    """(query tile, CTA, iteration) of pair (b, h)'s items in the launch's walk."""
    qt0 = first_query // lc.ATTN_QT
    n_qt = -(-S // lc.ATTN_QT) - qt0
    items = lc.attn_items(B, H, S, first_query)
    grid = min(items, _resident(train))
    out = []
    for qt in (range(qt0, qt0 + n_qt) if qtiles is None else qtiles):
        i = (qt0 + n_qt - 1 - qt) * B * H + b * H + h
        out.append((qt, i % grid, i // grid))
    return out


def _checked(L, name, *a, **k):
    """Call _lib.<name>, then hold every (batch, head) pair to the launch checker's fp64 bar.  Returns (result, worst ratio, worst pair)."""
    fn = getattr(L, name)
    before, check = lc.CHECKERS[name]
    ba = lc.bind(fn, *a, **k)
    st = before(ba, random.Random(0))
    result = fn(*a, **k)
    torch.cuda.synchronize()
    worst, where = -1.0, None
    for pair in [(b, h) for b in range(ba["B"]) for h in range(ba["H"])]:
        st["heads"] = [pair]
        r = check(ba, result, st)
        if r > worst:
            worst, where = r, pair
    return result, worst, where


def _report(tag, worst, pair, B, H, S, train, first_query=0):
    b, h = pair
    print(f"[fp64 {tag}] every (b, h) of {B} x {H}: worst ratio {worst:.3g} at b {b} h {h}, items (query tile, CTA, iteration) "
          f"{_items_of(b, h, B, H, S, train, first_query)}")
    assert worst <= 1.0, f"{tag}: (b {b}, h {h}) outside the fp64 bar, ratio {worst:.3g}"


def _same_bits(tag, got, want, where):
    """got == want bit for bit; on a mismatch the message names the first differing element through ``where(index)``."""
    assert got.dtype == want.dtype and got.shape == want.shape
    it = {2: torch.int16, 4: torch.int32}[got.element_size()]
    diff = (got.view(it) != want.view(it)).nonzero()
    assert diff.shape[0] == 0, f"{tag}: {diff.shape[0]} elements differ from the single-scene launch, first at {where(tuple(diff[0].tolist()))}"


def _rows_where(b, S, train, B, H, first_query=0):
    """Describes element (row, column) of scene b's [S, d] output by its query tile, head, CTA and iteration."""
    def where(ix):
        row, col = ix
        qt = row // lc.ATTN_QT
        return f"b {b} row {row} h {col // DH}: (query tile, CTA, iteration) {_items_of(b, col // DH, B, H, S, train, first_query, [qt])}"
    return where


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _operands(B, T, H, ns=1, seed=0, growing=False):
    """qk bf16 [B, ns S, 2d] (x 0.5, keys optionally growing from view to view) and V^T bf16 [B, d, ns S], as the kernel tests build them."""
    d, S = H * DH, T * BLK
    qk = torch.randn((B, ns * S, 2 * d), generator=_gen(seed), device="cuda") * 0.5
    if growing:                                  # later views: larger keys, so the row's reference maximum moves inside later items
        qk[..., d:] *= (1.0 + 0.9 * (torch.arange(ns * S, device="cuda") % S // BLK).float())[None, :, None]
    vt = torch.randn((B, d, ns * S), generator=_gen(seed + 1), device="cuda")
    return qk.bfloat16(), vt.bfloat16()


# ----------------------------------------------------------------------------------------------- a. single-stream inference
def _inference_case(L, tag, B, T, H, need, qk=None, vt=None):
    S, d = T * BLK, H * DH
    _walk(tag, B, H, S, False, need=need)
    if qk is None:
        qk, vt = _operands(B, T, H, seed=B + T)
    out, worst, pair = _checked(L, "attn_block_causal", qk, vt, B, S, H, d, BLK)
    _report(tag, worst, pair, B, H, S, False)
    _single(1, H, S, False)
    o = out.reshape(B, S, d)
    for b in range(B):
        one = L.attn_block_causal(qk[b:b + 1].contiguous(), vt[b:b + 1].contiguous(), 1, S, H, d, BLK)
        _same_bits(f"{tag} scene {b}", o[b], one, _rows_where(b, S, False, B, H))


@pytest.mark.parametrize("case", ["resident-1", "resident+1", "2resident+1"])
def test_inference_walk_at_the_resident_boundary(L, case):
    """B scenes of one 128-row query tile and one head, so items = B exactly: resident - 1 (the control, one item per CTA), resident + 1
    (CTA 0 walks a second item) and 2 resident + 1 (CTA 0 walks a third, whose Q sits in the buffer the first one used)."""
    R = _resident(False)
    B, need = {"resident-1": (R - 1, 1), "resident+1": (R + 1, 2), "2resident+1": (2 * R + 1, 3)}[case]
    _inference_case(L, f"inference {case} (B {B})", B, 2, 1, need)


@pytest.mark.parametrize("growing", [False, True], ids=["plain", "growing-logits"])
def test_inference_walk_at_the_benchmark_shape(L, growing):
    """The benchmark's attention launch: 32 scenes x 10 views (S = 640), 12 heads; growing keys make the reference maximum move inside
    the later items of every CTA."""
    B, T, H = 32, 10, 12
    qk, vt = _operands(B, T, H, seed=101, growing=growing)
    _inference_case(L, f"inference benchmark shape{' growing logits' if growing else ''}", B, T, H, 3, qk, vt)


# ----------------------------------------------------------------------------------------------- b. multi-end streams 1 and 2
@pytest.mark.parametrize("T", [10, 9])
def test_multiend_streams_walk(L, T):
    """Streams 1 and 2 of the branching attention (n_kt = q0 / 64 + 3, or + 1 for the last tile of an odd T) at 32 scenes x 12 heads."""
    B, H, ns = 32, 12, 3
    S, d = T * BLK, H * DH
    qk, vt = _operands(B, T, H, ns=ns, seed=200 + T)
    _single(1, H, S, False)
    for s in (1, 2):
        tag = f"multi-end stream {s} T {T}"
        _walk(tag, B, H, S, False, need=3)
        out, worst, pair = _checked(L, "attn_block_multiend", qk, vt, B, S, ns, s, H, d, BLK)
        _report(tag, worst, pair, B, H, S, False)
        o = out.reshape(B, S, d)
        for b in range(B):
            one = L.attn_block_multiend(qk[b:b + 1].contiguous(), vt[b:b + 1].contiguous(), 1, S, ns, s, H, d, BLK)
            _same_bits(f"{tag} scene {b}", o[b], one, _rows_where(b, S, False, B, H))


# ----------------------------------------------------------------------------------------------- c. KV-cache decode
@pytest.mark.parametrize("Tc", [9, 19, 10])
def test_kv_cache_decode_walk(L, Tc):
    """The padded KV-cache layout of MIGT.prefill_context at 32 scenes x 12 heads: Tc context views, an empty view slot full of huge values
    when Tc is odd (skip_view), the query view at the start of a 128-row tile (first_query); rows below that tile stay untouched."""
    B, H = 32, 12
    d, pad = H * DH, Tc % 2
    S = (Tc + pad + 1) * BLK
    r0 = (Tc + pad) * BLK
    skip = Tc if pad else -1
    qk = torch.full((B, S, 2 * d), 300.0, device="cuda")
    vt = torch.full((B, d, S), -77.0, device="cuda")
    cq, cv = _operands(B, Tc + 1, H, seed=300 + Tc)
    qk[:, :Tc * BLK], qk[:, r0:] = cq[:, :Tc * BLK], cq[:, Tc * BLK:]
    vt[:, :, :Tc * BLK], vt[:, :, r0:] = cv[:, :, :Tc * BLK], cv[:, :, Tc * BLK:]
    qk, vt = qk.bfloat16(), vt.bfloat16()
    tag = f"decode Tc {Tc}{' (empty slot)' if pad else ''}"
    _walk(tag, B, H, S, False, first_query=r0, need=2)
    out = torch.full((B * S, d), 7.0, dtype=torch.bfloat16, device="cuda")
    out, worst, pair = _checked(L, "attn_block_causal", qk, vt, B, S, H, d, BLK, first_query=r0, out=out, skip_view=skip)
    _report(tag, worst, pair, B, H, S, False, first_query=r0)
    _single(1, H, S, False, first_query=r0)
    o = out.reshape(B, S, d)
    for b in range(B):
        one = torch.full((S, d), 7.0, dtype=torch.bfloat16, device="cuda")
        L.attn_block_causal(qk[b:b + 1].contiguous(), vt[b:b + 1].contiguous(), 1, S, H, d, BLK, first_query=r0, out=one, skip_view=skip)
        _same_bits(f"{tag} scene {b}", o[b], one, _rows_where(b, S, False, B, H, r0))


# ----------------------------------------------------------------------------------------------- d., e. training forward and backward
TRAIN_B, TRAIN_T, TRAIN_H, TRAIN_NS, TRAIN_SEED = 5, 20, 12, 3, 4242       # scripts/bench_migt_train.py's step: 600 items per stream


@pytest.fixture(scope="module", params=[0.0, 0.1], ids=["rate0", "rate0.1"])
def train_forward(L, request):
    """qk, V^T and the training forward of every stream (O, out_f32, LSE) at B = 5, T = 20, 12 heads, 3 streams; the fp64 worst ratio
    per stream is measured in the test (the dropout hook is set per test)."""
    rate = request.param
    B, T, H, ns = TRAIN_B, TRAIN_T, TRAIN_H, TRAIN_NS
    S, d = T * BLK, H * DH
    qk, vt = _operands(B, T, H, ns=ns, seed=400)
    return dict(rate=rate, qk=qk, vt=vt, B=B, S=S, H=H, d=d, ns=ns)


def _train_forward_stream(L, f, s, out=None, lse=None, out_f32=None, B=None, qk=None, vt=None):
    B = f["B"] if B is None else B
    qk, vt = (f["qk"], f["vt"]) if qk is None else (qk, vt)
    S, H, d, ns = f["S"], f["H"], f["d"], f["ns"]
    if out is None:
        out = torch.empty((B * S, d), dtype=torch.bfloat16, device="cuda")
        lse = torch.empty((B, H, S), dtype=torch.float32, device="cuda")
        out_f32 = torch.empty((B * S, d), dtype=torch.float32, device="cuda")
    L.attn_multiend_train(qk, vt, B, S, ns, s, H, d, BLK, rate=f["rate"], seed=TRAIN_SEED + s, lse=lse, out_f32=out_f32, out=out)
    return out, lse, out_f32


def test_training_forward_walk(L, train_forward):
    """vf_attn_multiend_train on 132 resident CTAs: O, out_f32 and the LSE of every (b, h) and stream against fp64; at rate 0 also bit for
    bit against single-scene launches and against the inference instance at this size."""
    f = train_forward
    B, S, H, d, ns, rate = f["B"], f["S"], f["H"], f["d"], f["ns"], f["rate"]
    _single(1, H, S, True)
    o16 = torch.empty((ns, B * S, d), dtype=torch.bfloat16, device="cuda")
    o32 = torch.empty((ns, B * S, d), dtype=torch.float32, device="cuda")
    lse = torch.empty((ns, B, H, S), dtype=torch.float32, device="cuda")
    for s in range(ns):
        tag = f"training forward stream {s} rate {rate}"
        _walk(tag, B, H, S, True, need=2)
        _, worst, pair = _checked(L, "attn_multiend_train", f["qk"], f["vt"], B, S, ns, s, H, d, BLK, rate=rate, seed=TRAIN_SEED + s,
                                  lse=lse[s], out_f32=o32[s], out=o16[s])
        _report(tag, worst, pair, B, H, S, True)
        if rate > 0:
            continue
        o, l32, of = o16[s].reshape(B, S, d), lse[s], o32[s].reshape(B, S, d)
        for b in range(B):
            one, one_lse, one32 = _train_forward_stream(L, f, s, B=1, qk=f["qk"][b:b + 1].contiguous(), vt=f["vt"][b:b + 1].contiguous())
            where = _rows_where(b, S, True, B, H)
            _same_bits(f"{tag} scene {b} O", o[b], one, where)
            _same_bits(f"{tag} scene {b} out_f32", of[b], one32, where)
            _same_bits(f"{tag} scene {b} lse", l32[b], one_lse[0],
                       lambda ix, b=b: f"b {b} h {ix[0]} row {ix[1]}: (query tile, CTA, iteration) "
                                       f"{_items_of(b, ix[0], B, H, S, True, qtiles=[ix[1] // lc.ATTN_QT])}")
        inf = L.attn_block_multiend(f["qk"], f["vt"], B, S, ns, s, H, d, BLK)
        _same_bits(f"{tag} vs the inference instance", o16[s], inf, lambda ix: f"row {ix[0]} column {ix[1]}")


def test_training_backward_at_the_step_size(L, train_forward):
    """vf_attn_multiend_bwd (not persistent: one CTA per key view, stream and (b, h)) on the training forward's operands, every (b, h)
    against fp64.  dQ is summed with fp32 atomics, so no bit equality is asserted."""
    f = train_forward
    B, S, H, d, ns, rate = f["B"], f["S"], f["H"], f["d"], f["ns"], f["rate"]
    o32 = torch.empty((ns, B * S, d), dtype=torch.float32, device="cuda")
    lse = torch.empty((ns, B, H, S), dtype=torch.float32, device="cuda")
    for s in range(ns):
        _train_forward_stream(L, f, s, out=torch.empty((B * S, d), dtype=torch.bfloat16, device="cuda"), lse=lse[s], out_f32=o32[s])
    dout = torch.randn((ns, B * S, d), generator=_gen(500), device="cuda").bfloat16()
    tag = f"training backward rate {rate}"
    _, worst, pair = _checked(L, "attn_multiend_bwd", f["qk"], f["vt"], dout, o32, lse, B, S, ns, H, d, BLK, rate=rate, seed=TRAIN_SEED)
    print(f"[fp64 {tag}] every (b, h) of {B} x {H}, all {ns} streams: worst ratio {worst:.3g} at (b, h) {pair}")
    assert worst <= 1.0, f"{tag}: (b, h) {pair} outside the fp64 bar, ratio {worst:.3g}"


# ----------------------------------------------------------------------------------------------- f. the graphed benchmark step
def test_graphed_benchmark_step_equals_eager(L):
    """GraphedPredictions(32 scenes, 10 views), the step bench.py times, replayed once on the bench's own inputs == the eager
    generate_batch_predictions: generated codes and images bit for bit, cameras allclose (as tests/test_models_gpu.py at its toy size)."""
    import bench
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions, GraphedPredictions
    vcfg, tcfg = VQGANConfig(), MIGTConfig(localization_weight="0")
    cb = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, 0))
    tr = MIGT(tcfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(tcfg, 0))
    images, cams = bench.synth_inputs(32, 1234)
    S = bench.T_VIEWS * tcfg.token_image_size ** 2
    _walk("benchmark step attention", 32, tcfg.n_head, S, False, need=3)
    gp = GraphedPredictions(tr, cb, 32, bench.T_VIEWS)
    got = gp(images.pin_memory(), cams.pin_memory())
    got = {k: v.clone() for k, v in got.items() if isinstance(v, torch.Tensor)}
    want = generate_batch_predictions(tr, cb, images, cams)
    torch.cuda.synchronize()
    codes = int((got["generated_codes"] != want["generated_codes"]).sum())
    px = int((got["generated_images"] != want["generated_images"]).sum())
    print(f"[graphed benchmark step] launches per replay {gp.launches_per_replay}; differing codes {codes}, pixels {px}")
    assert torch.equal(got["generated_codes"], want["generated_codes"])
    assert torch.equal(got["generated_images"], want["generated_images"])
    assert torch.allclose(got["generated_cameras"], want["generated_cameras"])

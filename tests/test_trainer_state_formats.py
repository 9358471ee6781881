"""The two containers that carry trainer state, and the fine-tuning schedule, checked without a GPU against what can be run offline:
TensorFlow's generated ``TrackableObjectGraph`` proto (shipped inside tensorboard) for slot variables, real ``torch.optim.Adam`` for the
Lightning-layout ``optimizer_states``, and the reference's own ``AdamWeightDecay`` / ``WarmUp`` / ``MIGT`` / ``VQGAN`` objects (executed over
oracle/tf_shim.py; those parts skip where the reference sources are absent) for names, parameter order and the offset schedule.
Not checkable offline, and recorded as such in INTEGRATION.md: the names below TF 2.4's ``LossScaleOptimizer`` wrapper, whether TF 2.4
tracks a learning-rate schedule's variables, and pytorch-lightning's own reader."""
import hashlib
import math
import struct
import sys

import numpy as np
import pytest
import torch

from oracle import ref_loader
from oracle.make_golden import SMALL_VQ
from viewformer_b200 import tf_checkpoint as tfc
from viewformer_b200.config import MIGTConfig, VQGANConfig
from viewformer_b200.migt import MIGT
from viewformer_b200.train import adam_state_dict, read_adam_state_dict, trainable_names
from viewformer_b200.train_migt import warmup_cosine
from viewformer_b200.vqgan import VQGAN

pb = pytest.importorskip("tensorboard.compat.proto.trackable_object_graph_pb2")
needs_reference = pytest.mark.skipif(not ref_loader.migt_available(), reason="reference sources not present")

TINY = dict(n_layer=2, n_head=2, d_model=32, sequence_size=4, n_embeddings=64, token_image_size=2)


def _tiny_state(precision="bf16"):
    """(weights, MIGTTrainer.optimizer_state()-shaped dict) of the tiny model from integer-derived values (no generator involved)."""
    shapes = MIGT(MIGTConfig(**TINY)).param_shapes()
    fill = lambda s, i: torch.from_numpy(((np.arange(int(np.prod(s)), dtype=np.float32) % 251) * 0.5 - i).reshape(s))
    sd = {k: fill(s, i) for i, (k, s) in enumerate(shapes.items())}
    state = dict(m={k: v * 0.25 for k, v in sd.items()}, v={k: v * v for k, v in sd.items()}, iterations=12345, train_counter=45,
                 schedule_offset=12300, loss_scale=2.0 ** 13, loss_scale_counter=17, seed=3, precision=precision)
    return sd, state


def _graph(prefix):
    ck = tfc.Checkpoint(prefix)
    g = pb.TrackableObjectGraph()
    g.ParseFromString(ck.tensor(tfc.OBJECT_GRAPH_KEY))
    return ck, g


def _walk(g, path):
    nid = 0
    for part in path.split("/"):
        (nid,) = [c.node_id for c in g.nodes[nid].children if c.local_name == part]
    return nid


# ------------------------------------------------------------------------------------------------ 1. slot variables, both directions
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_slot_variables_written_here_parse_with_tensorflows_proto(tmp_path, precision):
    sd, state = _tiny_state(precision)
    tensors = {tfc.object_paths(k)[0]: v.numpy() for k, v in sd.items()}
    extra, slots = tfc.optimizer_entries(state)
    tensors.update(extra)
    prefix = str(tmp_path / "model")
    tfc.write_checkpoint(prefix, tensors, slots)
    ck, g = _graph(prefix)
    assert g.SerializeToString() == ck.tensor(tfc.OBJECT_GRAPH_KEY)          # canonical bytes for TensorFlow's generated code
    owner = "optimizer/base_optimizer" if precision == "bf16" else "optimizer"
    refs = g.nodes[_walk(g, owner)].slot_variables
    assert len(refs) == 2 * len(sd) and sum(len(n.slot_variables) for n in g.nodes) == len(refs)
    reachable = {c.node_id for n in g.nodes for c in n.children}
    by_ref = {(r.original_variable_node_id, r.slot_name): r.slot_variable_node_id for r in refs}
    for k in sd:
        path = tfc.object_paths(k)[0]
        for slot in ("m", "v"):
            nid = by_ref[(_walk(g, path), slot)]
            assert nid not in reachable                                      # a slot hangs off no parent: only the owner's reference leads to it
            (a,) = g.nodes[nid].attributes
            assert a.name == "VARIABLE_VALUE" and a.checkpoint_key == f"{path}/.OPTIMIZER_SLOT/{owner}/{slot}{tfc.VAR_SUFFIX}"
            assert np.array_equal(ck.tensor(a.checkpoint_key, verify_crc=True), state[slot][k].numpy())
            assert ck.slot(path, slot, owner) == a.checkpoint_key
    with pytest.raises(KeyError):
        ck.slot("ln_f/gamma", "vhat", owner)
    # the reader hands back what the writer was given, weights untouched by the extra entries
    back = tfc.load_optimizer_state(prefix, list(sd))
    want = {k: v for k, v in state.items() if precision == "bf16" or not k.startswith("loss_scale")}
    assert {k: v for k, v in back.items() if k not in ("m", "v")} == {k: v for k, v in want.items() if k not in ("m", "v")}
    assert all(torch.equal(back[s][k], state[s][k]) for s in ("m", "v") for k in sd)
    got = tfc.load_state_dict(prefix, list(sd))
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    with pytest.raises(KeyError, match="variable graph"):
        tfc.write_checkpoint(str(tmp_path / "bad"), {"a/w": np.zeros(2, np.float32)}, {("optimizer", "m", "a/w"): np.zeros(2, np.float32)})


def test_slot_variables_serialised_by_tensorflows_proto_are_resolved_here(tmp_path):
    """A graph decorated by TensorFlow's generated classes the way Keras lays an optimizer out — slot nodes appended behind the
    variables, referenced from the optimizer node only — spliced into a checkpoint written here."""
    rng = np.random.default_rng(7)
    tensors = {"h/0/mlp/c_fc/weight": rng.standard_normal((8, 32)).astype(np.float32), "ln_f/gamma": rng.standard_normal(8).astype(np.float32),
               "optimizer/iter": np.asarray(9, np.int64)}
    slot_vals = {(p, s): rng.standard_normal(tensors[p].shape).astype(np.float32) for p in list(tensors)[:2] for s in ("m", "v")}
    prefix = str(tmp_path / "keras")
    # the slot payloads travel as ordinary entries of a helper subtree; the graph below is what gives them their meaning
    tfc.write_checkpoint(prefix, dict(tensors, **{f"payload/{i}": v for i, v in enumerate(slot_vals.values())}))
    ck, g = _graph(prefix)
    opt = g.nodes[_walk(g, "optimizer")]
    for i, (p, s) in enumerate(slot_vals):
        opt.slot_variables.add(original_variable_node_id=_walk(g, p), slot_name=s, slot_variable_node_id=_walk(g, f"payload/{i}"))
    blob = g.SerializeToString()
    lens = tfc._put_varint(len(blob))
    sraw = lens + struct.pack("<I", tfc.masked_crc(lens)) + blob
    raw = tfc.read_index(prefix)
    data = open(prefix + ".data-00000-of-00001", "rb").read()
    raw[tfc.OBJECT_GRAPH_KEY] = tfc._msg(tfc._f_varint(1, 7), tfc._f_bytes(2, b""), tfc._f_varint(4, len(data)), tfc._f_varint(5, len(sraw)),
                                        tfc._f_fixed32(6, tfc.masked_crc(sraw)))
    open(prefix + ".data-00000-of-00001", "wb").write(data + sraw)
    items = sorted((k.encode(), v) for k, v in raw.items())
    with open(prefix + ".index", "wb") as f:
        off, size = tfc._emit_block(f, tfc._build_block(items))
        moff, msize = tfc._emit_block(f, tfc._build_block([]))
        ioff, isize = tfc._emit_block(f, tfc._build_block([(items[-1][0], tfc._put_varint(off) + tfc._put_varint(size))], restart_interval=1))
        footer = tfc._put_varint(moff) + tfc._put_varint(msize) + tfc._put_varint(ioff) + tfc._put_varint(isize)
        f.write(footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", tfc._MAGIC))
    ck = tfc.Checkpoint(prefix)
    nodes = ck.object_graph()
    for (p, s), val in slot_vals.items():
        assert np.array_equal(ck.tensor(ck.slot(p, s, nodes=nodes)), val)
    with pytest.raises(KeyError):
        ck.slot("optimizer/iter", "m", nodes=nodes)


# ------------------------------------------------------------------------------------------------ 2. the default file does not change
def test_weights_only_file_is_byte_identical_to_the_one_written_before_slots_existed(tmp_path):
    """SHA-256 of the two files the writer produced for these tensors before it knew slot variables; ``save_weights`` without
    ``include_optimizer`` must keep producing exactly them."""
    sd, _ = _tiny_state()
    m = MIGT(MIGTConfig(**TINY))
    m._sd = {k: v.clone() for k, v in sd.items()}                              # host copy only: the container needs no device
    prefix = str(tmp_path / "model")
    m.save_weights(prefix)
    digest = lambda ext: hashlib.sha256(open(prefix + ext, "rb").read()).hexdigest()
    assert digest(".index") == "53043ac30307bb06e486040f4f1510107744c79024c2ea030553675518391b6a"
    assert digest(".data-00000-of-00001") == "3b96624d0b290d9dd315de14d37392afc90679dbe579a8dfeb3ae88a087c8126"
    assert tfc.load_optimizer_state(prefix, list(sd)) is None
    with pytest.raises(RuntimeError, match="compiled"):
        m.save_weights(prefix, include_optimizer=True)


# ------------------------------------------------------------------------------------------------ 3. names the reference's objects carry
@pytest.fixture()
def tf():
    from oracle import tf_shim
    tf_shim.install()
    ref_loader.load_reference_migt()
    yield sys.modules["tensorflow"]
    tf_shim.uninstall()


@needs_reference
def test_optimizer_entry_names_are_the_reference_objects_names(tf):
    """Walks the reference's compiled MIGT: model.optimizer is its AdamWeightDecay, whose step counter is the variable 'iter' and whose
    learning_rate is the WarmUp holding the variable ``offset``; one training step creates one (m, v) pair per trained variable.  The
    shim's Adam keeps the pair unnamed — 'm' and 'v' are Keras Adam's add_slot names, which the shim cannot vouch for."""
    from oracle import synth, migt_oracle as mo
    kw = dict(n_layer=2, n_head=4, d_model=64, sequence_size=4, n_embeddings=40, token_image_size=2, n_loss_skip=1, dropout=0.0)
    cfg = MIGTConfig(**kw)
    sd = synth.make_migt_state_dict(cfg, 3)
    model = ref_loader.build_reference_migt(sd, **kw)
    utils = sys.modules["viewformer.models.utils"]
    opt, sched = utils.create_optimizer(1e-3, num_train_steps=10, num_warmup_steps=2, weight_decay_rate=cfg.weight_decay)
    model.compile(optimizer=opt)
    assert getattr(model, tfc.OPTIMIZER_ROOT) is opt and type(opt).__name__ == "AdamWeightDecay"
    scalars = {k: path for k, (path, _) in tfc.OPTIMIZER_SCALARS.items()}
    assert opt.iterations.name.split(":")[0] == scalars["iterations"] and opt.iterations.dtype == tf.int64
    obj = opt
    for part in scalars["schedule_offset"].split("/"):
        obj = getattr(obj, part)
    assert obj is sched.offset and type(sched).__name__ == "WarmUp" and obj.dtype == tf.int64
    codes = synth.make_codes(2, 4, n_embed=cfg.n_embeddings, side=2, seed=50)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(2, 4, seed=60))[0])
    model.train_step((cams, codes))
    assert int(opt.iterations) == 1 and all(len(pair) == len(tfc.SLOT_NAMES) for pair in opt._slots.values())
    _, slots = tfc.optimizer_entries(dict(m=sd, v=sd, iterations=1, train_counter=1, schedule_offset=0, seed=0, precision="fp32"))
    assert len(opt._slots) * len(tfc.SLOT_NAMES) == len(slots) == 2 * len(sd)
    assert {owner for owner, _, _ in slots} == {tfc.OPTIMIZER_ROOT}


# ------------------------------------------------------------------------------------------------ 4. optimizer_states[0] and real torch Adam
def _synthetic_moments(shapes, names):
    g = torch.Generator().manual_seed(5)
    return {k: torch.randn(shapes[k], generator=g) for k in names}, {k: torch.rand(shapes[k], generator=g) for k in names}


@pytest.mark.parametrize("quantizer", ["ema", "commit"])
def test_adam_state_loads_into_torch_adam_over_our_parameter_list(quantizer):
    """Runs everywhere: parameters created from ``param_shapes()`` in ``trainable_names`` order; real torch.optim.Adam accepts the
    state, and what it gives back after a step reads back through ``read_adam_state_dict``."""
    model = VQGAN(VQGANConfig(**SMALL_VQ), quantizer=quantizer)
    shapes, names = model.param_shapes(), trainable_names(model)
    assert ("quantize.embeddings" in names) == (quantizer == "commit") and not any("ema_" in k or k.endswith("counter") for k in names)
    m, v = _synthetic_moments(shapes, names)
    params = [torch.nn.Parameter(torch.zeros(shapes[k])) for k in names]
    opt = torch.optim.Adam(params, lr=1.0, betas=(0.9, 0.999))
    m0 = {k: t.clone() for k, t in m.items()}                                  # torch adopts the tensors it is given and updates them in place
    opt.load_state_dict(adam_state_dict(names, m, v, step=7, lr=2e-4, betas=(0.5, 0.9), eps=1e-8))
    (group,) = opt.param_groups
    assert group["lr"] == 2e-4 and tuple(group["betas"]) == (0.5, 0.9) and group["eps"] == 1e-8
    for k, p in zip(names, params):
        assert torch.equal(opt.state[p]["exp_avg"], m0[k]) and torch.equal(opt.state[p]["exp_avg_sq"], v[k]) and int(opt.state[p]["step"]) == 7
        p.grad = torch.zeros_like(p)
    opt.step()
    back = read_adam_state_dict(opt.state_dict(), names)
    assert back["step_count"] == 8 and back["lr"] == 2e-4 and back["betas"] == (0.5, 0.9)
    assert all(torch.equal(back["exp_avg"][k], m0[k] * 0.5) for k in names)          # zero gradient: m <- beta1 m
    fresh = read_adam_state_dict(torch.optim.Adam(params, lr=3e-4).state_dict(), names)
    assert fresh["step_count"] == 0 and not fresh["exp_avg"]
    with pytest.raises(RuntimeError, match="parameters"):
        read_adam_state_dict(opt.state_dict(), names[:-1])


@pytest.mark.skipif(not ref_loader.available(), reason="reference sources not present")
def test_adam_state_loads_into_torch_adam_over_the_reference_vqgan():
    """The reference's own module: ``trainable_names`` is the order of its ``parameters()``, and ``optimizer_states[0]`` loads into the
    optimizer its ``configure_optimizers()`` builds, every moment landing on the parameter it was named for."""
    ref = ref_loader.build_reference_vqgan(**SMALL_VQ)
    model = VQGAN(VQGANConfig(**SMALL_VQ))
    names = trainable_names(model)
    assert names == [n for n, _ in ref.named_parameters()]
    m, v = _synthetic_moments(model.param_shapes(), names)
    opt = ref.configure_optimizers()
    assert isinstance(opt, torch.optim.Adam)
    opt.load_state_dict(adam_state_dict(names, m, v, step=3, lr=ref.learning_rate, betas=(0.5, 0.9), eps=1e-8))
    for n, p in ref.named_parameters():
        st = opt.state[p]
        assert st["exp_avg"].shape == p.shape and torch.equal(st["exp_avg"], m[n]) and torch.equal(st["exp_avg_sq"], v[n]), n
    full = VQGAN(VQGANConfig())                                                # the full-size model: 342 parameters and 4 EMA buffers
    assert len(full.param_shapes()) == 346 and len(trainable_names(full)) == 342
    assert trainable_names(full) == [n for n, _ in ref_loader.build_reference_vqgan().named_parameters()]


# ------------------------------------------------------------------------------------------------ 5. the schedule under an offset
def _schedule_before_offsets(step, init, warm, total):
    """MIGTTrainer.learning_rate as it stood before ``schedule_offset`` existed."""
    if warm and step < warm:
        return init * (step / float(warm))
    decay_steps = max(1, total - warm)
    t = min(max(step - warm, 0), decay_steps) / float(decay_steps)
    return init * 0.5 * (1.0 + math.cos(math.pi * t))


def test_schedule_without_offset_is_value_for_value_the_one_before():
    for init, warm, total in ((1e-3, 2, 10), (8e-5, 2000, 200000), (1e-4, 0, 50), (1e-4, 30, 20)):
        for step in list(range(0, 40)) + [warm - 1, warm, warm + 1, total - 1, total, total + 7, 3 * total]:
            if step >= 0:
                assert warmup_cosine(step, init, warm, total) == _schedule_before_offsets(step, init, warm, total), (init, warm, total, step)


@needs_reference
def test_schedule_with_offset_equals_the_reference_warmup_at_that_offset(tf):
    utils = sys.modules["viewformer.models.utils"]
    init, warm, total = 3e-4, 20, 100
    for k in (0, 7, 1234):
        sched = utils.WarmUp(init, tf.keras.experimental.CosineDecay(init, total - warm), warm)
        sched.offset.assign(k)
        steps = sorted({0, max(k - 3, 0), k, k + 1, k + warm - 1, k + warm, k + warm + 1, k + (total + warm) // 2, k + total - 1, k + total, k + total + 9})
        for step in steps:
            want = float(sched(tf.Variable(step, dtype=tf.int64)))
            got = warmup_cosine(step, init, warm, total, offset=k)
            assert abs(got - want) <= 2e-6 * init, (k, step, got, want)
        assert warmup_cosine(k, init, warm, total, offset=k) == 0.0 and warmup_cosine(k + 5, init, warm, total, offset=k) == init * 5 / warm

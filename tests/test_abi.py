"""The C-ABI library loads on a CPU-only box and exports every symbol include/vf_b200.h declares; the ctypes binding in _lib.py holds
to the header: every function's parameter types, every parameter struct field by field, and every call site's argument count."""
import ast
import ctypes
import glob
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    src = open(os.path.join(ROOT, "include", "vf_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def declared_symbols():
    return sorted(set(re.findall(r"\b(vf_[a-z0-9_]+)\s*\(", header())))


def declared_prototypes():
    """{name: (return type, [(type, is pointer, parameter name)])} of every function the header declares."""
    out = {}
    for ret, name, params in re.findall(r"^(int|const char\*)\s+(vf_\w+)\s*\(([^)]*)\)\s*;", header(), flags=re.M):
        parsed = []
        for prm in params.split(","):
            if prm.strip() in ("", "void"):
                continue
            m = re.fullmatch(r"\s*(?:const\s+)?(\w+)\s*(\*?)\s*(\w+)\s*", prm)
            assert m, f"{name}: cannot parse parameter {prm!r}"
            parsed.append((m.group(1), bool(m.group(2)), m.group(3)))
        out[name] = (ret, parsed)
    return out


def declared_structs():
    """{typedef name: [(field, C type, is pointer, array length or None)]}: one entry per declarator, so `int N, H;` gives two."""
    out = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", header(), flags=re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            base, rest = re.fullmatch(r"(?:const\s+)?(\w+)\s*(.*)", decl, flags=re.S).groups()
            for d in rest.split(","):
                m = re.fullmatch(r"\s*(\*?)\s*(\w+)\s*(?:\[(\d+)\])?\s*", d)
                assert m, f"{name}: cannot parse declarator {d!r} of {decl!r}"
                fields.append((m.group(2), base, bool(m.group(1)), int(m.group(3)) if m.group(3) else None))
        out[name] = fields
    return out


def expected_argtype(func, ctype, pointer, pname):
    """The ctypes type _lib's mapping gives a header parameter."""
    from viewformer_b200 import _lib
    if not pointer:
        return {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "float": ctypes.c_float,
                "double": ctypes.c_double, "vf_stream_t": ctypes.c_void_p}[ctype]
    host = {"vf_simt_gemm_t": ctypes.POINTER(_lib.SimtGemm), "vf_tc_gemm_t": ctypes.POINTER(_lib.TcGemm)}   # parameter blocks
    if ctype in host:
        return host[ctype]
    if (func, pname) == ("vf_tc_gemm_plan", "plan"):                                                       # the plan array
        return ctypes.POINTER(ctypes.c_int)
    return _lib.DevPtr                                                                                    # everything else: device memory


def test_header_symbols_exported(lib):
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"libvf_b200.so does not export {s}"


def test_python_binding_lists_every_symbol():
    from viewformer_b200 import _lib
    assert set(declared_symbols()) == set(_lib.EXPORTS) == set(_lib.PROTOTYPES)


def test_prototype_table_matches_header():
    """Same functions; per function the same number of parameters (ctypes lets surplus arguments through) and, position by position,
    the ctypes type of the mapping; int returns except vf_last_error, as load() declares them."""
    from viewformer_b200 import _lib
    declared = declared_prototypes()
    assert sorted(declared) == declared_symbols(), "a declaration the prototype parser does not read"
    assert len(declared) == len(_lib.PROTOTYPES) == 70
    for name, (ret, params) in declared.items():
        assert ret == ("const char*" if name == "vf_last_error" else "int"), name
        got = _lib.PROTOTYPES[name]
        assert len(got) == len(params), f"{name}: {len(got)} argtypes, the header declares {len(params)} parameters"
        for k, (have, prm) in enumerate(zip(got, params)):
            want = expected_argtype(name, *prm)
            assert have is want, f"{name} parameter {k} {prm}: the table has {have.__name__}, the header wants {want.__name__}"


def test_struct_mirrors_match_header_field_by_field():
    from viewformer_b200 import _lib
    mirrors = {"vf_simt_gemm_t": _lib.SimtGemm, "vf_tc_gemm_t": _lib.TcGemm, "vf_conv_weights_bf16_t": _lib.ConvWeightsBf16,
               "vf_dense_weights_bf16_t": _lib.DenseWeightsBf16}
    declared = declared_structs()
    assert set(declared) == set(mirrors)
    scalar = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float}
    for name, fields in declared.items():
        got = mirrors[name]._fields_
        assert [f[0] for f in got] == [f[0] for f in fields], name
        for (fname, have), (_, ctype, pointer, n) in zip(got, fields):
            want = ctypes.c_void_p if pointer else scalar[ctype]
            if n is None:
                assert have is want, f"{name}.{fname}: mirror {have.__name__}, header {ctype}{'*' if pointer else ''}"
            else:
                assert issubclass(have, ctypes.Array) and have._type_ is want and have._length_ == n, f"{name}.{fname}[{n}]"


def test_struct_layouts_match(lib):
    from viewformer_b200 import _lib
    assert lib.vf_sizeof_simt_gemm() == ctypes.sizeof(_lib.SimtGemm)
    assert lib.vf_sizeof_tc_gemm() == ctypes.sizeof(_lib.TcGemm)


def test_weight_table_rows_are_the_struct_bytes():
    """A weight table row is the mirror's bytes read as int64: w_kn, fw, bw (NULL = 0), then the two sizes."""
    from viewformer_b200 import _lib
    for mirror in (_lib.ConvWeightsBf16, _lib.DenseWeightsBf16):
        rows = [mirror(0x7F0012340000, 0x7F0012350000, None, 128, 256), mirror(2 ** 40 + 64, 2 ** 40 + 128, 2 ** 40 + 192, 3, 5)]
        want = [[0x7F0012340000, 0x7F0012350000, 0, 128, 256], [2 ** 40 + 64, 2 ** 40 + 128, 2 ** 40 + 192, 3, 5]]
        assert _lib._device_table(mirror, rows, "cpu").tolist() == want
        assert tuple(_lib._device_table(mirror, [], "cpu").shape) == (0, 5)


def test_call_sites_pass_each_prototypes_argument_count():
    """Every `*.vf_name(...)` call of a declared function in the package, the tests, the scripts and the entry points passes exactly the
    prototype's argument count, positionally, with no *args."""
    from viewformer_b200 import _lib
    files = (glob.glob(os.path.join(ROOT, "viewformer_b200", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "tests", "*.py"))
             + glob.glob(os.path.join(ROOT, "scripts", "*.py")) + [os.path.join(ROOT, f) for f in ("bench.py", "__graft_entry__.py")])
    callers = {}
    for path in files:
        rel = os.path.relpath(path, ROOT)
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in _lib.PROTOTYPES):
                continue
            name, where = node.func.attr, f"{rel}:{node.lineno}"
            assert not node.keywords and not any(isinstance(a, ast.Starred) for a in node.args), f"{where}: {name} with keywords or *args"
            assert len(node.args) == len(_lib.PROTOTYPES[name]), f"{where}: {name} takes {len(_lib.PROTOTYPES[name])} arguments, got {len(node.args)}"
            callers[rel] = callers.get(rel, 0) + 1
    assert callers.get("viewformer_b200/_lib.py", 0) >= 60
    for rel in ("viewformer_b200/float_images.py", "viewformer_b200/cameras.py", "tests/test_train_bf16_gpu.py", "tests/test_exact_split_gpu.py",
                "tests/test_sevenscenes_gpu.py"):
        assert callers.get(rel), f"no call site found in {rel}"


class _ReportsCuda(torch.Tensor):
    """A CPU tensor that reports itself as a CUDA tensor: stands in for device memory so the conversion runs without a GPU."""

    @property
    def is_cuda(self):
        return True


def _passed_address(obj):
    """The address a DevPtr argument passes: from_param's result read back as a void* (it must be pointer-wide, not a C int)."""
    from viewformer_b200 import _lib
    return ctypes.cast(_lib.DevPtr.from_param(obj), ctypes.c_void_p).value


def test_device_pointer_argtype():
    from viewformer_b200 import _lib
    t = torch.zeros(4).as_subclass(_ReportsCuda)
    assert _passed_address(t) == t.data_ptr() != 0
    assert _passed_address(2 ** 40 + 256) == 2 ** 40 + 256
    assert _passed_address(None) is None
    assert _passed_address(ctypes.c_void_p(2 ** 40 + 512)) == 2 ** 40 + 512 == _passed_address(_lib._p(2 ** 40 + 512))   # explicit wrapping
    with pytest.raises(_lib.LibraryError, match="cpu tensor"):
        _lib.DevPtr.from_param(torch.zeros(4))
    with pytest.raises(TypeError):
        _lib.DevPtr.from_param(1.5)


@pytest.mark.gpu
def test_device_pointer_argtype_on_cuda_tensors():
    t = torch.zeros(4, device="cuda")
    assert _passed_address(t) == t.data_ptr()
    assert _passed_address(t[1:]) == t.data_ptr() + 4


def test_load_declares_every_prototype(lib):
    from viewformer_b200 import _lib
    for name, argtypes in _lib.PROTOTYPES.items():
        fn = getattr(lib, name)
        assert fn.argtypes is not None and tuple(fn.argtypes) == tuple(argtypes), name
        assert fn.restype is (ctypes.c_char_p if name == "vf_last_error" else ctypes.c_int), name


def test_version_and_error_string(lib):
    assert lib.vf_version() >= 100
    assert isinstance(lib.vf_last_error(), bytes)


def test_no_fallback_without_device():
    """Product path must fail loudly when there is no sm_90 device (no CPU fallback)."""
    from viewformer_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.LibraryError):
        _lib.load(require_device=True)
    from viewformer_b200 import VQGAN
    from oracle import synth
    m = VQGAN(ch=32, ch_mult=[1, 2], image_size=16, attn_resolutions=[8], embed_dim=16, z_channels=16, n_embed=32)
    with pytest.raises(_lib.LibraryError):
        m.load_state_dict(synth.make_vqgan_state_dict(m.config, 0))


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under viewformer_b200/ may import it."""
    pkg = os.path.join(ROOT, "viewformer_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f

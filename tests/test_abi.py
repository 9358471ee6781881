"""The C-ABI library loads on a CPU-only box and exports every symbol include/vf_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "vf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vf_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib):
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"libvf_b200.so does not export {s}"


def test_python_binding_lists_every_symbol():
    from viewformer_b200 import _lib
    assert set(declared_symbols()) == set(_lib.EXPORTS)


def test_struct_layouts_match(lib):
    from viewformer_b200 import _lib
    assert lib.vf_sizeof_simt_gemm() == ctypes.sizeof(_lib.SimtGemm)
    assert lib.vf_sizeof_tc_gemm() == ctypes.sizeof(_lib.TcGemm)


def test_version_and_error_string(lib):
    assert lib.vf_version() >= 100
    assert isinstance(lib.vf_last_error(), bytes)


def test_no_fallback_without_device():
    """Product path must fail loudly when there is no sm_90 device (no CPU fallback)."""
    import pytest
    import torch
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

"""Exact (split-fp16) tensor-core convs and GEMMs return the recorded bits (tests/golden/exact_conv_bits.json, recorded on an H100 by
scripts/record_exact_conv_bits.py): how operands are staged and where chunk sums live must not change the arithmetic."""
import importlib.util
import json
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("record_exact_conv_bits", os.path.join(ROOT, "scripts", "record_exact_conv_bits.py"))
rec = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(rec)

with open(rec.GOLDEN) as f:
    GOLDEN = json.load(f)["cases"]


def test_golden_covers_every_case():
    assert set(GOLDEN) == {rec.conv_id(c) for c in rec.CONVS} | {f"gemm_{k}" for k in rec.GEMMS}


@pytest.mark.gpu
@pytest.mark.parametrize("case", rec.CONVS, ids=rec.conv_id)
def test_exact_conv_bits(case):
    want = GOLDEN[rec.conv_id(case)]
    got = rec.run_conv(*case)
    assert got["sha256"] == want["sha256"]
    assert ("gn_sums" in got) == ("gn_sums" in want)
    if "gn_sums" in want:     # fp64 atomics: the summation order follows the tile schedule
        torch.testing.assert_close(torch.tensor(got["gn_sums"], dtype=torch.float64), torch.tensor(want["gn_sums"], dtype=torch.float64),
                                   rtol=1e-12, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", rec.GEMMS)
def test_exact_gemm_bits(kind):
    assert rec.run_gemm(kind)["sha256"] == GOLDEN[f"gemm_{kind}"]["sha256"]

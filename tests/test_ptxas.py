"""Compiler report of the tensor-core kernels (CPU only: nvcc cross-compiles for sm_90a without a GPU).

ptxas serializes warpgroup MMAs (every wgmma waits for the previous one) when their operand registers are written
after the wgmma fence, when too many registers are live across the asynchronous window, or when an MMA depends on a
compiler-inserted warpgroup arrive in a divergent path.  The kernels still compute the right result, only several
times slower, so nothing but the compiler's report shows it.  These tests read that report, and check that the
gradient-features kernels of dn_simt.cu and the classification-head kernels of dn_head.cu do not spill."""
import os
import re
import shutil
import subprocess

import pytest

import diffusion_net_b200 as dn

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CHECKED = ("rows_chain_kernel", "to_basis_kernel")

pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not found")


def _ptxas(tmp_path_factory, source, checked):
    """ptxas -v output of csrc/<source> compiled with the library's flags: {kernel: [lines]} for the checked kernels."""
    out = tmp_path_factory.mktemp("ptxas") / (source + ".o")
    flags = [f for f in dn._lib.NVCC_FLAGS if f != "-shared"]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(dn._lib._CSRC, source), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    per, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"function '(\w+)'", line)
        name = m.group(1) if m else None
        if "Compiling entry function" in line:
            cur = name
        key = name or cur
        if key and any(k in key for k in checked):
            per.setdefault(key, []).append(line)
    return per


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    per = _ptxas(tmp_path_factory, "dn_tc.cu", CHECKED)
    assert any("rows_chain_kernel" in k for k in per) and any("to_basis_kernel" in k for k in per), per.keys()
    return per


def _serialized(lines):
    return [l for l in lines if "wgmma.mma_async instructions are serialized" in l]


def test_chain_wgmma_not_serialized(report):
    bad = {k: _serialized(v) for k, v in report.items() if "rows_chain_kernel" in k and _serialized(v)}
    assert not bad, bad


def test_to_basis_wgmma_not_serialized(report):
    bad = {k: _serialized(v) for k, v in report.items() if "to_basis_kernel" in k and _serialized(v)}
    assert not bad, bad


def _assert_no_spills(report):
    for k, lines in report.items():
        spill = [l for l in lines if "spill stores" in l]
        assert spill, (k, lines)
        for l in spill:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and m.group(1) == "0" and m.group(2) == "0", (k, l)


def test_no_spills(report):
    _assert_no_spills(report)


def test_features_kernels_no_spills(tmp_path_factory):
    """Every instance of the gradient-features kernels keeps its state in registers, the block gather within the 128
    registers of its two CTAs per SM (with 64-bit row strides its C = 128 rotation instance spilled)."""
    per = _ptxas(tmp_path_factory, "dn_simt.cu", ("spmm_features", "features_bwd"))
    assert sum("spmm_features_blk_kernel" in k for k in per) == 4 and len(per) == 18, sorted(per)
    _assert_no_spills(per)


def test_head_kernels_no_spills(tmp_path_factory):
    """Every kernel of dn_head.cu keeps its state in registers: the forward, dX and dW kernels of the fused
    classification head on each engine (dX and dW hold two 64-float accumulators and run within a few registers of
    the cap), its partial reduction, and the element-mean forward and backward."""
    per = _ptxas(tmp_path_factory, "dn_head.cu", ("linear_nll", "element_mean"))
    assert len(per) == 12, sorted(per)
    assert sum(any(k in n for k in ("linear_nll_fwd", "linear_nll_dx", "linear_nll_dw")) for n in per) == 9, sorted(per)
    _assert_no_spills(per)

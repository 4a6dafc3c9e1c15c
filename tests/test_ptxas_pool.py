"""Compiler report of the global-mean pool kernels of dn_head.cu (CPU only: nvcc cross-compiles for sm_90a without a
GPU): its partial, reduction and backward kernels keep their state in registers.  The helpers are test_ptxas.py's."""
from test_ptxas import _assert_no_spills, _ptxas, pytestmark  # noqa: F401  (pytestmark: skip without nvcc)


def test_global_mean_pool_kernels_no_spills(tmp_path_factory):
    per = _ptxas(tmp_path_factory, "dn_head.cu", ("global_mean_pool",))
    assert sorted(k.split("global_mean_pool_")[1].split("_kernel")[0] for k in per) == ["bwd", "partial", "reduce"], \
        sorted(per)
    _assert_no_spills(per)

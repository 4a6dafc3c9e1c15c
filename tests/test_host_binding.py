"""CPU-side checks of the ctypes binding derived from include/diffusion_net_b200.h: every declaration is bound with
types from the closed set, the constants come from the header, and ``_lib.call`` passes tensors as their addresses and
raises as ``_lib.check`` does.  No GPU compute here."""
import ctypes as C
import types

import pytest
import torch

import diffusion_net_b200 as dn

L = dn._lib
STRUCTS = (L.dn_patches, L.dn_csr, L.dn_block_params, L.dn_mesh_batch, L.dn_gather_part, L.dn_slot_plan,
           L.dn_slot_elements, L.dn_eig_batch, L.dn_head)
SCALARS = (C.c_int, C.c_int64, C.c_double, C.c_float)


def test_every_declaration_bound_from_the_closed_set():
    lib = L.load()
    allowed_args = set(SCALARS) | {C.c_void_p} | {C.POINTER(s) for s in STRUCTS}
    assert len(L.SIGNATURES) == 73
    for name, (res, args) in L.SIGNATURES.items():
        assert res in (C.c_int, C.c_int64, C.c_char_p), name
        assert all(a in allowed_args for a in args), (name, args)
        fn = getattr(lib, name)
        assert fn.restype is res and list(fn.argtypes) == args, name


def test_spot_checks():
    S = L.SIGNATURES
    assert S["dn_linear_nll_ls_fwd"][1][-1] is C.c_float
    assert S["dn_linear_nll_ls_bwd"][1][-1] is C.c_float
    assert S["dn_mesh_laplacian"][1][4] is C.c_double                  # eps
    assert S["dn_workspace_bytes"] == (C.c_int64, [C.c_int64, C.c_int, C.c_int])
    assert S["dn_error_string"] == (C.c_char_p, [C.c_int])
    assert S["dn_abi_version"] == (C.c_int, [])
    assert S["dn_grad_spmm"][1][0] is C.POINTER(L.dn_csr)
    assert S["dn_csr_transpose"][1][0] is C.POINTER(L.dn_csr)
    assert S["dn_block_fwd_ex"][1][4:8] == [C.POINTER(L.dn_csr), C.POINTER(L.dn_block_params),
                                            C.POINTER(L.dn_mesh_batch), C.POINTER(L.dn_head)]
    assert S["dn_mini_mlp_fwd"][1][0] is C.c_void_p                    # const float* const* src_host
    assert S["dn_compute_hks"][1][-1] is C.c_void_p                    # dn_stream_t


def test_constants_from_the_header():
    assert L.ABI_VERSION == 5
    assert (L.ENGINE_SIMT, L.ENGINE_TC3X, L.ENGINE_TC1X, L.ENGINE_BF16) == (0, 1, 2, 3)
    assert (L.GATHER_COPY, L.GATHER_ADD_I32, L.GATHER_ADD_I64, L.GATHER_MAX_PARTS) == (0, 1, 2, 16)
    assert L.PROFILE_STAGES == 6 == len(dn.ops.PROFILE_STAGES)
    assert (L.OK, L.ERR_INVALID_ARGUMENT, L.ERR_UNSUPPORTED, L.ERR_WORKSPACE) == (0, -1, -2, -3)
    assert L.load().dn_abi_version() == L.ABI_VERSION


def test_parser_refuses_types_outside_the_set():
    sigs, consts = L.parse_header("enum dn_x { DN_A = 3, DN_B };\n#define DN_C -7\n"
                                  "int dn_ok(const float* a, int64_t n, double t, dn_stream_t s); /* int dn_no(); */")
    assert sigs == {"dn_ok": (C.c_int, [C.c_void_p, C.c_int64, C.c_double, C.c_void_p])}
    assert consts == {"DN_A": 3, "DN_B": 4, "DN_C": -7}
    for decl in ("int dn_bad(int32_t n);", "void dn_bad(int n);", "size_t dn_bad(void);", "int* dn_bad(void);"):
        with pytest.raises(RuntimeError, match="dn_bad"):
            L.parse_header(decl)


def test_call_raises_what_check_raises():
    with pytest.raises(RuntimeError) as want:
        L.check(L.ERR_INVALID_ARGUMENT, "dn_to_basis")
    lib = L.load()
    v, b, o = torch.ones(8, 4), torch.ones(8, 1), torch.empty(1, 4)
    # K = 0 is refused before the device is touched
    for values in (v, v.data_ptr(), None):
        raw = lib.dn_to_basis(values if not torch.is_tensor(values) else values.data_ptr(), b.data_ptr(), None, 8, 0,
                              4, o.data_ptr(), None, 0, L.ENGINE_SIMT, None)
        assert raw == L.ERR_INVALID_ARGUMENT
        with pytest.raises(RuntimeError) as got:
            L.call("dn_to_basis", values, b, None, 8, 0, 4, o, None, 0, L.ENGINE_SIMT, None)
        assert str(got.value) == str(want.value)


def test_call_passes_tensors_as_addresses(monkeypatch):
    seen = []
    fake = types.SimpleNamespace(dn_x=lambda *a: seen.append(a) or 0, dn_error_string=L.load().dn_error_string)
    monkeypatch.setattr(L, "_lib", fake)
    t, arr, ref = torch.zeros(3), (C.c_float * 2)(), C.byref(C.c_int(1))
    L.call("dn_x", t, 7, 2.5, None, arr, ref, t[1:])
    assert seen == [(t.data_ptr(), 7, 2.5, None, arr, ref, t.data_ptr() + 4)]

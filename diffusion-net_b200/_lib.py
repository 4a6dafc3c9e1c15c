"""ctypes binding of the C-ABI library (include/diffusion_net_b200.h).

The shared object is built IN-TREE (``diffusion-net_b200/libdiffusion_net_b200.so``)
with nvcc for sm_90a (H100) and loaded with ctypes -- plain pointers and sizes, no torch
types cross the boundary.  There is no CPU or library fallback: if the library is
missing or a call fails, a RuntimeError is raised.

The header is the only place a signature or constant is written: every ``dn_*``
declaration is bound from it (``SIGNATURES``), and its integer ``DN_*`` macros and
enum members are this module's names without the prefix (``ENGINE_TC3X``,
``GATHER_MAX_PARTS``, ``ERR_UNSUPPORTED``, ``ABI_VERSION``, ``PROFILE_STAGES``, ...).
"""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libdiffusion_net_b200.so")
SOURCES = ["dn_simt.cu", "dn_geom.cu", "dn_eig.cu", "dn_implicit.cu", "dn_implicit_batch.cu", "dn_batch_gather.cu",
           "dn_batch_rotate.cu", "dn_batch_plan.cu", "dn_fmap.cu", "dn_fmap_batch.cu", "dn_fmap_gt.cu", "dn_tc.cu",
           "dn_head.cu", "dn_capi.cu"]
HEADER = os.path.join(os.path.dirname(_HERE), "include", "diffusion_net_b200.h")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [HEADER]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu into the in-tree shared library (nvcc cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB_PATH] + [os.path.join(_CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd))
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


class dn_patches(C.Structure):
    _fields_ = [("n_patches", C.c_int32), ("max_src", C.c_int32), ("tgt_ptr", C.c_void_p), ("tgt", C.c_void_p),
                ("src_ptr", C.c_void_p), ("src_rows", C.c_void_p), ("ent_ptr", C.c_void_p), ("lcol", C.c_void_p),
                ("vals", C.c_void_p)]


class dn_csr(C.Structure):
    _fields_ = [("rowptr", C.c_void_p), ("colidx", C.c_void_p), ("vals", C.c_void_p), ("nnz", C.c_int64),
                ("patches", C.POINTER(dn_patches))]


class dn_block_params(C.Structure):
    _fields_ = [("diffusion_time", C.c_void_p), ("A_re", C.c_void_p), ("A_im", C.c_void_p),
                ("with_gradient_features", C.c_int), ("with_gradient_rotations", C.c_int),
                ("n_mlp_layers", C.c_int), ("mlp_weight_host", C.POINTER(C.c_void_p)),
                ("mlp_bias_host", C.POINTER(C.c_void_p)), ("mlp_dims_host", C.POINTER(C.c_int))]


class dn_mesh_batch(C.Structure):
    _fields_ = [("n_meshes", C.c_int32), ("n_tb_ctas", C.c_int32), ("tile_mesh", C.c_void_p), ("tb_rows", C.c_void_p),
                ("mesh_cta_begin", C.c_void_p)]


class dn_gather_part(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("op", C.c_int32), ("width", C.c_int32), ("range", C.c_int32),
                ("offset_range", C.c_int32), ("max_units", C.c_int64)]


class dn_slot_plan(C.Structure):
    _fields_ = [(name, C.c_void_p) for name in ("row_begin", "tile_mesh", "tb_rows", "mesh_cta_begin", "seg_begin",
                                                "seg_rows", "tile_seg", "table", "status")]


class dn_slot_elements(C.Structure):
    _fields_ = [("capacity", C.c_int64), ("tail", C.c_int64), ("k", C.c_int32), ("range", C.c_int32),
                ("csr_range", C.c_int32), ("begin", C.c_void_p), ("count", C.c_void_p), ("tile_seg", C.c_void_p)]



class dn_eig_batch(C.Structure):
    _fields_ = [("n_meshes", C.c_int32), ("n_tiles", C.c_int32), ("n_slices", C.c_int32), ("row_begin", C.c_void_p),
                ("tile_mesh", C.c_void_p), ("tile_begin", C.c_void_p), ("slice_mesh", C.c_void_p),
                ("slice_begin", C.c_void_p)]


class dn_head(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p), ("n_out", C.c_int32), ("out", C.c_void_p), ("ld_out", C.c_int64)]


_STRUCTS = {cls.__name__: cls for cls in (dn_patches, dn_csr, dn_block_params, dn_mesh_batch, dn_gather_part,
                                           dn_slot_plan, dn_slot_elements, dn_eig_batch, dn_head)}
_SCALARS = {"int": C.c_int, "int64_t": C.c_int64, "double": C.c_double, "float": C.c_float,
            "dn_stream_t": C.c_void_p}      # dn_stream_t is a typedef of void*


def _ctype(decl, ctype, structs, result=False):
    """The ctypes type of a header type: a scalar, a `const char*` return, a pointer to a header struct, or any
    other pointer (device data, host arrays, T* const*), passed as a plain address."""
    words = ctype.replace("*", " * ").split()
    base = [w for w in words if w not in ("const", "*")]
    stars = words.count("*")
    if stars == 0 and len(base) == 1 and base[0] in _SCALARS:
        return _SCALARS[base[0]]
    if result and words == ["const", "char", "*"]:
        return C.c_char_p
    if stars == 1 and len(base) == 1 and base[0] in structs:
        if base[0] not in _STRUCTS:
            raise RuntimeError("diffusion_net_b200: {}: struct {} has no ctypes class".format(decl, base[0]))
        return C.POINTER(_STRUCTS[base[0]])
    if stars and not result:
        return C.c_void_p
    raise RuntimeError("diffusion_net_b200: {}: unsupported type '{}' in {}".format(decl, " ".join(words), HEADER))


def parse_header(text):
    """(signatures, constants) of the C-ABI header: name -> (restype, argtypes) for every dn_* declaration, and
    name -> value for every integer #define and enum member named DN_*."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", "", text, flags=re.S)
    constants = {k: int(v) for k, v in re.findall(r"^#define[ \t]+(DN_\w+)[ \t]+(-?\d+)[ \t]*$", text, re.M)}
    for body in re.findall(r"\benum\s+\w+\s*\{([^}]*)\}", text):
        value = -1
        for member in filter(None, (m.strip() for m in body.split(","))):
            name, _, v = member.partition("=")
            value = int(v) if v.strip() else value + 1
            constants[name.strip()] = value
    structs = set(re.findall(r"\bstruct\s+(\w+)", text))
    signatures = {}
    for stmt in re.split(r"[;{}]", re.sub(r"^#[^\n]*", "", text, flags=re.M)):
        m = re.fullmatch(r"\s*([\w\s*]+?)\s*\b(dn_\w+)\s*\(([^()]*)\)\s*", stmt)
        if m is None:
            continue
        ret, name, params = m.groups()
        params = [] if params.strip() in ("", "void") else params.split(",")
        signatures[name] = (_ctype(name, ret, structs, result=True),
                            [_ctype(name, re.sub(r"\w+\s*$", "", p), structs) for p in params])
    return signatures, constants


with open(HEADER) as _fh:
    SIGNATURES, _constants = parse_header(_fh.read())
globals().update({k[len("DN_"):]: v for k, v in _constants.items()})

_lib = None


def load():
    """Load (building first if the .so is absent) and type the C-ABI library."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as e:  # fail loudly: there is no fallback path
        raise RuntimeError("diffusion_net_b200: cannot load {}: {}".format(LIB_PATH, e))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.dn_abi_version() != ABI_VERSION:
        raise RuntimeError("diffusion_net_b200: ABI version mismatch")
    _lib = lib
    return lib


def check(code: int, what: str = ""):
    if code != 0:
        msg = load().dn_error_string(code).decode()
        raise RuntimeError("diffusion_net_b200 {} failed ({}): {}".format(what, code, msg))


def addresses(args):
    """``args`` with every torch.Tensor replaced by its data_ptr(); every other argument (ints, floats, None, ctypes
    objects) as it is."""
    return [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]


def call(name, *args):
    """Call the entry point ``name``, whose int return is a status, with ``addresses(args)`` (the tensors stay
    referenced until the call returns), and raise as ``check`` does unless it is DN_OK."""
    check(getattr(load(), name)(*addresses(args)), name)


def ptr_array(ptrs):
    arr = (C.c_void_p * len(ptrs))()
    for i, p in enumerate(ptrs):
        arr[i] = p if p else None
    return arr


def int_array(vals):
    arr = (C.c_int * len(vals))()
    for i, v in enumerate(vals):
        arr[i] = int(v)
    return arr

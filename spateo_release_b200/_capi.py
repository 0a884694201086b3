"""ctypes binding of ``libspateo_b200.so`` (C ABI declared in ``include/spateo_b200.h``).

The header is the single source of truth: the two structs (``spb_scalars``, ``spb_em_params``) are parsed from it, so
the Python mirror cannot drift. There is **no CPU fallback**: if the shared library is missing or the machine has no
CUDA device, every entry point raises.
"""

from __future__ import annotations

import ctypes as C
import os
import re

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(_PKG_DIR)
HEADER = os.path.join(REPO_ROOT, "include", "spateo_b200.h")
LIB_PATH = os.path.join(_PKG_DIR, "libspateo_b200.so")

_SCALAR_TYPES = {
    "int32_t": C.c_int32,
    "uint32_t": C.c_uint32,
    "int64_t": C.c_int64,
    "uint64_t": C.c_uint64,
    "float": C.c_float,
    "double": C.c_double,
}


def _parse_struct(text: str, name: str):
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S)
    if m is None:
        raise RuntimeError(f"struct {name} not found in {HEADER}")
    fields = []
    for line in m.group(1).splitlines():
        line = re.sub(r"/\*.*?\*/", "", line).strip()
        if not line:
            continue
        fm = re.match(r"^(const\s+)?([A-Za-z_0-9]+)\s*(\*?)\s*([A-Za-z_0-9]+)(\[(\d+)\])?;$", line)
        if fm is None:
            raise RuntimeError(f"cannot parse field line {line!r} of {name}")
        base, ptr, fname, arr = fm.group(2), fm.group(3), fm.group(4), fm.group(6)
        if ptr:
            ctype = C.c_void_p
        else:
            ctype = _SCALAR_TYPES[base]
            if arr:
                ctype = ctype * int(arr)
        fields.append((fname, ctype))
    return fields


def header_text() -> str:
    with open(HEADER) as f:
        return f.read()


def declared_functions() -> list:
    """Names of every function the header declares (used by the CPU test that checks the exports)."""
    text = re.sub(r"/\*.*?\*/", "", header_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(?:int|int64_t)\s+(spb_[a-z_A-Z0-9]+)\s*\(", text)))


_hdr = header_text()


class SpbScalars(C.Structure):
    _fields_ = _parse_struct(_hdr, "spb_scalars")


class SpbEmParams(C.Structure):
    _fields_ = _parse_struct(_hdr, "spb_em_params")


class SpbFieldDesc(C.Structure):
    _fields_ = _parse_struct(_hdr, "spb_field_desc")


def _consts():
    out = {}
    for k, v in re.findall(r"#define (SPB_[A-Z_0-9]+)\s+\(?(-?\d+)\)?", _hdr):
        out[k] = int(v)
    return out


CONST = _consts()
ROW_TILE = CONST["SPB_ROW_TILE"]
COL_STAGE = CONST["SPB_COL_STAGE"]
MAX_K_FUSED = CONST["SPB_MAX_K_FUSED"]
TRACE_STRIDE = CONST["SPB_TRACE_STRIDE"]

_lib = None


class SpbError(RuntimeError):
    pass


def load_library():
    """Load the CUDA library; fails loudly when it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SpbError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). spateo_release_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    P, I32, I64, F, D = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double
    EP = C.POINTER(SpbEmParams)
    sig = {
        "spb_version": ([], C.c_int),
        "spb_launch_count": ([], C.c_int64),
        "spb_sizeof_em_params": ([], C.c_int),
        "spb_sizeof_scalars": ([], C.c_int),
        "spb_sizeof_field_desc": ([], C.c_int),
        "spb_kl_prepare_rows": ([P, I64, I64, I64, P, I64, P, I32, P, P], C.c_int),
        "spb_rows_sqnorm": ([P, I64, I64, I64, P, P], C.c_int),
        "spb_rows_normalize": ([P, I64, I64, I64, P, I64, P], C.c_int),
        "spb_split_tf32": ([P, P, P, I64, P], C.c_int),
        "spb_gene_cost_tc": ([P, P, I64, P, P, P, I64, P, I64, I64, I64, I32, I32, F, I32, P, I64, P], C.c_int),
        "spb_gather_rows": ([P, I64, I64, P, I64, P, I64, P], C.c_int),
        "spb_label_cost": ([P, P, P, I32, I64, I64, I32, P, I64, P], C.c_int),
        "spb_gather_cols": ([EP, I32, P], C.c_int),
        "spb_estep_col_lists": ([EP, P], C.c_int),
        "spb_estep_sweep1": ([EP, I32, P], C.c_int),
        "spb_col_finalize": ([EP, P], C.c_int),
        "spb_estep_sweep2": ([EP, I32, P], C.c_int),
        "spb_row_finalize": ([EP, P], C.c_int),
        "spb_row_fold": ([EP, I32, P], C.c_int),
        "spb_row_stats_finalize": ([EP, I32, P], C.c_int),
        "spb_row_stats_p2p": ([EP, I32, C.c_uint64, P], C.c_int),
        "spb_estep_col_select": ([EP, I32, P], C.c_int),
        "spb_sparse_P_emit": ([EP, I32, P, P, P], C.c_int),
        "spb_posterior_argmax_mapped": ([EP, I32, P, P, P, P], C.c_int),
        "spb_materialize_P": ([EP, I32, P, I64, P], C.c_int),
        "spb_posterior_transfer_rows": ([EP, I32, P, I64, I32, P, P, P], C.c_int),
        "spb_posterior_transfer_cols": ([EP, I32, P, I32, P, P, I64, P], C.c_int),
        "spb_iter_begin": ([EP, I32, P], C.c_int),
        "spb_update_gamma_alpha": ([EP, P], C.c_int),
        "spb_nonrigid_accumulate": ([EP, P], C.c_int),
        "spb_nonrigid_solve": ([EP, P], C.c_int),
        "spb_nonrigid_blend": ([EP, P], C.c_int),
        "spb_field_apply": ([EP, P], C.c_int),
        "spb_field_apply_lowrank": ([EP, P, I32, P, P], C.c_int),
        "spb_rigid_moments": ([EP, P], C.c_int),
        "spb_rigid_solve": ([EP, I32, P], C.c_int),
        "spb_row_update": ([EP, P], C.c_int),
        "spb_em_iteration": ([EP, I32, P], C.c_int),
        "spb_em_iteration_ex": ([EP, I32, I32, P], C.c_int),
        "spb_nonrigid_warm": ([], C.c_int),
        "spb_optimal_rigid": ([EP, P, P], C.c_int),
        "spb_rbf_kernel_T": ([P, I64, I64, P, I32, F, P, P], C.c_int),
        "spb_field_eval": ([P, I64, I32, P, P, I32, D, P, P], C.c_int),
        "spb_field_geometry": ([C.POINTER(SpbFieldDesc), P, I64, P, P, P, P, P, P, P, P, P, P, P, P, P], C.c_int),
        "spb_field_integrate": ([C.POINTER(SpbFieldDesc), P, I64, P, P, D, I32, D, D, D, P, P, P, P, P], C.c_int),
        "spb_voxel_count": ([P, I32, I64, I32, P, I32, P, I32, P, I32, D, P, P, P, P], C.c_int),
        "spb_voxel_accumulate": ([P, I32, I64, I32, P, I32, P, I32, P, I32, D, P, P, P, P, P, I64, I32, P, I64, P], C.c_int),
        "spb_inlier_from_nn": ([P, P, P, I64, I32, D, D, D, D, P, P, P, P, P], C.c_int),
        "spb_weighted_gram": ([P, I64, I64, I32, P, P, P, P, P], C.c_int),
        "spb_gram_tc_scratch_floats": ([I32, I32, I64, C.POINTER(C.c_int64)], C.c_int),
        "spb_gram_center": ([P, I64, I64, I32, P, P, P, P], C.c_int),
        "spb_gram_prepare": ([P, I64, I64, I32, P, P, P, I64, I32, P, P, P, P], C.c_int),
        "spb_gram_tc": ([P, P, P, P, I64, I64, I32, I32, P, P, P, I64, P, P, P], C.c_int),
        "spb_vfc_estep": ([P, I64, I64, I32, I32, P, P, D, D, D, D, D, P, P, P, P, P, P], C.c_int),
        "spb_field_eval_host": ([P, I64, I32, P, P, I32, D, P], C.c_int),
    }
    for name, (argtypes, restype) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    lib._spb_signatures = sig
    if lib.spb_sizeof_em_params() != C.sizeof(SpbEmParams) or lib.spb_sizeof_scalars() != C.sizeof(SpbScalars) or \
            lib.spb_sizeof_field_desc() != C.sizeof(SpbFieldDesc):
        raise SpbError("struct layout mismatch between include/spateo_b200.h and the built library: rebuild it")
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc == 0:
        return
    if rc == CONST["SPB_EINVAL"]:
        raise SpbError(f"{what}: invalid argument (SPB_EINVAL)")
    if rc == CONST["SPB_EUNSUPPORTED"]:
        raise SpbError(f"{what}: unsupported configuration (SPB_EUNSUPPORTED)")
    raise SpbError(f"{what}: CUDA error {rc}")


def ptr(t):
    """Device (or pinned host) pointer of a torch tensor / numpy array as c_void_p (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return C.c_void_p(t.data_ptr())
    return C.c_void_p(t.ctypes.data)


def current_stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise SpbError("spateo_release_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback.")

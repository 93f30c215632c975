"""ctypes binding of libnksr_b200.so (the C-ABI declared in include/nksr_b200.h).

This is the reference-side stub a maintainer would add (INTEGRATION.md): plain pointers and
sizes cross the boundary, torch only owns the memory and the stream.  There is NO fallback:
if the shared library is missing, or a call returns a non-zero code, we raise -- callers in the
reference treat RuntimeError as "skip / retry" (models/base_model.py:140-148).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

MAX_DEPTH = 8
ROW_STRIDE = 32
_LIB_NAME = "libnksr_b200.so"
_here = os.path.dirname(os.path.abspath(__file__))


class SvhT(C.Structure):
    _fields_ = [("depth", C.c_int32), ("voxel_size", C.c_float),
                ("n", C.c_int64 * MAX_DEPTH), ("offset", C.c_int64 * MAX_DEPTH),
                ("keys", C.c_void_p * MAX_DEPTH), ("parent", C.c_void_p * MAX_DEPTH),
                ("child8", C.c_void_p * MAX_DEPTH), ("nbr27", C.c_void_p * MAX_DEPTH),
                ("nbr125_top", C.c_void_p)]


class FeatT(C.Structure):
    _fields_ = [("channels", C.c_int32), ("z", C.c_void_p * MAX_DEPTH)]


class ConstraintsT(C.Structure):
    _fields_ = [("e_pos", C.c_void_p), ("range_pos", C.c_void_p), ("n_pos", C.c_int64), ("w_pos", C.c_float),
                ("e_nrm", C.c_void_p), ("range_nrm", C.c_void_p), ("t_nrm", C.c_void_p), ("n_nrm", C.c_int64),
                ("w_nrm", C.c_float), ("w_reg", C.c_float), ("nrm_compact", C.c_int32),
                ("mblocks", C.c_void_p), ("split_level", C.c_int32), ("mblock_off", C.c_int64 * MAX_DEPTH)]


class PlacementT(C.Structure):
    _fields_ = [("rank8", (C.c_void_p * MAX_DEPTH) * MAX_DEPTH), ("prefix", (C.c_void_p * MAX_DEPTH) * MAX_DEPTH)]


_T = {"p": C.c_void_p, "q": C.c_int64, "i": C.c_int32, "f": C.c_float, "z": C.c_size_t,
      "S": C.POINTER(SvhT), "F": C.POINTER(FeatT), "K": C.POINTER(ConstraintsT), "d": C.POINTER(C.c_double),
      "P": C.POINTER(PlacementT)}

# name -> (return kind, argument kinds); mirrors include/nksr_b200.h one to one
_SIGNATURES = {
    "nksr_version": ("s", ""),
    "nksr_error_string": ("s", "i"),
    "nksr_point_half_keys": ("i", "pqfppp"),
    "nksr_sort_workspace_bytes": ("z", "qi"),
    "nksr_sort_keys": ("i", "ppqpzp"),
    "nksr_sort_pairs": ("i", "ppppqpzp"),
    "nksr_unique_workspace_bytes": ("z", "q"),
    "nksr_unique_sorted": ("i", "pqipppzp"),
    "nksr_splat_candidates": ("i", "pqpp"),
    "nksr_parent_index": ("i", "pqpqppp"),
    "nksr_child_table": ("i", "ppqpqp"),
    "nksr_nbr27_search": ("i", "pqpp"),
    "nksr_nbr27_from_parent": ("i", "ppqpppp"),
    "nksr_decode_ijk": ("i", "pqipp"),
    "nksr_locate": ("i", "Spqpp"),
    "nksr_row_ranges": ("i", "pqpqp"),
    "nksr_pool27": ("i", "ppqipp"),
    "nksr_pool_children": ("i", "ppqipp"),
    "nksr_gather_gemm": ("i", "ppqippppiiiip"),
    "nksr_gather_gemm_wgrad_workspace_bytes": ("z", "qiiii"),
    "nksr_gather_gemm_wgrad": ("i", "ppqipiipppzip"),
    "nksr_transpose_taps": ("i", "pqiqppp"),
    "nksr_build_rows": ("i", "SFppqiipp"),
    "nksr_build_rows_voxel": ("i", "SFpppqiipp"),
    "nksr_gram_count": ("i", "Sppp"),
    "nksr_scan_workspace_bytes": ("z", "q"),
    "nksr_gram_rowptr": ("i", "ppqppzp"),
    "nksr_gram_fill": ("i", "SFKppppppp" + "p"),
    "nksr_gram_block_floats": ("q", "Si"),
    "nksr_gram_blocks": ("i", "SKpp"),
    "nksr_gram_sort_down": ("i", "ppppqippp"),
    "nksr_gram_count_own": ("i", "Spp"),
    "nksr_gram_place": ("i", "Siipppp" + "p"),
    "nksr_gram_fill_placed": ("i", "SFKppPppppp"),
    "nksr_gram_fill_placed_rows": ("i", "SFKppPqqppppp"),
    "nksr_gram_fill_brick": ("i", "SFKppPppppfp"),
    "nksr_gram_fill_grouped": ("i", "SFKppPppppp"),
    "nksr_gram_count_grouped": ("i", "Spp"),
    "nksr_nbr125_search": ("i", "pqpp"),
    "nksr_spmv": ("i", "pppppqp"),
    "nksr_pcg_workspace_bytes": ("z", "q"),
    "nksr_pcg_solve": ("i", "pppppp" + "qfiii" + "pzdp"),
    "nksr_pcg_stream_workspace_bytes": ("z", "qq"),
    "nksr_pcg_solve_stream": ("i", "pppppp" + "qqqqfiii" + "pzdp"),
    "nksr_spmv_plan_bytes": ("z", "q"),
    "nksr_spmv_stream": ("i", "ppppp" + "qqqq" + "pzp"),
    "nksr_dcg_workspace_bytes": ("z", ""),
    "nksr_dcg_init": ("i", "pppppppp" + "q" + "pz" + "pp"),
    "nksr_dcg_begin": ("i", "ppfip"),
    "nksr_dcg_spmv_dots": ("i", "ppppppp" + "q" + "ppp"),
    "nksr_dcg_update": ("i", "pppppppp" + "q" + "ppp"),
    "nksr_dcg_status": ("i", "pdp"),
    "nksr_gather_f32": ("i", "ppqpp"),
    "nksr_scatter_f32": ("i", "ppqpp"),
    "nksr_evaluate": ("i", "SFppqiippp"),
    "nksr_mesh_cell_flags": ("i", "Spp"),
    "nksr_mesh_stage0_cells": ("i", "Sppipp"),
    "nksr_mesh_leaf_flags": ("i", "Sipp"),
    "nksr_mesh_virtual_anchors": ("i", "Sipppp"),
    "nksr_mesh_anchor_flags": ("i", "Spqipp"),
    "nksr_mesh_split_cells": ("i", "pqiipp"),
    "nksr_mesh_corner_keys": ("i", "pqiiiipp"),
    "nksr_mesh_lattice_pos": ("i", "pqiiifipp"),
    "nksr_mesh_classify": ("i", "pqppqpppp"),
    "nksr_compact_rows": ("i", "pppqipp"),
    "nksr_scan32_workspace_bytes": ("z", "q"),
    "nksr_exclusive_scan32": ("i", "ppqpzp"),
    "nksr_mesh_cell_edges": ("i", "ppqiiiippp"),
    "nksr_run_heads": ("i", "pqpp"),
    "nksr_mesh_vertices": ("i", "ppqppifipp"),
    "nksr_mesh_triangles": ("i", "pppqpqpp"),
    "nksr_layer_mask": ("i", "Spqipp"),
    "nksr_voxel_moments": ("i", "pqppfpp"),
    "nksr_voxel_pca_normals": ("i", "ppqfpp"),
    "nksr_orient_normals": ("i", "ppppqfppp"),
    "nksr_knn_normals": ("i", "Spppp" + "qif" + "ppppp"),
    "nksr_nearest_point": ("i", "Sppqpqpippp"),
    "nksr_knn_mean_distance": ("i", "Sppqppqiipp"),
    "nksr_sdf_from_points": ("i", "Sppppqppqifiippp"),
}

_lib = None


class NksrError(RuntimeError):
    pass


def library_path() -> str:
    return os.path.join(_here, _LIB_NAME)


def load():
    """Load the CUDA library once.  Raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise NksrError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "or `make -C nksr_b200/csrc` -- nksr_b200 has no CPU or PyTorch fallback")
    lib = C.CDLL(path)
    for name, (ret, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch
        fn.restype = {"i": C.c_int, "z": C.c_size_t, "s": C.c_char_p, "q": C.c_int64}[ret]
        fn.argtypes = [_T[a] for a in args]
    _lib = lib
    return lib


def exported_symbols():
    return sorted(_SIGNATURES)


def _conv(kind, v):
    if kind == "p":
        if v is None:
            return None
        if isinstance(v, torch.Tensor):
            return v.data_ptr()
        return int(v)
    if kind in "SFKP":
        return C.byref(v)
    return v


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream if torch.device(device).type == "cuda" else 0


def call(name: str, *args):
    """Call an int-returning entry point; non-zero codes become NksrError."""
    lib = load()
    kinds = _SIGNATURES[name][1]
    if len(kinds) != len(args):
        raise TypeError(f"{name}: expected {len(kinds)} arguments, got {len(args)}")
    fn = getattr(lib, name)
    conv = [_conv(k, a) for k, a in zip(kinds, args)]
    # the library launches on the CURRENT device: make it the device that owns the tensors (the stream
    # argument already belongs to it), so cuda:1 fields work while cuda:0 is current
    dev = next((a.device for a in args if isinstance(a, torch.Tensor) and a.is_cuda), None)
    if dev is not None and dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):
            rc = fn(*conv)
    else:
        rc = fn(*conv)
    if _SIGNATURES[name][0] == "i" and rc != 0:
        raise NksrError(f"{name} failed: {lib.nksr_error_string(rc).decode()} ({rc})")
    return rc


def require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise NksrError(f"{what} must live on a CUDA device: nksr_b200 is a CUDA-only implementation "
                        "(no CPU path; the CPU oracle under oracle/ is test infrastructure)")


# ----------------------------------------------------------------------------- small helpers
def _ws(nbytes: int, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def sort_keys(keys: torch.Tensor) -> torch.Tensor:
    n = keys.numel()
    out = torch.empty_like(keys)
    if n:
        nb = call("nksr_sort_workspace_bytes", n, 0)
        ws = _ws(nb, keys.device)
        call("nksr_sort_keys", keys, out, n, ws, nb, stream_ptr(keys.device))
    return out


def sort_pairs(keys: torch.Tensor, vals: torch.Tensor):
    n = keys.numel()
    ko, vo = torch.empty_like(keys), torch.empty_like(vals)
    if n:
        nb = call("nksr_sort_workspace_bytes", n, 1)
        ws = _ws(nb, keys.device)
        call("nksr_sort_pairs", keys, ko, vals, vo, n, ws, nb, stream_ptr(keys.device))
    return ko, vo


def unique_sorted(keys: torch.Tensor, shift: int = 0) -> torch.Tensor:
    n = keys.numel()
    out = torch.empty_like(keys)
    cnt = torch.zeros(1, dtype=torch.int64, device=keys.device)
    if n:
        nb = call("nksr_unique_workspace_bytes", n)
        ws = _ws(nb, keys.device)
        call("nksr_unique_sorted", keys, n, shift, out, cnt, ws, nb, stream_ptr(keys.device))
    return out[: int(cnt.item())]


def exclusive_scan32(flags: torch.Tensor) -> torch.Tensor:
    n = flags.numel()
    out = torch.empty(n + 1, dtype=torch.int64, device=flags.device)
    nb = call("nksr_scan32_workspace_bytes", max(n, 1))
    ws = _ws(nb, flags.device)
    call("nksr_exclusive_scan32", flags, out, n, ws, nb, stream_ptr(flags.device))
    return out


def compact_rows(rows: torch.Tensor, flags: torch.Tensor, scan: torch.Tensor, count: int) -> torch.Tensor:
    n = flags.numel()
    row_bytes = rows.element_size() * (rows.numel() // max(n, 1)) if n else rows.element_size()
    out = torch.empty((count,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
    if n and count:
        call("nksr_compact_rows", rows, flags, scan, n, row_bytes, out, stream_ptr(rows.device))
    return out


class StageTimer:
    """CUDA-event stage timer (no syncs until .report()); enabled by NKSR_STAGE_TIMES=1 or explicitly."""

    def __init__(self, device, enabled=None):
        self.enabled = bool(int(os.environ.get("NKSR_STAGE_TIMES", "0"))) if enabled is None else enabled
        self.device, self.marks = device, []
        self.mark("start")

    def mark(self, name):
        if self.enabled:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(torch.cuda.current_stream(self.device))
            self.marks.append((name, ev))

    def report(self):
        if not self.enabled or len(self.marks) < 2:
            return {}
        torch.cuda.synchronize(self.device)
        out = {}
        for (_, a), (name, b) in zip(self.marks[:-1], self.marks[1:]):
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out

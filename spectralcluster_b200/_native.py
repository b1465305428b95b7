"""ctypes binding of libspectralcluster_b200.so (the C ABI in include/spectralcluster_b200.h).

There is NO CPU fallback: if the library is missing this module raises, and if no H100 is
visible `context()` raises.  torch tensors are used only as device buffers (`data_ptr()`).
"""

from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libspectralcluster_b200.so")

c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_dbl = ctypes.c_double
c_ptr = ctypes.c_void_p
GATHER_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int)   # sc_gather_fn
PICK_FN = ctypes.CFUNCTYPE(ctypes.c_int64, ctypes.c_void_p, ctypes.POINTER(ctypes.c_double),
                           ctypes.c_int64, ctypes.POINTER(ctypes.c_void_p))   # sc_pick_fn

# name -> argtypes (every function returns int except the two noted); this table is also what
# tests/test_abi.py checks against include/spectralcluster_b200.h.
PROTOTYPES = {
    "sc_abi_version": [],
    "sc_last_error": [],
    "sc_launch_count": [],
    "sc_context_create": [c_int, ctypes.POINTER(c_ptr)],
    "sc_context_destroy": [c_ptr],
    "sc_context_sm_count": [c_ptr],
    "sc_context_set_gemm_sm_limit": [c_ptr, c_int],
    "sc_normalize_rows": [c_ptr, c_ptr, c_int, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr, c_ptr,
                          c_i64, c_ptr],
    "sc_normalize_rows_typed": [c_ptr, c_ptr, c_int, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr,
                                c_ptr, c_i64, c_ptr],
    "sc_affinity_cosine": [c_ptr, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr, c_i64, c_i64, c_i64,
                           c_ptr, c_i64, c_ptr, c_ptr],
    "sc_crop_diagonal": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_ptr],
    "sc_crop_diagonal_values": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr],
    "sc_gaussian_blur": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_ptr, c_i64, c_ptr, c_ptr],
    "sc_gaussian_blur_rowmax": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_int, c_ptr, c_ptr],
    "sc_row_threshold": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_dbl, c_dbl, c_int, c_int, c_ptr,
                         c_i64, c_ptr],
    "sc_symmetrize": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_ptr, c_i64, c_ptr],
    "sc_blur_threshold_symmetrize": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_ptr, c_dbl,
                                     c_dbl, c_int, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr,
                                     c_i64, c_ptr],
    "sc_blur_upper_rowmax": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_int, c_ptr, c_i64, c_ptr,
                             c_ptr],
    "sc_threshold_symmetrize_upper": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_dbl, c_int, c_int,
                                      c_int, c_ptr, c_i64, c_ptr, c_ptr, c_i64, c_ptr],
    "sc_blur_threshold_symmetrize_upper": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_dbl, c_ptr, c_dbl,
                                           c_dbl, c_int, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr,
                                           c_i64, c_ptr],
    "sc_split_planes": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_i64, c_ptr],
    "sc_diffuse": [c_ptr, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64,
                   c_ptr, c_ptr, c_ptr],
    "sc_row_group_bounds": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_gather_rows_f16": [c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_ptr],
    "sc_diffuse_tile_list": [c_ptr, c_ptr, c_i64, c_ptr, c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_diffuse_rowmax_tiles": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_bound_order": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_int, c_ptr, c_ptr],
    "sc_bound_order_hubs": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_int, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_diffuse_hub_tiles": [c_ptr, c_ptr, c_int, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_diffuse_tile_list_rows": [c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_ptr, c_ptr, c_int, c_ptr,
                                  c_ptr, c_ptr, c_ptr],
    "sc_diffuse_rowmax_tiles_fold": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_row_stats": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_affinity_stats": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr],
    "sc_affinity_stats_rows": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr],
    "sc_affinity_stats_finish": [c_ptr, c_ptr, c_i64, c_ptr, c_ptr],
    "sc_row_normalize": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_ptr],
    "sc_laplacian": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_dbl, c_ptr, c_i64, c_ptr],
    "sc_affinity_cosine_block": [c_ptr, c_int, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64,
                                 c_ptr, c_i64, c_ptr, c_ptr],
    "sc_gaussian_blur_rowmax_block": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                                      c_ptr, c_dbl, c_int, c_ptr, c_ptr],
    "sc_blur_threshold_symmetrize_block": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                                           c_ptr, c_dbl, c_ptr, c_dbl, c_dbl, c_int, c_int, c_int,
                                           c_ptr, c_i64, c_ptr, c_ptr, c_i64, c_ptr],
    "sc_row_stats_block": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_transpose": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr],
    "sc_gemm_nt_planes": [c_ptr, c_int, c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_i64, c_i64,
                          c_i64, c_ptr, c_i64, c_ptr, c_i64, c_ptr],
    "sc_diffuse_stats_block": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_i64, c_i64, c_ptr,
                               c_ptr, c_ptr],
    "sc_constraint_combine": [c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_i64, c_int, c_ptr, c_i64, c_ptr],
    "sc_scale_shift": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_dbl, c_dbl, c_ptr, c_i64, c_ptr],
    "sc_gemm_nt_f32": [c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr],
    "sc_ipc_export": [c_ptr, c_ptr, c_ptr, ctypes.POINTER(c_i64)],
    "sc_ipc_open": [c_ptr, c_ptr, c_i64, ctypes.POINTER(c_ptr)],
    "sc_ipc_close_all": [c_ptr],
    "sc_memcpy_async": [c_ptr, c_ptr, c_ptr, c_i64, c_ptr],
    "sc_eigh_dense": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_dbl, c_int, c_i64,
                      c_i64, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_extremal": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_dbl, c_int, c_i64,
                         c_i64, c_dbl, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_extremal_locked": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_dbl, c_int,
                                c_i64, c_dbl, c_i64, c_dbl, c_ptr, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_eigh_mapback": [c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_block_size": [c_i64],
    "sc_eigh_extremal_sharded": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr,
                                 c_dbl, c_int, c_i64, c_i64, c_dbl, c_i64, c_ptr, c_int, c_i64,
                                 c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_extremal_locked_sharded": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr,
                                        c_ptr, c_dbl, c_int, c_i64, c_dbl, c_i64, c_dbl, c_ptr,
                                        c_i64, c_ptr, c_int, c_i64, c_ptr, c_ptr, c_ptr, c_ptr,
                                        c_ptr],
    "sc_eigh_extremal_factored_sharded": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr,
                                          c_ptr, c_dbl, c_int, c_i64, c_i64, c_dbl, c_i64, c_ptr,
                                          c_int, c_i64, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_extremal_locked_factored_sharded": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr,
                                                 c_ptr, c_ptr, c_dbl, c_int, c_i64, c_dbl, c_i64,
                                                 c_dbl, c_ptr, c_i64, c_ptr, c_int, c_i64, c_ptr,
                                                 c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_block_product": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr, c_i64, ctypes.c_int, c_ptr, c_i64,
                         c_ptr],
    "sc_block_product_f16": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr, c_i64, ctypes.c_int, c_ptr,
                             c_i64, c_ptr],
    "sc_eigh_extremal_factored": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_dbl, c_int,
                                  c_i64, c_i64, c_dbl, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_eigh_extremal_locked_factored": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_dbl,
                                         c_int, c_i64, c_dbl, c_i64, c_dbl, c_ptr, c_i64, c_ptr,
                                         c_ptr, c_ptr],
    "sc_affinity_cosine_panel": [c_ptr, c_int, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64,
                                 c_ptr, c_i64, c_ptr, c_ptr],
    "sc_blur_upper_rowmax_block": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_ptr,
                                   c_dbl, c_int, c_ptr, c_i64, c_ptr, c_ptr],
    "sc_threshold_symmetrize_upper_block": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_dbl,
                                            c_dbl, c_int, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr,
                                            c_i64, c_ptr],
    "sc_krylov_matvec": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_krylov_orthogonalize": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_krylov_scale": [c_ptr, c_ptr, c_i64, c_dbl, c_ptr, c_ptr],
    "sc_krylov_random": [c_ptr, c_ptr, c_i64, c_i64, c_ptr],
    "sc_krylov_combine": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_i64, c_ptr, c_ptr],
    "sc_krylov_columns": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr],
    "sc_row_renorm": [c_ptr, c_ptr, c_i64, c_i64, c_ptr],
    "sc_kmeans": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr, c_i64, c_int, c_i64, c_dbl,
                  c_ptr, c_ptr, c_ptr],
    "sc_cosine_distances_f64": [c_ptr, c_ptr, c_int, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr,
                                c_ptr],
    "sc_cluster_centroids": [c_ptr, c_ptr, c_int, c_i64, c_i64, c_i64, c_ptr, c_i64, c_ptr, c_i64,
                             c_ptr],
    "sc_complete_linkage": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_average_linkage": [c_ptr, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_nn_chain_small": [c_ptr, c_ptr, c_i64, c_i64, c_int, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_gmm_band_pass": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_int, c_ptr, c_ptr, c_ptr, c_ptr],
    "sc_gmm_band_pass_packed": [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_int, c_ptr, c_ptr, c_ptr,
                                c_ptr],
    "sc_gmm_band_pack": [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr],
    "sc_naive_cluster": [c_ptr, c_ptr, c_int, c_i64, c_i64, c_i64, c_dbl, c_dbl, c_i64, c_ptr,
                         c_i64, c_ptr, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr],
}

# enum values of include/spectralcluster_b200.h
THRESHOLD_ROWMAX, THRESHOLD_PERCENTILE = 0, 1
SYMMETRIZE_MAX, SYMMETRIZE_AVERAGE = 0, 1
LAPLACIAN_AFFINITY, LAPLACIAN_UNNORMALIZED, LAPLACIAN_RANDOMWALK, LAPLACIAN_GRAPHCUT = 0, 1, 2, 3
GEMM_TCGEN05, GEMM_SIMT = 0, 1
GEMM_SPLIT3, GEMM_SINGLE, GEMM_SPLIT2 = 0, 1, 2
ABI_VERSION = 2
EIG_LARGEST, EIG_SMALLEST = 0, 1
DTYPE_F32, DTYPE_F64, DTYPE_F16, DTYPE_BF16 = 0, 1, 2, 3
LINKAGE_COMPLETE, LINKAGE_AVERAGE = 0, 1
NN_SMALL_MAX = 2048           # SC_NN_SMALL_MAX: the largest n sc_nn_chain_small takes

_lib = None
_lock = threading.Lock()


class NativeError(RuntimeError):
  """A C-ABI call returned non-zero; the message is sc_last_error()."""


def load():
  """dlopen the in-tree shared library; raise (never fall back) if it is absent."""
  global _lib
  with _lock:
    if _lib is not None:
      return _lib
    if not os.path.exists(LIB_PATH):
      raise ImportError(
          "spectralcluster_b200: %s is missing. Build it with `python -m spectralcluster_b200.build`"
          " (or __graft_entry__.build()). There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in PROTOTYPES.items():
      fn = getattr(lib, name)
      fn.argtypes = args
      fn.restype = (ctypes.c_char_p if name == "sc_last_error" else
                    ctypes.c_longlong if name == "sc_launch_count" else ctypes.c_int)
    if lib.sc_abi_version() != ABI_VERSION:
      raise ImportError("spectralcluster_b200: ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
  msg = load().sc_last_error()
  return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, exc=NativeError):
  if rc != 0:
    raise exc(last_error())


def call(name: str, *args, exc=NativeError):
  """Invoke a C-ABI function, raising `exc` with sc_last_error() on failure."""
  check(getattr(load(), name)(*args), exc)


_contexts = {}


def context(device: int = 0):
  """The sc_context* for a CUDA device (created once per process and device)."""
  with _lock:
    ctx = _contexts.get(device)
  if ctx is not None:
    return ctx
  lib = load()
  out = c_ptr()
  check(lib.sc_context_create(int(device), ctypes.byref(out)))
  with _lock:
    _contexts[device] = out
  return out

"""Device side of the hot path: buffers (torch tensors used only as HBM allocations), thin
wrappers over the C ABI, and the refinement planner that fuses the reference's operator
sequence (spectral_clusterer.py:131-135) into kernel launches.

Layout in HBM: every N x N matrix is fp32 row-major with a padded leading dimension
(`ld` = N rounded up to 64 elements, so rows start on 256-byte boundaries and 128-bit
loads/TMA boxes are aligned); the GEMM operands additionally exist as two fp16 planes
(hi, lo) of the same shape, i.e. the same 4 bytes per element.  Row statistics, scaling
vectors, eigenvectors and the k-means state are fp64 vectors / N x k arrays.
"""

from __future__ import annotations

import ctypes
import os
import typing

import numpy as np

from . import _native as nat

_torch = None

# MMAs per product of the Diffuse GEMM inside predict(), picked by N from the error of each scheme
# (tests/diffuse_precision_study.py measures it): the rounding of the fp16 operand planes is a
# zero-mean perturbation per product that averages down with sqrt(K) = sqrt(N), so the parity
# tolerance (|dw| <= 1e-5 |w| + 1e-6 max|w|) allows one MMA from N = 16,384, two from N = 4,096 and
# needs three below (the parity tests pin these sizes).
AUTO_SINGLE_FROM, AUTO_SPLIT2_FROM = 16384, 4096

# The stored route keeps about this many bytes per element of the N x ld matrices alive at its
# peak: A and B (fp32) while the blur writes Y (fp16 hi plane), then S (fp32) beside A and Y.
STORED_ROUTE_BYTES_PER_ELEMENT = 10
# Device memory the route choice leaves for the CUDA context, the allocator and the vectors.
FACTORED_ROUTE_RESERVE = 4 << 30
# The factored route builds the affinity and the blur in row panels of about this many bytes.
FACTORED_PANEL_BYTES = 1 << 30
# Panel origins sit on the affinity's 128-row tiles (which also aligns them with the 64-row tiles
# of the threshold pass and the 32-row bands of the blur); the blur reads 4 rows on either side.
PANEL_ALIGN, BLUR_HALO = 128, 4
# Bounded Diffuse (sc_diffuse_tile_list): the column groups of its row bounds, its output tile, and
# the row order -- spherical k-means on the device (sc_bound_order) with this many clusters and
# assignment passes on the rows' group-norm profiles (the order only decides which tiles are
# skipped, never a value; on the bench's speaker turns at N = 65,536 the tile count is the same
# from 3 to 20 passes).
BOUND_GROUP_COLS, LIST_BM, LIST_BN = 256, 128, 192
BOUND_ORDER_CLUSTERS, BOUND_ORDER_ITERS = 16, 4
# predict() takes the bounded Diffuse from this N (tools/time_bounded_diffuse.py, H100 80GB HBM3,
# 700 W, measured with the earlier host k-means row order): at 16,384 its fixed costs (mostly that
# order, 5.5 ms) left it 25 % slower than the storing Diffuse + stored solve (11.7 against 9.4 ms);
# at 32,768 it is 40 % faster (33 against 56).
BOUNDED_FROM = 32768


def stored_route_peak_bytes(n: int) -> int:
  """Peak device bytes of predict()'s stored route at n, computed from shapes."""
  return STORED_ROUTE_BYTES_PER_ELEMENT * n * round_up(n, 64)


def bounded_tile_count(n: int) -> int:
  """Tiles of the symmetric single-MMA Diffuse launch (those that reach the upper triangle)."""
  tiles_n = -(-n // LIST_BN)
  return sum(tiles_n - max(0, -(-(LIST_BM * m - LIST_BN + 1) // LIST_BN))
             for m in range(-(-n // LIST_BM)))


def nn_chain_entry(linkage: int, n: int) -> str:
  """The NN-chain kernel for n rows, chosen by n alone: one thread block up to nat.NN_SMALL_MAX
  (DESIGN.md §5 has the measured crossing), the cooperative grid above."""
  if n <= nat.NN_SMALL_MAX:
    return "sc_nn_chain_small"
  return {nat.LINKAGE_COMPLETE: "sc_complete_linkage",
          nat.LINKAGE_AVERAGE: "sc_average_linkage"}[linkage]


def panel_rows_for(n: int) -> int:
  """Rows per panel of the factored route: about FACTORED_PANEL_BYTES of fp32 rows, a multiple of
  PANEL_ALIGN, chosen from n alone."""
  rows = FACTORED_PANEL_BYTES // (4 * round_up(n, 64)) // PANEL_ALIGN * PANEL_ALIGN
  return max(PANEL_ALIGN, min(rows, round_up(n, PANEL_ALIGN)))


def panel_plan(n: int, rows: int):
  """[(r0, r1, a0, a1)]: the factored route's panels produce the rows [r0, r1) (every row once,
  r0 a multiple of `rows`) from the affinity rows [a0, a1) = the blur halo [r0 - 4, r1 + 4) clipped
  at 0 and n, with a0 moved down to a multiple of PANEL_ALIGN."""
  assert rows > 0 and rows % PANEL_ALIGN == 0
  plan = []
  for r0 in range(0, n, rows):
    r1 = min(n, r0 + rows)
    a0 = max(0, r0 - BLUR_HALO) // PANEL_ALIGN * PANEL_ALIGN
    plan.append((r0, r1, a0, min(n, r1 + BLUR_HALO)))
  return plan


def torch():
  global _torch
  if _torch is None:
    import torch as _t
    _torch = _t
  return _torch


def _ptr(t) -> ctypes.c_void_p:
  return ctypes.c_void_p(0 if t is None else t.data_ptr())


def round_up(x: int, m: int) -> int:
  return (x + m - 1) // m * m


def dtype_code(x) -> int:
  """The sc_dtype of a device tensor that sc_normalize_rows_typed reads."""
  t = torch()
  return {t.float32: nat.DTYPE_F32, t.float64: nat.DTYPE_F64, t.float16: nat.DTYPE_F16,
          t.bfloat16: nat.DTYPE_BF16}[x.dtype]


def device_embeddings(x):
  """A CUDA tensor handed to predict() as embeddings -> the tensor predict() reads: detached,
  float16 / bfloat16 / float32 / float64 (anything else widened to float64, as host arrays are),
  with unit column stride and rows that do not overlap (anything else made contiguous once)."""
  t = torch()
  x = x.detach()
  if x.dtype not in (t.float16, t.bfloat16, t.float32, t.float64):
    x = x.to(t.float64)
  n, d = int(x.shape[0]), int(x.shape[1])
  if (d > 1 and x.stride(1) != 1) or (n > 1 and x.stride(0) < d):
    x = x.contiguous()
  return x


def host_twin(x) -> np.ndarray:
  """The ndarray a CUDA tensor stands for: x.cpu().numpy(), through float32 for bfloat16 (exact),
  which numpy lacks.  Only where the reference hands the embeddings to user code."""
  t = torch()
  return (x.float() if x.dtype == t.bfloat16 else x).detach().cpu().numpy()


def twin(x):
  """A device tensor as fp32 / fp64 in the dtype its host twin reaches predict()'s arithmetic in:
  float16 rows widen to float64 (predict() widens an fp16 ndarray so), bfloat16 rows to float32 (the
  twin of a bf16 tensor is its exact fp32 upcast); fp32 / fp64 tensors are returned as they are."""
  t = torch()
  if x.dtype == t.float16:
    return x.to(t.float64)
  if x.dtype == t.bfloat16:
    return x.to(t.float32)
  return x


def blur_radius(sigma: float) -> int:
  """scipy.ndimage.gaussian_filter's radius int(truncate * sigma + 0.5), truncate = 4; sigma <=
  1e-15 copies the input (radius 0).  The blur kernels apply the same rule."""
  return int(4.0 * sigma + 0.5) if sigma > 1e-15 else 0


class DeferredBlur(typing.NamedTuple):
  """Pass 1 of the symmetric blur pair without a stored B: what pass 2 needs to blur the upper
  tiles of `a` (with `diag` substituted on read) again."""
  a: typing.Any
  diag: typing.Any
  sigma: float


class Engine:
  """One per CUDA device: the sc_context plus allocation / launch helpers."""

  _instances: typing.Dict[int, "Engine"] = {}

  # matrices smaller than this use the SIMT fp64-accumulate GEMM (a 128x128 tensor-core tile would
  # be mostly padding); everything else goes through the tensor-core kernel.
  simt_below = 64
  # force the dense (full-spectrum) eigensolver up to this N even when Lanczos would do (tests)
  dense_eig_max = 0

  def __init__(self, device: int = 0):
    t = torch()
    if not t.cuda.is_available():
      raise RuntimeError(
          "spectralcluster_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    self.device_index = device
    self.device = t.device("cuda", device)
    self.ctx = nat.context(device)
    self.gemm_precision = nat.GEMM_SPLIT3       # affinity: its entries feed a threshold
    # Diffuse inside predict() (K = N): an sc_gemm_precision to use at every N, or None for the
    # N-based policy above.  The operator-level API (refinement.Diffuse) always uses split3.
    self.diffuse_precision = None
    # predict() takes the factored route (no N x N fp32 matrix) when the stored route's peak,
    # stored_route_peak_bytes(n), exceeds this many bytes and the call is within its scope.
    # Computed from the device's total memory, never from what is free, so that one GPU model
    # always takes the same route for the same call.
    self.factored_above_bytes = (t.cuda.get_device_properties(device).total_memory -
                                 FACTORED_ROUTE_RESERVE)
    self.profile = None

  @classmethod
  def get(cls, device: typing.Optional[int] = None) -> "Engine":
    if device is None:
      device = torch().cuda.current_device() if torch().cuda.is_available() else 0
    eng = cls._instances.get(device)
    if eng is None:
      eng = cls(device)
      cls._instances[device] = eng
    return eng

  def diffuse_precision_for(self, n: int) -> int:
    """The sc_gemm_precision predict() uses for an n x n Diffuse (None = decide by n)."""
    if self.diffuse_precision is not None:
      return self.diffuse_precision
    if n >= AUTO_SINGLE_FROM:
      return nat.GEMM_SINGLE
    return nat.GEMM_SPLIT2 if n >= AUTO_SPLIT2_FROM else nat.GEMM_SPLIT3

  # ---- buffers
  @property
  def stream(self) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch().cuda.current_stream(self.device).cuda_stream)

  def matrix(self, n: int, dtype=None):
    t = torch()
    return t.empty((n, round_up(n, 64)), dtype=dtype or t.float32, device=self.device)

  def planes(self, n: int, cols: typing.Optional[int] = None):
    t = torch()
    ld = round_up(cols if cols is not None else n, 64)
    return (t.empty((n, ld), dtype=t.float16, device=self.device),
            t.empty((n, ld), dtype=t.float16, device=self.device))

  def vector(self, n: int, dtype=None, zero=False):
    t = torch()
    f = t.zeros if zero else t.empty
    return f((n,), dtype=dtype or t.float64, device=self.device)

  def upload_matrix(self, a: np.ndarray):
    """Host [n, n] array -> device fp32 matrix with padded rows."""
    t = torch()
    n = a.shape[0]
    m = self.matrix(n)
    src = t.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    m[:, :n].copy_(src, non_blocking=False)
    return m

  def download_matrix(self, m, n: int) -> np.ndarray:
    return m[:, :n].to("cpu").numpy().astype(np.float64)

  # C-ABI entry point -> the reference function whose work it does (NVTX range names)
  REFERENCE_NAMES = {
      "sc_normalize_rows": "utils.compute_affinity_matrix", "sc_affinity_cosine": "utils.compute_affinity_matrix",
      "sc_crop_diagonal": "refinement.CropDiagonal", "sc_crop_diagonal_values": "refinement.CropDiagonal",
      "sc_gaussian_blur": "refinement.GaussianBlur", "sc_gaussian_blur_rowmax": "refinement.GaussianBlur",
      "sc_blur_upper_rowmax": "refinement.GaussianBlur",
      "sc_blur_threshold_symmetrize": "refinement.RowWiseThreshold+Symmetrize",
      "sc_threshold_symmetrize_upper": "refinement.RowWiseThreshold+Symmetrize",
      "sc_blur_threshold_symmetrize_upper": "refinement.RowWiseThreshold+Symmetrize",
      "sc_row_threshold": "refinement.RowWiseThreshold", "sc_symmetrize": "refinement.Symmetrize",
      "sc_diffuse": "refinement.Diffuse", "sc_gemm_nt_planes": "refinement.Diffuse",
      "sc_row_normalize": "refinement.RowWiseNormalize", "sc_row_stats": "refinement.RowWiseNormalize",
      "sc_laplacian": "laplacian.compute_laplacian",
      "sc_eigh_dense": "utils.compute_sorted_eigenvectors",
      "sc_eigh_extremal": "utils.compute_sorted_eigenvectors",
      "sc_eigh_extremal_sharded": "utils.compute_sorted_eigenvectors",
      "sc_eigh_extremal_locked": "utils.compute_sorted_eigenvectors",
      "sc_eigh_extremal_locked_sharded": "utils.compute_sorted_eigenvectors",
      "sc_eigh_extremal_locked_factored": "utils.compute_sorted_eigenvectors",
      "sc_eigh_mapback": "utils.compute_sorted_eigenvectors",
      "sc_kmeans": "custom_distance_kmeans.run_kmeans", "sc_row_renorm": "spectral_clusterer.row_wise_renorm",
      "sc_affinity_stats": "fallback_clusterer.check_single_cluster",
      "sc_affinity_stats_rows": "fallback_clusterer.check_single_cluster",
      "sc_affinity_stats_finish": "fallback_clusterer.check_single_cluster",
      "sc_gmm_band_pass": "fallback_clusterer.check_single_cluster",
      "sc_gmm_band_pass_packed": "fallback_clusterer.check_single_cluster",
      "sc_gmm_band_pack": "fallback_clusterer.check_single_cluster",
      "sc_constraint_combine": "constraint.adjust_affinity", "sc_scale_shift": "constraint.adjust_affinity",
      "sc_normalize_rows_typed": "utils.compute_affinity_matrix",
      "sc_cluster_centroids": "utils.get_cluster_centroids",
      "sc_cosine_distances_f64": "AgglomerativeClustering(cosine)",
      "sc_complete_linkage": "AgglomerativeClustering(cosine, complete)",
      "sc_average_linkage": "AgglomerativeClustering(cosine, average)",
      "sc_nn_chain_small": "AgglomerativeClustering(cosine)",
      "sc_naive_cluster": "naive_clusterer.NaiveClusterer",
  }
  nvtx = os.environ.get("SCB_NVTX") == "1"

  def call(self, name, *args, exc=nat.NativeError):
    """One C-ABI call on the current stream; with `profile` on, bracketed by CUDA events; with
    SCB_NVTX=1 inside an NVTX range named after the reference function it replaces."""
    if self.nvtx:
      torch().cuda.nvtx.range_push("%s [%s]" % (self.REFERENCE_NAMES.get(name, name), name))
      try:
        return self._call(name, *args, exc=exc)
      finally:
        torch().cuda.nvtx.range_pop()
    return self._call(name, *args, exc=exc)

  def _call(self, name, *args, exc=nat.NativeError):
    if self.profile is None:
      nat.call(name, self.ctx, *args, exc=exc)
      return
    t = torch()
    start, stop = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
    start.record()
    nat.call(name, self.ctx, *args, exc=exc)
    stop.record()
    self.profile.append((name, start, stop))

  def start_profile(self):
    self.profile = []

  def stop_profile(self) -> typing.Dict[str, float]:
    """Milliseconds per C-ABI entry point since start_profile() (device time, CUDA events)."""
    torch().cuda.synchronize(self.device)
    out: typing.Dict[str, float] = {}
    for name, start, stop in self.profile or []:
      out[name] = out.get(name, 0.0) + start.elapsed_time(stop)
    self.profile = None
    return out

  # ---- operators (device in / device out)
  def gemm_engine(self, n: int) -> int:
    return nat.GEMM_SIMT if n < self.simt_below else nat.GEMM_TCGEN05

  def affinity(self, x_dev, want_crop_vector: bool):
    """utils.compute_affinity_matrix on a device [n, d] fp16/bf16/fp32/fp64 tensor (row stride
    free, unit column stride), read in place."""
    t = torch()
    n, d = int(x_dev.shape[0]), int(x_dev.shape[1])
    engine = self.gemm_engine(n)
    a = self.matrix(n)
    crop = self.vector(n, t.float32, zero=True) if want_crop_vector else None
    code = dtype_code(x_dev)
    if engine == nat.GEMM_SIMT:
      xn = t.empty((n, round_up(d, 4)), dtype=t.float32, device=self.device)
      self.call("sc_normalize_rows_typed", _ptr(x_dev), code, n, d, x_dev.stride(0), _ptr(xn),
                xn.stride(0), None, None, 0, self.stream)
      self.call("sc_affinity_cosine", engine, self.gemm_precision, _ptr(xn), xn.stride(0), None,
                None, 0, n, d, _ptr(a), a.stride(0), _ptr(crop), self.stream)
    else:
      hi, lo = self.planes(n, d)
      self.call("sc_normalize_rows_typed", _ptr(x_dev), code, n, d, x_dev.stride(0), None, 0,
                _ptr(hi), _ptr(lo), hi.stride(0), self.stream)
      self.call("sc_affinity_cosine", engine, self.gemm_precision, None, 0, _ptr(hi), _ptr(lo),
                hi.stride(0), n, d, _ptr(a), a.stride(0), _ptr(crop), self.stream)
    return a, crop

  def crop_diagonal(self, a, n):
    out = self.matrix(n)
    self.call("sc_crop_diagonal", _ptr(a), n, a.stride(0), _ptr(out), out.stride(0), self.stream)
    return out

  def crop_values(self, a, n):
    d = self.vector(n, torch().float32)
    self.call("sc_crop_diagonal_values", _ptr(a), n, a.stride(0), _ptr(d), self.stream)
    return d

  def gaussian_blur(self, a, n, sigma, diag=None):
    out = self.matrix(n)
    self.call("sc_gaussian_blur", _ptr(a), n, a.stride(0), _ptr(diag), float(sigma), _ptr(out),
              out.stride(0), None, self.stream)
    return out

  def row_threshold(self, a, n, type_, p, mult, binarize, preserve_diag):
    out = self.matrix(n)
    self.call("sc_row_threshold", _ptr(a), n, a.stride(0), int(type_), float(p), float(mult),
              int(bool(binarize)), int(bool(preserve_diag)), _ptr(out), out.stride(0),
              self.stream, exc=ValueError)
    return out

  def symmetrize(self, a, n, type_):
    out = self.matrix(n)
    self.call("sc_symmetrize", _ptr(a), n, a.stride(0), int(type_), _ptr(out), out.stride(0),
              self.stream, exc=ValueError)
    return out

  def blur_rowmax(self, a, n, sigma, diag, zero_diag):
    t = torch()
    m = self.vector(n, t.float32, zero=True)
    self.call("sc_gaussian_blur_rowmax", _ptr(a), n, a.stride(0), _ptr(diag), float(sigma),
              int(bool(zero_diag)), _ptr(m), self.stream)
    return m

  def blur_threshold_symmetrize(self, a, n, sigma, diag, rowmax, p, mult, binarize,
                                preserve_diag, sym_type, want_f32, want_planes):
    y = self.matrix(n) if want_f32 else None
    hi, lo = self.planes(n) if want_planes else (None, None)
    self.call("sc_blur_threshold_symmetrize", _ptr(a), n, a.stride(0), _ptr(diag), float(sigma),
              _ptr(rowmax), float(p), float(mult), int(bool(binarize)), int(bool(preserve_diag)),
              int(sym_type), _ptr(y), 0 if y is None else y.stride(0), _ptr(hi), _ptr(lo),
              0 if hi is None else hi.stride(0), self.stream)
    return y, hi, lo

  def blur_upper_rowmax(self, a, n, sigma, diag, zero_diag, store_b=False):
    """Symmetric pass 1: (b, m = row maxima of blur(a)).  b is a DeferredBlur record, and
    threshold_symmetrize_upper blurs a's upper tiles again; with store_b it is a matrix whose upper
    tiles hold blur(a)."""
    t = torch()
    b = self.matrix(n) if store_b else None
    m = self.vector(n, t.float32)
    self.call("sc_blur_upper_rowmax", _ptr(a), n, a.stride(0), _ptr(diag), float(sigma),
              int(bool(zero_diag)), _ptr(b), 0 if b is None else b.stride(0), _ptr(m), self.stream)
    return (b if store_b else DeferredBlur(a, diag, float(sigma))), m

  def threshold_symmetrize_upper(self, b, n, rowmax, p, mult, binarize, preserve_diag, sym_type,
                                 want_f32, want_planes, want_lo=True):
    """Symmetric pass 2: Y and its mirror from b, a DeferredBlur record (the blur is recomputed)
    or a matrix holding the upper tiles of blur(a)."""
    t = torch()
    y = self.matrix(n) if want_f32 else None
    hi = lo = None
    if want_planes and want_lo:
      hi, lo = self.planes(n)
    elif want_planes:      # a single-MMA Diffuse reads only the hi plane: 2 B/element less to write
      hi = t.empty((n, round_up(n, 64)), dtype=t.float16, device=self.device)
    rule = (_ptr(rowmax), float(p), float(mult), int(bool(binarize)), int(bool(preserve_diag)),
            int(sym_type), _ptr(y), 0 if y is None else y.stride(0), _ptr(hi), _ptr(lo),
            0 if hi is None else hi.stride(0), self.stream)
    if isinstance(b, DeferredBlur):
      self.call("sc_blur_threshold_symmetrize_upper", _ptr(b.a), n, b.a.stride(0), _ptr(b.diag),
                b.sigma, *rule)
    else:
      self.call("sc_threshold_symmetrize_upper", _ptr(b), n, b.stride(0), *rule)
    return y, hi, lo

  @staticmethod
  def upper_pass_ok(sigma: float) -> bool:
    """The symmetric blur pair covers radius-4 filters (sigma ~ 1, every BASELINE config)."""
    return blur_radius(sigma) == 4

  def split_planes(self, a, n):
    hi, lo = self.planes(n)
    self.call("sc_split_planes", _ptr(a), n, a.stride(0), _ptr(hi), _ptr(lo), hi.stride(0),
              self.stream)
    return hi, lo

  def diffuse(self, n, y=None, hi=None, lo=None, want_stats=False, precision=None):
    """S = Y Y^T.  With want_stats (tensor-core engine) also returns (rowmax fp32, rowsum fp64) of S
    from the GEMM epilogue; otherwise (None, None).  `precision` defaults to the fp32-accurate
    three-MMA split (the operator-level API); predict() passes `diffuse_precision`."""
    t = torch()
    precision = self.gemm_precision if precision is None else precision
    engine = self.gemm_engine(n)
    s = self.matrix(n)
    if engine == nat.GEMM_SIMT:
      assert y is not None
      self.call("sc_diffuse", engine, precision, _ptr(y), y.stride(0), None, None, 0,
                n, _ptr(s), s.stride(0), None, None, self.stream)
      return s, None, None
    if hi is None:
      hi, lo = self.split_planes(y, n)
    mx = self.vector(n, t.float32) if want_stats else None
    sm = self.vector(n, t.float64) if want_stats else None
    self.call("sc_diffuse", engine, precision, None, 0, _ptr(hi), _ptr(lo),
              hi.stride(0), n, _ptr(s), s.stride(0), _ptr(mx), _ptr(sm), self.stream)
    return s, mx, sm

  def diffuse_stats(self, n, hi):
    """(rowmax fp32, rowsum fp64) of S = Y Y^T from the single-MMA Diffuse on the hi plane of Y,
    without storing S (bitwise the statistics of the storing call)."""
    t = torch()
    mx, sm = self.vector(n, t.float32), self.vector(n, t.float64)
    self.call("sc_diffuse", nat.GEMM_TCGEN05, nat.GEMM_SINGLE, None, 0, _ptr(hi), None,
              hi.stride(0), n, None, 0, _ptr(mx), _ptr(sm), self.stream)
    return mx, sm

  def row_group_bounds(self, hi, n):
    """(norms fp32 [n, G], diagonal lower bounds fp64, row sums fp64) of the fp16 plane `hi`; the
    row sums carry a zero pad to an even length, the block product's operand alignment."""
    t = torch()
    g = -(-n // BOUND_GROUP_COLS)
    norms = t.empty((n, g), dtype=t.float32, device=self.device)
    diag, c = self.vector(n), self.vector(round_up(n, 2), zero=True)
    self.call("sc_row_group_bounds", _ptr(hi), n, hi.stride(0), _ptr(norms), g, _ptr(diag), _ptr(c),
              self.stream)
    return norms, diag, c

  def bound_order(self, norms):
    """Row order of the bounded Diffuse (device int32): stable sort by the labels of a spherical
    k-means of the profiles, computed and applied on the device without a host synchronisation.
    The same order on every call; profiles that are all alike keep the natural order."""
    t = torch()
    n = int(norms.shape[0])
    perm = t.empty(n, dtype=t.int32, device=self.device)
    self.call("sc_bound_order", _ptr(norms), n, int(norms.shape[1]), BOUND_ORDER_CLUSTERS,
              BOUND_ORDER_ITERS, _ptr(perm), self.stream)
    return perm

  def rowmax_tiles(self, hi, n, norms, diag, perm):
    """Row maxima (fp32) of S = hi hi^T from the tiles of the product of hi[perm] that can hold
    one, and (computed, total) tile counts as a device int32 [2]."""
    t = torch()
    yp = t.empty_like(hi)
    self.call("sc_gather_rows_f16", _ptr(hi), hi.stride(0), _ptr(perm), n, hi.shape[1], _ptr(yp),
              yp.stride(0), self.stream)
    tiles = t.empty(-(-n // LIST_BM) * -(-n // LIST_BN), dtype=t.int32, device=self.device)
    counts = t.empty(2, dtype=t.int32, device=self.device)
    self.call("sc_diffuse_tile_list", _ptr(norms), int(norms.shape[1]), _ptr(diag), _ptr(perm), n,
              _ptr(tiles), _ptr(counts), _ptr(counts[1:]), self.stream)
    mx = self.vector(n, t.float32)
    self.call("sc_diffuse_rowmax_tiles", _ptr(yp), yp.stride(0), n, _ptr(tiles), _ptr(counts),
              _ptr(perm), _ptr(mx), self.stream)
    del yp
    return mx, counts

  def bound_order_hubs(self, norms, diag):
    """Hub-first row order of the bounded Diffuse: the clusters of bound_order, each re-sorted by
    its diagonal descending (ties by row), as (perm, starts) device int32 tensors; starts[c] is the
    first position of cluster c and starts[-1] = n.  No host synchronisation."""
    t = torch()
    n = int(norms.shape[0])
    perm = t.empty(n, dtype=t.int32, device=self.device)
    starts = t.empty(BOUND_ORDER_CLUSTERS + 1, dtype=t.int32, device=self.device)
    self.call("sc_bound_order_hubs", _ptr(norms), n, int(norms.shape[1]), BOUND_ORDER_CLUSTERS,
              BOUND_ORDER_ITERS, _ptr(diag), _ptr(perm), _ptr(starts), self.stream)
    return perm, starts

  def hub_rowmax_tiles(self, hi, n, norms, perm, starts, want_phase1=False):
    """Row maxima (fp32) of S = hi hi^T in two listed launches over hi[perm]: phase 1 pairs every
    cluster's rows with its hub, phase 2 computes the tiles the per-row rule keeps against the
    maxima phase 1 found.  Also the tile counts (phase 1, phase 2, total) as a device int32 [3],
    and with want_phase1 a copy of the phase-1 maxima."""
    t = torch()
    yp = t.empty_like(hi)
    self.call("sc_gather_rows_f16", _ptr(hi), hi.stride(0), _ptr(perm), n, hi.shape[1], _ptr(yp),
              yp.stride(0), self.stream)
    k = int(starts.shape[0]) - 1
    size = -(-n // LIST_BM) * -(-n // LIST_BN)
    tiles1 = t.empty(size, dtype=t.int32, device=self.device)
    tiles2 = t.empty(size, dtype=t.int32, device=self.device)
    counts = t.empty(3, dtype=t.int32, device=self.device)
    mx = self.vector(n, t.float32)
    self.call("sc_diffuse_hub_tiles", _ptr(starts), k, n, _ptr(tiles1), _ptr(counts), self.stream)
    self.call("sc_diffuse_rowmax_tiles", _ptr(yp), yp.stride(0), n, _ptr(tiles1), _ptr(counts),
              _ptr(perm), _ptr(mx), self.stream)
    phase1 = mx.clone() if want_phase1 else None
    self.call("sc_diffuse_tile_list_rows", _ptr(norms), int(norms.shape[1]), _ptr(perm), n,
              _ptr(mx), _ptr(starts), k, _ptr(tiles2), _ptr(counts[1:]), _ptr(counts[2:]),
              self.stream)
    self.call("sc_diffuse_rowmax_tiles_fold", _ptr(yp), yp.stride(0), n, _ptr(tiles2),
              _ptr(counts[1:]), _ptr(perm), _ptr(mx), self.stream)
    del yp
    if want_phase1:
      return mx, counts, phase1
    return mx, counts

  def bounded_diffuse(self, n, hi, want_max=True):
    """Statistics of S = Y Y^T (Y >= 0 and bitwise symmetric, `hi` its fp16 plane), S never formed:
    (rowmax fp32 or None, rowsum fp64, tile counts).  rowsum = Y (Y 1) by two passes over Y; the
    row maxima, when wanted, from the hub-first tile lists (bit for bit those of sc_diffuse).  The
    counts are an int32 tensor [2] (computed in both phases, total): on the device, or on the host
    (0 computed) when no GEMM runs."""
    t = torch()
    norms, diag, c = self.row_group_bounds(hi, n)
    rowsum = t.empty((1, n), dtype=t.float64, device=self.device)
    self.block_product_f16(hi, n, n, c.view(1, -1), 1, rowsum)
    if not want_max:
      return None, rowsum.view(n), t.tensor([0, bounded_tile_count(n)], dtype=t.int32)
    perm, starts = self.bound_order_hubs(norms, diag)
    mx, counts = self.hub_rowmax_tiles(hi, n, norms, perm, starts)
    return mx, rowsum.view(n), t.stack((counts[0] + counts[1], counts[2]))

  # ---- row panels of the factored route
  def normalized_planes(self, x_dev):
    """Split fp16 planes of the row-normalised embeddings (the affinity GEMM's operands) of a
    device [n, d] fp16/bf16/fp32/fp64 tensor."""
    n, d = int(x_dev.shape[0]), int(x_dev.shape[1])
    hi, lo = self.planes(n, d)
    self.call("sc_normalize_rows_typed", _ptr(x_dev), dtype_code(x_dev), n, d, x_dev.stride(0),
              None, 0, _ptr(hi), _ptr(lo), hi.stride(0), self.stream)
    return hi, lo

  def affinity_panel(self, hi, lo, n, d, a0, a1, crop=None):
    """Rows [a0, a1) of the affinity (bitwise those of affinity()); with `crop` (fp32, length n)
    their CropDiagonal values also land in crop[a0:a1]."""
    t = torch()
    panel = t.empty((a1 - a0, round_up(n, 64)), dtype=t.float32, device=self.device)
    self.call("sc_affinity_cosine_panel", self.gemm_precision, _ptr(hi), _ptr(lo), hi.stride(0),
              n, d, a0, a1 - a0, _ptr(panel), panel.stride(0),
              None if crop is None else _ptr(crop[a0:]), self.stream)
    return panel

  def blur_upper_rowmax_block(self, panel, a0, n, r0, r1, sigma, diag, zero_diag, b, m):
    """Pass 1 of the symmetric blur pair on a panel: b <- upper tiles of rows [r0, r1), and their
    row and column maxima folded into m."""
    self.call("sc_blur_upper_rowmax_block", _ptr(panel), n, panel.stride(0), a0,
              int(panel.shape[0]), r0, r1, _ptr(diag), float(sigma), int(bool(zero_diag)), _ptr(b),
              b.stride(0), _ptr(m), self.stream)

  def threshold_symmetrize_upper_block(self, b, n, r0, r1, rowmax, p, mult, binarize,
                                       preserve_diag, sym_type, hi):
    """Pass 2 on a panel: Y_hi (full size) <- the tile pairs whose rows lie in [r0, r1)."""
    self.call("sc_threshold_symmetrize_upper_block", _ptr(b), n, b.stride(0), r0, r1,
              _ptr(rowmax), float(p), float(mult), int(bool(binarize)), int(bool(preserve_diag)),
              int(sym_type), None, 0, _ptr(hi), None, hi.stride(0), self.stream)

  def block_product_f16(self, s, rows, n, t_, b, y):
    self.call("sc_block_product_f16", _ptr(s), rows, n, s.stride(0), _ptr(t_), t_.stride(0), b,
              _ptr(y), y.stride(0), self.stream)

  def eigh_factored(self, y_hi, n, delta, left, right, sign, which, n_values, n_vectors, tol=1e-9,
                    max_matvecs=0):
    """eigh() of the block Lanczos solver on S = Y_hi Y_hi^T, S never formed."""
    t = torch()
    w = np.empty(max(n_values, 1), dtype=np.float64)
    v = t.empty((n, max(n_vectors, 1)), dtype=t.float64, device=self.device)
    stats = np.zeros(4, dtype=np.int64)
    self.call("sc_eigh_extremal_factored", _ptr(y_hi), n, y_hi.stride(0), _ptr(delta), _ptr(left),
              _ptr(right), float(sign), int(which), n_values, n_vectors, float(tol),
              int(max_matvecs), w.ctypes.data_as(ctypes.c_void_p), _ptr(v),
              stats.ctypes.data_as(ctypes.c_void_p), self.stream)
    return w[:n_values], v[:, :n_vectors], stats

  def row_stats(self, a, n, want_max=True, want_sum=True):
    mx = self.vector(n) if want_max else None
    sm = self.vector(n) if want_sum else None
    self.call("sc_row_stats", _ptr(a), n, a.stride(0), _ptr(mx), _ptr(sm), self.stream)
    return mx, sm

  def row_normalize(self, a, n):
    out = self.matrix(n)
    self.call("sc_row_normalize", _ptr(a), n, a.stride(0), _ptr(out), out.stride(0), self.stream)
    return out

  def laplacian(self, w, n, type_, eps=1e-10):
    out = self.matrix(n)
    self.call("sc_laplacian", _ptr(w), n, w.stride(0), int(type_), float(eps), _ptr(out),
              out.stride(0), self.stream, exc=ValueError)
    return out

  def eigh(self, s, n, delta, left, right, sign, which, n_values, n_vectors, dense, tol=1e-9,
           max_matvecs=0):
    """Sorted extremal eigenvalues (host fp64) and eigenvectors (device fp64 [n, n_vectors])."""
    t = torch()
    w = np.empty(max(n_values, 1), dtype=np.float64)
    v = t.empty((n, max(n_vectors, 1)), dtype=t.float64, device=self.device)
    wp = w.ctypes.data_as(ctypes.c_void_p)
    stats = np.zeros(4, dtype=np.int64)
    if dense:
      self.call("sc_eigh_dense", _ptr(s), n, s.stride(0), _ptr(delta), _ptr(left), _ptr(right),
                float(sign), int(which), n_values, n_vectors, wp, _ptr(v), None, None, self.stream)
    else:
      self.call("sc_eigh_extremal", _ptr(s), n, s.stride(0), _ptr(delta), _ptr(left),
                _ptr(right), float(sign), int(which), n_values, n_vectors, float(tol),
                int(max_matvecs), wp, _ptr(v), stats.ctypes.data_as(ctypes.c_void_p),
                self.stream)
    return w[:n_values], v[:, :n_vectors], stats

  def eigh_window(self, s, n, delta, left, right, sign, which, n_values, locked, n_locked, scale,
                  tol=1e-9, max_matvecs=0):
    """The next n_values extremal eigenvalues (host fp64) on the complement of locked[:n_locked]
    (device fp64 [capacity, n]); their symmetrised-space vectors land in locked[n_locked:].  The
    operand decides the operator: an fp32 `s` is S itself, an fp16 `s` is Y_hi of the factored
    operator S = Y_hi Y_hi^T (sc_eigh_extremal_locked_factored), never formed."""
    w = np.empty(n_values, dtype=np.float64)
    stats = np.zeros(4, dtype=np.int64)
    assert locked.shape[0] >= n_locked + n_values and locked.shape[1] == n and locked.is_contiguous()
    entry = ("sc_eigh_extremal_locked_factored" if s.dtype == torch().float16
             else "sc_eigh_extremal_locked")
    self.call(entry, _ptr(s), n, s.stride(0), _ptr(delta), _ptr(left),
              _ptr(right), float(sign), int(which), n_values, float(tol), int(max_matvecs),
              float(scale), _ptr(locked), n_locked, w.ctypes.data_as(ctypes.c_void_p),
              stats.ctypes.data_as(ctypes.c_void_p), self.stream)
    return w, stats

  def eigh_mapback(self, u, n, cols, left, right):
    """Eigenvectors (device fp64 [n, len(cols)]) of the operator from the symmetrised-space
    vectors u[cols] (device fp64 [*, n])."""
    t = torch()
    idx = np.ascontiguousarray(cols, dtype=np.int32)
    v = t.empty((n, max(len(idx), 1)), dtype=t.float64, device=self.device)
    if len(idx):
      assert int(idx.min()) >= 0 and int(idx.max()) < u.shape[0] and u.is_contiguous()
      self.call("sc_eigh_mapback", _ptr(u), n, idx.ctypes.data_as(ctypes.c_void_p), len(idx),
                _ptr(left), _ptr(right), _ptr(v), self.stream)
    return v[:, :len(idx)]

  def eigh_dense_pick(self, s, n, delta, left, right, sign, which, picker):
    """Full spectrum by the dense solver; `picker(w) -> count` (host) decides from the sorted
    eigenvalues how many eigenvectors are computed.  Returns (w[n], v device [n, count])."""
    t = torch()
    w = np.empty(n, dtype=np.float64)
    box = {}

    def pick(_user, w_ptr, n_values, out_ptr):
      try:
        count = int(picker(np.ctypeslib.as_array(w_ptr, shape=(int(n_values),)).copy()))
        count = max(0, min(count, int(n_values)))
        box["v"] = t.empty((n, max(count, 1)), dtype=t.float64, device=self.device)
        out_ptr[0] = box["v"].data_ptr()
        box["count"] = count
        return count
      except Exception as e:                         # never unwind through the C frame
        box["error"] = e
        return -1

    callback = nat.PICK_FN(pick)
    try:
      self.call("sc_eigh_dense", _ptr(s), n, s.stride(0), _ptr(delta), _ptr(left), _ptr(right),
                float(sign), int(which), n, 0, w.ctypes.data_as(ctypes.c_void_p), None, callback,
                None, self.stream)
    except nat.NativeError:
      if "error" in box:
        raise box["error"]
      raise
    return w, box["v"][:, :box["count"]]

  def row_renorm(self, e):
    self.call("sc_row_renorm", _ptr(e), int(e.shape[0]), int(e.shape[1]), self.stream)

  def kmeans(self, e, k, metric, max_iter, tol=0.001):
    """run_kmeans on a contiguous device fp64 [n, k_dim] array -> (host int64 labels, passes).
    `metric` is an SC_KMEANS_* code.  Errors are ValueError, except a singular mahalanobis
    covariance: numpy.linalg.LinAlgError("Singular matrix"), as np.linalg.inv raises it."""
    n, kd = int(e.shape[0]), int(e.shape[1])
    # scikit-learn's draws: RandomState(0).choice(n, p=uniform) then uniform(size=trials) per
    # additional centre (sklearn/cluster/_kmeans.py:231, :249).  Host RNG logic only.
    rs = np.random.RandomState(0)
    first = int(rs.choice(n, p=np.full(n, 1.0 / n)))
    trials = 2 + int(np.log(k))
    u = np.ascontiguousarray(
        [rs.uniform(size=trials) for _ in range(k - 1)], dtype=np.float64).reshape(-1)
    labels = np.empty(n, dtype=np.int64)
    iters = np.zeros(1, dtype=np.int64)
    try:
      self.call("sc_kmeans", _ptr(e), n, kd, int(k), first,
                u.ctypes.data_as(ctypes.c_void_p) if u.size else None, trials, int(metric),
                int(max_iter), float(tol), labels.ctypes.data_as(ctypes.c_void_p),
                iters.ctypes.data_as(ctypes.c_void_p), self.stream, exc=ValueError)
    except ValueError as err:
      if str(err) == "Singular matrix":
        raise np.linalg.LinAlgError("Singular matrix") from None
      raise
    return labels, int(iters[0])

  def cosine_distances(self, x_dev):
    """scipy pdist(x, "cosine") of a device [n, d] fp32/fp64 tensor as a full symmetric fp64
    [n, ld] device matrix, and a device int32 flag that is 1 iff an entry is not finite."""
    t = torch()
    n, d = int(x_dev.shape[0]), int(x_dev.shape[1])
    dist = self.matrix(n, t.float64)
    flag = t.empty((1,), dtype=t.int32, device=self.device)
    self.call("sc_cosine_distances_f64", _ptr(x_dev), 1 if x_dev.dtype == t.float64 else 0, n, d,
              x_dev.stride(0), _ptr(dist), dist.stride(0), _ptr(flag), self.stream)
    return dist, flag

  def cluster_centroids(self, x_dev, labels: np.ndarray):
    """utils.get_cluster_centroids bit for bit on a device [n, d] fp32/fp64 tensor and host labels
    -> device fp64 [max(labels) + 1, d] (NaN rows for ids without a member)."""
    t = torch()
    labels = np.asarray(labels).astype(np.int64)
    if labels.shape != (x_dev.shape[0],):
      raise ValueError("labels must hold one id per embedding")
    if labels.size and labels.min() < 0:
      raise ValueError("'list' argument must have no negative elements")   # np.bincount's error
    n, d = int(x_dev.shape[0]), int(x_dev.shape[1])
    k = int(labels.max()) + 1
    lab = t.from_numpy(labels).to(self.device)
    out = t.empty((k, d), dtype=t.float64, device=self.device)
    self.call("sc_cluster_centroids", _ptr(x_dev), 1 if x_dev.dtype == t.float64 else 0, n, d,
              x_dev.stride(0), _ptr(lab), k, _ptr(out), out.stride(0), self.stream)
    return out

  def complete_linkage(self, dist, n: int):
    """Complete-linkage NN-chain over the device distance matrix (overwritten) -> host
    (xy int64 [n-1, 2], distance fp64 [n-1], size int64 [n-1]), in chain order."""
    return self.nn_chain(nn_chain_entry(nat.LINKAGE_COMPLETE, n), dist, n, nat.LINKAGE_COMPLETE)

  def average_linkage(self, dist, n: int):
    """Average-linkage NN-chain over the device distance matrix (overwritten) -> host
    (xy int64 [n-1, 2], distance fp64 [n-1], size int64 [n-1]), in chain order."""
    return self.nn_chain(nn_chain_entry(nat.LINKAGE_AVERAGE, n), dist, n, nat.LINKAGE_AVERAGE)

  def naive_cluster(self, x_dev, threshold: float, adaptation_threshold: float, stop_at: int = 0,
                    means=None, counts=None):
    """NaiveClusterer over the rows of a device [n, d] fp32/fp64 tensor (row stride free, unit
    column stride) in one launch, continuing from device means (fp64 [c0, d]) / counts (int64
    [c0]) when given; stop_at > 0 stops once that many clusters are open.  -> (labels int64
    device [processed], processed, clusters, means fp64 device [clusters, d], counts int64 device
    [clusters])."""
    t = torch()
    n, d = int(x_dev.shape[0]), int(x_dev.shape[1])
    c0 = 0 if means is None else int(means.shape[0])
    grow = n if stop_at <= 0 else min(n, max(int(stop_at) - c0, 0))
    cap = c0 + grow
    m = t.empty((max(cap, 1), d), dtype=t.float64, device=self.device)
    c = t.empty((max(cap, 1),), dtype=t.int64, device=self.device)
    if c0:
      m[:c0].copy_(means)
      c[:c0].copy_(counts)
    labels = t.empty((max(n, 1),), dtype=t.int64, device=self.device)
    processed, clusters = ctypes.c_int64(), ctypes.c_int64()
    self.call("sc_naive_cluster", _ptr(x_dev), 1 if x_dev.dtype == t.float64 else 0, n, d,
              x_dev.stride(0), float(threshold), float(adaptation_threshold), int(stop_at),
              _ptr(m), m.stride(0), _ptr(c), cap, c0, _ptr(labels), ctypes.byref(processed),
              ctypes.byref(clusters), self.stream)
    k = clusters.value
    return labels[:processed.value], processed.value, k, m[:k], c[:k]

  def nn_chain(self, entry: str, dist, n: int, linkage: int):
    """The NN-chain entry `entry` (one of nn_chain_entry's answers) for an nat.LINKAGE_* linkage;
    complete_linkage / average_linkage choose the entry by n."""
    xy = np.empty((n - 1, 2), dtype=np.int64)
    md = np.empty(n - 1, dtype=np.float64)
    ms = np.empty(n - 1, dtype=np.int64)
    head = (_ptr(dist), n, dist.stride(0)) + ((linkage,) if entry == "sc_nn_chain_small" else ())
    self.call(entry, *head, xy.ctypes.data_as(ctypes.c_void_p),
              md.ctypes.data_as(ctypes.c_void_p), ms.ctypes.data_as(ctypes.c_void_p), self.stream)
    return xy, md, ms


class Refined:
  """Result of the refinement sequence in the structured form the eigensolver wants:
  the matrix is diag(row_scale) * S with S fp32 on the device (`row_scale` None = ones).
  `symmetric` tells whether S is symmetric (up to rounding).  On the factored route S is not
  stored: `s` is None and S = y_hi y_hi^T with y_hi the fp16 hi plane of Y."""

  def __init__(self, s, n, symmetric, row_scale=None, rowsum=None, y_hi=None, tiles=None):
    self.s = s
    self.n = n
    self.symmetric = symmetric
    self.row_scale = row_scale
    self.rowsum = rowsum      # fp64 row sums of S when the Diffuse epilogue produced them
    self.y_hi = y_hi
    # bounded Diffuse (stored front end): its (computed, total) tile counts, an int32 tensor [2]
    self.tiles = tiles


def factored_sequence_ok(eng: Engine, options) -> bool:
  """Whether options.refinement_sequence is [CropDiagonal] GaussianBlur RowWiseThreshold(RowMax)
  Symmetrize Diffuse [RowWiseNormalize] with a radius-4 blur: the chain the factored route runs."""
  from . import refinement as rf
  RN = rf.RefinementName
  names = list(options.refinement_sequence or [])
  if names[:1] == [RN.CropDiagonal]:
    names = names[1:]
  if names[-1:] == [RN.RowWiseNormalize]:
    names = names[:-1]
  return (names == [RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize, RN.Diffuse] and
          options.thresholding_type == rf.ThresholdType.RowMax and
          isinstance(options.symmetrize_type, rf.SymmetrizeType) and
          eng.upper_pass_ok(float(options.gaussian_blur_sigma)))


class FactoredAffinity:
  """The affinity of the factored route: never stored, rebuilt in row panels from the split planes
  of the normalised embeddings.  The blur's row maxima m do not depend on p_percentile, so pass 1
  runs once per predict() and every AutoTune evaluation reuses it."""

  def __init__(self, eng: Engine, x_dev, panel_rows: typing.Optional[int] = None):
    self.n, self.d = int(x_dev.shape[0]), int(x_dev.shape[1])
    self.hi, self.lo = eng.normalized_planes(x_dev)
    self.panel_rows = panel_rows or panel_rows_for(self.n)
    self.symmetric = True
    self.crop_vector = None
    self._m = None

  def _panels(self, eng: Engine, options):
    """Yield (r0, r1, affinity panel, its first row a0, crop values by global row or None,
    B panel) over panel_plan()."""
    from . import refinement as rf
    t = torch()
    crop_first = list(options.refinement_sequence or [])[:1] == [rf.RefinementName.CropDiagonal]
    diag = eng.vector(self.n, t.float32) if crop_first else None
    b = t.empty((self.panel_rows, round_up(self.n, 64)), dtype=t.float32, device=eng.device)
    for r0, r1, a0, a1 in panel_plan(self.n, self.panel_rows):
      panel = eng.affinity_panel(self.hi, self.lo, self.n, self.d, a0, a1, diag)
      yield r0, r1, panel, a0, diag, b
      del panel

  def _rows(self, eng: Engine, stop: typing.Optional[int] = None):
    """Yield (r0, r1, affinity rows [r0, r1)) over panel_plan(), without the blur halo, for the
    panels that start below `stop`."""
    for r0, r1, _, _ in panel_plan(self.n, self.panel_rows):
      if stop is not None and r0 >= stop:
        break
      panel = eng.affinity_panel(self.hi, self.lo, self.n, self.d, r0, r1)
      yield r0, r1, panel
      del panel

  def statistics(self, eng: Engine) -> typing.Dict[str, float]:
    """{min, neighbor_min, std} of the affinity for the single-cluster checks: the per-row partials
    of sc_affinity_stats over one sweep of row panels, finished in its order, so the values are
    those of the stored affinity bit for bit."""
    n = self.n
    part = eng.vector(4 * n + 4)
    for r0, r1, panel in self._rows(eng):
      eng.call("sc_affinity_stats_rows", _ptr(panel), r1 - r0, n, panel.stride(0), r0, _ptr(part),
               eng.stream)
    from . import fallback_clusterer
    out = np.zeros(4, dtype=np.float64)
    eng.call("sc_affinity_stats_finish", _ptr(part), n, out.ctypes.data_as(ctypes.c_void_p),
             eng.stream)
    return fallback_clusterer.statistics_from_sums(out, n)

  def upper_band(self, eng: Engine, offset: int):
    """(band, row_off): the packed band affinity[np.triu_indices(n, offset)] of the AffinityGmmBic
    check (gmm_bic.packed_row_offsets; fp32, NaN in its padding slots) and its device row offsets,
    from one sweep of row panels."""
    from . import gmm_bic
    t = torch()
    n = self.n
    off = gmm_bic.packed_row_offsets(n, offset)
    band = t.empty((max(int(off[-1]), 4),), dtype=t.float32, device=eng.device)
    row_off = t.from_numpy(off).to(eng.device)
    for r0, r1, panel in self._rows(eng, stop=gmm_bic.band_rows(n, offset)):
      eng.call("sc_gmm_band_pack", _ptr(panel), panel.stride(0), r0, r1 - r0, n, int(offset),
               _ptr(row_off), _ptr(band), eng.stream)
    return band, row_off

  def rowmax(self, eng: Engine, options):
    """m of the symmetric blur pair (pass 1 over every panel), computed once."""
    if self._m is None:
      m = eng.vector(self.n, torch().float32, zero=True)
      zero_diag = bool(options.thresholding_preserve_diagonal)
      sigma = float(options.gaussian_blur_sigma)
      for r0, r1, panel, a0, diag, b in self._panels(eng, options):
        eng.blur_upper_rowmax_block(panel, a0, self.n, r0, r1, sigma, diag, zero_diag, b, m)
      self._m = m
    return self._m

  def refine(self, eng: Engine, options) -> Refined:
    """The refinement sequence on the factored route: Y_hi by pass 2 over every panel, then the
    statistics-only Diffuse."""
    from . import refinement as rf
    t = torch()
    n = self.n
    m = self.rowmax(eng, options)
    scratch = eng.vector(n, t.float32, zero=True)   # pass 2 re-folds maxima that are already in m
    y_hi = t.empty((n, round_up(n, 64)), dtype=t.float16, device=eng.device)
    sym_type = (nat.SYMMETRIZE_MAX if options.symmetrize_type == rf.SymmetrizeType.Max
                else nat.SYMMETRIZE_AVERAGE)
    zero_diag = bool(options.thresholding_preserve_diagonal)
    sigma = float(options.gaussian_blur_sigma)
    for r0, r1, panel, a0, diag, b in self._panels(eng, options):
      eng.blur_upper_rowmax_block(panel, a0, n, r0, r1, sigma, diag, zero_diag, b, scratch)
      eng.threshold_symmetrize_upper_block(
          b, n, r0, r1, m, options.p_percentile, options.thresholding_soft_multiplier,
          options.thresholding_with_binarization, zero_diag, sym_type, y_hi)
    del scratch
    mx, sm = eng.diffuse_stats(n, y_hi)
    names = list(options.refinement_sequence)
    row_scale = 1.0 / mx.double() if names[-1] == rf.RefinementName.RowWiseNormalize else None
    return Refined(None, n, True, row_scale, sm, y_hi=y_hi)



def run_refinement(eng: Engine, a, n: int, options, crop_vector=None, a_symmetric=True,
                   diffuse_precision=None, bounded=False) -> Refined:
  """Apply options.refinement_sequence to the device affinity `a`.

  Fusions (all exact restatements, SURVEY.md A.3):
    [CropDiagonal] GaussianBlur? RowWiseThreshold(RowMax) Symmetrize  on a symmetric input
        -> crop vector + blur statistics pass + blur/threshold/symmetrize pass (12 B/element),
           emitting fp16 planes directly when Diffuse follows;
    RowWiseNormalize as the last operator -> kept as a row scaling for the eigensolver.
  Anything else runs operator by operator.
  `bounded` (the caller checked the scope: a single-MMA Diffuse closing the fused chain): S is not
  stored; the result carries Y_hi, the row sums Y (Y 1) and the bounded Diffuse's row maxima.
  """
  from . import refinement as rf
  names = list(options.refinement_sequence or [])
  RN = rf.RefinementName
  cur = a
  sym = a_symmetric
  planes = None          # (hi, lo) of `cur` when available
  cur_is_planes_only = False
  row_scale = None
  stats = None           # (rowmax fp32, rowsum fp64) of `cur` straight from the Diffuse epilogue
  y_hi = tiles = None    # the bounded Diffuse's operand and tile counts
  i = 0
  while i < len(names):
    name = names[i]
    if not isinstance(name, RN):
      raise ValueError("Unknown refinement operation: {}".format(name))
    # ---- fused chain
    j = i
    has_crop = names[j] == RN.CropDiagonal
    if has_crop:
      j += 1
    has_blur = j < len(names) and names[j] == RN.GaussianBlur
    if has_blur:
      j += 1
    fusable = (sym and row_scale is None and not cur_is_planes_only and
               j + 1 < len(names) and names[j] == RN.RowWiseThreshold and
               names[j + 1] == RN.Symmetrize and
               options.thresholding_type == rf.ThresholdType.RowMax and
               isinstance(options.symmetrize_type, rf.SymmetrizeType))
    if fusable:
      sigma = float(options.gaussian_blur_sigma) if has_blur else 0.0
      diag = None
      if has_crop:
        if crop_vector is not None and i == 0:
          diag = crop_vector
        else:
          diag = eng.crop_values(cur, n)
      zero_diag = bool(options.thresholding_preserve_diagonal)
      next_is_diffuse = j + 2 < len(names) and names[j + 2] == RN.Diffuse
      use_tc = eng.gemm_engine(n) == nat.GEMM_TCGEN05
      want_planes = next_is_diffuse and use_tc
      want_f32 = not want_planes
      sym_type = (nat.SYMMETRIZE_MAX if options.symmetrize_type == rf.SymmetrizeType.Max
                  else nat.SYMMETRIZE_AVERAGE)
      if eng.upper_pass_ok(sigma):
        # blur(A) is symmetric: pass 1 keeps only the row maxima of its upper tiles, pass 2 blurs
        # them again and writes Y and its mirror
        b, m = eng.blur_upper_rowmax(cur, n, sigma, diag, zero_diag)
        want_lo = (diffuse_precision if diffuse_precision is not None
                   else eng.gemm_precision) != nat.GEMM_SINGLE
        y, hi, lo = eng.threshold_symmetrize_upper(
            b, n, m, options.p_percentile, options.thresholding_soft_multiplier,
            options.thresholding_with_binarization, zero_diag, sym_type, want_f32, want_planes,
            want_lo)
        del b
      else:
        m = eng.blur_rowmax(cur, n, sigma, diag, zero_diag)
        y, hi, lo = eng.blur_threshold_symmetrize(
            cur, n, sigma, diag, m, options.p_percentile, options.thresholding_soft_multiplier,
            options.thresholding_with_binarization, zero_diag, sym_type, want_f32, want_planes)
      cur = y
      planes = (hi, lo) if want_planes else None
      cur_is_planes_only = want_planes
      sym = True
      i = j + 2
      continue
    # ---- single operators
    if name == RN.Diffuse:
      if row_scale is not None:
        cur, row_scale = _materialise_scale(eng, cur, n, row_scale), None
      # the row reductions of a closing RowWiseNormalize / of the Laplacian degree come out of the
      # GEMM epilogue when Diffuse is the last matrix-valued operator of the sequence
      tail = names[i + 1:]
      fuse_stats = (tail in ([], [RN.RowWiseNormalize]) and
                    eng.gemm_engine(n) == nat.GEMM_TCGEN05)
      if bounded and fuse_stats and planes is not None and planes[1] is None:
        mx, sm, tiles = eng.bounded_diffuse(n, planes[0], want_max=tail == [RN.RowWiseNormalize])
        y_hi, cur = planes[0], None
      elif planes is not None:
        cur, mx, sm = eng.diffuse(n, hi=planes[0], lo=planes[1], want_stats=fuse_stats,
                                  precision=diffuse_precision)
      else:
        cur, mx, sm = eng.diffuse(n, y=cur, want_stats=fuse_stats, precision=diffuse_precision)
      stats = (mx, sm) if sm is not None else None
      planes, cur_is_planes_only, sym = None, False, True
      i += 1
      continue
    if cur_is_planes_only:
      raise AssertionError("internal: planes-only matrix consumed by a non-GEMM operator")
    if name == RN.RowWiseNormalize and i == len(names) - 1 and row_scale is None:
      if stats is not None:
        mx = stats[0].double()
      else:
        mx, _ = eng.row_stats(cur, n, want_max=True, want_sum=False)
      row_scale = 1.0 / mx
      i += 1
      continue
    stats = None
    if row_scale is not None:
      cur, row_scale = _materialise_scale(eng, cur, n, row_scale), None
      sym = False
    if name == RN.CropDiagonal:
      cur = eng.crop_diagonal(cur, n)
    elif name == RN.GaussianBlur:
      cur = eng.gaussian_blur(cur, n, options.gaussian_blur_sigma)
    elif name == RN.RowWiseThreshold:
      if not isinstance(options.thresholding_type, rf.ThresholdType):
        raise TypeError("thresholding_type must be a ThresholdType")
      cur = eng.row_threshold(
          cur, n, nat.THRESHOLD_ROWMAX if options.thresholding_type == rf.ThresholdType.RowMax
          else nat.THRESHOLD_PERCENTILE, options.p_percentile,
          options.thresholding_soft_multiplier, options.thresholding_with_binarization,
          options.thresholding_preserve_diagonal)
      sym = False
    elif name == RN.Symmetrize:
      if options.symmetrize_type == rf.SymmetrizeType.Max:
        cur = eng.symmetrize(cur, n, nat.SYMMETRIZE_MAX)
      elif options.symmetrize_type == rf.SymmetrizeType.Average:
        cur = eng.symmetrize(cur, n, nat.SYMMETRIZE_AVERAGE)
      else:
        raise ValueError("Unsupported symmetrize_type.")
      sym = True
    elif name == RN.RowWiseNormalize:
      cur = eng.row_normalize(cur, n)
      sym = False
    else:
      raise ValueError("Unknown refinement operation: {}".format(name))
    i += 1
  return Refined(cur, n, sym, row_scale, stats[1] if stats is not None else None, y_hi=y_hi,
                 tiles=tiles)


def _materialise_scale(eng: Engine, s, n: int, row_scale):
  # diag(row_scale) S : only reached by sequences that keep refining after RowWiseNormalize
  return eng.row_normalize(s, n)

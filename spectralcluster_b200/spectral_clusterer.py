"""SpectralClusterer -- drop-in mirror of the reference orchestrator
(/root/reference/spectralcluster/spectral_clusterer.py: __init__ :29-106,
_compute_eigenvectors_ncluster :108-168, predict :201-314) whose arithmetic runs on an H100.

predict(): one H2D copy of the [N, d] embeddings (none when they come as a CUDA tensor, which is
read in place as its host twin would be), every N x N intermediate stays in HBM
(affinity GEMM -> fused refinement -> Diffuse GEMM -> row statistics -> symmetric eigensolve ->
k-means), one D2H copy of N labels.  The callers around the path follow the reference: the
fallback clusterer for tiny inputs is host code (scikit-learn, as in the reference); the
max_spectral_size AHC pre-clustering runs on the device (agglomerative.py: fp64 cosine distances and
the complete-linkage NN-chain, scikit-learn's labels integer for integer); the single-cluster checks
are device reductions over the resident affinity.
"""

from __future__ import annotations

import typing

import numpy as np

from . import _native as nat
from . import agglomerative
from . import autotune as autotune_lib
from . import constraint as constraint_lib
from . import custom_distance_kmeans
from . import device as dev
from . import eigen_windows
from . import fallback_clusterer
from . import laplacian as laplacian_lib
from . import naive_clusterer
from . import refinement
from . import utils

AutoTune = autotune_lib.AutoTune
AutoTuneProxy = autotune_lib.AutoTuneProxy
ConstraintName = constraint_lib.ConstraintName
ConstraintOptions = constraint_lib.ConstraintOptions
FallbackOptions = fallback_clusterer.FallbackOptions
LaplacianType = laplacian_lib.LaplacianType
RefinementName = refinement.RefinementName
RefinementOptions = refinement.RefinementOptions
EigenGapType = utils.EigenGapType


# The block Lanczos solver (sc_eigh_extremal) finds at most this many eigenpairs.
LANCZOS_MAX_PAIRS = 32
# The dense solver (sc_eigh_dense) takes n x n operators up to this n; above it, more pairs than
# one Lanczos solve finds come from the windowed solve (eigen_windows.py).
DENSE_MAX_N = 32768


def lanczos_basis(limit: int) -> int:
  """Basis vectors the block Lanczos solver is sized for when `limit` eigenpairs are wanted."""
  return max(2 * limit + 32, 64)


def lanczos_fits(n: int, limit: int) -> bool:
  """Whether the block Lanczos solver takes `limit` eigenpairs of an n x n operator: it reads S a
  handful of times but needs n >= 4 x its basis."""
  return limit <= LANCZOS_MAX_PAIRS and n >= 4 * lanczos_basis(limit)


class DeviceAffinity:
  """An affinity matrix resident in HBM (what predict() passes between its stages)."""

  def __init__(self, matrix, n: int, crop_vector=None, symmetric: bool = True):
    self.matrix = matrix
    self.n = n
    self.crop_vector = crop_vector
    self.symmetric = symmetric


class SpectralClusterer:
  """Spectral clustering of embeddings; same constructor and attributes as the reference."""

  def __init__(self,
               min_clusters: typing.Optional[int] = None,
               max_clusters: typing.Optional[int] = None,
               refinement_options: typing.Optional[RefinementOptions] = None,
               autotune: typing.Optional[AutoTune] = None,
               fallback_options: typing.Optional[FallbackOptions] = None,
               laplacian_type: typing.Optional[LaplacianType] = None,
               stop_eigenvalue: float = 1e-2,
               row_wise_renorm: bool = False,
               custom_dist: typing.Union[str, typing.Callable] = "cosine",
               max_iter: int = 300,
               constraint_options=None,
               eigengap_type: EigenGapType = EigenGapType.Ratio,
               max_spectral_size: typing.Optional[int] = None,
               affinity_function: typing.Callable = utils.compute_affinity_matrix,
               post_eigen_cluster_function: typing.Callable = (
                   custom_distance_kmeans.run_kmeans)):
    self.min_clusters = min_clusters
    self.max_clusters = max_clusters
    self.refinement_options = refinement_options or RefinementOptions()
    self.autotune = autotune
    self.fallback_options = fallback_options or FallbackOptions()
    self.laplacian_type = laplacian_type
    self.row_wise_renorm = row_wise_renorm
    self.stop_eigenvalue = stop_eigenvalue
    self.custom_dist = custom_dist
    self.max_iter = max_iter
    self.constraint_options = constraint_options
    self.eigengap_type = eigengap_type
    self.max_spectral_size = max_spectral_size
    self.affinity_function = affinity_function
    self.post_eigen_cluster_function = post_eigen_cluster_function
    # Diagnostics of the last predict(): eigenvalues used by the eigengap, cluster count, solver.
    self.last_details: typing.Dict[str, typing.Any] = {}
    # Set collect_timings to get, after every predict(), last_timings = {C-ABI entry point: ms of
    # device time (CUDA events)} -- the per-stage breakdown bench.py prints.
    self.collect_timings = False
    self.last_timings: typing.Dict[str, float] = {}
    # Set to a torch.distributed process group (or True for the default group) to spread the
    # AutoTune grid over the ranks, one p_percentile evaluation at a time per GPU
    # (BASELINE.json configs[4]); every rank must call predict() with the same embeddings.
    self.autotune_group = None

  # ------------------------------------------------------------------ eigen stage
  def _constrain(self, eng, affinity: "DeviceAffinity", constraint_matrix) -> "DeviceAffinity":
    """constraint_operator.adjust_affinity on the resident affinity."""
    q_host = np.asarray(constraint_matrix, dtype=np.float64)
    op = self.constraint_options.constraint_operator
    op.check_input(np.empty((affinity.n, affinity.n), dtype=np.bool_), q_host)
    q = eng.upload_matrix(q_host)
    out = op.adjust_on_device(eng, affinity.matrix, q, affinity.n)
    sym = affinity.symmetric and bool(np.array_equal(q_host, q_host.T))
    return DeviceAffinity(out, affinity.n, None, sym)

  def _eigen_on_device(self, eng, affinity: DeviceAffinity, constraint_matrix=None):
    """Refinement + Laplacian terms + eigensolve; returns (w host, V device [n, nv], k, gap)."""
    n = affinity.n
    if isinstance(affinity, dev.FactoredAffinity):
      refined = affinity.refine(eng, self.refinement_options)
    else:
      refined = dev.run_refinement(eng, affinity.matrix, n, self.refinement_options,
                                   crop_vector=affinity.crop_vector,
                                   a_symmetric=affinity.symmetric,
                                   diffuse_precision=eng.diffuse_precision_for(n),
                                   bounded=affinity.symmetric and
                                   self._bounded_route(eng, n, constraint_matrix))
    if (self.constraint_options and not self.constraint_options.apply_before_refinement and
        constraint_matrix is not None):
      # constraint on the refined affinity (spectral_clusterer.py:137-142)
      s = refined.s
      if refined.row_scale is not None:
        s = eng.row_normalize(s, n)
      adjusted = self._constrain(eng, DeviceAffinity(s, n, None, refined.symmetric and
                                                      refined.row_scale is None), constraint_matrix)
      refined = dev.Refined(adjusted.matrix, n, adjusted.symmetric)
    delta, left, right, sign, which = laplacian_lib.operator_terms(eng, refined,
                                                                   self.laplacian_type)
    descend = which == nat.EIG_LARGEST
    limit = n
    if self.max_clusters and self.max_clusters + 1 < limit:
      limit = self.max_clusters + 1
    n_vectors = min(n, max(limit, self.min_clusters or 0))
    op = (refined.s, n, delta, left, right, sign)
    counted = None          # (k, gap) when the solver already ran the eigengap
    fallback = None         # why a Lanczos solve gave way to the dense solver
    top = None              # lambda_max when w is a prefix of an ascending spectrum
    if not refined.symmetric:
      # not symmetric nor diagonally similar to a symmetric matrix (e.g. RowWiseThreshold without
      # Symmetrize): np.linalg.eig + .real semantics (utils.py:59-61) by Krylov-Schur
      from . import arnoldi
      solver = "krylov-schur"
      if limit == n and n > arnoldi.FULL_SPECTRUM_LIMIT:
        # max_clusters=None: only the prefix that settles the eigengap (eigen_windows.py)
        w, v, stats, top = eigen_windows.grow_krylov_schur(
            eng, op, descend, self.min_clusters, self.stop_eigenvalue, self.eigengap_type)
        top_solve = None
      else:
        w, v, stats = arnoldi.eig_extremal_device(eng, *op, not descend, limit, n_vectors)
        top_solve = lambda: arnoldi.eig_extremal_device(eng, *op, False, 1, 0)[0]
    elif refined.y_hi is not None and lanczos_fits(n, limit):
      # factored operator, one solve (the bounded route and _factored_route): S = Y_hi Y_hi^T is
      # never stored.  `solver` names the route's choice: one Lanczos solve after the bounded
      # Diffuse of the stored front end, "lanczos-factored" on the panel route.
      solver = "lanczos" if refined.tiles is not None else "lanczos-factored"
      fop = (refined.y_hi,) + op[1:]
      w, v, stats = eng.eigh_factored(*fop, which, limit, n_vectors)
      stats = stats.tolist()
      top_solve = lambda: eng.eigh_factored(*fop, nat.EIG_LARGEST, 1, 0)[0]
    elif n > eng.dense_eig_max and lanczos_fits(n, limit):
      solver = "lanczos"
      try:
        w, v, stats = eng.eigh(*op, which, limit, n_vectors, False)
        stats = stats.tolist()
        top_solve = lambda: eng.eigh(*op, nat.EIG_LARGEST, 1, 0, False)[0]
      except nat.NativeError as e:
        # a wanted pair did not converge within the product budget: the values next to it crowd
        # within tol * lambda_max (as the nonzero Laplacian values of the near-complete components
        # Diffuse leaves do).  The dense solver takes any stored S up to DENSE_MAX_N, as on the
        # dense route below.
        if n > DENSE_MAX_N or "eigenpairs converged" not in str(e):
          raise
        solver, stats, top_solve, fallback = "dense", None, None, str(e)
        w, v, _ = eng.eigh(*op, which, n, n_vectors, True)
    elif n > DENSE_MAX_N or refined.y_hi is not None:
      # more pairs than one Lanczos solve finds, above the dense solver's n: windows of block
      # Lanczos on the complement of the pairs found, until the eigengap is decided; on the
      # stored S, or on the factored operator of _factored_windows_route
      factored = refined.y_hi is not None
      solver = "lanczos-factored-windows" if factored else "lanczos-windows"
      top_solve = None
      ops = eigen_windows.DeviceOps(eng, *((refined.y_hi,) + op[1:] if factored else op), which,
                                    capacity=eigen_windows.capacity(
                                        n, self.max_clusters, self.min_clusters),
                                    factored=factored)
      prefix = eigen_windows.solve(ops, descend, self.max_clusters, self.min_clusters,
                                   self.stop_eigenvalue, self.eigengap_type, n=n)
      w, top = prefix.values[:limit], prefix.lambda_max
      counted = self._count_clusters(w, descend, top)
      columns = min(len(w), max(counted[0], self.min_clusters or 0, 1))
      v = ops.vectors(prefix.order[:columns])
      stats = ops.stats
    else:
      # the dense solver (Householder tridiagonalisation, 4/3 n^3): small matrices, and
      # max_clusters=None / > 31 (every eigenvalue, or more pairs than Lanczos finds, is needed)
      solver, stats, top_solve = "dense", None, None
      if limit == n and n > 256:
        # every eigenvalue is needed (max_clusters=None scans the whole spectrum, utils.py:100-102)
        # but only the columns predict() will select: the eigengap runs between the two phases
        def picker(values):
          nonlocal counted
          counted = self._count_clusters(values, descend)
          return max(counted[0], self.min_clusters or 0, 1)

        w, v = eng.eigh_dense_pick(*op, which, picker)
      else:
        w, v, _ = eng.eigh(*op, which, n, n_vectors, True)
    if (top_solve is not None and limit < n and not descend and
        self.eigengap_type == EigenGapType.NormalizedDiff):
      # np.max(eigenvalues) of the full spectrum (utils.py:109): one more extremal solve
      w = np.concatenate([w, top_solve()])
    k, gap = counted or self._count_clusters(w, descend, top)
    self.last_details = dict(eigenvalues=np.array(w[:limit]), n_clusters_raw=k, max_gap=gap,
                             solver=solver, lanczos_stats=stats)
    if fallback is not None:
      self.last_details["lanczos_fallback"] = fallback
    if refined.tiles is not None:
      computed, total = refined.tiles.tolist()
      self.last_details["diffuse"] = dict(tiles=computed, of=total, operator="factored")
    return w, v, k, gap

  def _operator_scope(self, eng, n: int, constraint_matrix=None, single_check=False) -> bool:
    """The options every route that never stores S serves: the default affinity, the fused chain
    closed by a single-MMA Diffuse (dev.factored_sequence_ok), no constraint, min_clusters != 1 and
    no autotune_group.  `single_check`: min_clusters == 1 is served too (the factored route's
    single-cluster check, _factored_single_cluster_route)."""
    return (self.affinity_function is utils.compute_affinity_matrix and
            (self.min_clusters != 1 or single_check) and
            not (self.constraint_options and constraint_matrix is not None) and
            self.autotune_group is None and
            dev.factored_sequence_ok(eng, self.refinement_options) and
            eng.gemm_engine(n) == nat.GEMM_TCGEN05 and
            eng.diffuse_precision_for(n) == nat.GEMM_SINGLE)

  def _lanczos_scope(self, eng, n: int, constraint_matrix=None, single_check=False) -> bool:
    """The calls of _operator_scope that one Lanczos solve serves (bounded max_clusters <
    LANCZOS_MAX_PAIRS that lanczos_fits): those of the two one-solve routes below."""
    limit = (self.max_clusters or 0) + 1
    return (self.max_clusters is not None and self.max_clusters < LANCZOS_MAX_PAIRS and
            (self.min_clusters or 0) <= limit and
            n > limit and n > eng.dense_eig_max and lanczos_fits(n, limit) and
            self._operator_scope(eng, n, constraint_matrix, single_check))

  def _factored_route(self, eng, n: int, constraint_matrix=None, single_check=False) -> bool:
    """Whether predict() on n embeddings takes the factored route with one Lanczos solve: the
    stored route's peak (computed from shapes) exceeds eng.factored_above_bytes and every option
    is one _lanczos_scope accepts.  _factored_windows_route covers the eigen options one solve
    cannot serve, _factored_single_cluster_route the calls with min_clusters == 1; any other call
    keeps the stored route."""
    return (self._lanczos_scope(eng, n, constraint_matrix, single_check) and
            dev.stored_route_peak_bytes(n) > eng.factored_above_bytes)

  def _factored_windows_route(self, eng, n: int, constraint_matrix=None,
                              single_check=False) -> bool:
    """Whether predict() on n embeddings takes the factored route with the windowed solve
    (eigen_windows.py on the factored operator): as _factored_route, but for max_clusters=None or
    more pairs than one Lanczos solve finds.  Disjoint from _factored_route."""
    return ((self.max_clusters is None or self.max_clusters + 1 > LANCZOS_MAX_PAIRS) and
            n > DENSE_MAX_N and dev.stored_route_peak_bytes(n) > eng.factored_above_bytes and
            self._operator_scope(eng, n, constraint_matrix, single_check))

  def _factored_single_cluster_route(self, eng, n: int, constraint_matrix=None) -> bool:
    """Whether predict() on n embeddings with min_clusters == 1 takes the factored route: the calls
    _factored_route or _factored_windows_route would take if min_clusters were not 1.  The
    single-cluster check runs on panels of the affinity (FactoredAffinity.statistics /
    upper_band), then the eigen stage as on those routes.  Disjoint from the other three routes,
    which refuse min_clusters == 1."""
    return self.min_clusters == 1 and (
        self._factored_route(eng, n, constraint_matrix, single_check=True) or
        self._factored_windows_route(eng, n, constraint_matrix, single_check=True))

  def _bounded_route(self, eng, n: int, constraint_matrix=None) -> bool:
    """Whether the stored front end (a resident affinity) replaces the storing Diffuse and the
    stored Lanczos solve by the bounded Diffuse and one Lanczos solve on the factored operator:
    the calls of _lanczos_scope from N = dev.BOUNDED_FROM that do not take the factored route."""
    return (n >= dev.BOUNDED_FROM and self._lanczos_scope(eng, n, constraint_matrix) and
            dev.stored_route_peak_bytes(n) <= eng.factored_above_bytes)

  def _count_clusters(self, eigenvalues, descend: bool, max_eigenvalue=None):
    """utils.compute_number_of_clusters with this clusterer's options -> (k, max gap); only a
    descending spectrum stops at stop_eigenvalue.  `max_eigenvalue`: lambda_max of a spectrum of
    which `eigenvalues` is an ascending prefix."""
    stop = dict(stop_eigenvalue=self.stop_eigenvalue) if descend else {}
    return utils.compute_number_of_clusters(eigenvalues, max_clusters=self.max_clusters,
                                            eigengap_type=self.eigengap_type, descend=descend,
                                            max_eigenvalue=max_eigenvalue, **stop)

  def _compute_eigenvectors_ncluster(self, affinity, constraint_matrix=None):
    """(eigenvectors, n_clusters, max eigengap) for an affinity matrix.

    `affinity` is a host ndarray (reference signature) or a DeviceAffinity.  Eigenvectors come
    back as a host ndarray [n, n_vec] in the first case, a device fp64 tensor in the second;
    n_vec covers every column predict() can select (all n when max_clusters is None)."""
    eng = dev.Engine.get()
    if isinstance(affinity, (DeviceAffinity, dev.FactoredAffinity)):
      _, v, k, gap = self._eigen_on_device(eng, affinity, constraint_matrix)
      return v, k, gap
    a = np.asarray(affinity)
    if a.ndim != 2:
      raise ValueError("affinity must be 2-dimensional")
    if a.shape[0] != a.shape[1]:
      raise ValueError("affinity must be a square matrix")
    sym = bool(np.allclose(a, a.T, rtol=1e-6, atol=1e-9))
    da = DeviceAffinity(eng.upload_matrix(a), a.shape[0], None, sym)
    _, v, k, gap = self._eigen_on_device(eng, da, constraint_matrix)
    return v.to("cpu").numpy(), k, gap

  def _reduce_size_and_predict(self, embeddings) -> np.ndarray:
    """spectral_clusterer.py:170-199: complete-linkage cosine AHC down to `max_spectral_size`
    clusters (the reference's own lossy answer to large N, on the device with scikit-learn's labels
    -- see agglomerative.py; BASELINE configs[3] shards the exact problem instead), spectral
    clustering of the cluster centroids on the device, labels chained back.  A CUDA tensor stays on
    the device: its centroids are a device fp64 tensor (sc_cluster_centroids), clustered in turn."""
    on_device = not isinstance(embeddings, np.ndarray)
    x = dev.twin(embeddings) if on_device else embeddings
    pre = agglomerative.CosineCompleteLinkage(n_clusters=self.max_spectral_size).fit_predict(x)
    return utils.chain_labels(pre, self.predict(utils.get_cluster_centroids(x, pre)))

  # ------------------------------------------------------------------ predict
  def predict(self, embeddings, constraint_matrix=None) -> np.ndarray:
    """Cluster the rows of `embeddings` -> int64 labels (a host ndarray).

    `embeddings` is an [n_samples, n_features] ndarray, or a CUDA tensor on the device
    Engine.get() serves (float16, bfloat16, float32 or float64; integer and bool tensors are
    widened to float64; any row stride).  A CUDA tensor X is clustered in place, never copied to
    the host except where a user `affinity_function` or scikit-learn must receive an ndarray, and
    gives what its host twin gives, bit for bit: X.cpu().numpy(), or X.float().cpu().numpy() for
    bfloat16."""
    if self.collect_timings and dev.torch().cuda.is_available():
      eng = dev.Engine.get()
      if eng.profile is None:
        eng.start_profile()
        try:
          return self._predict(embeddings, constraint_matrix)
        finally:
          self.last_timings = eng.stop_profile()
    return self._predict(embeddings, constraint_matrix)

  def _predict(self, embeddings, constraint_matrix=None) -> np.ndarray:
    num_embeddings = embeddings.shape[0]
    on_device = naive_clusterer._is_cuda_tensor(embeddings)
    if not on_device and not isinstance(embeddings, np.ndarray):
      raise TypeError("embeddings must be a numpy array")
    if len(embeddings.shape) != 2:
      raise ValueError("embeddings must be 2-dimensional")
    if on_device:
      serves = dev.torch().cuda.current_device()
      if embeddings.device.index != serves:
        raise ValueError("embeddings are on %s, but predict() runs on cuda:%d (the current device)"
                         % (embeddings.device, serves))
      given, embeddings = embeddings, dev.device_embeddings(embeddings)
    if num_embeddings < self.fallback_options.spectral_min_embeddings:
      # too few embeddings for a spectrum (spectral_clusterer.py:230-234): the fallback clusterer
      return fallback_clusterer.FallbackClusterer(self.fallback_options).predict(embeddings)
    if self.max_spectral_size is not None and num_embeddings > self.max_spectral_size:
      if constraint_matrix is not None:
        raise RuntimeError("Cannot handle constraint_matrix when max_spectral_size is set")
      if (self.max_spectral_size < 2 or
          (self.max_clusters and self.max_spectral_size <= self.max_clusters) or
          (self.min_clusters and self.max_spectral_size <= self.min_clusters)):
        raise ValueError("max_spectral_size should be a relatively big number")
      return self._reduce_size_and_predict(embeddings)
    eng = dev.Engine.get()
    t = dev.torch()
    sequence = list(self.refinement_options.refinement_sequence or [])
    builtin = self.affinity_function is utils.compute_affinity_matrix
    if builtin and on_device:
      x_dev = embeddings
    elif builtin:
      x = np.ascontiguousarray(embeddings)
      if x.dtype not in (np.float32, np.float64):
        x = x.astype(np.float64)
      x_dev = t.from_numpy(x).to(eng.device, non_blocking=True)
    if (self._factored_route(eng, num_embeddings, constraint_matrix) or
        self._factored_windows_route(eng, num_embeddings, constraint_matrix) or
        self._factored_single_cluster_route(eng, num_embeddings, constraint_matrix)):
      affinity = dev.FactoredAffinity(eng, x_dev)
    elif builtin:
      crop_first = bool(sequence) and sequence[0] == RefinementName.CropDiagonal
      a, crop = eng.affinity(x_dev, want_crop_vector=crop_first)
      affinity = DeviceAffinity(a, num_embeddings, crop, True)
    else:
      # the reference hands the user's function an ndarray: a CUDA tensor's host twin
      x_dev = dev.twin(embeddings) if on_device else None
      host = np.asarray(self.affinity_function(
          dev.host_twin(given) if on_device else embeddings))
      affinity = DeviceAffinity(eng.upload_matrix(host), num_embeddings, None,
                                bool(np.allclose(host, host.T, rtol=1e-6, atol=1e-9)))

    single_details = {}
    if self.min_clusters == 1:
      # single-vs-multi cluster decision (spectral_clusterer.py:253-256) on the resident affinity,
      # or on affinity panels and the packed upper band on the factored route
      if fallback_clusterer.check_single_cluster(self.fallback_options,
                                                 None if on_device else embeddings, affinity,
                                                 single_details, embeddings_dev=x_dev):
        if single_details:
          self.last_details = dict(single_cluster=single_details)
        return np.array([0] * num_embeddings)

    if (self.constraint_options and self.constraint_options.apply_before_refinement and
        constraint_matrix is not None):
      # constraint on the raw affinity (spectral_clusterer.py:258-264), on the device
      affinity = self._constrain(eng, affinity, constraint_matrix)

    if self.autotune:
      if RefinementName.RowWiseThreshold not in sequence:
        raise ValueError("AutoTune is only effective when the refinement sequence"
                         "contains RowWiseThreshold")
      proxy = self.autotune.proxy

      def p_percentile_to_ratio(p_percentile: float):
        self.refinement_options.p_percentile = p_percentile   # shared state, as the reference
        vectors, k, gap = self._compute_eigenvectors_ncluster(affinity, constraint_matrix)
        if proxy == AutoTuneProxy.PercentileSqrtOverNME:
          return np.sqrt(1 - p_percentile) / gap, vectors, k
        if proxy == AutoTuneProxy.PercentileOverNME:
          return (1 - p_percentile) / gap, vectors, k
        raise ValueError("Unsupported value of AutoTuneProxy")

      if self.autotune_group is not None:
        labels = self._predict_parallel_autotune(eng, affinity, p_percentile_to_ratio)
        if single_details:
          self.last_details["single_cluster"] = single_details
        return labels
      eigenvectors, n_clusters, best_p = self.autotune.tune(p_percentile_to_ratio)
      self.last_details["best_p_percentile"] = best_p
    else:
      eigenvectors, n_clusters, _ = self._compute_eigenvectors_ncluster(affinity, constraint_matrix)
    del affinity
    if single_details:
      self.last_details["single_cluster"] = single_details

    return self._cluster_embeddings(eng, eigenvectors, n_clusters)

  def _cluster_embeddings(self, eng, eigenvectors, n_clusters):
    """spectral_clusterer.py:295-313: clamp k, slice, optional row renorm, k-means."""
    if self.min_clusters is not None:
      n_clusters = max(n_clusters, self.min_clusters)
    self.last_details["n_clusters"] = n_clusters

    spectral = eigenvectors[:, :n_clusters].contiguous()
    if self.row_wise_renorm and n_clusters > 0:
      eng.row_renorm(spectral)
    if self.post_eigen_cluster_function is custom_distance_kmeans.run_kmeans:
      return custom_distance_kmeans.run_kmeans(
          spectral_embeddings=spectral, n_clusters=n_clusters, custom_dist=self.custom_dist,
          max_iter=self.max_iter)
    return self.post_eigen_cluster_function(
        spectral_embeddings=spectral.to("cpu").numpy(), n_clusters=n_clusters,
        custom_dist=self.custom_dist, max_iter=self.max_iter)

  def _predict_parallel_autotune(self, eng, affinity, p_percentile_to_ratio):
    """One p_percentile per rank: rank r evaluates grid[r::world] on its own copy of the base
    affinity; the (ratio, k) pairs are all-gathered, every rank picks the same winner, the rank
    that evaluated it runs k-means and broadcasts the labels."""
    import torch.distributed as dist
    from . import sharded
    t = dev.torch()
    if self.autotune.search_level != 1:
      raise NotImplementedError("parallel AutoTune supports search_level == 1")
    group = None if self.autotune_group is True else self.autotune_group
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    grid = self.autotune.get_percentile_range()
    kept = {}

    def evaluate(p):
      ratio, vectors, k = p_percentile_to_ratio(p)
      if not kept or ratio < kept["ratio"]:
        kept.update(ratio=ratio, vectors=vectors, k=k, p=p)
      return ratio, k

    best, best_p, ratio, k, owner = sharded.parallel_autotune(
        evaluate, grid, dist=dist, group=group, world=world, rank=rank)
    if len(grid) > 1 and self.autotune.search_step >= autotune_lib.MIN_SEARCH_STEP:
      self.autotune.narrow(grid, best)          # the reference stores the narrowed range (A.4-2)
    self.last_details["best_p_percentile"] = best_p
    n = affinity.n
    on_gpu = dist.get_backend(group) == "nccl"
    labels = t.empty((n,), dtype=t.int64, device=eng.device if on_gpu else "cpu")
    if rank == owner:
      assert kept["p"] == best_p
      labels.copy_(t.from_numpy(self._cluster_embeddings(eng, kept["vectors"], kept["k"])))
    dist.broadcast(labels, src=dist.get_global_rank(group, owner) if group is not None else owner,
                   group=group)
    return labels.cpu().numpy()

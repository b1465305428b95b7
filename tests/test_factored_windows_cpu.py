"""CPU: the windowed solve on the factored operator -- which predict() calls take that route (a
fake engine stands in for an 80 GB H100), and that a factored DeviceOps and the eigen stage call
the factored C entries with the locked set (a recording engine stands in for the library)."""

import ctypes

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import eigen_windows as ew

RN = scb.RefinementName
H100_80GB = 85_520_809_984          # torch.cuda.get_device_properties(0).total_memory
ICASSP = [RN.CropDiagonal, RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize, RN.Diffuse,
          RN.RowWiseNormalize]


class FakeEngine:
  """What the route predicates read from an Engine, for a device with `total` bytes."""

  dense_eig_max = 0
  upper_pass_ok = staticmethod(dev.Engine.upper_pass_ok)
  diffuse_precision_for = dev.Engine.diffuse_precision_for

  def __init__(self, total=H100_80GB):
    self.factored_above_bytes = total - dev.FACTORED_ROUTE_RESERVE
    self.diffuse_precision = None

  def gemm_engine(self, n):
    return nat.GEMM_SIMT if n < dev.Engine.simt_below else nat.GEMM_TCGEN05


def _seq(*names, sigma=1.0, **kw):
  return scb.RefinementOptions(gaussian_blur_sigma=sigma, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               thresholding_type=kw.pop("ttype", scb.ThresholdType.RowMax),
                               refinement_sequence=list(names), **kw)


def clusterer(**kw):
  args = dict(min_clusters=2, max_clusters=None,
              refinement_options=scb.configs.icassp2018_refinement_options,
              laplacian_type=scb.LaplacianType.GraphCut, custom_dist="cosine")
  args.update(kw)
  return scb.SpectralClusterer(**args)


@pytest.mark.parametrize("max_clusters", [None, 32, 64, 511])
@pytest.mark.parametrize("laplacian", [None, scb.LaplacianType.GraphCut])
def test_windowed_options_take_the_factored_windows_route(max_clusters, laplacian):
  eng = FakeEngine()
  c = clusterer(max_clusters=max_clusters, laplacian_type=laplacian)
  assert c._factored_windows_route(eng, 131072)
  assert not c._factored_route(eng, 131072) and not c._bounded_route(eng, 131072)
  c.max_clusters = 10                      # the one-solve route: the two are disjoint
  assert c._factored_route(eng, 131072) and not c._factored_windows_route(eng, 131072)


def test_windowed_route_follows_the_byte_formula():
  eng = FakeEngine()
  c = clusterer()
  assert not c._factored_windows_route(eng, 65536)
  assert not c._factored_route(eng, 65536)
  n = 90000
  eng.factored_above_bytes = dev.stored_route_peak_bytes(n)
  assert not c._factored_windows_route(eng, n)
  eng.factored_above_bytes -= 1
  assert c._factored_windows_route(eng, n)


def test_windowed_route_needs_more_than_the_dense_solvers_n():
  eng = FakeEngine()
  eng.factored_above_bytes = 0
  c = clusterer()
  assert c._factored_windows_route(eng, scb.spectral_clusterer.DENSE_MAX_N + 1)
  assert not c._factored_windows_route(eng, scb.spectral_clusterer.DENSE_MAX_N)


def _not_affinity(x):
  return x


@pytest.mark.parametrize("change", [
    dict(min_clusters=1), dict(affinity_function=_not_affinity), dict(constraint=True),
    dict(refinement_options=_seq(*ICASSP, sigma=2.0)),
    dict(refinement_options=_seq(*ICASSP, ttype=scb.ThresholdType.Percentile)),
    dict(diffuse_precision=nat.GEMM_SPLIT2), dict(autotune_group=True)])
def test_out_of_scope_calls_keep_the_stored_route(change):
  change = dict(change)
  eng = FakeEngine()
  eng.diffuse_precision = change.pop("diffuse_precision", None)
  constraint = change.pop("constraint", False)
  group = change.pop("autotune_group", None)
  c = clusterer(**change)
  c.autotune_group = group
  matrix = None
  if constraint:
    c.constraint_options = scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=False)
    matrix = [[0]]
  for max_clusters in (None, 64):
    c.max_clusters = max_clusters
    assert not c._factored_windows_route(eng, 131072, matrix)
    assert not c._factored_route(eng, 131072, matrix)


# ---- the C entries a factored DeviceOps and the eigen stage call


def _doubles(ptr, count):
  return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_double)), shape=(count,))


def _int64s(ptr, count):
  return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_int64)), shape=(count,))


class RecordingEngine(dev.Engine):
  """The real Engine wrappers over a library that records each call and answers with a spectrum
  that falls under stop_eigenvalue at its fourth value: 5, 4, 3, 0.5, 0.25, ..."""

  device = "cpu"
  stream = None

  def __init__(self):                          # no CUDA context
    self.calls = []
    self.profile = None

  @staticmethod
  def spectrum(first, count, which):
    i = np.arange(first, first + count)
    w = np.where(i < 3, 5.0 - i, 0.5 ** (i - 2.0))
    return w if which == nat.EIG_LARGEST else 5.0 - w

  def _call(self, name, *args, exc=None):
    self.calls.append((name, args))
    if name in ("sc_eigh_extremal_locked", "sc_eigh_extremal_locked_factored"):
      which, count, n_locked = args[7], args[8], args[13]
      _doubles(args[14], count)[:] = self.spectrum(n_locked, count, which)
      _int64s(args[15], 4)[:] = (16 * count, 0, count, 7)
    elif name in ("sc_eigh_extremal", "sc_eigh_extremal_factored"):
      count = args[8]
      _doubles(args[12], count)[:] = [9.0] * count
      _int64s(args[14], 4)[:] = (4, 0, 1, 300)


def _args(call, *names):
  order = ("operand", "n", "ld", "delta", "left", "right", "sign", "which", "n_values", "tol",
           "max_matvecs", "scale", "locked", "n_locked")
  return tuple(call[1][order.index(k)] for k in names)


@pytest.mark.parametrize("factored", [True, False])
def test_device_ops_call_the_entry_of_their_operator(factored):
  t = dev.torch()
  eng, n = RecordingEngine(), 1000
  operand = t.zeros((n, 1024), dtype=t.float16 if factored else t.float32)
  ops = ew.DeviceOps(eng, operand, n, None, None, None, -1.0, nat.EIG_SMALLEST, capacity=48,
                     factored=factored)
  w1 = ops.window(16)
  ops.window(16)
  top = ops.lambda_max()
  names = [c[0] for c in eng.calls]
  if factored:
    assert names == ["sc_eigh_extremal_locked_factored"] * 2 + ["sc_eigh_extremal_factored"]
  else:
    assert names == ["sc_eigh_extremal_locked"] * 2 + ["sc_eigh_extremal"]
  first, second, single = eng.calls
  for call, n_locked, scale in ((first, 0, 0.0), (second, 16, float(np.abs(w1).max()))):
    ptr, locked, count, sc, which, values = _args(call, "operand", "locked", "n_locked", "scale",
                                                  "which", "n_values")
    assert ptr.value == operand.data_ptr() and locked.value == ops.locked.data_ptr()
    assert (count, sc, which, values) == (n_locked, scale, nat.EIG_SMALLEST, 16)
  assert single[1][0].value == operand.data_ptr()
  assert single[1][7:10] == (nat.EIG_LARGEST, 1, 0)           # which, n_values, n_vectors
  assert top == 9.0 and ops.scale == 9.0
  assert ops.stats == dict(windows=2, passes=7 + 7 + 300, matvecs=512, restarts=0)


def test_device_ops_refuse_a_factored_operand_that_is_not_fp16():
  t = dev.torch()
  with pytest.raises(AssertionError):
    ew.DeviceOps(RecordingEngine(), t.zeros((64, 64)), 64, None, None, None, 1.0,
                 nat.EIG_LARGEST, capacity=16, factored=True)


class FakeFactoredAffinity(dev.FactoredAffinity):
  """A FactoredAffinity whose refinement is a zero Y_hi: the eigen stage reads only its shape."""

  def __init__(self, n):
    t = dev.torch()
    self.n, self.symmetric, self.crop_vector = n, True, None
    self.y_hi = t.zeros((n, dev.round_up(n, 64)), dtype=t.float16)
    self.refined = 0

  def refine(self, eng, options):
    self.refined += 1
    return dev.Refined(None, self.n, True, y_hi=self.y_hi)


@pytest.mark.parametrize("max_clusters,windows", [(None, 1), (40, 3)])
def test_eigen_stage_runs_windows_on_a_factored_refinement(max_clusters, windows):
  eng, n = RecordingEngine(), 1000
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=max_clusters)
  affinity = FakeFactoredAffinity(n)
  w, v, k, _ = c._eigen_on_device(eng, affinity)
  names = [call[0] for call in eng.calls]
  assert names == ["sc_eigh_extremal_locked_factored"] * windows + ["sc_eigh_mapback"]
  for call in eng.calls[:-1]:
    assert call[1][0].value == affinity.y_hi.data_ptr()
  assert c.last_details["solver"] == "lanczos-factored-windows"
  assert k == 3 and tuple(v.shape) == (n, 3) and affinity.refined == 1
  assert c.last_details["lanczos_stats"]["windows"] == windows
  want = RecordingEngine.spectrum(0, 16 * windows, nat.EIG_LARGEST)
  np.testing.assert_array_equal(w, want[:max_clusters + 1] if max_clusters else want)

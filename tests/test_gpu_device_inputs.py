"""GPU: SpectralClusterer.predict and FallbackClusterer.predict on CUDA tensors.

predict(X) must return what predict(H) returns for the host twin H = X.cpu().numpy() (for bfloat16,
X.float().cpu().numpy()), bit for bit: labels, their dtype and type, and last_details.  The kernels
behind it: sc_normalize_rows_typed against sc_normalize_rows on the upcast twin, and
sc_cluster_centroids against utils.get_cluster_centroids."""

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import utils
from conftest import golden_names, load_golden
from oracle import spectral_oracle as orc

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16, torch.float32, torch.float64]
SCC = scb.SingleClusterCondition
FCT = scb.FallbackClustererType


def host_twin(x):
  return (x.float() if x.dtype == torch.bfloat16 else x).cpu().numpy()


def upcast(x):
  """The tensor sc_normalize_rows reads for the twin of x (fp16 rows via fp64, bf16 via fp32)."""
  return dev.twin(x).contiguous()


def details_equal(a, b, path="last_details"):
  assert type(a) is type(b) or (np.isscalar(a) and np.isscalar(b)), path
  if isinstance(a, dict):
    assert a.keys() == b.keys(), path
    for key in a:
      details_equal(a[key], b[key], "%s[%r]" % (path, key))
  elif isinstance(a, (list, tuple)):
    assert len(a) == len(b), path
    for i, (u, v) in enumerate(zip(a, b)):
      details_equal(u, v, "%s[%d]" % (path, i))
  elif isinstance(a, np.ndarray):
    assert a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True), path
  else:
    assert a == b or (a != a and b != b), path


def assert_twin_equal(make, x, **kw):
  """make() -> a fresh clusterer (AutoTune and refinement options hold state)."""
  h = host_twin(x)
  got_c, want_c = make(), make()
  np.random.seed(0)
  got = got_c.predict(x, **kw)
  np.random.seed(0)
  want = want_c.predict(h, **kw)
  assert type(got) is np.ndarray and got.dtype == want.dtype and got.shape == want.shape
  assert np.array_equal(got, want)
  details_equal(got_c.last_details, want_c.last_details)
  return got, got_c


def dvectors(n, d=128, speakers=4, seed=0, dtype=torch.float32):
  x = orc.synthetic_dvectors(n, d, speakers, seed=seed).astype(np.float32)
  return torch.from_numpy(x).cuda().to(dtype)


def icassp(**kw):
  args = dict(min_clusters=2, max_clusters=7,
              refinement_options=scb.RefinementOptions(
                  gaussian_blur_sigma=1, p_percentile=0.95, thresholding_soft_multiplier=0.01,
                  thresholding_type=scb.ThresholdType.RowMax,
                  refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE)))
  args.update(kw)
  return lambda: scb.SpectralClusterer(**args)


def graphcut(**kw):
  return icassp(max_clusters=10, laplacian_type=scb.LaplacianType.GraphCut, **kw)


# ---------------------------------------------------------------- kernels
def typed_planes(engine, x, n, d, out_f32):
  t = torch
  if out_f32:
    xn = t.zeros((n, dev.round_up(d, 4)), dtype=t.float32, device=engine.device)
    engine.call("sc_normalize_rows_typed", dev._ptr(x), dev.dtype_code(x), n, d, x.stride(0),
                dev._ptr(xn), xn.stride(0), None, None, 0, engine.stream)
    return (xn[:, :d],)
  hi, lo = (t.zeros((n, dev.round_up(d, 64)), dtype=t.float16, device=engine.device)
            for _ in range(2))
  engine.call("sc_normalize_rows_typed", dev._ptr(x), dev.dtype_code(x), n, d, x.stride(0), None,
              0, dev._ptr(hi), dev._ptr(lo), hi.stride(0), engine.stream)
  return hi[:, :d], lo[:, :d]


def reference_planes(engine, x, n, d, out_f32):
  t = torch
  if out_f32:
    xn = t.zeros((n, dev.round_up(d, 4)), dtype=t.float32, device=engine.device)
    engine.call("sc_normalize_rows", dev._ptr(x), int(x.dtype == t.float64), n, d, x.stride(0),
                dev._ptr(xn), xn.stride(0), None, None, 0, engine.stream)
    return (xn[:, :d],)
  hi, lo = (t.zeros((n, dev.round_up(d, 64)), dtype=t.float16, device=engine.device)
            for _ in range(2))
  engine.call("sc_normalize_rows", dev._ptr(x), int(x.dtype == t.float64), n, d, x.stride(0), None,
              0, dev._ptr(hi), dev._ptr(lo), hi.stride(0), engine.stream)
  return hi[:, :d], lo[:, :d]


def bits(a):
  return a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32)


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("dtype", DTYPES)
def test_typed_normalisation_equals_the_upcast_twin(engine, dtype, strided):
  g = torch.Generator(device="cuda").manual_seed(3)
  for n in (1, 127, 1000, 4097):
    for d in (1, 3, 64, 256, 257):
      wide = torch.randn((n, d + 13 if strided else d), generator=g, device="cuda",
                         dtype=torch.float64).to(dtype)
      x = wide[:, 5:5 + d] if strided else wide
      assert x.stride(1) == 1 and (x.stride(0) == d + 13 if strided else x.is_contiguous())
      for out_f32 in (True, False):
        got = typed_planes(engine, x, n, d, out_f32)
        want = reference_planes(engine, upcast(x), n, d, out_f32)
        for a, b in zip(got, want):
          assert torch.equal(bits(a), bits(b)), (dtype, strided, n, d, out_f32)


@pytest.mark.parametrize("x_dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,k,d", [(1, 1, 5), (1000, 37, 3), (5000, 1024, 64), (65536, 1024, 257),
                                   (65536, 3, 130)])
def test_cluster_centroids_equal_the_host_function(engine, x_dtype, n, k, d):
  rng = np.random.default_rng(n + k + d)
  labels = rng.integers(0, k, n)
  labels[labels % 7 == 3] = 0                     # ids without a member: NaN rows
  labels[-1] = k - 1
  wide = torch.from_numpy(rng.standard_normal((n, d + 9)) * 10.0 ** rng.integers(-3, 4, (n, 1)))
  x = wide.to(x_dtype).cuda()[:, 4:4 + d]
  got = engine.cluster_centroids(x, labels).cpu().numpy()
  with np.errstate(invalid="ignore"):
    want = utils.get_cluster_centroids(x.cpu().numpy(), labels)
  assert got.shape == want.shape == (k, d) and got.dtype == want.dtype == np.float64
  nan = np.isnan(want)
  assert np.array_equal(np.isnan(got), nan)
  assert nan.any() == (k > 7 and n > 100)
  assert np.array_equal(got[~nan].view(np.int64), want[~nan].view(np.int64))


# ---------------------------------------------------------------- predict() branches
@pytest.mark.parametrize("name", golden_names())
def test_golden_fixtures(name):
  from test_gpu_predict import make_clusterer
  case = load_golden(name)
  x = torch.from_numpy(np.ascontiguousarray(case["embeddings"])).cuda()
  labels, _ = assert_twin_equal(lambda: make_clusterer(case["options"]), x)
  np.testing.assert_array_equal(utils.enforce_ordered_labels(labels),
                                utils.enforce_ordered_labels(case["labels"]))


@pytest.mark.parametrize("dtype", DTYPES)
def test_icassp_every_dtype(dtype):
  _, c = assert_twin_equal(icassp(), dvectors(1000, dtype=dtype))
  assert c.last_details["n_clusters"] == 4


def test_icassp_strided_rows():
  wide = dvectors(1000, 160)
  x = wide[:, 16:144]
  assert x.stride(0) == 160
  assert_twin_equal(icassp(), x)
  assert_twin_equal(icassp(), dvectors(1000, 128, dtype=torch.float16).t().contiguous().t())


def test_integer_tensor_is_widened_like_an_ndarray():
  x = (dvectors(600) * 100).round().to(torch.int32)
  assert_twin_equal(icassp(), x)


def test_graphcut_without_max_clusters():
  assert_twin_equal(icassp(max_clusters=None, laplacian_type=scb.LaplacianType.GraphCut),
                    dvectors(1536, 256, 6, seed=1))


def test_bounded_route():
  _, c = assert_twin_equal(graphcut(), dvectors(32768, 256, 6, seed=2))
  assert c.last_details["solver"] == "lanczos" and "diffuse" in c.last_details


def test_factored_route(engine):
  saved = engine.factored_above_bytes
  engine.factored_above_bytes = 0
  try:
    _, c = assert_twin_equal(graphcut(), dvectors(16384, 256, 6, seed=3))
  finally:
    engine.factored_above_bytes = saved
  assert c.last_details["solver"] == "lanczos-factored"


@pytest.mark.parametrize("speakers", [1, 3])
@pytest.mark.parametrize("cond,kind", [(SCC.AffinityGmmBic, FCT.Naive), (SCC.AllAffinity, FCT.Naive),
                                       (SCC.NeighborAffinity, FCT.Naive),
                                       (SCC.AffinityStd, FCT.Naive),
                                       (SCC.FallbackClusterer, FCT.Naive),
                                       (SCC.FallbackClusterer, FCT.Agglomerative)])
def test_single_cluster_checks(cond, kind, speakers):
  options = scb.FallbackOptions(single_cluster_condition=cond, fallback_clusterer_type=kind,
                                single_cluster_affinity_threshold=0.6, naive_threshold=0.6,
                                agglomerative_threshold=0.6)
  for dtype in (torch.float32, torch.float16):
    assert_twin_equal(icassp(min_clusters=1, fallback_options=options),
                      dvectors(600, 64, speakers, seed=4, dtype=dtype))


def test_max_spectral_size():
  labels, _ = assert_twin_equal(icassp(max_spectral_size=300), dvectors(1500, 64, 4, seed=5))
  assert labels.dtype == np.float64


@pytest.mark.parametrize("kind", [FCT.Naive, FCT.Agglomerative])
def test_below_spectral_min_embeddings(kind):
  options = scb.FallbackOptions(spectral_min_embeddings=100, fallback_clusterer_type=kind)
  for dtype in DTYPES:
    x = dvectors(40, 64, 3, seed=6, dtype=dtype)
    assert_twin_equal(icassp(fallback_options=options), x)
    got = scb.fallback_clusterer.FallbackClusterer(options).predict(x)
    want = scb.fallback_clusterer.FallbackClusterer(options).predict(host_twin(x))
    assert type(got) is np.ndarray and got.dtype == want.dtype and np.array_equal(got, want)


@pytest.mark.parametrize("before", [True, False])
def test_constraint_propagation(before):
  n = 800
  rng = np.random.default_rng(7)
  q = np.zeros((n, n))
  for i, j in rng.integers(0, n, (200, 2)):
    q[i, j] = q[j, i] = rng.choice([-1.0, 1.0])
  make = icassp(constraint_options=scb.ConstraintOptions(
      constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=before,
      constraint_propagation_alpha=0.6), laplacian_type=scb.LaplacianType.GraphCut)
  assert_twin_equal(make, dvectors(n, 64, 4, seed=7), constraint_matrix=q)


def test_autotune():
  make = icassp(autotune=scb.AutoTune(p_percentile_min=0.6, p_percentile_max=0.95,
                                      init_search_step=0.05, search_level=1),
                laplacian_type=scb.LaplacianType.GraphCut)
  _, c = assert_twin_equal(make, dvectors(1000, 128, 4, seed=8))
  assert "best_p_percentile" in c.last_details


def test_custom_dist_cityblock():
  assert_twin_equal(icassp(custom_dist="cityblock"), dvectors(1000, 128, 4, seed=9))


def test_row_wise_renorm():
  assert_twin_equal(icassp(row_wise_renorm=True), dvectors(1000, 128, 4, seed=10))


def test_user_affinity_function_gets_the_host_twin():
  x = dvectors(700, 64, 3, seed=11, dtype=torch.bfloat16)
  h = host_twin(x)
  seen = []

  def affinity(embeddings):
    assert isinstance(embeddings, np.ndarray) and np.array_equal(embeddings, h)
    assert embeddings.dtype == h.dtype
    seen.append(1)
    return utils.compute_affinity_matrix(embeddings)

  assert_twin_equal(icassp(affinity_function=affinity), x)
  assert len(seen) == 2


# ---------------------------------------------------------------- no host copy, errors
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_builtin_affinity_never_copies_the_embeddings_to_the_host(monkeypatch, dtype):
  x = dvectors(1000, dtype=dtype)
  want = icassp()().predict(host_twin(x))
  storage = x.untyped_storage().data_ptr()

  def guard(name):
    original = getattr(torch.Tensor, name)

    def wrapped(self, *a, **kw):
      to_host = name != "to" or "cpu" in str(a) + str(kw)
      if to_host and self.untyped_storage().data_ptr() == storage:
        raise AssertionError("the embeddings were copied to the host (Tensor.%s)" % name)
      return original(self, *a, **kw)
    monkeypatch.setattr(torch.Tensor, name, wrapped)

  for name in ("cpu", "numpy", "__array__", "to"):
    guard(name)
  got = icassp()().predict(x)
  monkeypatch.undo()
  assert np.array_equal(got, want)


def test_errors():
  c = icassp()()
  with pytest.raises(TypeError):
    c.predict(torch.zeros(10, 4))
  for shape in ((10,), (10, 4, 2)):
    with pytest.raises(ValueError, match="2-dimensional"):
      c.predict(torch.zeros(shape, device="cuda"))


def test_tensor_on_another_gpu():
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  x = dvectors(100).to("cuda:1")
  with pytest.raises(ValueError, match="cuda:1.*cuda:0"):
    icassp()().predict(x)


# ---------------------------------------------------------------- at scale
def test_factored_route_at_131072_with_no_more_memory(engine):
  n = 131072
  if engine.factored_above_bytes > 90e9:
    pytest.skip("sized for an 80 GB device")
  x = dvectors(n, 256, 6, seed=12)
  h = host_twin(x)
  peaks, outs = [], []
  for arg in (x, h):
    c = graphcut()()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    np.random.seed(0)
    outs.append((c.predict(arg), c.last_details))
    torch.cuda.synchronize()
    peaks.append(torch.cuda.max_memory_allocated())
  (got, got_d), (want, want_d) = outs
  assert got_d["solver"] == "lanczos-factored"
  assert np.array_equal(got, want)
  details_equal(got_d, want_d)
  assert peaks[0] <= peaks[1], peaks


def test_user_affinity_function_gets_the_tensor_dtype():
  for x in (dvectors(300, 32, 3, seed=13, dtype=torch.float16),
            (dvectors(300, 32, 3, seed=13) * 50).round().to(torch.int16)):
    h = x.cpu().numpy()

    def affinity(embeddings):
      assert embeddings.dtype == h.dtype and np.array_equal(embeddings, h)
      return utils.compute_affinity_matrix(embeddings)

    assert_twin_equal(icassp(affinity_function=affinity), x)

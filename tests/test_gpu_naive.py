"""GPU: the naive online clusterer in one device launch (`sc_naive_cluster`) against the host
NaiveClusterer: labels, counts and fp64 running means bit for bit on synthetic speaker-turn data
with one, a few and thousands of clusters (past the shared-memory capacity of the cluster of CTAs,
into the global-memory slots), fp32 and fp64 input; reference labels; continuation of state in
both directions; zero rows; stop mode; and predict(min_clusters=1) with the FallbackClusterer /
Naive single-cluster check."""

import os

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import fallback_clusterer as fb
from spectralcluster_b200 import naive_clusterer as nc
from spectralcluster_b200 import synthetic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callers")


def assert_same_state(dev_c, host_c):
  assert dev_c._counts == host_c._counts
  np.testing.assert_array_equal(dev_c._means.view(np.int64), host_c._means.view(np.int64))


def run_both(x, thr, adapt=None):
  host = nc.NaiveClusterer(thr, adapt)
  want = host.predict(x)
  device = nc.NaiveClusterer(thr, adapt)
  got = device.predict(torch.from_numpy(x).cuda())
  np.testing.assert_array_equal(got, want)
  assert got.dtype == want.dtype
  assert_same_state(device, host)
  return device, want


def test_reference_labels():
  z = np.load(os.path.join(GOLDEN, "naive.npz"))
  for (thr, adapt), want in zip(z["thresholds"], z["labels"]):
    c = nc.NaiveClusterer(thr, None if adapt < 0 else adapt)
    np.testing.assert_array_equal(c.fit_predict(torch.from_numpy(z["x"]).cuda()), want)


# (n, threshold, adaptation) -> clusters on speaker_turn_dvectors(n, 256, 8, seed=n): -0.5 gives
# one cluster, 0.5 a few (one per speaker), 0.85 at n = 2,048 gives 467, 0.87 gives 1,880 (one of
# them with 169 members) and 0.88 gives 2,048, every embedding its own cluster.  A 16-CTA cluster
# holds 111 centroids per CTA in shared memory at d = 256 (1,776 in all); the rest live in global
# memory.
CASES = [(2048, -0.5, None, 1), (2048, 0.5, None, 7), (2048, 0.5, 0.7, None), (2048, 0.85, None, 467),
         (2048, 0.87, None, 1880), (2048, 0.88, None, 2048), (16384, -0.5, None, 1),
         (16384, 0.5, None, 8), (16384, 0.5, 0.9, None), (65536, -0.5, None, 1),
         (65536, 0.5, None, 8)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,thr,adapt,clusters", CASES)
def test_synthetic_bitwise(n, thr, adapt, clusters, dtype):
  x = synthetic.speaker_turn_dvectors(n, 256, 8, seed=n).astype(dtype)
  device, _ = run_both(x, thr, adapt)
  if clusters is not None:
    assert len(device._counts) == clusters


@pytest.mark.parametrize("a", [1, 700])
def test_continuation(a):
  x = synthetic.speaker_turn_dvectors(2048, 256, 8, seed=3)
  host = nc.NaiveClusterer(0.5, 0.8)
  want = host.predict(x)
  # device on [0, a), host on [a, n)
  c = nc.NaiveClusterer(0.5, 0.8)
  head = c.predict(torch.from_numpy(x[:a]).cuda())
  tail = [c.predict_next(e) for e in x[a:]]
  np.testing.assert_array_equal(np.concatenate([head, tail]), want)
  assert_same_state(c, host)
  # host on [0, a), device continuing that state on [a, n)
  c = nc.NaiveClusterer(0.5, 0.8)
  head = c.predict(x[:a])
  tail = c.predict(torch.from_numpy(x[a:]).cuda())
  np.testing.assert_array_equal(np.concatenate([head, tail]), want)
  assert_same_state(c, host)
  assert [e.count for e in c.centroids] == host._counts


def test_merges_into_global_memory_slots():
  """2,000 host-opened clusters continued on the device: the embeddings are noisy copies of
  centroids 1,700..1,999, which sit past the shared-memory slots (centroid c is slot c // 16 of a
  16-CTA cluster, 111 slots at d = 256), so they merge in global memory; fresh directions open
  clusters beyond that."""
  rng = np.random.default_rng(12)
  base = rng.standard_normal((2000, 256))
  picks = rng.integers(1700, 2000, 600)
  tail = base[picks] + 0.3 * rng.standard_normal((600, 256))
  tail[::50] = rng.standard_normal((12, 256))
  host = nc.NaiveClusterer(0.5, 0.6)
  host.predict(base)
  assert len(host._counts) == 2000
  c = nc.NaiveClusterer(0.5, 0.6)
  c.predict(base)
  want = host.predict(tail)
  np.testing.assert_array_equal(c.predict(torch.from_numpy(tail).cuda()), want)
  assert_same_state(c, host)
  assert max(host._counts[1700:]) > 1 and len(host._counts) > 2000


@pytest.mark.parametrize("rows", [[0], [5, 900]])
def test_zero_rows(rows):
  """A zero row gives NaN cosines: np.argmax picks the first NaN, nothing opens or merges.  A zero
  first row opens a zero centroid whose cosine is NaN for every later embedding."""
  x = synthetic.speaker_turn_dvectors(1024, 64, 4, seed=7)
  x[rows] = 0.0
  with np.errstate(invalid="ignore", divide="ignore"):
    run_both(x, 0.5)


@pytest.mark.parametrize("n,thr", [(2048, -0.5), (2048, 0.5), (2048, 0.88), (16384, 0.5)])
def test_stop_mode(engine, n, thr):
  x = synthetic.speaker_turn_dvectors(n, 256, 8, seed=n)
  xd = torch.from_numpy(x).cuda()
  full, _, k, _, _ = engine.naive_cluster(xd, thr, thr)
  labels, processed, k2, means, counts = engine.naive_cluster(xd, thr, thr, stop_at=2)
  assert (k2 == 1) == (k == 1)
  assert processed == (n if k == 1 else int(np.flatnonzero(full.cpu().numpy() == 1)[0]) + 1)
  assert labels.shape[0] == processed and k2 == min(k, 2)
  np.testing.assert_array_equal(labels.cpu().numpy(), full[:processed].cpu().numpy())
  host = nc.NaiveClusterer(thr)
  host.predict(x[:processed])
  np.testing.assert_array_equal(means.cpu().numpy().view(np.int64), host._means.view(np.int64))
  assert counts.cpu().tolist() == host._counts


def naive_options(thr):
  return scb.FallbackOptions(single_cluster_condition=scb.SingleClusterCondition.FallbackClusterer,
                             fallback_clusterer_type=scb.FallbackClustererType.Naive,
                             naive_threshold=thr)


@pytest.mark.parametrize("speakers", [1, 4])
def test_predict_min_clusters_1(monkeypatch, speakers):
  """predict() with the device check against predict() with the host check (the host path reads
  only the embeddings: any ndarray affinity selects it)."""
  x = synthetic.speaker_turn_dvectors(16384, 256, speakers, seed=11)
  opts = naive_options(0.5)
  want_single = fb.check_single_cluster(opts, x, np.zeros((1, 1)))
  assert want_single == (speakers == 1)
  c = scb.SpectralClusterer(min_clusters=1, max_clusters=7,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            fallback_options=opts)
  got = c.predict(x)
  details = c.last_details["single_cluster"]
  assert (details["n_clusters"] == 1) == want_single
  if want_single:
    assert details["processed"] == 16384
  check = fb.check_single_cluster
  monkeypatch.setattr(fb, "check_single_cluster",
                      lambda o, e, a, d=None, embeddings_dev=None: check(o, e, np.zeros((1, 1))))
  np.testing.assert_array_equal(got, c.predict(x))

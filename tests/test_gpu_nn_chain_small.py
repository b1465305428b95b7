"""GPU: the one-block NN-chain (sc_nn_chain_small) against scipy `linkage(..., "complete" /
"average")` on Z bit for bit, and against the cooperative entries (sc_complete_linkage /
sc_average_linkage) on the same matrix: the same merges in the same chain order, the same
distances and sizes.  Random data, exact-tie matrices and duplicated points, at the warp edges,
at a stream's sizes and at the cutoff NN_SMALL_MAX."""

import numpy as np
import pytest
from scipy.cluster import hierarchy
from scipy.spatial import distance

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import agglomerative as agg
from spectralcluster_b200 import device as dev

pytestmark = pytest.mark.gpu

SIZES = [2, 3, 31, 32, 33, 100, 600, nat.NN_SMALL_MAX]
LINKAGE = {"complete": nat.LINKAGE_COMPLETE, "average": nat.LINKAGE_AVERAGE}
COOPERATIVE = {"complete": "sc_complete_linkage", "average": "sc_average_linkage"}


def upload(engine, dist):
  t = dev.torch()
  n = dist.shape[0]
  dm = engine.matrix(n, t.float64).fill_(float("nan"))
  dm[:, :n].copy_(t.from_numpy(np.ascontiguousarray(dist)))
  return dm


def assert_bitwise(a, b, msg=""):
  np.testing.assert_array_equal(np.asarray(a).view(np.int64), np.asarray(b).view(np.int64),
                                err_msg=msg)


def check(engine, dist, method, want_z):
  n = dist.shape[0]
  small = engine.nn_chain("sc_nn_chain_small", upload(engine, dist), n, LINKAGE[method])
  grid = engine.nn_chain(COOPERATIVE[method], upload(engine, dist), n, LINKAGE[method])
  np.testing.assert_array_equal(small[0], grid[0], err_msg="merges, n = %d" % n)
  assert_bitwise(small[1], grid[1], "distances, n = %d" % n)
  np.testing.assert_array_equal(small[2], grid[2], err_msg="sizes, n = %d" % n)
  assert_bitwise(agg.linkage_matrix(small[0], small[1], n), want_z, "Z, n = %d" % n)


@pytest.mark.parametrize("method", ["complete", "average"])
@pytest.mark.parametrize("n", SIZES)
def test_random_data(engine, n, method):
  x = np.random.default_rng(n).standard_normal((n, 24))
  y = distance.pdist(x, "cosine")
  check(engine, distance.squareform(y), method, hierarchy.linkage(y, method))


@pytest.mark.parametrize("method", ["complete", "average"])
@pytest.mark.parametrize("n", SIZES)
def test_exact_ties(engine, n, method):
  rng = np.random.default_rng(n + 1)
  d = np.triu(rng.integers(1, 2 + n % 4, size=(n, n)).astype(np.float64), 1)
  d = d + d.T
  check(engine, d, method, hierarchy.linkage(distance.squareform(d, checks=False), method))


@pytest.mark.parametrize("method", ["complete", "average"])
@pytest.mark.parametrize("n", SIZES)
def test_duplicated_points(engine, n, method):
  rng = np.random.default_rng(n + 2)
  base = rng.standard_normal((max(1, n // 8), 8))
  x = base[rng.integers(0, base.shape[0], size=n)]     # zero distances tie
  y = distance.pdist(x, "cosine")
  check(engine, distance.squareform(y), method, hierarchy.linkage(y, method))


def test_refuses_what_it_cannot_serve(engine):
  t = dev.torch()
  n = nat.NN_SMALL_MAX + 1
  dm = engine.matrix(n, t.float64)
  with pytest.raises(nat.NativeError, match="above SC_NN_SMALL_MAX"):
    engine.nn_chain("sc_nn_chain_small", dm, n, nat.LINKAGE_COMPLETE)
  with pytest.raises(nat.NativeError, match="bad arguments"):
    engine.nn_chain("sc_nn_chain_small", dm, 1, nat.LINKAGE_COMPLETE)
  # no chain top of an all-NaN matrix has a nearest neighbour: an error, not a merge
  dm = engine.matrix(5, t.float64).fill_(float("nan"))
  with pytest.raises(nat.NativeError, match="no nearest neighbour"):
    engine.nn_chain("sc_nn_chain_small", dm, 5, nat.LINKAGE_AVERAGE)

"""CPU: the Python wiring of the device naive clusterer with a fake engine: the FallbackClusterer /
Naive single-cluster check on a device affinity asks the engine for a run that stops at the second
cluster and records what it processed; a host ndarray affinity never touches the device; and
NaiveClusterer.predict on a device tensor hands the engine its state and takes the engine's state
back, so that predict_next continues where a host run would."""

import numpy as np
import pytest
import torch

from spectralcluster_b200 import device as dev
from spectralcluster_b200 import fallback_clusterer as fb
from spectralcluster_b200 import naive_clusterer as nc


class _FakeEngine:
  """Engine.naive_cluster restated with the host NaiveClusterer on CPU tensors."""
  device = torch.device("cpu")

  def __init__(self):
    self.calls = []

  def naive_cluster(self, x_dev, threshold, adaptation_threshold, stop_at=0, means=None,
                    counts=None):
    self.calls.append(dict(n=int(x_dev.shape[0]), threshold=threshold,
                           adaptation=adaptation_threshold, stop_at=stop_at,
                           means=None if means is None else means.numpy().copy(),
                           counts=None if counts is None else counts.tolist()))
    c = nc.NaiveClusterer(threshold, adaptation_threshold)
    if means is not None:
      c._means, c._counts = means.numpy().copy(), counts.tolist()
    labels = []
    for e in x_dev.numpy():
      if stop_at > 0 and len(c._counts) >= stop_at:
        break
      labels.append(c.predict_next(e))
    k = len(c._counts)
    m = torch.from_numpy(c._means) if k else torch.empty((0, x_dev.shape[1]), dtype=torch.float64)
    return (torch.tensor(labels, dtype=torch.int64), len(labels), k, m,
            torch.tensor(c._counts, dtype=torch.int64))


class _NoDevice(Exception):
  pass


def _no_device(cls, device=None):
  raise _NoDevice()


class _FakeDeviceAffinity:
  n = 300


def _options(thr, adapt=None):
  return fb.FallbackOptions(single_cluster_condition=fb.SingleClusterCondition.FallbackClusterer,
                            fallback_clusterer_type=fb.FallbackClustererType.Naive,
                            naive_threshold=thr, naive_adaptation_threshold=adapt)


def _blobs(n, k, seed):
  rng = np.random.default_rng(seed)
  centres = np.eye(6)[:k]
  return centres[np.arange(n) * k // n] + 0.1 * rng.standard_normal((n, 6))


@pytest.mark.parametrize("k", [1, 3])
def test_device_affinity_runs_the_engine_until_a_second_cluster(monkeypatch, k):
  x = _blobs(300, k, 2)
  eng = _FakeEngine()
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: eng))
  details = {}
  got = fb.check_single_cluster(_options(0.5, 0.7), x, _FakeDeviceAffinity(), details)
  assert got == (k == 1)
  assert len(eng.calls) == 1
  call = eng.calls[0]
  assert (call["n"], call["threshold"], call["adaptation"], call["stop_at"]) == (300, 0.5, 0.7, 2)
  assert call["means"] is None
  second = 300 // k + 1 if k > 1 else 300                # the first row of the second blob opens it
  assert details == dict(processed=second, n_clusters=min(k, 2))
  # an ndarray affinity takes the host clusterer and never asks for an engine
  monkeypatch.setattr(dev.Engine, "get", classmethod(_no_device))
  assert fb.check_single_cluster(_options(0.5, 0.7), x, np.eye(300)) == got
  with pytest.raises(_NoDevice):
    fb.check_single_cluster(_options(0.5, 0.7), x, _FakeDeviceAffinity())


def test_device_affinity_uses_the_uploaded_embeddings(monkeypatch):
  x = _blobs(40, 2, 3)
  eng = _FakeEngine()
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: eng))
  xd = torch.from_numpy(x[::-1].copy())
  fb.check_single_cluster(_options(0.5), None, _FakeDeviceAffinity(), embeddings_dev=xd)
  assert eng.calls[0]["n"] == 40 and eng.calls[0]["adaptation"] == 0.5
  with pytest.raises(ValueError):                       # the host clusterer's parameter check
    fb.check_single_cluster(_options(0.8, 0.5), x, _FakeDeviceAffinity())


def test_state_is_handed_over_both_ways(monkeypatch):
  x = _blobs(200, 3, 4)
  host = nc.NaiveClusterer(0.5, 0.8)
  want = host.predict(x)
  eng = _FakeEngine()
  monkeypatch.setattr(dev.Engine, "get", classmethod(lambda cls, device=None: eng))
  monkeypatch.setattr(nc, "_is_cuda_tensor", lambda e: isinstance(e, torch.Tensor))
  c = nc.NaiveClusterer(0.5, 0.8)
  head = c.predict(torch.from_numpy(x[:90]))            # "device" on [0, 90)
  assert eng.calls[-1]["means"] is None
  tail = [c.predict_next(e) for e in x[90:150]]         # host on [90, 150)
  state = (c._means.copy(), list(c._counts))
  rest = c.fit_predict(torch.from_numpy(x[150:]))       # "device" again, from the host state
  np.testing.assert_array_equal(eng.calls[-1]["means"], state[0])
  assert eng.calls[-1]["counts"] == state[1] and eng.calls[-1]["stop_at"] == 0
  np.testing.assert_array_equal(np.concatenate([head, tail, rest]), want)
  np.testing.assert_array_equal(c._means, host._means)
  assert c._counts == host._counts and isinstance(c._counts[0], int)
  # an ndarray stays on the host
  monkeypatch.setattr(dev.Engine, "get", classmethod(_no_device))
  c.reset()
  np.testing.assert_array_equal(c.predict(x), want)

"""CPU: what a CUDA-tensor input to predict() leaves unchanged for every other input, the dtype
rules that define a CUDA tensor's host twin, and the summation order sc_cluster_centroids restates.
No device calls."""

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import utils


def test_non_ndarray_inputs_fail_as_before():
  c = scb.SpectralClusterer()
  with pytest.raises(AttributeError):
    c.predict([[1.0, 2.0]])                 # .shape is read before the type check
  with pytest.raises(ValueError, match="2-dimensional"):
    c.predict(np.zeros(3))
  for x in (torch.zeros(10, 4), torch.zeros(10), torch.zeros(10, 4, dtype=torch.float16)):
    with pytest.raises(TypeError, match="numpy array"):
      c.predict(x)                           # CPU tensors stay refused


@pytest.mark.parametrize("dtype,want", [(torch.float16, torch.float64),
                                        (torch.bfloat16, torch.float32),
                                        (torch.float32, torch.float32),
                                        (torch.float64, torch.float64)])
def test_twin_dtype(dtype, want):
  x = torch.randn(5, 3).to(dtype)
  y = dev.twin(x)
  assert y.dtype == want
  assert np.array_equal(y.numpy(), (x.float() if dtype == torch.bfloat16 else x).numpy()
                        .astype(np.float64 if dtype == torch.float16 else None))
  if dtype in (torch.float32, torch.float64):
    assert y is x


def test_device_embeddings_layout_rules():
  w = torch.randn(6, 10, requires_grad=True)
  x = dev.device_embeddings(w[:, 2:7])
  assert not x.requires_grad and x.stride() == (10, 1)          # row stride kept, no copy
  assert x.untyped_storage().data_ptr() == w.untyped_storage().data_ptr()
  x = dev.device_embeddings(torch.randn(5, 6).t())
  assert x.is_contiguous()
  assert dev.device_embeddings(torch.arange(12).reshape(3, 4)).dtype == torch.float64
  assert dev.device_embeddings(torch.ones(3, 4, dtype=torch.bool)).dtype == torch.float64
  x = torch.randn(4, 1).expand(4, 3)                            # overlapping rows
  assert dev.device_embeddings(x).is_contiguous()
  for dtype in (torch.float16, torch.bfloat16):
    assert dev.device_embeddings(torch.randn(3, 4).to(dtype)).dtype == dtype


def centroids_in_kernel_order(x, labels):
  """sc_cluster_centroids restated: a stable sort of the rows by id, then per (id, column) a
  sequential fp64 sum from 0.0 in increasing row index, over the member count."""
  labels = np.asarray(labels, dtype=np.int64)
  k = int(labels.max()) + 1
  order = np.argsort(labels, kind="stable")
  off = np.concatenate([[0], np.cumsum(np.bincount(labels, minlength=k))])
  out = np.empty((k, x.shape[1]), dtype=np.float64)
  with np.errstate(invalid="ignore"):
    for c in range(k):
      rows = order[off[c]:off[c + 1]]
      assert np.all(np.diff(rows) > 0)
      s = np.zeros(x.shape[1], dtype=np.float64)
      for r in rows:
        s = s + x[r].astype(np.float64)
      out[c] = s / np.float64(len(rows))
  return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,k,d", [(1, 1, 3), (50, 9, 7), (700, 40, 33)])
def test_centroid_summation_order_matches_get_cluster_centroids(dtype, n, k, d):
  rng = np.random.default_rng(n * k + d)
  labels = rng.integers(0, k, n)
  labels[labels % 4 == 1] = 0            # ragged sizes and ids without a member
  labels[-1] = k - 1
  x = (rng.standard_normal((n, d)) * 10.0 ** rng.integers(-4, 5, (n, 1))).astype(dtype)
  got = centroids_in_kernel_order(x, labels)
  with np.errstate(invalid="ignore"):
    want = utils.get_cluster_centroids(x, labels)
  nan = np.isnan(want)
  assert np.array_equal(np.isnan(got), nan)
  assert nan.any() == (k > 1 and n > 1)
  assert np.array_equal(got[~nan].view(np.int64), want[~nan].view(np.int64))

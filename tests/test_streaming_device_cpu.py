"""CPU: the NN-chain kernel choice (by n alone, one thread block up to NN_SMALL_MAX), and the host
logic of MultiStageClusterer.streaming_predict on CUDA tensors: the type checks that refuse a
mixed stream before any state changes, and the cache's dtype, which follows np.vstack on the host
twins.  No device calls: a CPU tensor that reports a CUDA device stands in for a CUDA tensor."""

import os
import re

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "spectralcluster_b200.h")


# ---- the kernel choice

def test_header_and_binding_agree_on_the_cutoff_and_the_linkage_codes():
  text = open(HEADER).read()
  assert int(re.search(r"SC_NN_SMALL_MAX\s*=\s*(\d+)", text).group(1)) == nat.NN_SMALL_MAX
  assert int(re.search(r"SC_LINKAGE_COMPLETE\s*=\s*(\d+)", text).group(1)) == nat.LINKAGE_COMPLETE
  assert int(re.search(r"SC_LINKAGE_AVERAGE\s*=\s*(\d+)", text).group(1)) == nat.LINKAGE_AVERAGE


class _Matrix:
  """What Engine.nn_chain reads of a device matrix: its address and its row stride."""

  def __init__(self, n):
    self.ld = dev.round_up(n, 64)

  def data_ptr(self):
    return 4096

  def stride(self, dim):
    return self.ld if dim == 0 else 1


def routed(monkeypatch, method, n):
  calls = []
  eng = object.__new__(dev.Engine)
  monkeypatch.setattr(dev.Engine, "stream", property(lambda self: None))
  monkeypatch.setattr(dev.Engine, "call", lambda self, name, *args, **kw: calls.append((name, args)))
  xy, md, ms_ = getattr(eng, method)(_Matrix(n), n)
  assert xy.shape == (n - 1, 2) and md.shape == ms_.shape == (n - 1,)
  (name, args), = calls
  return name, args


@pytest.mark.parametrize("method,linkage,cooperative", [
    ("complete_linkage", nat.LINKAGE_COMPLETE, "sc_complete_linkage"),
    ("average_linkage", nat.LINKAGE_AVERAGE, "sc_average_linkage")])
def test_route_chooses_by_n_alone(monkeypatch, method, linkage, cooperative):
  cut = nat.NN_SMALL_MAX
  for n in (2, 3, 100, 600, cut - 1, cut):
    name, args = routed(monkeypatch, method, n)
    assert name == "sc_nn_chain_small" == dev.nn_chain_entry(linkage, n), n
    assert args[1:4] == (n, dev.round_up(n, 64), linkage)
  for n in (cut + 1, 65536):
    name, args = routed(monkeypatch, method, n)
    assert name == cooperative == dev.nn_chain_entry(linkage, n), n
    assert args[1:3] == (n, dev.round_up(n, 64)) and len(args) == 7
  # nothing else decides: not the environment, not free device memory
  monkeypatch.setenv("SCB_NVTX", "1")
  monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (0, 0))
  assert routed(monkeypatch, method, cut)[0] == "sc_nn_chain_small"
  assert routed(monkeypatch, method, cut + 1)[0] == cooperative


# ---- streaming_predict on CUDA tensors

class FakeCuda(torch.Tensor):
  """A CPU tensor that reports itself as a CUDA tensor on cuda:<index>."""

  @property
  def is_cuda(self):
    return True

  @property
  def device(self):
    return torch.device("cuda", getattr(self, "index", 0))


def fake(x, index=0):
  t = torch.as_tensor(x).as_subclass(FakeCuda)
  t.index = index
  return t


def twin(x):
  return (x.float() if x.dtype == torch.bfloat16 else x).as_subclass(torch.Tensor).numpy()


def stream(seen=None, U1=100):
  """A MultiStageClusterer whose main clusterer records what it is given and returns zeros."""
  main = scb.SpectralClusterer()

  def predict(x):
    if seen is not None:
      seen.append(x)
    return np.zeros(x.shape[0], dtype=np.int64)
  main.predict = predict
  return ms.MultiStageClusterer(main, U1=U1)


def state(s):
  return (s.num_embeddings, s.cache, s.previous_output, s.compression_labels, s.stream_device)


def assert_state_is(s, before):
  after = state(s)
  assert after[0] == before[0] and after[4] == before[4]
  for a, b in zip(after[1:4], before[1:4]):
    assert a is b


@pytest.fixture
def current_device_0(monkeypatch):
  monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def test_mixed_streams_raise_type_error_and_change_nothing(current_device_0):
  rng = np.random.default_rng(0)
  host = stream()
  host.streaming_predict(rng.standard_normal(8))
  host.streaming_predict(rng.standard_normal(8))
  before = state(host)
  for e in (fake(rng.standard_normal(8)), fake(rng.standard_normal((1, 8)), 1)):
    with pytest.raises(TypeError, match="host arrays"):
      host.streaming_predict(e)
    assert_state_is(host, before)

  on_device = stream()
  on_device.streaming_predict(fake(rng.standard_normal(8)))
  on_device.streaming_predict(fake(rng.standard_normal(8)))
  before = state(on_device)
  assert before[4] == torch.device("cuda", 0)
  for e in (rng.standard_normal(8), torch.zeros(8), fake(rng.standard_normal(8), 1)):
    with pytest.raises(TypeError, match="CUDA tensors on cuda:0"):
      on_device.streaming_predict(e)
    assert_state_is(on_device, before)


def test_a_tensor_off_the_current_device_is_refused_before_the_first_step(current_device_0):
  s = stream()
  with pytest.raises(ValueError, match="current device"):
    s.streaming_predict(fake(np.ones(4), 1))
  assert s.num_embeddings == 0 and s.cache is None and s.stream_device is None


@pytest.mark.parametrize("dtypes", [
    [torch.float16] * 5,
    [torch.float32] * 5,
    [torch.float64] * 5,
    [torch.float16, torch.float16, torch.float32, torch.float16, torch.float64, torch.float16],
    [torch.float32, torch.float16, torch.float64, torch.float32],
    [torch.bfloat16, torch.bfloat16, torch.float16, torch.bfloat16],
    [torch.float64, torch.bfloat16, torch.float16]])
def test_cache_dtype_follows_vstack_of_the_twins(current_device_0, dtypes):
  rng = np.random.default_rng(len(dtypes))
  seen_dev, seen_host = [], []
  on_device, host = stream(seen_dev), stream(seen_host)
  for i, dtype in enumerate(dtypes):
    row = rng.standard_normal(6) if i % 2 == 0 else rng.standard_normal((1, 6))
    e = fake(torch.from_numpy(row).to(dtype))
    on_device.streaming_predict(e)
    host.streaming_predict(twin(e))
    got, want = twin(on_device.cache), host.cache
    assert got.dtype == want.dtype and got.shape == want.shape, i
    np.testing.assert_array_equal(got, want)
    assert isinstance(on_device.cache, FakeCuda) and on_device.cache.is_cuda
  assert len(seen_dev) == len(seen_host) == len(dtypes) - 1
  for a, b in zip(seen_dev, seen_host):
    assert twin(a).dtype == b.dtype


@pytest.mark.parametrize("cache_dtype", [torch.float16, torch.float32, torch.float64])
@pytest.mark.parametrize("row_dtype", [torch.float16, torch.bfloat16, torch.float32, torch.float64])
def test_append_rows_after_a_compression(cache_dtype, row_dtype):
  """After a compression the cache is the fp64 centroids; before, any twin dtype."""
  cache = torch.randn(5, 3, dtype=torch.float64).to(cache_dtype)
  row = torch.randn(3).to(row_dtype)
  got = ms.append_rows(cache, row)
  want = np.vstack([twin(cache), twin(row)])
  assert twin(got).dtype == want.dtype
  np.testing.assert_array_equal(twin(got), want)


def test_host_streams_never_touch_torch_cuda(monkeypatch):
  def refuse():
    raise AssertionError("a host stream asked for the current device")
  monkeypatch.setattr(torch.cuda, "current_device", refuse)
  s = stream()
  for e in np.random.default_rng(3).standard_normal((4, 5)).astype(np.float16):
    s.streaming_predict(e)
  assert s.cache.dtype == np.float16 and s.cache.shape == (4, 5) and s.stream_device is None

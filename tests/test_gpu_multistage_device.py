"""GPU: MultiStageClusterer.streaming_predict on a stream of CUDA tensors.  The reference's labels
(tests/golden/callers/multistage.npz) for every deflicker mode from fp32 and fp64 rows, and a
1,500-step stream (L = 50, U1 = 100, U2 = 600: two compressions) whose every step returns what the
same stream of host twins returns: labels, previous_output, compression_labels, main.last_details
and the cache itself, for fp16, bf16, fp32 and fp64 rows, with min_clusters = 2 and with
min_clusters = 1 (the average-linkage single-cluster check on every step)."""

import os

import numpy as np
import pytest
import torch

import spectralcluster_b200 as scb
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import multi_stage_clusterer as ms
from spectralcluster_b200 import synthetic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callers")
ordered = scb.utils.enforce_ordered_labels


def refinement():
  return scb.RefinementOptions(gaussian_blur_sigma=0, p_percentile=0.9,
                               refinement_sequence=list(scb.ICASSP2018_REFINEMENT_SEQUENCE))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("mode", ["NoDeflicker", "OrderBased", "Hungarian"])
def test_golden_stream_of_cuda_tensors(mode, dtype):
  z = np.load(os.path.join(GOLDEN, "multistage.npz"))
  xd = torch.from_numpy(z["x"].astype(dtype)).cuda()
  main = scb.SpectralClusterer(min_clusters=1, max_clusters=5, refinement_options=refinement())
  clusterer = ms.MultiStageClusterer(main, fallback_threshold=0.5, L=8, U1=30, U2=60,
                                     deflicker=getattr(ms.Deflicker, mode))
  for i in range(xd.shape[0]):
    labels = clusterer.streaming_predict(xd[i])
    assert isinstance(labels, np.ndarray)
    if i + 1 in z["checkpoints"]:
      want = z["%s_%d" % (mode, i + 1)]
      if mode == "NoDeflicker":       # raw k-means ids: compare as partitions
        np.testing.assert_array_equal(ordered(labels), ordered(want), err_msg=str(i + 1))
      else:
        np.testing.assert_array_equal(labels, want, err_msg=str(i + 1))
  assert clusterer.cache.is_cuda and clusterer.cache.dtype == torch.float64   # compressed


def assert_same(got, want, what):
  """Equal values of equal types, arrays bit for bit (NaN included), dicts key by key."""
  if isinstance(want, dict):
    assert isinstance(got, dict) and sorted(got) == sorted(want), what
    for k in want:
      assert_same(got[k], want[k], "%s[%r]" % (what, k))
  elif isinstance(want, np.ndarray):
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype and got.shape == want.shape, what
    assert got.tobytes() == want.tobytes(), what
  elif isinstance(want, float):
    assert type(got) is type(want) and np.float64(got).tobytes() == np.float64(want).tobytes(), what
  else:
    assert type(got) is type(want) and got == want, what


STREAMS = [("float16", 2, "Hungarian"), ("bfloat16", 2, "OrderBased"),
           ("float32", 2, "NoDeflicker"), ("float64", 2, "Hungarian"),
           ("float16", 1, "OrderBased"), ("bfloat16", 1, "Hungarian"),
           ("float32", 1, "Hungarian"), ("float64", 1, "NoDeflicker")]


@pytest.mark.parametrize("dtype,min_clusters,mode", STREAMS)
def test_stream_equals_the_host_twin_stream(dtype, min_clusters, mode):
  steps = 1500
  x = synthetic.speaker_turn_dvectors(steps, 128, 4, seed=min_clusters)
  xd = torch.from_numpy(x).cuda().to(getattr(torch, dtype))

  def stream():
    main = scb.SpectralClusterer(min_clusters=min_clusters, max_clusters=7,
                                 refinement_options=refinement())
    return ms.MultiStageClusterer(main, fallback_threshold=0.5, L=50, U1=100, U2=600,
                                  deflicker=getattr(ms.Deflicker, mode))

  on_device, host = stream(), stream()
  compressions = 0
  for i in range(steps):
    e = xd[i] if i % 3 else xd[i:i + 1]              # (d,) and (1, d) rows
    got = on_device.streaming_predict(e)
    want = host.streaming_predict(dev.host_twin(e))
    what = "step %d" % (i + 1)
    assert_same(got, want, what)
    assert_same(on_device.previous_output, host.previous_output, what)
    assert_same(on_device.compression_labels, host.compression_labels, what)
    assert_same(on_device.main.last_details, host.main.last_details, what)
    assert on_device.cache.is_cuda
    assert_same(dev.host_twin(on_device.cache), host.cache, what + " cache")
    compressions += i + 1 > 100 and host.cache.shape[0] == 100
  assert compressions >= 2
  assert len(np.unique(got)) > 1

"""Engine.blur_upper_rowmax / threshold_symmetrize_upper route by what pass 1 returned: a
DeferredBlur record runs the recomputing pass 2, a stored B the element-wise one.  No GPU: the
C-ABI calls are recorded, not made."""

import torch

from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev


class RecordingEngine(dev.Engine):
  stream = None

  def __init__(self):            # no device, no context
    self.calls = []
    self.device = "cpu"
    self.profile = None

  def call(self, name, *args, exc=None):
    self.calls.append((name, args))

  def matrix(self, n, dtype=None):
    return torch.zeros((n, dev.round_up(n, 64)), dtype=dtype or torch.float32)

  def planes(self, n, cols=None):
    return (torch.zeros((n, dev.round_up(n, 64)), dtype=torch.float16),
            torch.zeros((n, dev.round_up(n, 64)), dtype=torch.float16))

  def vector(self, n, dtype=None, zero=False):
    return torch.zeros(n, dtype=dtype or torch.float32)


def thrsym(eng, b, n, m):
  return eng.threshold_symmetrize_upper(b, n, m, 0.95, 0.01, False, True, nat.SYMMETRIZE_MAX,
                                        False, True, True)


def test_record_runs_the_recomputing_pass():
  eng, n = RecordingEngine(), 100
  a, crop = eng.matrix(n), torch.zeros(n)
  rec, m = eng.blur_upper_rowmax(a, n, 1.0, crop, True)
  assert isinstance(rec, dev.DeferredBlur)
  assert rec.a is a and rec.diag is crop and rec.sigma == 1.0
  name, args = eng.calls[-1]
  assert name == "sc_blur_upper_rowmax"
  assert args[6].value is None and args[7] == 0          # no B: pass 1 keeps the row maxima only
  _, hi, lo = thrsym(eng, rec, n, m)
  name, args = eng.calls[-1]
  assert name == "sc_blur_threshold_symmetrize_upper"
  assert args[0].value == a.data_ptr() and args[2] == a.stride(0)
  assert args[3].value == crop.data_ptr() and args[4] == 1.0
  assert args[5].value == m.data_ptr()
  assert args[11].value is None and args[13].value == hi.data_ptr() and args[14].value == lo.data_ptr()


def test_stored_b_runs_the_elementwise_pass():
  eng, n = RecordingEngine(), 100
  a = eng.matrix(n)
  b, m = eng.blur_upper_rowmax(a, n, 1.0, None, False, store_b=True)
  assert isinstance(b, torch.Tensor)
  name, args = eng.calls[-1]
  assert name == "sc_blur_upper_rowmax" and args[6].value == b.data_ptr()
  thrsym(eng, b, n, m)
  name, args = eng.calls[-1]
  assert name == "sc_threshold_symmetrize_upper"
  assert args[0].value == b.data_ptr() and args[2] == b.stride(0)
  assert args[3].value == m.data_ptr()


def test_recomputing_pass_has_an_nvtx_name():
  assert "sc_blur_threshold_symmetrize_upper" in nat.PROTOTYPES
  assert "sc_blur_threshold_symmetrize_upper" in dev.Engine.REFERENCE_NAMES

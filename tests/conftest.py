import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


_BUILD_ERROR = None


def pytest_configure(config):
  global _BUILD_ERROR
  config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")
  # The C-ABI library is a build artefact (git-ignored): make sure it exists and is current
  # before any test imports it (incremental: a no-op when the sources are unchanged).  A box
  # without nvcc can still run the host-logic / oracle tests: the failure is remembered and only
  # the tests that need the library are skipped.
  try:
    from spectralcluster_b200 import build
    build.build()
  except Exception as e:                                   # no nvcc, or a compile error
    _BUILD_ERROR = "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")
    if os.environ.get("SCB_REQUIRE_BUILD") == "1":
      raise


def _cuda_available():
  try:
    import torch
    return torch.cuda.is_available()
  except Exception:
    return False


def pytest_collection_modifyitems(config, items):
  """`pytest tests` on a machine without CUDA skips the GPU tests instead of failing them."""
  have_gpu = _cuda_available()
  skip_gpu = pytest.mark.skip(reason="needs a CUDA device (H100); there is no CPU fallback")
  skip_lib = pytest.mark.skip(reason="C-ABI library could not be built: %s" % _BUILD_ERROR)
  for item in items:
    needs_gpu = item.get_closest_marker("gpu") is not None or "engine" in getattr(item, "fixturenames", ())
    if needs_gpu and not have_gpu:
      item.add_marker(skip_gpu)
    elif _BUILD_ERROR is not None and (needs_gpu or item.module.__name__.endswith("test_abi")):
      item.add_marker(skip_lib)


def golden_names():
  return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def load_golden(name):
  """Fixture written by tests/golden/make_golden.py from the unmodified reference."""
  from oracle import spectral_oracle as orc
  z = np.load(os.path.join(GOLDEN, name + ".npz"))
  case = {k: z[k] for k in z.files}
  case["options"] = eval(str(z["options"]), {"__builtins__": {}}, {})
  if "embeddings" not in case:
    n, d, speakers, seed = (int(v) for v in z["synthetic_args"])
    x = orc.synthetic_dvectors(n, d, speakers, seed=seed)
    import hashlib
    digest = hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()
    assert digest == str(z["embeddings_sha256"]), "synthetic generator drifted from the fixture"
    case["embeddings"] = x
  return case


@pytest.fixture(scope="session")
def engine():
  from spectralcluster_b200 import device
  return device.Engine.get()

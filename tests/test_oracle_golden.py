"""CPU: the oracle reproduces every fixture the unmodified reference produced
(tests/golden/make_golden.py) -- labels bit for bit, leading eigenvalues to the last few bits
(LAPACK's rounding depends on the kernels OpenBLAS picks for the host CPU)."""

import numpy as np
import pytest

from conftest import golden_names, load_golden
from oracle import spectral_oracle as orc


@pytest.mark.parametrize("name", golden_names())
def test_oracle_matches_reference_fixture(name):
  case = load_golden(name)
  opt = case["options"]
  x = case["embeddings"]
  if opt["autotune"]:
    _, _, k, p_best, trace = orc.autotune(orc.affinity(x), opt)
    np.testing.assert_array_equal(np.array(trace), case["autotune_trace"])
    assert p_best == float(case["p_best"])
    assert k == int(case["n_clusters_raw"])
  labels, det = orc.predict(x, opt, return_details=True)
  np.testing.assert_array_equal(labels, case["labels"])
  if "eigenvalues_head" in case:
    head = case["eigenvalues_head"]
    np.testing.assert_allclose(det["eigenvalues"][:len(head)], head, rtol=1e-11,
                               atol=1e-12 * np.abs(head).max())

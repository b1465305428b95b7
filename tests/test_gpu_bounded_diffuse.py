"""GPU: the bounded Diffuse against the storing one on the same Y_hi -- row maxima bit for bit (on
speaker data, identical rows and a block-diagonal Y), row sums within the epilogue's fp32 rounding,
the device tile count against the NumPy rule -- and predict() against the storing route."""

import numpy as np
import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev
from spectralcluster_b200 import spectral_clusterer as sc_mod
from oracle import spectral_oracle as orc

import bounded_diffuse_numpy as bd
from test_gpu_factored import assert_routes_agree, embeddings, icassp, stored_front

pytestmark = pytest.mark.gpu
SIZES = [16384, 40003, 65536]


def bits(t):
  return t.contiguous().view(dev.torch().int32)


def edge_y(engine, n, kind):
  t = dev.torch()
  hi = t.zeros((n, dev.round_up(n, 64)), dtype=t.float16, device=engine.device)
  if kind == "identical":
    hi[:, :n] = 0.125
  else:                                   # block-diagonal: 6 blocks of symmetric positive values
    g = t.Generator(device=engine.device).manual_seed(n)
    edges = np.linspace(0, n, 7).astype(int)
    for a, b in zip(edges[:-1], edges[1:]):
      blk = t.rand((b - a, b - a), generator=g, device=engine.device) * 0.9 + 0.1
      hi[a:b, a:b] = t.maximum(blk, blk.T).half()
  return hi


def check_rowmax(engine, n, hi, expect_all=False):
  t = dev.torch()
  mx_ref, sm_ref = engine.diffuse_stats(n, hi)
  norms, diag, c = engine.row_group_bounds(hi, n)
  perm = engine.bound_order(norms)
  mx, counts = engine.rowmax_tiles(hi, n, norms, diag, perm)
  assert t.equal(bits(mx), bits(mx_ref))
  computed, total = counts.tolist()
  assert total == dev.bounded_tile_count(n)
  if expect_all:
    assert computed == total
  want = bd.kept_tiles(norms.double().cpu().numpy(), diag.cpu().numpy(), perm.cpu().numpy())
  assert computed == len(want)
  _, sm, _ = engine.bounded_diffuse(n, hi, want_max=False)
  rel = ((sm - sm_ref).abs() / sm_ref.abs().clamp_min(1e-300)).max().item()
  assert rel <= 2 * 191 * 2.0 ** -24, rel
  return computed, total


@pytest.mark.parametrize("n", SIZES)
def test_rowmax_bitwise_on_speaker_data(engine, n):
  _, _, _, hi = stored_front(engine, embeddings(engine, n, speakers=6), icassp())
  check_rowmax(engine, n, hi)


@pytest.mark.parametrize("kind", ["identical", "block"])
@pytest.mark.parametrize("n", SIZES)
def test_rowmax_bitwise_on_edge_inputs(engine, n, kind):
  hi = edge_y(engine, n, kind)
  check_rowmax(engine, n, hi, expect_all=kind == "identical")


@pytest.mark.parametrize("n", [dev.BOUNDED_FROM, 40003, 65536])
def test_predict_equals_the_storing_route(engine, n, monkeypatch):
  x = orc.synthetic_dvectors(n, 256, 6, seed=3).astype(np.float32)
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=10,
                            refinement_options=scb.configs.icassp2018_refinement_options,
                            laplacian_type=scb.LaplacianType.GraphCut, custom_dist="cosine")
  got = c.predict(x)
  det = dict(c.last_details)
  assert det["solver"] == "lanczos" and det["diffuse"]["operator"] == "factored"
  assert 0 < det["diffuse"]["tiles"] <= det["diffuse"]["of"] == dev.bounded_tile_count(n)
  monkeypatch.setattr(sc_mod.SpectralClusterer, "_bounded_route", lambda *a, **k: False)
  want = c.predict(x)
  assert "diffuse" not in c.last_details and c.last_details["solver"] == "lanczos"
  assert det["n_clusters"] == c.last_details["n_clusters"]
  assert np.array_equal(got, want)
  assert_routes_agree(det["eigenvalues"], c.last_details["eigenvalues"])

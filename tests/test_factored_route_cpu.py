"""CPU: the factored route's host logic -- which predict() calls take it (a fake engine stands in
for an 80 GB H100) and the row-panel plan its kernels run over."""

import pytest

import spectralcluster_b200 as scb
from spectralcluster_b200 import _native as nat
from spectralcluster_b200 import device as dev

RN = scb.RefinementName
H100_80GB = 85_520_809_984          # torch.cuda.get_device_properties(0).total_memory


class FakeEngine:
  """What _factored_route reads from an Engine, for a device with `total` bytes."""

  dense_eig_max = 0
  upper_pass_ok = staticmethod(dev.Engine.upper_pass_ok)

  def __init__(self, total=H100_80GB):
    self.factored_above_bytes = total - dev.FACTORED_ROUTE_RESERVE
    self.diffuse_precision = None

  def gemm_engine(self, n):
    return nat.GEMM_SIMT if n < dev.Engine.simt_below else nat.GEMM_TCGEN05

  diffuse_precision_for = dev.Engine.diffuse_precision_for


def icassp_clusterer(**kw):
  return scb.SpectralClusterer(min_clusters=2, max_clusters=10,
                               refinement_options=scb.configs.icassp2018_refinement_options,
                               custom_dist="cosine", **kw)


def test_80gb_routes_65536_stored_and_131072_factored():
  c, eng = icassp_clusterer(), FakeEngine()
  assert not c._factored_route(eng, 65536)
  assert c._factored_route(eng, 131072)
  assert c._factored_route(eng, 98304)


def test_threshold_follows_the_byte_formula():
  eng = FakeEngine()
  c = icassp_clusterer()
  n = 90000
  peak = 10 * n * dev.round_up(n, 64)
  assert dev.stored_route_peak_bytes(n) == peak
  eng.factored_above_bytes = peak
  assert not c._factored_route(eng, n)
  eng.factored_above_bytes = peak - 1
  assert c._factored_route(eng, n)


def _seq(*names, sigma=1.0, **kw):
  return scb.RefinementOptions(gaussian_blur_sigma=sigma, p_percentile=0.95,
                               thresholding_soft_multiplier=0.01,
                               thresholding_type=kw.pop("ttype", scb.ThresholdType.RowMax),
                               refinement_sequence=list(names), **kw)


ICASSP = [RN.CropDiagonal, RN.GaussianBlur, RN.RowWiseThreshold, RN.Symmetrize, RN.Diffuse,
          RN.RowWiseNormalize]


@pytest.mark.parametrize("opts", [
    _seq(*ICASSP), _seq(*ICASSP[1:]), _seq(*ICASSP[:-1]), _seq(*ICASSP[1:-1]),
    _seq(*ICASSP, symmetrize_type=scb.SymmetrizeType.Average)])
@pytest.mark.parametrize("laplacian", [None, scb.LaplacianType.GraphCut,
                                       scb.LaplacianType.RandomWalk])
def test_in_scope_calls_take_the_factored_route(opts, laplacian):
  c = scb.SpectralClusterer(min_clusters=2, max_clusters=31, refinement_options=opts,
                            laplacian_type=laplacian,
                            eigengap_type=scb.EigenGapType.NormalizedDiff,
                            row_wise_renorm=True, custom_dist="cityblock",
                            autotune=scb.AutoTune())
  assert c._factored_route(FakeEngine(), 131072)


def _not_affinity(x):
  return x


@pytest.mark.parametrize("change", [
    dict(min_clusters=1), dict(max_clusters=None), dict(max_clusters=32),
    dict(affinity_function=_not_affinity), dict(autotune_group=True),
    dict(refinement_options=_seq(*ICASSP, sigma=2.0)),
    dict(refinement_options=_seq(RN.CropDiagonal, RN.RowWiseThreshold, RN.Symmetrize,
                                 RN.Diffuse, RN.RowWiseNormalize)),
    dict(refinement_options=_seq(*ICASSP, ttype=scb.ThresholdType.Percentile)),
    dict(refinement_options=_seq(*ICASSP[:-1], RN.CropDiagonal)),
    dict(refinement_options=_seq(RN.RowWiseThreshold, RN.Symmetrize)),
    dict(refinement_options=_seq(*ICASSP, RN.Diffuse)),
    dict(constraint=True), dict(diffuse_precision=nat.GEMM_SPLIT2), dict(dense_eig_max=1 << 20)])
def test_out_of_scope_calls_keep_the_stored_route(change):
  change = dict(change)
  eng = FakeEngine()
  eng.diffuse_precision = change.pop("diffuse_precision", None)
  if "dense_eig_max" in change:
    eng.dense_eig_max = change.pop("dense_eig_max")
  constraint = change.pop("constraint", False)
  group = change.pop("autotune_group", None)
  kw = dict(min_clusters=2, max_clusters=10,
            refinement_options=scb.configs.icassp2018_refinement_options)
  kw.update(change)
  c = scb.SpectralClusterer(custom_dist="cosine", **kw)
  c.autotune_group = group
  matrix = None
  if constraint:
    c.constraint_options = scb.ConstraintOptions(
        constraint_name=scb.ConstraintName.ConstraintPropagation, apply_before_refinement=False)
    matrix = [[0]]
  assert not c._factored_route(eng, 131072, matrix)


@pytest.mark.parametrize("n", [4097, 16384, 65536, 98304, 131072, 131000])
@pytest.mark.parametrize("rows", [128, 384, 2048, None])
def test_panel_plan(n, rows):
  rows = rows or dev.panel_rows_for(n)
  plan = dev.panel_plan(n, rows)
  covered = []
  for r0, r1, a0, a1 in plan:
    covered.extend(range(r0, r1))
    assert r0 % dev.PANEL_ALIGN == 0 and a0 % dev.PANEL_ALIGN == 0
    assert r0 % 64 == 0 and r0 % 32 == 0           # the threshold tiles and the blur bands
    assert a0 <= max(0, r0 - dev.BLUR_HALO) and a0 > r0 - dev.BLUR_HALO - dev.PANEL_ALIGN
    assert a1 == min(n, r1 + dev.BLUR_HALO)
    assert r1 - r0 == rows or r1 == n
  assert covered == list(range(n))                    # every row exactly once, in order
  assert plan[0][2] == 0 and plan[-1][3] == n         # halos clipped at 0 and n
  if n % rows:
    assert plan[-1][1] - plan[-1][0] == n % rows      # a short last panel


def test_panel_height_depends_on_n_alone():
  for n in (65536, 98304, 131072, 190000):
    rows = dev.panel_rows_for(n)
    assert rows % dev.PANEL_ALIGN == 0
    assert 4 * rows * dev.round_up(n, 64) <= dev.FACTORED_PANEL_BYTES
    assert 4 * (rows + dev.PANEL_ALIGN) * dev.round_up(n, 64) > dev.FACTORED_PANEL_BYTES
  assert dev.panel_rows_for(1000) == 1024

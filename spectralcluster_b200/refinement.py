"""Affinity refinement operators -- device-backed mirror of the reference's refinement module.

Same public names, dataclass fields, defaults, enum member names and exceptions as
/root/reference/spectralcluster/refinement.py (enums :11-36, RefinementOptions :71-133,
operators :136-245).  Each operator's `refine(ndarray) -> ndarray` uploads the matrix, runs the
CUDA kernel behind the C ABI and downloads the result (fp32 arithmetic, returned as float64);
`SpectralClusterer.predict` does not go through these host round trips -- it keeps the matrix in
HBM and lets `device.run_refinement` fuse the sequence.
"""

from __future__ import annotations

import abc
import dataclasses
import enum
import typing

import numpy as np

from . import _native as nat
from . import device as dev


class RefinementName(enum.Enum):
  CropDiagonal = enum.auto()
  GaussianBlur = enum.auto()
  RowWiseThreshold = enum.auto()
  Symmetrize = enum.auto()
  Diffuse = enum.auto()
  RowWiseNormalize = enum.auto()


class ThresholdType(enum.Enum):
  RowMax = enum.auto()        # clear values below row_max * p_percentile
  Percentile = enum.auto()    # clear the p_percentile*100 % smallest values of each row


class SymmetrizeType(enum.Enum):
  Max = enum.auto()           # max(A, A^T)
  Average = enum.auto()       # (A + A^T) / 2


def _square(affinity: np.ndarray):
  dims = affinity.shape
  if len(dims) != 2:
    raise ValueError("affinity must be 2-dimensional")
  if dims[0] != dims[1]:
    raise ValueError("affinity must be a square matrix")
  return dims[0]


class AffinityRefinementOperation(metaclass=abc.ABCMeta):
  """Base class: validates the input and moves it through the device."""

  def check_input(self, affinity: np.ndarray):
    _square(affinity)

  def _on_device(self, affinity: np.ndarray, fn) -> np.ndarray:
    n = _square(affinity)
    eng = dev.Engine.get()
    a = eng.upload_matrix(affinity)
    return eng.download_matrix(fn(eng, a, n), n)

  @abc.abstractmethod
  def refine(self, affinity: np.ndarray) -> np.ndarray:
    """Returns a new matrix of the same shape."""


class CropDiagonal(AffinityRefinementOperation):
  """Diagonal <- largest off-diagonal value of the row (reference :136-151)."""

  def refine(self, affinity):
    return self._on_device(affinity, lambda eng, a, n: eng.crop_diagonal(a, n))


class GaussianBlur(AffinityRefinementOperation):
  """scipy.ndimage.gaussian_filter semantics (reference :154-162)."""

  def __init__(self, sigma: int = 1):
    self.sigma = sigma

  def refine(self, affinity):
    return self._on_device(affinity, lambda eng, a, n: eng.gaussian_blur(a, n, self.sigma))


class RowWiseThreshold(AffinityRefinementOperation):
  """Soft/hard row-wise thresholding (reference :165-210)."""

  def __init__(self, p_percentile: float = 0.95, thresholding_soft_multiplier: float = 0.01,
               thresholding_type: ThresholdType = ThresholdType.RowMax,
               thresholding_with_binarization: bool = False,
               thresholding_preserve_diagonal: bool = False):
    if not isinstance(thresholding_type, ThresholdType):
      raise TypeError("thresholding_type must be a ThresholdType")
    self.p_percentile = p_percentile
    self.multiplier = thresholding_soft_multiplier
    self.thresholding_type = thresholding_type
    self.thresholding_with_binarization = thresholding_with_binarization
    self.thresholding_preserve_diagonal = thresholding_preserve_diagonal

  def refine(self, affinity):
    if self.thresholding_type == ThresholdType.RowMax:
      kind = nat.THRESHOLD_ROWMAX
    elif self.thresholding_type == ThresholdType.Percentile:
      kind = nat.THRESHOLD_PERCENTILE
    else:
      raise ValueError("Unsupported thresholding_type")
    return self._on_device(affinity, lambda eng, a, n: eng.row_threshold(
        a, n, kind, self.p_percentile, self.multiplier, self.thresholding_with_binarization,
        self.thresholding_preserve_diagonal))


class Symmetrize(AffinityRefinementOperation):
  """max(A, A^T) or their average (reference :213-226)."""

  def __init__(self, symmetrize_type: SymmetrizeType = SymmetrizeType.Max):
    self.symmetrize_type = symmetrize_type

  def refine(self, affinity):
    if self.symmetrize_type == SymmetrizeType.Max:
      kind = nat.SYMMETRIZE_MAX
    elif self.symmetrize_type == SymmetrizeType.Average:
      kind = nat.SYMMETRIZE_AVERAGE
    else:
      raise ValueError("Unsupported symmetrize_type.")
    return self._on_device(affinity, lambda eng, a, n: eng.symmetrize(a, n, kind))


class Diffuse(AffinityRefinementOperation):
  """A A^T (reference :229-234) on the wgmma GEMM."""

  def refine(self, affinity):
    return self._on_device(affinity, lambda eng, a, n: eng.diffuse(n, y=a)[0])


class RowWiseNormalize(AffinityRefinementOperation):
  """Rows divided by their maximum (reference :237-245)."""

  def refine(self, affinity):
    return self._on_device(affinity, lambda eng, a, n: eng.row_normalize(a, n))


@dataclasses.dataclass
class RefinementOptions:
  """Option bag of the refinement sequence; fields and defaults as reference :76-100."""

  gaussian_blur_sigma: int = 1
  p_percentile: float = 0.95
  thresholding_soft_multiplier: float = 0.01
  thresholding_type: ThresholdType = ThresholdType.RowMax
  thresholding_with_binarization: bool = False
  thresholding_preserve_diagonal: bool = False
  symmetrize_type: SymmetrizeType = SymmetrizeType.Max
  refinement_sequence: typing.Optional[typing.Sequence[RefinementName]] = None

  def get_refinement_operator(self, name: RefinementName) -> AffinityRefinementOperation:
    """Operator object for `name`, configured from this bag (reference :102-133)."""
    makers = {
        RefinementName.CropDiagonal: lambda: CropDiagonal(),
        RefinementName.GaussianBlur: lambda: GaussianBlur(self.gaussian_blur_sigma),
        RefinementName.RowWiseThreshold: lambda: RowWiseThreshold(
            self.p_percentile, self.thresholding_soft_multiplier, self.thresholding_type,
            self.thresholding_with_binarization, self.thresholding_preserve_diagonal),
        RefinementName.Symmetrize: lambda: Symmetrize(self.symmetrize_type),
        RefinementName.Diffuse: lambda: Diffuse(),
        RefinementName.RowWiseNormalize: lambda: RowWiseNormalize(),
    }
    maker = makers.get(name) if isinstance(name, RefinementName) else None
    if maker is None:
      raise ValueError("Unknown refinement operation: {}".format(name))
    return maker()

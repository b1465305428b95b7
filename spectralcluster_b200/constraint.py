"""Constrained clustering operators -- device-backed mirror of
/root/reference/spectralcluster/constraint.py (ConstraintOptions :26-48, AffinityIntegration
:95-117, ConstraintPropagation :120-164, ConstraintMatrix :167-201).

ConstraintPropagation's closed form  F = (1-a)^2 (I - a Abar)^-1 Q (I - a Abar)^-1  (Abar =
D^-1/2 A D^-1/2) is evaluated on the device without a factorisation: the inverse comes from the
Newton-Schulz iteration X <- X (2I - M X), M = I - a Abar, which starts at X = I with residual
a Abar (spectral radius a < 1) and squares it every step -- ceil(log2(ln 1e-9 / ln a)) steps of
two dense products each, on the same GEMM engines as Diffuse (wgmma split-fp16 planes, or the
SIMT fp64-accumulate engine below 64 rows).  The reference calls np.linalg.inv (:151).

From X = I the iteration diverges for |a| >= 1 (the reference still inverts I - a Abar there), and
M is held in fp32, so the error of the inverse grows with cond(M) <= (1 + |a|) / (1 - |a|).
|a| <= MAX_ABS_ALPHA is the range measured against the float64 inverse on an H100
(tests/test_gpu_constraint_kernels.py); any other alpha raises NotImplementedError before a launch.
"""

from __future__ import annotations

import abc
import dataclasses
import enum
import math
import typing

import numpy as np

from . import _native as nat
from . import device as dev

EPS = 1e-10
# Newton-Schulz: stop once the residual's spectral radius |a|^(2^steps) is below this
RESIDUAL_TARGET = 1e-9
# largest |alpha| whose propagation was measured within the test tolerance on an H100 (80 GB HBM3,
# 700 W): 0.999 stays inside it at N = 63 and 1,000; 0.9999 at N = 1,000 is 1.6x outside it
MAX_ABS_ALPHA = 0.999


def newton_schulz_steps(alpha: float) -> int:
  """Steps of X <- X (2I - M X) from X = I until |alpha|^(2^steps) <= RESIDUAL_TARGET (the
  spectral radius of the residual alpha Abar is |alpha|); raises NotImplementedError for the
  alphas the device path does not serve."""
  alpha = float(alpha)
  if not abs(alpha) <= MAX_ABS_ALPHA:
    raise NotImplementedError(
        "ConstraintPropagation alpha={!r}: the device inverts I - alpha Abar by a Newton-Schulz "
        "iteration, which diverges for |alpha| >= 1 and is measured accurate in fp32 only for "
        "|alpha| <= {}".format(alpha, MAX_ABS_ALPHA))
  if alpha == 0.0:
    return 0                                                           # M = I: X = I is exact
  return max(1, int(math.ceil(math.log2(math.log(RESIDUAL_TARGET) / math.log(abs(alpha))))))


class ConstraintName(enum.Enum):
  AffinityIntegration = enum.auto()
  ConstraintPropagation = enum.auto()


class IntegrationType(enum.Enum):
  Max = enum.auto()
  Average = enum.auto()


@dataclasses.dataclass
class ConstraintOptions:
  """Which operator, and whether it acts before or after the affinity refinement."""
  constraint_name: ConstraintName
  apply_before_refinement: bool
  integration_type: typing.Optional[IntegrationType] = None
  constraint_propagation_alpha: float = 0.6

  def __post_init__(self):
    if self.constraint_name == ConstraintName.AffinityIntegration:
      self.constraint_operator = AffinityIntegration(self.integration_type)
    elif self.constraint_name == ConstraintName.ConstraintPropagation:
      self.constraint_operator = ConstraintPropagation(self.constraint_propagation_alpha)


def _matmul(eng, a, b, n):
  """a @ b for device fp32 [n, ld] matrices (b need not be symmetric: its transpose is formed)."""
  t = dev.torch()
  bt = eng.matrix(n)
  eng.call("sc_transpose", dev._ptr(b), n, n, b.stride(0), dev._ptr(bt), bt.stride(0), eng.stream)
  c = eng.matrix(n)
  if eng.gemm_engine(n) == nat.GEMM_SIMT:
    eng.call("sc_gemm_nt_f32", dev._ptr(a), a.stride(0), dev._ptr(bt), bt.stride(0), n, n, n,
             dev._ptr(c), c.stride(0), eng.stream)
  else:
    ah, al = eng.split_planes(a, n)
    bh, bl = eng.split_planes(bt, n)
    eng.call("sc_gemm_nt_planes", nat.GEMM_SPLIT3, dev._ptr(ah), dev._ptr(al), ah.stride(0), n,
             dev._ptr(bh), dev._ptr(bl), bh.stride(0), n, n, dev._ptr(c), c.stride(0), None, 0,
             eng.stream)
  return c


def _scale_shift(eng, x, n, alpha, beta, rows=None, cols=None):
  out = eng.matrix(n)
  eng.call("sc_scale_shift", dev._ptr(x), x.stride(0), n, dev._ptr(rows), dev._ptr(cols),
           float(alpha), float(beta), dev._ptr(out), out.stride(0), eng.stream)
  return out


class ConstraintOperation(metaclass=abc.ABCMeta):

  def check_input(self, affinity, constraint_matrix):
    """constraint.py:53-75 (same messages)."""
    if len(affinity.shape) != 2:
      raise ValueError("affinity must be 2-dimensional")
    if affinity.shape[0] != affinity.shape[1]:
      raise ValueError("affinity must be a square matrix")
    if len(constraint_matrix.shape) != 2:
      raise ValueError("constraint matrix must be 2-dimensional")
    if constraint_matrix.shape[0] != constraint_matrix.shape[1]:
      raise ValueError("constraint matrix must be a square matrix")
    if affinity.shape != constraint_matrix.shape:
      raise ValueError("affinity and constraint matrix must have the same shape")

  def adjust_affinity(self, affinity: np.ndarray, constraint_matrix: np.ndarray) -> np.ndarray:
    """Host arrays in, host array out (the reference signature); the arithmetic runs on the device."""
    self.check_input(affinity, constraint_matrix)
    eng = dev.Engine.get()
    n = affinity.shape[0]
    out = self.adjust_on_device(eng, eng.upload_matrix(affinity), eng.upload_matrix(constraint_matrix), n)
    return eng.download_matrix(out, n)

  @abc.abstractmethod
  def adjust_on_device(self, eng, a, q, n):
    """Device fp32 matrices in, a new device matrix out."""


class AffinityIntegration(ConstraintOperation):
  """Element-wise max / average of the affinity and the constraint matrix (constraint.py:95-117)."""

  def __init__(self, integration_type: IntegrationType = IntegrationType.Max):
    self.integration_type = integration_type

  def adjust_on_device(self, eng, a, q, n):
    if self.integration_type == IntegrationType.Max:
      mode = 0
    elif self.integration_type == IntegrationType.Average:
      mode = 1
    else:
      raise ValueError("Unsupported integration type: {}".format(self.integration_type))
    out = eng.matrix(n)
    eng.call("sc_constraint_combine", dev._ptr(a), a.stride(0), dev._ptr(q), q.stride(0), n, mode,
             dev._ptr(out), out.stride(0), eng.stream)
    return out


class ConstraintPropagation(ConstraintOperation):
  """Exhaustive and efficient constraint propagation (Lu & Ip, ECCV 2010), constraint.py:120-164."""

  def __init__(self, alpha: float = 0.6):
    self.alpha = alpha

  def check_input(self, affinity, constraint_matrix):
    super().check_input(affinity, constraint_matrix)
    newton_schulz_steps(self.alpha)

  def adjust_on_device(self, eng, a, q, n):
    alpha = float(self.alpha)
    steps = newton_schulz_steps(alpha)
    _, rowsum = eng.row_stats(a, n, want_max=False, want_sum=True)
    dn = 1.0 / (dev.torch().sqrt(rowsum) + EPS)                       # :144
    m = _scale_shift(eng, a, n, -alpha, 1.0, rows=dn, cols=dn)         # M = I - alpha Abar
    x = _scale_shift(eng, m, n, 0.0, 1.0)                              # X0 = I
    for _ in range(steps):                                             # X <- X (2I - M X)
      r = _scale_shift(eng, _matmul(eng, m, x, n), n, -1.0, 2.0)
      x = _matmul(eng, x, r, n)
    f = _matmul(eng, _matmul(eng, x, q, n), x, n)                      # :152-153
    f = _scale_shift(eng, f, n, (1.0 - alpha) ** 2, 0.0)
    out = eng.matrix(n)
    eng.call("sc_constraint_combine", dev._ptr(a), a.stride(0), dev._ptr(f), f.stride(0), n, 2,
             dev._ptr(out), out.stride(0), eng.stream)
    return out


class ConstraintMatrix:
  """Pairwise constraints between neighbouring turns from speaker-turn confidence scores
  (constraint.py:167-201): score 0 between turns i and i+1 -> must-link (+1), a score above the
  threshold -> cannot-link (-1); scores[0] is unused."""

  def __init__(self, speaker_turn_scores: typing.Sequence[float], threshold: float = 1):
    if any(score < 0 for score in speaker_turn_scores):
      raise ValueError("Speaker turn score must be larger or equal to 0.")
    self.speaker_turn_scores = speaker_turn_scores
    self.threshold = threshold

  def compute_diagonals(self) -> np.ndarray:
    scores = np.asarray(self.speaker_turn_scores, dtype=np.float64)
    n = len(scores)
    link = np.where(scores[1:] == 0, 1.0, np.where(scores[1:] > self.threshold, -1.0, 0.0))
    out = np.zeros((n, n))
    idx = np.arange(n - 1)
    out[idx, idx + 1] = link
    out[idx + 1, idx] = link
    return out

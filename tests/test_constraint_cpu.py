"""CPU: the step rule and the loop of ConstraintPropagation.adjust_on_device restated in float64.

The device inverts M = I - alpha Abar (Abar = D^-1/2 A D^-1/2, spectral radius 1 for a non-negative
affinity) by Newton-Schulz from X = I.  The residual I - M X starts at alpha Abar and is squared
every step, so after s steps its spectral radius is |alpha|^(2^s).  Every alpha the device path
accepts must reach the 1e-9 residual target; every other alpha must raise NotImplementedError
before the engine is touched."""

import re

import numpy as np
import pytest

from spectralcluster_b200 import constraint as ct

ACCEPTED = [0.0, 1e-12, -1e-6, 0.1, 0.4, 0.6, 0.9, 0.99, 0.995, 0.999, ct.MAX_ABS_ALPHA, -0.6,
            -0.99, -ct.MAX_ABS_ALPHA]
REFUSED = [1.0, -1.0, 1.2, -1.5, 0.9999, -0.9999, float("nan"), float("inf")]


def propagation_inputs(n=128, d=16, seed=0):
  """Random unit vectors, affinity (x x^T + 1) / 2, and a +-1/0 neighbour constraint matrix."""
  rng = np.random.default_rng(seed)
  x = rng.standard_normal((n, d))
  x /= np.linalg.norm(x, axis=1, keepdims=True)
  a = (x @ x.T + 1.0) / 2.0
  link = rng.choice([1.0, -1.0, 0.0], n - 1)
  q = np.diag(link, 1) + np.diag(link, -1)
  return a, q


def abar(a):
  dn = 1.0 / (np.sqrt(a.sum(axis=1)) + ct.EPS)                 # constraint.py:143-146
  return dn[:, None] * a * dn[None, :]


def test_step_counts_of_the_fixture_alphas_are_unchanged():
  assert ct.newton_schulz_steps(0.4) == 5
  assert ct.newton_schulz_steps(0.6) == 6
  assert ct.newton_schulz_steps(0.0) == 0


@pytest.mark.parametrize("alpha", ACCEPTED)
def test_step_rule_reaches_the_residual_target(alpha):
  """|alpha|^(2^s) <= 1e-9 with the fewest steps s that reach it."""
  s = ct.newton_schulz_steps(alpha)
  assert abs(alpha) ** (2 ** s) <= ct.RESIDUAL_TARGET
  if s > 1:
    assert abs(alpha) ** (2 ** (s - 1)) > ct.RESIDUAL_TARGET


@pytest.mark.parametrize("alpha", ACCEPTED)
def test_newton_schulz_loop_in_float64(alpha):
  """The device loop X <- X (2I - M X) in float64: the residual ||I - M X||_2 reaches 1e-9, up to
  float64 rounding of the iteration (a few n cond(M) 2^-53), and F = (1-a)^2 X Q X matches the
  one computed with np.linalg.inv to the same relative accuracy."""
  a, q = propagation_inputs()
  n = a.shape[0]
  m = np.eye(n) - alpha * abar(a)
  x = np.eye(n)
  for _ in range(ct.newton_schulz_steps(alpha)):
    x = x @ (2.0 * np.eye(n) - m @ x)
  cond = np.linalg.cond(m)
  floor = 4 * n * cond * 2.0 ** -53
  assert np.linalg.norm(np.eye(n) - m @ x, 2) <= ct.RESIDUAL_TARGET + floor
  inv = np.linalg.inv(m)
  f_ref = (1 - alpha) ** 2 * inv @ q @ inv
  f = (1 - alpha) ** 2 * x @ q @ x
  # |dF| <= 2 |dX| ||Q|| ||X|| (1-a)^2 with ||dX|| <= ||X|| (residual + floor), ||Q||_2 <= 2
  bound = 2 * 2 * (ct.RESIDUAL_TARGET + floor) * (1 - alpha) ** 2 * np.linalg.norm(inv, 2) ** 2
  assert np.abs(f - f_ref).max() <= bound


@pytest.mark.parametrize("alpha", REFUSED)
def test_unserved_alpha_raises_before_device_work(alpha):
  a, q = propagation_inputs(8)
  name = re.escape(repr(float(alpha)))
  with pytest.raises(NotImplementedError, match=name):
    ct.newton_schulz_steps(alpha)
  op = ct.ConstraintPropagation(alpha)
  # host API: raised by the input check, before an engine (which needs a GPU) is created
  with pytest.raises(NotImplementedError, match=name):
    op.adjust_affinity(a, q)

  class NoEngine:
    def __getattr__(self, attr):
      raise AssertionError("device work started: Engine.%s" % attr)

  with pytest.raises(NotImplementedError, match=name):
    op.adjust_on_device(NoEngine(), None, None, 8)


def test_the_old_twelve_step_cap_missed_the_target():
  """Why the cap went: 12 steps leave a residual of 0.999^4096 ~ 1.7e-2."""
  assert ct.newton_schulz_steps(0.999) > 12
  assert 0.999 ** (2 ** 12) > 1e-2
  assert ct.newton_schulz_steps(0.999) == 15

"""NumPy restatement of the bounded Diffuse (sc_row_group_bounds + sc_diffuse_tile_list): the row
bounds of a non-negative fp16 Y, the tiles of the symmetric single-MMA launch in its rasterised
order, and the rule that keeps a tile.  Shared by the CPU and GPU tests."""

import numpy as np

BM, BN, GROUP_M, GROUP_COLS = 128, 192, 16, 256
EPS = 2.0 ** -10


def row_bounds(y16):
  """(group norms [n, G] fp64, diagonal fp64, row sums fp64) of a non-negative fp16 [n, n] Y."""
  y = y16.astype(np.float64)
  n = y.shape[0]
  g = -(-n // GROUP_COLS)
  pad = np.zeros((n, g * GROUP_COLS))
  pad[:, :n] = y
  norms = np.sqrt((pad.reshape(n, g, GROUP_COLS) ** 2).sum(axis=2))
  return norms, (y * y).sum(axis=1), y.sum(axis=1)


def rasterised_tiles(n):
  """[(m, c)] of the symmetric launch (TileCursor): groups of GROUP_M row blocks, column blocks
  from the group's first reaching one, the group's valid row blocks innermost."""
  tm, tn = -(-n // BM), -(-n // BN)
  out = []
  for g in range(-(-tm // GROUP_M)):
    for c in range(g * GROUP_M * BM // BN, tn):
      for m in range(g * GROUP_M, min(tm, (g + 1) * GROUP_M)):
        if BM * m <= BN * c + BN - 1:
          out.append((m, c))
  return out


def kept_tiles(norms, diag, perm):
  """The tiles of the product of the rows Y[perm] the rule keeps, in rasterised order."""
  n = len(perm)
  pn, pd = norms[perm], diag[perm]
  keep = []
  for m, c in rasterised_tiles(n):
    r0, r1, c0, c1 = BM * m, min(n, BM * m + BM), BN * c, min(n, BN * c + BN)
    if c0 < BM * m + BM:                       # straddles the diagonal
      keep.append((m, c))
      continue
    u = float(pn[r0:r1].max(axis=0) @ pn[c0:c1].max(axis=0))
    l = min(pd[r0:r1].min(), pd[c0:c1].min())
    if not u * (1 + EPS) < l * (1 - EPS):
      keep.append((m, c))
  return keep

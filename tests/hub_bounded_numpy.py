"""NumPy restatement of the hub-first bounded Diffuse (sc_bound_order_hubs, sc_diffuse_hub_tiles,
sc_diffuse_tile_list_rows): the row order with each cluster's largest diagonal first, the phase-1
tiles that pair every cluster's rows with its hub, the row maxima those tiles fold, and the per-row
rule that keeps a phase-2 tile.  Shared by the CPU and GPU tests and tools/count_hub_tiles.py."""

import numpy as np

from bounded_diffuse_numpy import BM, BN, EPS, rasterised_tiles


def diag_key(diag):
  """The diagonal as the order compares it: fp32, rounded down (towards zero)."""
  d32 = diag.astype(np.float32)
  over = d32.astype(np.float64) > diag
  d32[over] = np.nextafter(d32[over], np.float32(0))
  return d32


def hub_order(diag, labels, k):
  """(perm, starts): rows sorted by (label, fp32 diagonal descending, index); starts[c] is the
  first position of cluster c (starts[k] = n), so cluster c's hub is perm[starts[c]] when it is
  not empty."""
  n = len(diag)
  perm = np.lexsort((np.arange(n), -diag_key(diag).astype(np.float64), labels))
  starts = np.concatenate([[0], np.cumsum(np.bincount(labels, minlength=k))]).astype(np.int64)
  return perm, starts


def hub_tiles(starts, n):
  """Phase 1 in rasterised order: for each non-empty cluster [s, e), the tiles of the hub's row
  block against every column block that holds a row of the cluster."""
  want = set()
  for s, e in zip(starts[:-1], starts[1:]):
    if e > s:
      want.update((s // BM, c) for c in range(s // BN, (e - 1) // BN + 1))
  return [t for t in rasterised_tiles(n) if t in want]


def fold(sp, tiles, n, into=None):
  """Row maxima (in the permuted order) of the elements of `tiles` of the permuted product `sp`,
  folded as the launch folds them: row r takes columns c >= r of a tile, column c the rows r < c."""
  mx = np.zeros(n) if into is None else into.copy()
  for m, c in tiles:
    r0, r1, c0, c1 = BM * m, min(n, BM * m + BM), BN * c, min(n, BN * c + BN)
    b = sp[r0:r1, c0:c1]
    rr = np.arange(r0, r1)[:, None]
    cc = np.arange(c0, c1)[None, :]
    mx[r0:r1] = np.maximum(mx[r0:r1], np.where(cc >= rr, b, 0.0).max(axis=1))
    mx[c0:c1] = np.maximum(mx[c0:c1], np.where(rr < cc, b, 0.0).max(axis=0))
  return mx


def block_max(pn, rows):
  """Maxima of the group norms over each block of `rows` rows of the permuted norms pn."""
  n, g = pn.shape
  nb = -(-n // rows)
  pad = np.zeros((nb * rows, g))
  pad[:n] = pn
  return pad.reshape(nb, rows, g).max(axis=1)


def _any_over_blocks(flag, rows):
  n, t = flag.shape
  nb = -(-n // rows)
  pad = np.zeros((nb * rows, t), dtype=bool)
  pad[:n] = flag
  return pad.reshape(nb, rows, t).any(axis=1)


def row_rule_flags(pn, big_l):
  """(row_keep [tiles_m, tiles_n], col_keep [tiles_n, tiles_m]): some row i of row block m has
  (1 + eps) u_iJ >= L_i against column block J, and the same with the roles swapped."""
  n = pn.shape[0]
  ur = pn @ block_max(pn, BN).T                      # u_iJ  [n, tiles_n]
  uc = pn @ block_max(pn, BM).T                      # u_Ij  [n, tiles_m]
  row_keep = _any_over_blocks(ur * (1 + EPS) >= big_l[:, None], BM)
  col_keep = _any_over_blocks(uc * (1 + EPS) >= big_l[:, None], BN)
  return row_keep, col_keep


def phase2_tiles(pn, big_l, phase1):
  """The tiles phase 2 computes, in rasterised order: every tile that straddles the diagonal or
  passes the per-row rule, except those phase 1 computed.  pn and big_l are in the permuted order."""
  n = pn.shape[0]
  row_keep, col_keep = row_rule_flags(pn, big_l)
  done = set(phase1)
  out = []
  for m, c in rasterised_tiles(n):
    if (m, c) in done:
      continue
    if BN * c < BM * m + BM or row_keep[m, c] or col_keep[c, m]:
      out.append((m, c))
  return out

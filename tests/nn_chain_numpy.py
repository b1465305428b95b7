"""NumPy restatement of scipy's `_hierarchy.nn_chain` for complete linkage, with the rules the
device kernel (sc_complete_linkage) follows: the chain starts at the lowest active index; the
nearest neighbour of the chain top is found by a strict `<` scan in index order that starts from
the previous chain element (so it wins ties, and otherwise the lowest index does); mutual
neighbours x < y merge into y.  Returns the merges in chain order, unsorted and unrelabelled."""

import numpy as np


def nn_chain_complete(dist):
  d = np.array(dist, dtype=np.float64, copy=True)
  n = d.shape[0]
  size = np.ones(n, dtype=np.int64)
  xy = np.empty((n - 1, 2), dtype=np.int64)
  md = np.empty(n - 1, dtype=np.float64)
  ms = np.empty(n - 1, dtype=np.int64)
  chain = []
  for k in range(n - 1):
    if not chain:
      chain.append(int(np.flatnonzero(size)[0]))
    while True:
      x = chain[-1]
      if len(chain) > 1:
        y, best = chain[-2], d[x, chain[-2]]
      else:
        y, best = -1, np.inf
      cand = np.flatnonzero(size)
      cand = cand[cand != x]
      j = int(np.argmin(d[x, cand]))            # first index holding the minimum
      if d[x, cand[j]] < best:
        y, best = int(cand[j]), d[x, cand[j]]
      if len(chain) > 1 and y == chain[-2]:
        break
      chain.append(y)
    del chain[-2:]
    a, b = min(x, y), max(x, y)
    xy[k] = a, b
    md[k] = best
    ms[k] = size[a] + size[b]
    size[b] += size[a]
    size[a] = 0
    keep = size > 0
    keep[b] = False
    d[b, keep] = d[keep, b] = np.maximum(d[a, keep], d[b, keep])
  return xy, md, ms

"""Row-sharded refinement across the GPUs of one box (SURVEY.md 8(e), BASELINE.json configs[3]).

One process per GPU (torch.distributed: NCCL on GPUs, gloo in the CPU tests).  Rank g owns the
row block [row_begin, row_end) of every N x N matrix:

  1. embeddings are replicated; every rank normalises all N rows (N*d work, no traffic);
  2. affinity rows of the block PLUS the blur halo (R rows each side) are computed locally --
     the halo is recomputed from the embeddings, not exchanged; CropDiagonal is row-local;
  3. blur statistics pass -> row maxima of the owned rows -> ALL-GATHER of N floats
     (the fused threshold/symmetrize rule needs m_i and m_j, SURVEY.md A.3);
  4. blur + threshold + symmetrize pass -> owned rows of Y as split fp16 planes;
  5. Diffuse: S = Y Y^T is symmetric, so rank g computes only S(g,g) and the blocks S(g, g+o),
     o = 1..G/2.  On NVLink (transport "peer": CUDA IPC mappings of the peers' buffers) the Y row
     blocks it multiplies against are pulled by the copy engines on a side stream while the
     tensor cores work on the own diagonal block -- no SM is taken from the persistent GEMM --
     and the other half of every rank's row block is written by the peers' GEMM epilogues
     themselves: each off-diagonal product stores its transposed tiles straight into the
     owner's S over NVLink (compute and exchange in one kernel).  Transport "nccl"/"gloo" (CPU
     tests, boxes without IPC) moves the same blocks with batched send/recv instead;
  6. row maxima / sums of S_block (RowWiseNormalize, Laplacian degree) are row-local.

Above the size where those per-rank buffers fit (sharded_stored_peak_bytes), the factored route
(FactoredShardedRefiner) keeps only the owned rows of Y's fp16 hi plane and never stores S: the
front end runs in row panels, S's row statistics are streamed over chunks of the peers' Y rows,
and the eigensolver applies S = Y Y^T as two half-products per pass.

The orchestration below is backend-agnostic: `DeviceBackend` runs the CUDA kernels through the C
ABI; the CPU tests plug in a NumPy backend and run the same code under gloo with 2 ranks.
"""

from __future__ import annotations

import ctypes
import math
import typing

import numpy as np


def _round_up(x: int, m: int) -> int:
  return (x + m - 1) // m * m


# The factored route streams the peers' Y rows through two staging buffers of about this many
# bytes each: a fixed size, whatever N and the world size.
STAGING_BYTES = 1 << 28


def sharded_stored_peak_bytes(n: int, world: int) -> int:
  """Per-rank device bytes of the stored sharded route's N x N-scale buffers, computed from shapes:
  both fp16 planes of Y at full size (world * block rows) and the fp32 arena that holds the halo'd
  affinity block and then S's row block (block + blur halo + 2 x 64 rows)."""
  from .device import BLUR_HALO, round_up
  block = _round_up(int(math.ceil(n / world)), 128)
  ld = round_up(n, 64)
  return 4 * world * block * ld + 4 * (block + 2 * BLUR_HALO + 2 * 64) * ld


def sharded_factored_peak_bytes(n: int, world: int) -> int:
  """Per-rank device bytes of the factored sharded route's large buffers, computed from shapes:
  the owned rows of Y_hi (fp16), one fp32 affinity panel with its halo, and the two staging
  buffers.  Nothing in it is N x N."""
  from .device import panel_rows_for, round_up
  block = _round_up(int(math.ceil(n / world)), 128)
  ld = round_up(n, 64)
  panel = min(panel_rows_for(n), block)
  staging = 2 * 2 * staging_rows_for(n) * ld if world > 1 else 0
  return 2 * block * ld + 4 * (panel + 2 * 64) * ld + staging


def staging_rows_for(n: int) -> int:
  """Rows of peer Y_hi per staging buffer: about STAGING_BYTES of fp16 rows, a multiple of 128."""
  from .device import round_up
  return max(128, STAGING_BYTES // (2 * round_up(n, 64)) // 128 * 128)


def factored_sharded_route(eng, n: int, world: int) -> bool:
  """Whether predict_sharded() takes the factored route: the stored sharded route's per-rank peak
  (computed from shapes) exceeds eng.factored_above_bytes, and Diffuse is the single-MMA product
  whose operand is Y's hi plane alone.  Decided from n, the world size, the options and the
  device's total memory, never from what is free, as predict()'s own route choice."""
  from . import _native as nat
  return (sharded_stored_peak_bytes(n, world) > eng.factored_above_bytes and
          eng.diffuse_precision_for(n) == nat.GEMM_SINGLE)


class RowPanel(typing.NamedTuple):
  """Output rows [row_begin, row_end) of one front-end panel, computed from the affinity rows
  [halo_begin, halo_end) (the blur halo clipped at 0 and n)."""
  row_begin: int
  row_end: int
  halo_begin: int
  halo_end: int

  @property
  def halo_rows(self) -> int:
    return self.halo_end - self.halo_begin


class ShardPlan:
  """Row partition of an n x n problem over `world` ranks, with the blur halo of `radius`.

  Block schedule of the symmetric product S = Y Y^T (G x G blocks of `block` rows): every
  off-diagonal block pair {S(a,b), S(b,a) = S(a,b)^T} is computed exactly once and mirrored to the
  other owner as a transposed copy (compute_jobs / mirror_jobs): G/2 block products per rank,
  diagonal block included.  Only the Y rows a rank multiplies against are fetched.
  """

  def __init__(self, n: int, world: int, rank: int, radius: int, align: int = 128):
    if world < 1 or not 0 <= rank < world:
      raise ValueError("bad world/rank")
    self.n, self.world, self.rank, self.radius = n, world, rank, radius
    self.block = _round_up(int(math.ceil(n / world)), align)
    if (world - 1) * self.block >= n:
      raise ValueError("n=%d is too small to give each of %d ranks a row block of %d"
                       % (n, world, self.block))
    self.row_begin, self.row_end = self.rows_of(rank)
    self.halo_begin = max(0, self.row_begin - radius)
    self.halo_end = min(n, self.row_end + radius)

  def rows_of(self, rank: int) -> typing.Tuple[int, int]:
    lo = rank * self.block
    return lo, min(lo + self.block, self.n)

  @property
  def rows(self) -> int:
    return self.row_end - self.row_begin

  @property
  def halo_rows(self) -> int:
    return self.halo_end - self.halo_begin

  def split_row(self, rank: int) -> int:
    """Row (relative to the block) at which rank's block is halved for the offset-G/2 pairing."""
    lo, hi = self.rows_of(rank)
    return min(hi - lo, _round_up((hi - lo + 1) // 2, 128))

  def compute_jobs(self, rank: typing.Optional[int] = None):
    """Off-diagonal products of `rank`: [(peer, (r0, r1), (c0, c1))] meaning
    S(rank, peer)[r0:r1, c0:c1] = Y_rank[r0:r1] * Y_peer[c0:c1]^T, indices relative to the blocks.

    Rank g takes the whole blocks at offsets 1 .. ceil(G/2)-1.  For even G the offset-G/2 block
    pair {a < b} is split between its two owners: a computes the top half of its rows against
    all of b, b computes all of its rows against the bottom half of a's rows -- together they
    cover S(a, b) once.  Everything else reaches a rank as a transposed copy (mirror_jobs)."""
    g = self.rank if rank is None else rank
    G = self.world
    rows_g = self.rows_of(g)[1] - self.rows_of(g)[0]
    jobs = []
    for o in range(1, (G + 1) // 2):
      p = (g + o) % G
      jobs.append((p, (0, rows_g), (0, self.rows_of(p)[1] - self.rows_of(p)[0])))
    if G % 2 == 0 and G > 1:
      p = (g + G // 2) % G
      rows_p = self.rows_of(p)[1] - self.rows_of(p)[0]
      if g < p:
        jobs.append((p, (0, self.split_row(g)), (0, rows_p)))
      else:
        jobs.append((p, (0, rows_g), (self.split_row(p), rows_p)))
    return [j for j in jobs if j[1][1] > j[1][0] and j[2][1] > j[2][0]]

  def mirror_jobs(self):
    """Blocks other ranks compute for this rank: [(source, (r0, r1), (c0, c1))] meaning source
    sends S(source, rank)[r0:r1, c0:c1] transposed; it lands at my rows c0:c1, source's
    columns r0:r1."""
    out = []
    for q in range(self.world):
      if q != self.rank:
        out += [(q, rr, cc) for p, rr, cc in self.compute_jobs(q) if p == self.rank]
    return out

  def y_requests(self):
    """Y rows other ranks need from this rank: [(consumer, (c0, c1))]."""
    return [(q, cc) for q, _, cc in self.mirror_jobs()]


class _Once:
  """A work handle whose wait() is idempotent (gloo hangs on a second wait of the same op)."""

  def __init__(self, work, after=None):
    self.work, self.done, self.after = work, False, after or []

  def wait(self):
    if not self.done:
      self.work.wait()
      for fn in self.after:
        fn()
      self.done = True


class ShardedRefiner:
  """[CropDiagonal] [GaussianBlur] RowWiseThreshold(RowMax) Symmetrize Diffuse on row blocks.

  `backend` supplies the arithmetic, `dist` is torch.distributed (or None for world == 1).
  run() returns the owned rows of S = Y Y^T together with their row maxima / sums.
  """

  def __init__(self, backend, options, dist=None, group=None):
    from . import refinement as rf
    self.backend, self.options, self.dist, self.group = backend, options, dist, group
    names = list(options.refinement_sequence or [])
    RN = rf.RefinementName
    self.has_crop = bool(names) and names[0] == RN.CropDiagonal
    rest = names[1:] if self.has_crop else names
    self.has_blur = bool(rest) and rest[0] == RN.GaussianBlur
    rest = rest[1:] if self.has_blur else rest
    tail = [RN.RowWiseThreshold, RN.Symmetrize, RN.Diffuse]
    if rest[:3] != tail or rest[3:] not in ([], [RN.RowWiseNormalize]):
      raise NotImplementedError(
          "the sharded pipeline covers [CropDiagonal] [GaussianBlur] RowWiseThreshold "
          "Symmetrize Diffuse [RowWiseNormalize] (the ICASSP-2018 family)")
    if options.thresholding_type != rf.ThresholdType.RowMax:
      raise NotImplementedError("sharded pipeline: RowMax thresholding only")
    self.sigma = float(options.gaussian_blur_sigma) if self.has_blur else 0.0
    self.sym_max = options.symmetrize_type == rf.SymmetrizeType.Max
    self.trace = None              # set to [] to collect (label, backend.mark()) pairs

  def _mark(self, label):
    if self.trace is not None:
      self.trace.append((label, self.backend.mark()))

  def _p2p(self, sends, recvs):
    """Post point-to-point transfers [(tensor, peer), ...]; returns one work handle per recv."""
    d = self.dist
    if not sends and not recvs:
      return [], []
    # gloo cannot send/recv device tensors: the single-GPU test configuration (two ranks sharing
    # one GPU over gloo) stages them through host memory; NCCL moves them GPU to GPU.
    staged = d.get_backend(self.group) == "gloo"
    if self.group is not None:      # P2POp wants GLOBAL ranks; the plan speaks group-local ranks
      sends = [(t, d.get_global_rank(self.group, peer)) for t, peer in sends]
      recvs = [(t, d.get_global_rank(self.group, peer)) for t, peer in recvs]
    ops, landing = [], []
    for t, peer in recvs:
      if staged and t.is_cuda:
        host = t.new_empty(t.shape, device="cpu")
        landing.append([lambda t=t, host=host: t.copy_(host)])
        ops.append(d.P2POp(d.irecv, host, peer, self.group))
      else:
        landing.append([])
        ops.append(d.P2POp(d.irecv, t, peer, self.group))
    for t, peer in sends:
      ops.append(d.P2POp(d.isend, t.cpu() if (staged and t.is_cuda) else t, peer, self.group))
    raw = d.batch_isend_irecv(ops)
    if len(raw) == len(ops):                         # gloo: one work per op
      works = [_Once(w, landing[i] if i < len(recvs) else None) for i, w in enumerate(raw)]
      return works[:len(recvs)], works
    works = [_Once(w) for w in raw]                  # NCCL: a single work for the whole group
    return [works[-1]] * len(recvs), works

  def run(self, embeddings, world: int = 1, rank: int = 0):
    from .device import blur_radius
    be, opt = self.backend, self.options
    n = int(embeddings.shape[0])
    plan = ShardPlan(n, world, rank, blur_radius(self.sigma))
    self._mark("start")
    planes = be.normalize(embeddings)
    # affinity of the owned rows + halo; CropDiagonal values for exactly those rows
    a_ext, crop = be.affinity_block(planes, n, plan.halo_begin, plan.halo_rows, self.has_crop)
    # blur statistics -> row maxima of the owned rows, gathered into a full-length vector
    m_full = be.new_row_vector(world * plan.block)
    be.blur_rowmax_block(a_ext, n, plan, crop, self.sigma,
                         bool(opt.thresholding_preserve_diagonal), m_full)
    if world > 1:
      self._all_gather_blocks(m_full, plan)
    self._mark("rowmax gathered")
    # owned rows of Y straight into the full-size planes (the fetched peer blocks land beside them)
    y_full = be.new_planes(world * plan.block, n)
    be.thrsym_block(a_ext, n, plan, crop, self.sigma, m_full, opt, self.sym_max, y_full)
    del a_ext
    self._mark("Y block done")

    def yblk(p):
      return [plane[p * plan.block:(p + 1) * plan.block] for plane in y_full]

    jobs = plan.compute_jobs() if world > 1 else []
    transport = be.transport(self.dist, self.group) if world > 1 else "local"
    self.last_transport = transport
    if transport == "peer":
      s_block = self._diffuse_peer(plan, y_full, jobs, n, yblk)
    else:
      s_block = self._diffuse_sendrecv(plan, y_full, jobs, n, yblk, world, rank)
    self._mark("mirrored blocks")
    rowmax, rowsum = be.row_stats_block(s_block, plan.rows, n)
    self._mark("row stats")
    return dict(plan=plan, s_block=s_block, rowmax=rowmax, rowsum=rowsum, y_planes=y_full)

  def _diffuse_peer(self, plan, y_full, jobs, n, yblk):
    """NVLink peer-memory schedule (one process per GPU, buffers mapped with CUDA IPC)."""
    be, rank = self.backend, plan.rank
    s_block = be.new_block(plan.rows, n)
    peers = be.peer_buffers(self.dist, self.group, y_full, s_block)
    # Everybody's Y block is written and everybody is done with the affinity arena (S lives in
    # it): a one-element all-reduce, stream-ordered, no host stall.
    be.stream_barrier(self.dist, self.group)
    self._mark("Y blocks visible")
    n_planes = be.b_planes_needed(n)               # split2 / single read only the hi plane of B
    pulls = []
    for p, _, (c0, c1) in jobs:
      lo = plan.rows_of(p)[0]
      pulls.append(be.pull_rows([pl for pl in y_full[:n_planes]], peers[p]["y"][:n_planes],
                                lo + c0, c1 - c0))
    be.gemm_block(y_full, plan.row_begin, plan.rows, plan.row_begin, plan.rows, n, s_block, 0)
    self._mark("own block")
    ld = s_block.stride(0)
    for (p, (r0, r1), (c0, c1)), ready in zip(jobs, pulls):
      be.wait_pull(ready)
      lo = plan.rows_of(p)[0]
      # S(p, rank)[c0:c1, r0:r1] = S(rank, p)[r0:r1, c0:c1]^T, stored by this GEMM's epilogue
      mirror = peers[p]["s"] + 4 * (c0 * ld + plan.row_begin + r0)
      be.gemm_block(y_full, plan.row_begin + r0, r1 - r0, lo + c0, c1 - c0, n, s_block, r0,
                    mirror=mirror, ldm=ld)
    self._mark("computed blocks")
    be.stream_barrier(self.dist, self.group)      # every peer's mirrored tiles have landed
    return s_block

  def _diffuse_sendrecv(self, plan, y_full, jobs, n, yblk, world, rank):
    """send/recv schedule (NCCL without IPC, gloo in the CPU tests, and world == 1)."""
    be = self.backend
    recv_works, all_works = [], []
    be.reserve_comm_sms(world > 1)     # leave SMs to the send/recv kernels during the GEMMs
    try:
      if world > 1:
        recvs = [(t[c0:c1], p) for p, _, (c0, c1) in jobs for t in yblk(p)]
        sends = [(t[c0:c1], q) for q, (c0, c1) in plan.y_requests() for t in yblk(rank)]
        recv_works, all_works = self._p2p(sends, recvs)
      s_block = be.new_block(plan.rows, n)
      be.gemm_block(y_full, plan.row_begin, plan.rows, plan.row_begin, plan.rows, n, s_block, 0)
      self._mark("own block")
      for idx, (p, (r0, r1), (c0, c1)) in enumerate(jobs):
        for w in recv_works[idx * len(y_full):(idx + 1) * len(y_full)]:
          w.wait()                                   # stream-ordered on CUDA, blocking on gloo
        lo = plan.rows_of(p)[0]
        be.gemm_block(y_full, plan.row_begin + r0, r1 - r0, lo + c0, c1 - c0, n, s_block, r0)
      for w in all_works:
        w.wait()
    finally:
      be.reserve_comm_sms(False)
    self._mark("computed blocks")
    if world > 1:
      outgoing = []                                  # S(rank, p)[r0:r1, c0:c1]^T -> rank p
      for p, (r0, r1), (c0, c1) in jobs:
        lo = plan.rows_of(p)[0]
        outgoing.append((be.transposed_block(s_block, r0, r1 - r0, lo + c0, c1 - c0), p))
      incoming = [(be.new_dense(c1 - c0, r1 - r0), q) for q, (r0, r1), (c0, c1) in plan.mirror_jobs()]
      _, all_w = self._p2p(outgoing, incoming)
      for w in all_w:
        w.wait()
      for (buf, q), (_, (r0, r1), (c0, c1)) in zip(incoming, plan.mirror_jobs()):
        be.place_block(s_block, c0, plan.rows_of(q)[0] + r0, buf)
    return s_block

  def _all_gather_blocks(self, full, plan):
    """full[p*block:(p+1)*block] <- rank p's slice (equal, padded blocks)."""
    mine = full[plan.rank * plan.block:(plan.rank + 1) * plan.block].clone()
    self.dist.all_gather_into_tensor(full, mine, group=self.group)


class FactoredShardedRefiner(ShardedRefiner):
  """The refinement of ShardedRefiner with S never stored and Y kept for the owned rows only.

  1. front end in row panels of the owned rows (two passes, as device.FactoredAffinity): pass 1
     computes each panel's affinity rows plus the blur halo and folds the blur row maxima into m,
     which is all-gathered (N floats); pass 2 recomputes the panel's affinity and writes its rows
     of Y's fp16 hi plane (no lo plane) into a rows x ld buffer;
  2. S's row maxima and sums of the owned rows: the own block by the symmetric statistics-only
     GEMM, then every peer's Y rows in chunks through two fixed-size staging buffers (send/recv),
     each chunk's statistics folded by the statistics-only GEMM.  S(g, :) is computed in full
     by every rank: twice the flops of the stored route's symmetric split.
  run() returns the owned Y_hi rows with the row maxima / sums."""

  def __init__(self, backend, options, dist=None, group=None, panel_rows=None):
    super().__init__(backend, options, dist=dist, group=group)
    self.panel_rows = panel_rows

  def panels(self, plan):
    from .device import panel_rows_for
    step = self.panel_rows or panel_rows_for(plan.n)
    out = []
    for r0 in range(plan.row_begin, plan.row_end, step):
      r1 = min(plan.row_end, r0 + step)
      out.append(RowPanel(r0, r1, max(0, r0 - plan.radius), min(plan.n, r1 + plan.radius)))
    return out

  def run(self, embeddings, world: int = 1, rank: int = 0):
    from .device import blur_radius
    be, opt = self.backend, self.options
    n = int(embeddings.shape[0])
    plan = ShardPlan(n, world, rank, blur_radius(self.sigma))
    panels = self.panels(plan)
    capacity = max(p.halo_rows for p in panels)
    zero_diag = bool(opt.thresholding_preserve_diagonal)
    self._mark("start")
    planes = be.normalize(embeddings)
    m_full = be.new_row_vector(world * plan.block)
    for p in panels:
      a, crop = be.affinity_block(planes, n, p.halo_begin, p.halo_rows, self.has_crop, capacity)
      be.blur_rowmax_block(a, n, p, crop, self.sigma, zero_diag, m_full)
    if world > 1:
      self._all_gather_blocks(m_full, plan)
    self._mark("rowmax gathered")
    y_rows = be.new_rows(plan.rows, n)
    for p in panels:
      a, crop = be.affinity_block(planes, n, p.halo_begin, p.halo_rows, self.has_crop, capacity)
      be.thrsym_rows(a, n, p, crop, self.sigma, m_full, opt, self.sym_max, y_rows, None,
                     plan.row_begin)
    del a
    self._mark("Y rows done")
    rowmax, rowsum = self._row_stats(plan, y_rows, n)
    self._mark("row stats")
    return dict(plan=plan, y_rows=y_rows, rowmax=rowmax, rowsum=rowsum)

  def _row_stats(self, plan, y_rows, n):
    """Row maxima and sums of S(g, :) = Y[R_g] Y^T, S never stored."""
    be, world, rank = self.backend, plan.world, plan.rank
    mx, sm = be.new_stats(plan.rows)
    be.stats_block(y_rows, plan.rows, y_rows, plan.rows, n, mx, sm)     # own block, symmetric
    self.last_transport = self.dist.get_backend(self.group) if world > 1 else "local"
    if world == 1:
      return mx, sm
    staging, chunk = be.staging(n)
    be.reserve_comm_sms(True)        # leave SMs to the send/recv kernels during the GEMMs
    try:
      for o in range(1, world):
        # step o: receive the rows of rank + o, send mine to rank - o (every pair matches)
        src, dst = (rank + o) % world, (rank - o) % world
        lo, hi = plan.rows_of(src)
        recv = [(c0, min(c0 + chunk, hi - lo)) for c0 in range(0, hi - lo, chunk)]
        send = [(c0, min(c0 + chunk, plan.rows)) for c0 in range(0, plan.rows, chunk)]

        def post(j):
          sends = [(y_rows[send[j][0]:send[j][1]], dst)] if j < len(send) else []
          recvs = ([(staging[j % 2][:recv[j][1] - recv[j][0]], src)] if j < len(recv) else [])
          return self._p2p(sends, recvs)

        steps = max(len(recv), len(send))
        pending, works = post(0), []
        for j in range(steps):
          recv_w, all_w = pending
          works += all_w
          # chunk j + 1 lands in the other buffer while chunk j is multiplied; the GEMM of chunk
          # j - 1, which read that buffer, is already ordered before it on the stream
          pending = post(j + 1) if j + 1 < steps else ([], [])
          for w in recv_w:
            w.wait()
          if j < len(recv):
            c0, c1 = recv[j]
            be.stats_block(y_rows, plan.rows, staging[j % 2], c1 - c0, n, mx, sm)
        for w in works:
          w.wait()
    finally:
      be.reserve_comm_sms(False)
    return mx, sm


class DeviceBackend:
  """The CUDA kernels behind the C ABI (wgmma GEMMs, fused blur passes)."""

  def __init__(self, engine):
    from . import _native as nat
    from . import device as dev
    self.eng, self.nat, self.dev = engine, nat, dev
    self.t = dev.torch()
    # The N x N-scale buffers are allocated once and reused by every run(): at N = 131,072 they
    # add up to >100 GB per GPU and re-allocating them costs ~1 s of cudaMalloc/cudaFree per step.
    # (A result that must survive the next run() has to be cloned by the caller.)
    self._buffers = {}
    self._peer_ok, self.peer_error = None, None
    self._peer_maps, self._flag, self._copy_stream = {}, None, None

  def _buffer(self, tag, shape, dtype):
    key = (tag, tuple(shape), dtype)
    buf = self._buffers.get(key)
    if buf is None:
      for k in [k for k in self._buffers if k[0] == tag]:
        del self._buffers[k]                      # shape changed: drop the stale buffer first
      buf = self.t.empty(shape, dtype=dtype, device=self.eng.device)
      self._buffers[key] = buf
    return buf

  def _p(self, t):
    return self.dev._ptr(t)

  def normalize(self, x):
    eng, t = self.eng, self.t
    n, d = int(x.shape[0]), int(x.shape[1])
    hi, lo = eng.planes(n, d)
    eng.call("sc_normalize_rows", self._p(x), 1 if x.dtype == t.float64 else 0, n, d,
             x.stride(0), None, 0, self._p(hi), self._p(lo), hi.stride(0), eng.stream)
    return hi, lo, d

  def affinity_block(self, planes, n, row_begin, row_count, want_crop, capacity=None):
    """Affinity rows [row_begin, +row_count) in the arena; `capacity` (rows) keeps one arena for
    panels of different heights."""
    eng, t = self.eng, self.t
    hi, lo, d = planes
    ld = self.dev.round_up(n, 64)
    # the halo'd affinity block is dead before S_block is written: both live in one arena
    arena = self._buffer("arena", (max(row_count, capacity or 0, 1) + 2 * 64, ld), t.float32)
    a = arena[:row_count]
    crop = t.zeros((n,), dtype=t.float32, device=eng.device) if want_crop else None
    eng.call("sc_affinity_cosine_block", eng.gemm_precision, self._p(hi), self._p(lo),
             hi.stride(0), n, d, row_begin, row_count, self._p(a), a.stride(0),
             None if crop is None else self.dev.ctypes.c_void_p(crop.data_ptr() + 4 * row_begin),
             eng.stream)
    return a, crop

  def new_row_vector(self, length):
    return self.t.zeros((length,), dtype=self.t.float32, device=self.eng.device)

  def new_planes(self, rows, n):
    t, ld = self.t, self.dev.round_up(n, 64)
    return (self._buffer("y_hi", (rows, ld), t.float16), self._buffer("y_lo", (rows, ld), t.float16))

  def new_block(self, rows, n):
    ld = self.dev.round_up(n, 64)
    arena = next((b for k, b in self._buffers.items() if k[0] == "arena" and b.shape[1] == ld
                  and b.shape[0] >= rows), None)
    if arena is None:
      arena = self._buffer("arena", (rows + 2 * 64, ld), self.t.float32)
    return arena[:rows]

  def blur_rowmax_block(self, a_ext, n, plan, crop, sigma, zero_diag, m_full):
    eng = self.eng
    eng.call("sc_gaussian_blur_rowmax_block", self._p(a_ext), n, a_ext.stride(0),
             plan.halo_begin, plan.halo_rows, plan.row_begin, plan.row_end, self._p(crop),
             float(sigma), int(zero_diag), self._p(m_full), eng.stream)

  def thrsym_block(self, a_ext, n, plan, crop, sigma, m_full, opt, sym_max, y_full):
    self.thrsym_rows(a_ext, n, plan, crop, sigma, m_full, opt, sym_max, y_full[0], y_full[1], 0)

  def thrsym_rows(self, a_ext, n, rows, crop, sigma, m_full, opt, sym_max, hi, lo, first_row):
    """Y rows [rows.row_begin, rows.row_end) into planes whose row 0 is global row first_row
    (`lo` None: the hi plane only)."""
    eng, nat = self.eng, self.nat
    off = (rows.row_begin - first_row) * hi.stride(0) * 2
    c = self.dev.ctypes.c_void_p
    eng.call("sc_blur_threshold_symmetrize_block", self._p(a_ext), n, a_ext.stride(0),
             rows.halo_begin, rows.halo_rows, rows.row_begin, rows.row_end, self._p(crop),
             float(sigma), self._p(m_full), float(opt.p_percentile),
             float(opt.thresholding_soft_multiplier), int(bool(opt.thresholding_with_binarization)),
             int(bool(opt.thresholding_preserve_diagonal)),
             nat.SYMMETRIZE_MAX if sym_max else nat.SYMMETRIZE_AVERAGE, None, 0,
             c(hi.data_ptr() + off), None if lo is None else c(lo.data_ptr() + off), hi.stride(0),
             eng.stream)

  # ---- factored route: owned Y_hi rows, S's row statistics streamed
  def new_rows(self, rows, n):
    """The owned rows of Y's hi plane.  The stored route's full-size planes are released first:
    the two routes never run on the same call."""
    self.release("y_hi", "y_lo")
    return self._buffer("y_rows", (rows, self.dev.round_up(n, 64)), self.t.float16)

  def release(self, *tags):
    for k in [k for k in self._buffers if k[0] in tags]:
      del self._buffers[k]

  def new_stats(self, rows):
    t = self.t
    return (t.zeros((rows,), dtype=t.float32, device=self.eng.device),
            t.zeros((rows,), dtype=t.float64, device=self.eng.device))

  def stats_block(self, a, a_rows, b, b_rows, n, mx, sm):
    """mx / sm (rows of a) <- max / + the row maxima / sums of a[:a_rows] b[:b_rows]^T (K = n)."""
    self.eng.call("sc_diffuse_stats_block", self._p(a), a.stride(0), a_rows, self._p(b),
                  b.stride(0), b_rows, n, self._p(mx), self._p(sm), self.eng.stream)

  def staging(self, n):
    """Two staging buffers for peer Y_hi rows, and their height in rows."""
    rows = staging_rows_for(n)
    buf = self._buffer("staging", (2, rows, self.dev.round_up(n, 64)), self.t.float16)
    return [buf[0], buf[1]], rows

  def gemm_block(self, y_full, a_row, a_rows, b_row, b_rows, n, s_block, s_row, mirror=None,
                 ldm=0):
    """s_block[s_row:s_row+a_rows, b_row:b_row+b_rows] = Y[a_row:+a_rows] Y[b_row:+b_rows]^T;
    `mirror` (a raw device address, possibly in a peer GPU) also receives the transpose."""
    eng = self.eng
    hi, lo = y_full
    ld = hi.stride(0)
    c = self.dev.ctypes.c_void_p
    eng.call("sc_gemm_nt_planes", eng.diffuse_precision_for(n),
             c(hi.data_ptr() + 2 * a_row * ld), c(lo.data_ptr() + 2 * a_row * ld), ld, a_rows,
             c(hi.data_ptr() + 2 * b_row * ld), c(lo.data_ptr() + 2 * b_row * ld), ld, b_rows, n,
             c(s_block.data_ptr() + 4 * (s_row * s_block.stride(0) + b_row)), s_block.stride(0),
             c(mirror) if mirror else None, int(ldm), eng.stream)

  # ---- NVLink peer memory (CUDA IPC) -------------------------------------------------------
  def transport(self, dist, group):
    """"peer" (IPC-mapped buffers, copy-engine pulls + epilogue pushes) when every rank of the
    group drives its own GPU of this box over NCCL; else "nccl" / "gloo" send/recv."""
    import os
    backend = dist.get_backend(group)
    if backend != "nccl":
      return backend
    if os.environ.get("SCB_SHARDED_TRANSPORT", "peer") != "peer":
      return "nccl"
    if self._peer_ok is None:
      self._peer_ok = self._probe_peer(dist, group)
    return "peer" if self._peer_ok else "nccl"

  def _probe_peer(self, dist, group):
    """All ranks on distinct devices of one host, and an IPC round trip works."""
    import socket
    t = self.t
    world = dist.get_world_size(group)
    info = [None] * world
    dist.all_gather_object(info, (socket.gethostname(), self.eng.device_index), group=group)
    ok = len(set(h for h, _ in info)) == 1 and len(set(d for _, d in info)) == world
    if ok:
      try:
        probe = self._buffer("ipc_probe", (1 << 18,), t.float32)
        self._open_all(dist, group, [probe])
      except Exception as e:                      # IPC unavailable (container policy, driver)
        self.peer_error = str(e)
        ok = False
    flag = t.tensor([1 if ok else 0], device=self.eng.device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
    return bool(int(flag[0]))

  def _open_all(self, dist, group, tensors):
    """[{name index: raw address in this process} per rank] for the given local tensors."""
    import ctypes
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    mine = []
    for tn in tensors:
      handle = ctypes.create_string_buffer(64)
      off = ctypes.c_int64(0)
      self.nat.call("sc_ipc_export", self.eng.ctx, self._p(tn), handle, ctypes.byref(off))
      mine.append((handle.raw, int(off.value)))
    everyone = [None] * world
    dist.all_gather_object(everyone, mine, group=group)
    out = []
    for q in range(world):
      if q == rank:
        out.append([tn.data_ptr() for tn in tensors])
        continue
      addrs = []
      for raw, off in everyone[q]:
        ptr = ctypes.c_void_p()
        self.nat.call("sc_ipc_open", self.eng.ctx, ctypes.create_string_buffer(raw, 64), off,
                      ctypes.byref(ptr))
        addrs.append(int(ptr.value))
      out.append(addrs)
    return out

  def peer_buffers(self, dist, group, y_full, s_block):
    """{rank: {"y": [hi address, lo address], "s": address}} of every rank's persistent Y planes
    and S row block, mapped once per buffer set."""
    key = (y_full[0].data_ptr(), y_full[1].data_ptr(), s_block.data_ptr())
    cached = self._peer_maps.get(key)
    if cached is None:
      addrs = self._open_all(dist, group, [y_full[0], y_full[1], s_block])
      cached = [dict(y=a[:2], s=a[2]) for a in addrs]
      self._peer_maps = {key: cached}             # buffers changed shape: older maps are stale
    return cached

  def stream_barrier(self, dist, group):
    if self._flag is None:
      self._flag = self.t.zeros((1,), dtype=self.t.float32, device=self.eng.device)
    dist.all_reduce(self._flag, group=group)

  def b_planes_needed(self, n):
    return 2 if self.eng.diffuse_precision_for(n) == self.nat.GEMM_SPLIT3 else 1

  def pull_rows(self, local_planes, peer_addrs, row, rows):
    """Copy rows [row, row+rows) of the peer's planes into the same rows of the local planes on
    the copy stream; returns the event the consumer waits for."""
    t = self.t
    if self._copy_stream is None:
      self._copy_stream = t.cuda.Stream(device=self.eng.device)
    side = self._copy_stream
    side.wait_stream(t.cuda.current_stream(self.eng.device))
    c = self.dev.ctypes.c_void_p
    for plane, addr in zip(local_planes, peer_addrs):
      off = row * plane.stride(0) * plane.element_size()
      self.nat.call("sc_memcpy_async", self.eng.ctx, c(plane.data_ptr() + off), c(addr + off),
                    rows * plane.stride(0) * plane.element_size(), c(side.cuda_stream))
    ev = t.cuda.Event()
    ev.record(side)
    return ev

  def wait_pull(self, ev):
    self.t.cuda.current_stream(self.eng.device).wait_event(ev)

  comm_sms = 16

  def reserve_comm_sms(self, on):
    import ctypes
    limit = (self.nat.load().sc_context_sm_count(self.eng.ctx) - self.comm_sms) if on else 0
    self.nat.call("sc_context_set_gemm_sm_limit", self.eng.ctx, ctypes.c_int(limit))

  def mark(self):
    e = self.t.cuda.Event(enable_timing=True)
    e.record()
    return e

  def new_dense(self, rows, cols):
    return self.t.empty((rows, cols), dtype=self.t.float32, device=self.eng.device)

  def transposed_block(self, s_block, row_begin, rows, col_begin, cols):
    """Contiguous [cols, rows] copy of s_block[row_begin:+rows, col_begin:+cols]^T."""
    eng = self.eng
    out = self.new_dense(cols, rows)
    c = self.dev.ctypes.c_void_p
    eng.call("sc_transpose", c(s_block.data_ptr() + 4 * (row_begin * s_block.stride(0) + col_begin)),
             rows, cols, s_block.stride(0), self._p(out), out.stride(0), eng.stream)
    return out

  def place_block(self, s_block, row_begin, col_begin, dense):
    r, c = dense.shape
    s_block[row_begin:row_begin + r, col_begin:col_begin + c].copy_(dense)

  def row_stats_block(self, s_block, rows, n):
    eng, t = self.eng, self.t
    mx = t.empty((rows,), dtype=t.float64, device=eng.device)
    sm = t.empty((rows,), dtype=t.float64, device=eng.device)
    eng.call("sc_row_stats_block", self._p(s_block), rows, n, s_block.stride(0), self._p(mx),
             self._p(sm), eng.stream)
    return mx, sm


class ShardedOps:
  """The eigensolver on a row-sharded S: the operator diag(delta) + sign * diag(left) S diag(right)
  with this rank's row block of S (factored: its rows of Y_hi, S = Y Y^T applied as Y (Y^T T):
  Y^T T summed over the ranks, then Y T' all-gathered).  Every block product streams the local rows and all-gathers the
  slabs (b N doubles per pass over S); everything else -- Gram-Schmidt, the locked set, the Ritz
  pairs -- runs replicated on full-length vectors, so every rank returns bitwise identical values.

  extremal() is one sc_eigh_extremal_sharded solve.  window / lambda_max / vectors are the ops
  eigen_windows.solve drives, as eigen_windows.DeviceOps on one GPU; their locked set of
  `capacity` full-length vectors is replicated on every rank."""

  def __init__(self, eng, s_block, plan, n, delta, left, right, sign, which, width: int,
               dist=None, group=None, capacity: int = 0, factored: bool = False):
    from . import _native as nat
    from . import device as dev
    t = dev.torch()
    self.eng, self.nat, self.ptr = eng, nat, dev._ptr
    self.s_block, self.plan, self.n = s_block, plan, n
    self.delta, self.left, self.right, self.sign, self.which = delta, left, right, sign, which
    # factored: s_block is this rank's rows of Y_hi (fp16) and S = Y Y^T is never formed
    self.entry = "sc_eigh_extremal_factored_sharded" if factored else "sc_eigh_extremal_sharded"
    self.window_entry = ("sc_eigh_extremal_locked_factored_sharded" if factored
                         else "sc_eigh_extremal_locked_sharded")
    world, rank = plan.world, plan.rank
    # block products land in slabs [rank][vector][block]: one all-gather of contiguous slabs per
    # pass over S completes all `width` (or fewer) vectors on every rank
    y_slabs = t.zeros((world * width * plan.block,), dtype=t.float64, device=eng.device)

    def gather(_user, count):
      try:
        if world > 1 and count < 0:
          # factored operator: sum this rank's share of Y^T T (-count vectors of length n)
          dist.all_reduce(y_slabs[:-count * n], group=group)
        elif world > 1:
          per = count * plan.block
          dist.all_gather_into_tensor(y_slabs[:world * per], y_slabs[rank * per:(rank + 1) * per].clone(),
                                      group=group)
        return 0
      except Exception:                                  # never unwind through the C frame
        return 1

    self.y_slabs, self.callback = y_slabs, nat.GATHER_FN(gather)
    self.locked = t.empty((capacity, n), dtype=t.float64, device=eng.device) if capacity else None
    self.count, self.scale = 0, 0.0
    self.stats = dict(windows=0, passes=0, matvecs=0, restarts=0)

  def _slab_args(self):
    return (self.ptr(self.y_slabs), self.plan.rank, self.plan.block, self.callback, None)

  def extremal(self, which, n_values, n_vectors):
    """The n_values extremal eigenvalues (host fp64), eigenvectors for the first n_vectors of
    them (device fp64 [n, n_vectors]) and the solver's stats[4]."""
    from . import device as dev
    t = dev.torch()
    s, plan, ptr = self.s_block, self.plan, self.ptr
    w = np.empty(n_values, dtype=np.float64)
    v = t.empty((self.n, n_vectors), dtype=t.float64, device=self.eng.device)
    stats = np.zeros(4, dtype=np.int64)
    self.eng.call(self.entry, ptr(s), plan.rows, plan.row_begin, self.n,
                  s.stride(0), ptr(self.delta), ptr(self.left), ptr(self.right), float(self.sign),
                  int(which), n_values, n_vectors, 1e-9, 0, *self._slab_args(),
                  w.ctypes.data_as(ctypes.c_void_p), ptr(v) if n_vectors else None,
                  stats.ctypes.data_as(ctypes.c_void_p), self.eng.stream)
    return w, v, stats

  def window(self, count):
    s, plan, ptr = self.s_block, self.plan, self.ptr
    assert self.count + count <= self.locked.shape[0]
    w = np.empty(count, dtype=np.float64)
    st = np.zeros(4, dtype=np.int64)
    self.eng.call(self.window_entry, ptr(s), plan.rows, plan.row_begin, self.n,
                  s.stride(0), ptr(self.delta), ptr(self.left), ptr(self.right), float(self.sign),
                  int(self.which), count, 1e-9, 0, float(self.scale), ptr(self.locked), self.count,
                  *self._slab_args(), w.ctypes.data_as(ctypes.c_void_p),
                  st.ctypes.data_as(ctypes.c_void_p), self.eng.stream)
    self.count += count
    self.scale = max(self.scale, float(np.abs(w).max()))
    self.stats["windows"] += 1
    self.stats["matvecs"] += int(st[0])
    self.stats["restarts"] += int(st[1])
    self.stats["passes"] += int(st[3])
    return w

  def lambda_max(self):
    w, _, st = self.extremal(self.nat.EIG_LARGEST, 1, 0)
    self.scale = max(self.scale, abs(float(w[0])))
    self.stats["passes"] += int(st[3])
    return float(w[0])

  def vectors(self, cols):
    return self.eng.eigh_mapback(self.locked, self.n, cols, self.left, self.right)


def windowed(clusterer) -> bool:
  """Whether predict_sharded() solves in windows: max_clusters None or more pairs than one
  Lanczos solve finds."""
  from .spectral_clusterer import LANCZOS_MAX_PAIRS
  return not clusterer.max_clusters or clusterer.max_clusters + 1 > LANCZOS_MAX_PAIRS


def check_sharded_options(clusterer, num_embeddings: int):
  """The argument / option checks of predict() that also apply to predict_sharded(): a clusterer
  configured with something this path does not implement must fail here, not silently return
  labels that differ from predict() and from the reference."""
  from . import custom_distance_kmeans, utils
  if clusterer.autotune:
    raise NotImplementedError("predict_sharded: AutoTune is not sharded")
  if clusterer.affinity_function is not utils.compute_affinity_matrix:
    raise NotImplementedError("predict_sharded: only the built-in cosine affinity is sharded")
  if num_embeddings < clusterer.fallback_options.spectral_min_embeddings:
    raise NotImplementedError("predict_sharded: the fallback clusterer is not sharded")
  if clusterer.max_spectral_size is not None and num_embeddings > clusterer.max_spectral_size:
    raise NotImplementedError("predict_sharded: max_spectral_size pre-clustering is not sharded "
                              "(sharding is the exact alternative to it)")
  if clusterer.min_clusters == 1:
    raise NotImplementedError("predict_sharded: single-cluster detection is not sharded")
  if clusterer.constraint_options:
    raise NotImplementedError("predict_sharded: constraints are not sharded")
  from . import eigen_windows as ew
  from .spectral_clusterer import lanczos_basis, lanczos_fits
  if not windowed(clusterer):
    limit = clusterer.max_clusters + 1
    if not lanczos_fits(num_embeddings, limit):
      raise ValueError("predict_sharded: n=%d is too small for the Lanczos basis (%d vectors); "
                       "use predict()" % (num_embeddings, lanczos_basis(limit)))
    return
  if clusterer.max_clusters and clusterer.max_clusters + 1 > ew.MAX_WINDOW_PAIRS:
    raise ew._cap_error(clusterer.max_clusters, ew.MAX_WINDOW_PAIRS)
  # the last window starts with up to capacity - WINDOW_PAIRS vectors locked
  capacity = ew.capacity(num_embeddings, clusterer.max_clusters, clusterer.min_clusters)
  locked = max(capacity - ew.WINDOW_PAIRS, 0)
  if num_embeddings - locked < 2 * ew.WINDOW_BASIS:
    raise ValueError("predict_sharded: n=%d is too small for the windowed Lanczos basis (%d "
                     "locked + %d vectors); use predict()"
                     % (num_embeddings, locked, 2 * ew.WINDOW_BASIS))


def predict_sharded(clusterer, embeddings, dist=None, group=None) -> np.ndarray:
  """SpectralClusterer.predict() with every N x N matrix row-sharded over the ranks of `group`
  (BASELINE.json configs[3]: N = 131,072 does not fit one GPU).  Every rank passes the same
  embeddings (a host ndarray, or a float32/float64 tensor already on this rank's GPU) and
  receives the same labels.

  Refinement as in ShardedRefiner, or FactoredShardedRefiner when factored_sharded_route() says
  the stored route's per-rank buffers do not fit; row maxima / sums all-gathered (2 N doubles); eigensolve by the
  sharded thick-restart Lanczos (each matvec streams the local row block and all-gathers N
  doubles), in windows with a replicated locked set when max_clusters is None or >= 32; eigengap
  and k-means replicated on the [N, k] eigenvectors."""
  from . import _native as nat
  from . import eigen_windows as ew
  from . import custom_distance_kmeans, device as dev, laplacian as lap, utils
  from . import refinement as rf
  t = dev.torch()
  on_device = t.is_tensor(embeddings) and embeddings.is_cuda
  if not on_device and not isinstance(embeddings, np.ndarray):
    raise TypeError("embeddings must be a numpy array")
  if len(embeddings.shape) != 2:
    raise ValueError("embeddings must be 2-dimensional")
  check_sharded_options(clusterer, int(embeddings.shape[0]))
  world = dist.get_world_size(group) if dist is not None else 1
  rank = dist.get_rank(group) if dist is not None else 0
  eng = dev.Engine.get()
  be = getattr(eng, "_sharded_backend", None)
  if be is None:                 # persistent: N x N-scale buffers and the peers' IPC mappings
    be = eng._sharded_backend = DeviceBackend(eng)
  if on_device:
    x_dev = embeddings
  else:
    x = np.ascontiguousarray(embeddings)
    if x.dtype not in (np.float32, np.float64):
      x = x.astype(np.float64)
    x_dev = t.from_numpy(x).to(eng.device, non_blocking=True)
  n = int(x_dev.shape[0])
  opt = clusterer.refinement_options
  # the stored route's per-rank buffers do not fit: keep only the owned rows of Y_hi
  factored = factored_sharded_route(eng, n, world)
  refiner = (FactoredShardedRefiner if factored else ShardedRefiner)(
      be, opt, dist=dist if world > 1 else None, group=group)
  res = refiner.run(x_dev, world, rank)
  plan = res["plan"]
  length = world * plan.block

  def gathered(local):
    full = t.zeros((length,), dtype=t.float64, device=eng.device)
    full[plan.row_begin:plan.row_end] = local
    if world > 1:
      dist.all_gather_into_tensor(full, full[rank * plan.block:(rank + 1) * plan.block].clone(),
                                  group=group)
    return full[:n].contiguous()

  rowmax, rowsum = gathered(res["rowmax"]), gathered(res["rowsum"])
  normalized = list(opt.refinement_sequence)[-1] == rf.RefinementName.RowWiseNormalize
  r = (1.0 / rowmax) if normalized else None
  delta, left, right, sign, which = lap.terms_from_row_sums(rowsum, r, clusterer.laplacian_type)
  descend = which == nat.EIG_LARGEST
  op = (eng, res["y_rows"] if factored else res["s_block"], plan, n, delta, left, right, sign,
        which)
  dist_args = dict(dist=dist if world > 1 else None, group=group, factored=factored)
  route = "factored-sharded" if factored else "sharded"
  if windowed(clusterer):
    # max_clusters None or >= 32: windows of block Lanczos on the complement of the pairs found,
    # until the eigengap is decided (as predict() above the dense solver's n).  Every decision is
    # made on w, which is bitwise the same on every rank.
    limit = min(n, clusterer.max_clusters + 1) if clusterer.max_clusters else n
    ops = ShardedOps(*op, width=int(nat.load().sc_eigh_block_size(ew.WINDOW_PAIRS)),
                     capacity=ew.capacity(n, clusterer.max_clusters, clusterer.min_clusters),
                     **dist_args)
    prefix = ew.solve(ops, descend, clusterer.max_clusters, clusterer.min_clusters,
                      clusterer.stop_eigenvalue, clusterer.eigengap_type, n=n)
    w = prefix.values[:limit]
    k, gap = clusterer._count_clusters(w, descend, prefix.lambda_max)
    columns = min(len(w), max(k, clusterer.min_clusters or 0, 1))
    v = ops.vectors(prefix.order[:columns])
    solver, stats = "lanczos-windows-%s x%d" % (route, world), ops.stats
  else:
    limit = min(n, clusterer.max_clusters + 1)
    n_vectors = min(n, max(limit, clusterer.min_clusters or 0))
    ops = ShardedOps(*op, width=int(nat.load().sc_eigh_block_size(limit)), **dist_args)
    w, v, stats = ops.extremal(which, limit, n_vectors)
    if not descend and clusterer.eigengap_type == utils.EigenGapType.NormalizedDiff:
      # np.max(eigenvalues) of the full spectrum (utils.py:109): one more extremal solve
      w = np.concatenate([w, ops.extremal(nat.EIG_LARGEST, 1, 0)[0]])
    k, gap = clusterer._count_clusters(w, descend)
    solver, stats = "lanczos-%s x%d" % (route, world), stats.tolist()
  clusterer.last_details = dict(eigenvalues=np.array(w[:limit]), n_clusters_raw=k, max_gap=gap,
                                solver=solver,
                                transport=getattr(refiner, "last_transport", "local"),
                                lanczos_stats=stats)
  return clusterer._cluster_embeddings(eng, v, k)


def parallel_autotune(evaluate: typing.Callable[[float], typing.Tuple[float, int]],
                      grid: typing.Sequence[float], dist=None, group=None, world: int = 1,
                      rank: int = 0):
  """AutoTune with one p_percentile per rank (BASELINE.json configs[4]).

  Every rank holds the base affinity; rank r evaluates grid[r::world] with `evaluate(p) ->
  (ratio, n_clusters)`; the (ratio, k) pairs are all-gathered and every rank picks the same
  winner: the smallest ratio, the lowest grid index on ties (autotune.py:106-111 keeps the
  first strict minimum of an ascending scan).  Returns (best_index, best_p, ratio, k, owner).
  """
  mine = [(idx, evaluate(grid[idx])) for idx in range(rank, len(grid), world)]
  table = np.full((len(grid), 2), np.inf)
  for idx, (ratio, k) in mine:
    table[idx] = (ratio, k)
  if world > 1:
    import torch as t
    local = t.from_numpy(table)
    device = None
    if dist.get_backend(group) == "nccl":
      device = t.device("cuda", t.cuda.current_device())
      local = local.to(device)
    gathered = [t.empty_like(local) for _ in range(world)]
    dist.all_gather(gathered, local, group=group)
    table = t.stack(gathered).min(dim=0).values.cpu().numpy()   # unevaluated entries are +inf
  best = int(np.argmin(table[:, 0]))          # first minimum == lowest index on ties
  return best, grid[best], float(table[best, 0]), int(table[best, 1]), best % world

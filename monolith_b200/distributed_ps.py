"""FID-hash sharded tables across the GPUs of one box — replacement of the reference's
distributed_ps path for the embedding hot path.

Mirrors PartitionedHashTable._lookup_gpu / _apply_gradients_gpu (ref: native_training/
distributed_ps.py:1501-1760, 1762-2001) and DistributedMultiTypeHashTableMpi (ref:
distributed_ps_sync.py:95-512): owner(fid) = fid mod N (ref: distributed_ps.py:289;
fused_reorder_by_indices.cc:121-123), and per step

  forward : 1 dedup + bucket FIDs by owner (FusedReorderByIndices layout: shard-major, table-minor)
            2 all-to-all of the per-(shard, table) counts           int32[N*K]   (ref :1586-1588)
            3 all-to-all of the deduplicated FIDs                   int64        (ref :1582-1601)
            4 owner: fused lookup of everything received                        (ref :1619-1621)
            5 all-to-all of the rows                                float32      (ref :1680-1703)
            6 requester: gather + per-row pool from the received buffer         (ref :1745-1756)
  backward: 7 requester: scatter pooled grads to the unique rows                (ref :1792-1805)
            8 all-to-all of the row grads (reverse splits)                      (ref :1884-1899)
            9 owner: fused optimizer update, shards applied in order            (ref :1981-1990)

The reference runs these as Horovod/BytePS alltoalls with host staging; here they are NCCL
all-to-all-v calls (torch.distributed.all_to_all_single) over NVLink/NVSwitch on a dedicated
communication stream, so that the caller's dense tower can run concurrently on its own stream.

The compute steps come from a `backend` object so that the exchange logic (splits, offsets,
ordering) is testable on CPU with the gloo backend; the default backend is the CUDA engine.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import _lib
from .clip_ops import scale_ptr


class CudaBackend:
  """The engine's kernels behind the five compute steps of the exchange."""

  def __init__(self, table):
    from . import distribution_ops
    self.t = table
    self.dops = distribution_ops
    # 16-byte aligned rows everywhere in the fused buffers <=> every table dim is a multiple of 4
    self.vec_ok = all(d % 4 == 0 for d in table.get_table_dim_sizes())

  def reorder(self, fids_list, num_shards, dims):
    out, shard_sizes, slot_sizes, _, offs = self.dops.fused_reorder_by_indices(fids_list, num_shards, dims,
                                                                               rank0_empty_shard=False)
    return out, shard_sizes, slot_sizes, offs

  def fused_lookup(self, ids, slot_sizes, num_shards):
    return self.t.fused_lookup(ids, slot_sizes, num_shards)[0]

  def fused_apply(self, ids, slot_sizes, grads, num_shards, req_time):
    _, _, id_off, emb_off = self.t.fused_offsets(slot_sizes, num_shards)
    self.t.fused_apply_gradient(ids, ids, slot_sizes, grads, id_off, emb_off, 0, req_time, num_shards)

  def gather_pool(self, rows, offs, dim, row_offsets, pooling, out):
    return self.dops.gather_pool(rows, offs, dim, row_offsets, pooling, out=out)

  def gather_pool_grad_into(self, grad_buf, pooled_grad, offs, dim, row_offsets, pooling, scale=None):
    """Fills grad_buf (pre-zeroed, shared by all tables of the step).  dim % 4 == 0 and <= 128: the
    deterministic sort-based scatter; otherwise the float-atomic kernel (like the reference GPU path).
    pooled_grad is float32 or bfloat16 (the bf16 kernels widen it exactly); grad_buf is float32.  scale (a
    one-element float32 device tensor, or None): pooled_grad is multiplied by it in float32 first (the _scaled
    kernels, no extra pass)."""
    if self.vec_ok and dim <= 128:
      self.dops.scatter_grad_rows(pooled_grad, offs, dim, grad_buf, row_offsets, pooling, scale=scale)
    else:
      self.dops._gather_pool_grad_into(grad_buf, pooled_grad, offs, dim, row_offsets, pooling, 0, scale)

  def zeros(self, n, like):
    return torch.zeros(n, dtype=torch.float32, device=like.device)


def _a2a(out: torch.Tensor, inp: torch.Tensor, out_splits: Sequence[int], in_splits: Sequence[int], group):
  dist.all_to_all_single(out, inp, output_split_sizes=list(out_splits), input_split_sizes=list(in_splits), group=group)


class StepContext:
  """What the backward needs from the forward (ref: the tensors _lookup_gpu stashes in auxiliary_bundle)."""
  __slots__ = ("uniq", "shard_sizes", "slot_sizes", "offs", "recv_ids", "recv_slot", "send_row_splits",
               "recv_row_splits", "names", "row_offsets", "poolings", "occ_splits", "n_rows_total")


class _Phases:
  """Optional per-phase device timing (MONO_TIMING=1): CUDA events around each step of the exchange."""

  def __init__(self, enabled):
    import os
    self.enabled = enabled
    self.level = int(os.environ.get("MONO_TIMING", "0") or 0)
    self.marks = []
    self.acc = {}
    self.skip = int(os.environ.get("MONO_TIMING_SKIP", "5"))  # warm-up steps left out of the averages

  def fine(self, name):
    """extra marks inside a phase (MONO_TIMING=2): kernel time vs the barrier wait that follows"""
    if self.enabled and self.level >= 2:
      self.mark(name)

  def mark(self, name):
    if self.enabled:
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      self.marks.append((name, e))

  def flush(self):
    if not self.enabled or len(self.marks) < 2:
      self.marks = []
      return
    torch.cuda.synchronize()
    if self.skip > 0:
      self.skip -= 1
      self.marks = []
      return
    for (n0, e0), (n1, e1) in zip(self.marks[:-1], self.marks[1:]):
      t, c = self.acc.get(n1, (0.0, 0))
      self.acc[n1] = (t + e0.elapsed_time(e1), c + 1)
    self.marks = []

  def report(self):
    return {k: round(t / c, 4) for k, (t, c) in self.acc.items()}


class PartitionedHashTable:
  """Sharded view over one MultiHashTable per rank (ref: PartitionedHashTable, distributed_ps.py:581-2001)."""

  def __init__(self, table, world_size: int, rank: int, group=None, backend=None, dims: Optional[Sequence[int]] = None,
               names: Optional[Sequence[str]] = None):
    self.table = table
    self.N = world_size
    self.rank = rank
    self.group = group
    self.backend = backend if backend is not None else CudaBackend(table)
    self.names = tuple(names) if names is not None else tuple(table.table_names)
    self.dims = list(dims) if dims is not None else list(table.get_table_dim_sizes())
    self.K = len(self.names)
    import os
    self.phases = _Phases(os.environ.get("MONO_TIMING", "0") == "1" and backend is None)
    self.comm_stream = None
    if torch.cuda.is_available() and backend is None:
      self.comm_stream = torch.cuda.Stream(device=table.device)

  # -- helpers ------------------------------------------------------------------------------
  def _row_splits(self, slot_sizes: Sequence[int]) -> List[int]:
    """floats exchanged with each peer: sum_k slot[n][k] * D_k (ref: recv_emb_splits, distributed_ps.py:1514-1523)."""
    return [sum(slot_sizes[n * self.K + k] * self.dims[k] for k in range(self.K)) for n in range(self.N)]

  def lookup(self, slot_to_fids: Dict[str, torch.Tensor], row_offsets: Optional[Dict[str, torch.Tensor]] = None,
             pooling: Optional[Dict[str, str]] = None, outs: Optional[Dict[str, torch.Tensor]] = None,
             dtype: torch.dtype = torch.float32):
    """Forward steps 1-6.  Returns ({table: pooled [rows, D]}, ctx).  dtype: of the pooled rows this call
    allocates, float32 or bfloat16 (the float32 rows rounded once; the exchanged rows stay float32)."""
    if dtype not in (torch.float32, torch.bfloat16):
      raise ValueError(f"dtype must be torch.float32 or torch.bfloat16, not {dtype}")
    be, N, K = self.backend, self.N, self.K
    row_offsets = row_offsets or {}
    pooling = pooling or {}
    lists = []
    for name in self.names:
      f = slot_to_fids.get(name)
      lists.append(f.reshape(-1) if f is not None else torch.empty(0, dtype=torch.int64, device=self._dev(slot_to_fids)))
    dev = lists[0].device
    ph = self.phases
    ph.mark("start")
    # 1 dedup + bucket by owner
    uniq, shard_sizes, slot_sizes, offs = be.reorder(lists, N, self.dims)
    ph.mark("f1_reorder")
    # 2 counts
    send_cnt = torch.tensor(slot_sizes, dtype=torch.int64, device=dev)
    recv_cnt = torch.empty_like(send_cnt)
    _a2a(recv_cnt, send_cnt, [K] * N, [K] * N, self.group)
    recv_slot = [int(x) for x in recv_cnt.cpu().tolist()]  # [requester n][table k]: ids I own
    recv_id_splits = [sum(recv_slot[n * K:(n + 1) * K]) for n in range(N)]
    ph.mark("f2_a2a_counts")
    # 3 FIDs
    recv_ids = torch.empty(sum(recv_id_splits), dtype=torch.int64, device=dev)
    _a2a(recv_ids, uniq, recv_id_splits, shard_sizes, self.group)
    ph.mark("f3_a2a_ids")
    # 4 owner-side fused lookup (rows laid out requester-major / table-minor)
    rows = be.fused_lookup(recv_ids, recv_slot, N)
    ph.mark("f4_owner_lookup")
    # 5 rows back
    send_row_splits = self._row_splits(recv_slot)
    recv_row_splits = self._row_splits(slot_sizes)
    recv_rows = torch.empty(sum(recv_row_splits), dtype=torch.float32, device=dev)
    _a2a(recv_rows, rows, recv_row_splits, send_row_splits, self.group)
    ph.mark("f5_a2a_rows")
    # 6 requester-side gather + pool, table by table (offs covers the occurrences list by list)
    pooled, occ_splits, pos = {}, [], 0
    for k, name in enumerate(self.names):
      n_occ = lists[k].numel()
      occ_splits.append((pos, pos + n_occ))
      if name in slot_to_fids:
        ro = row_offsets.get(name)
        out = None if outs is None else outs.get(name)
        if out is None and dtype != torch.float32:
          out = torch.empty(n_occ if ro is None else ro.numel() - 1, self.dims[k], dtype=dtype, device=dev)
        pooled[name] = be.gather_pool(recv_rows, offs[pos:pos + n_occ], self.dims[k], ro, pooling.get(name, "sum"), out)
      pos += n_occ
    ph.mark("f6_gather_pool")
    ctx = StepContext()
    ctx.uniq, ctx.shard_sizes, ctx.slot_sizes, ctx.offs = uniq, shard_sizes, slot_sizes, offs
    ctx.recv_ids, ctx.recv_slot = recv_ids, recv_slot
    ctx.send_row_splits, ctx.recv_row_splits = send_row_splits, recv_row_splits
    ctx.row_offsets, ctx.poolings, ctx.occ_splits = row_offsets, pooling, occ_splits
    return pooled, ctx

  def apply_gradients(self, ctx: StepContext, pooled_grads: Dict[str, torch.Tensor], req_time: int = 0,
                      grad_scale: Optional[torch.Tensor] = None):
    """Backward steps 7-9.  pooled_grads are float32 or bfloat16; the exchanged row gradients are float32.
    grad_scale (ref: PartitionedHashTable.apply_gradients' grad_scale, distributed_ps.py:1283-1329): a one-element
    float32 tensor on the gradients' device, e.g. clip_ops.global_norm_scale's scale.  Every pooled gradient is then
    multiplied by it in float32 inside the scatter of step 7; the backend receives it only when it is given."""
    be, N = self.backend, self.N
    some = next(iter(pooled_grads.values()))
    scale_ptr(grad_scale, some.device, "grad_scale")
    extra = {} if grad_scale is None else {"scale": grad_scale}
    ph = self.phases
    ph.mark("bwd_start")
    # 7 scatter pooled grads to the unique rows, in the layout of the received row buffer
    grad_rows = be.zeros(sum(ctx.recv_row_splits), some)
    for k, name in enumerate(self.names):
      if name not in pooled_grads:
        continue
      lo, hi = ctx.occ_splits[k]
      be.gather_pool_grad_into(grad_rows, pooled_grads[name], ctx.offs[lo:hi], self.dims[k], ctx.row_offsets.get(name),
                               ctx.poolings.get(name, "sum"), **extra)
    ph.mark("b7_scatter_grads")
    # 8 grads to the owners (reverse of step 5)
    owner_grads = torch.empty(sum(ctx.send_row_splits), dtype=torch.float32, device=grad_rows.device)
    _a2a(owner_grads, grad_rows, ctx.send_row_splits, ctx.recv_row_splits, self.group)
    ph.mark("b8_a2a_grads")
    # 9 owner-side fused optimizer (same FID from several requesters: applied in requester order)
    be.fused_apply(ctx.recv_ids, ctx.recv_slot, owner_grads, N, req_time)
    ph.mark("b9_owner_apply")
    ph.flush()

  @staticmethod
  def _dev(d):
    return next(iter(d.values())).device


class HostCounts:
  """Per-step exchange of small host-side integer rows between the ranks of ONE node through a shared
  /dev/shm mapping (every rank ends up with the full world x width matrix).  It replaces the count
  all-to-all + device-to-host read of the NCCL path: the counts are already on the host (the grouping
  returns them), so they never need to touch a GPU.  Double-buffered by step parity; a rank can run at
  most one exchange ahead of the slowest one, because exchange e+1 completes only after every rank has
  published e+1, which each does after reading all of e."""

  def __init__(self, world: int, rank: int, width: int, group=None):
    import mmap
    import os
    import platform
    import uuid
    import numpy as np
    if platform.machine() not in ("x86_64", "AMD64"):
      # payload-then-epoch publication below relies on x86 total store order; a weakly ordered host (aarch64)
      # needs release/acquire atomics here -- use exchange="nccl" there
      raise RuntimeError("HostCounts needs an x86-64 host (store ordering); use the NCCL exchange on this platform")
    self.world, self.rank, self.width, self.epoch = world, rank, width, 0
    nbytes = 2 * world * (width + 1) * 8
    name = [f"/dev/shm/mono_counts_{os.getpid()}_{uuid.uuid4().hex}" if rank == 0 else None]
    if rank == 0:
      with open(name[0], "wb") as f:
        f.write(b"\0" * nbytes)
    if world > 1:
      dist.broadcast_object_list(name, src=0, group=group)
    self._f = open(name[0], "r+b")
    self._mm = mmap.mmap(self._f.fileno(), nbytes)
    self.arr = np.frombuffer(self._mm, dtype=np.int64).reshape(2, world, width + 1)
    if world > 1:
      dist.barrier(group=group)
    if rank == 0:
      os.unlink(name[0])

  def exchange(self, row, timeout_s: float = 120.0):
    import time
    import numpy as np
    self.epoch += 1
    e, buf = self.epoch, self.arr[self.epoch & 1]
    buf[self.rank, 1:] = np.asarray(row, dtype=np.int64)
    buf[self.rank, 0] = e            # published after the payload (x86 store order)
    t0 = None
    while not bool((buf[:, 0] == e).all()):
      if t0 is None:
        t0 = time.monotonic()
      elif time.monotonic() - t0 > timeout_s:
        raise RuntimeError(f"HostCounts: rank {self.rank} timed out at exchange {e}")
    return buf[:, 1:].copy()


def exchange_plan(cnt, me: int):
  """Offsets of the peer-window exchange for rank `me`, from the N x N count matrix cnt[r][o] = number of
  distinct FIDs requester r sends to owner o (identical on every rank).  All in items (FIDs / rows):
    recv[r]        what this rank, as an owner, receives from requester r
    bucket_at[o]   where this rank's bucket for owner o starts in its own bucketed unique list (= rows_in)
    seg_at[o]      where this rank's items start inside owner o's received list (ids_in / grads_in of o)
    rows_dst[r]    as an owner: where requester r's bucket for this rank starts in r's rows_in
    recv_at[r]     as an owner: where requester r's items start in this rank's received list
  so that the received lists are compact, requester-major — exactly an all-to-all-v result."""
  import numpy as np
  cnt = np.asarray(cnt, dtype=np.int64)
  N = cnt.shape[0]
  col_pre = np.concatenate([np.zeros((1, N), np.int64), np.cumsum(cnt, axis=0)])          # [r][o] = sum_{r' < r} cnt[r'][o]
  row_pre = np.concatenate([np.zeros((N, 1), np.int64), np.cumsum(cnt, axis=1)], axis=1)  # [r][o] = sum_{o' < o} cnt[r][o']
  return {"recv": cnt[:, me].copy(), "bucket_at": row_pre[me, :N].copy(), "seg_at": col_pre[me, :].copy(),
          "rows_dst": row_pre[:N, me].copy(), "recv_at": col_pre[:N, me].copy()}


class _FlatSource:
  """What the peer and NCCL exchanges of ShardedStep.step() group, pool and reduce: one FID list, one pooling, one
  output tensor and its gradient."""

  def __init__(self, st, fids, pooled_grad, out, row_offsets, pooling, grad_scale):
    self.st, self.fids, self.grad, self.out = st, fids, pooled_grad, out
    self.row_offsets, self.pooling, self.grad_scale = row_offsets, pooling, grad_scale
    self.n_fids, self.device = fids.numel(), fids.device

  def build(self, N, D):
    return self.st.grouping.build(self.fids, N, D)

  def pool(self, rows, offs):
    self.st.dops.gather_pool(rows, offs, self.st.dim, self.row_offsets, self.pooling, out=self.out)

  def take_grads(self):
    if callable(self.grad):
      self.grad = self.grad()

  def reduce(self, out_rows):
    self.st.grouping.reduce(self.grad, out_rows, self.row_offsets, self.pooling, grad_scale=self.grad_scale)

  def reduce_push(self, counts, window, region_off, dst_row_off):
    self.st.grouping.reduce_push(self.grad, counts, window, region_off, dst_row_off, self.row_offsets, self.pooling,
                                 grad_scale=self.grad_scale)


class _PartsSource:
  """What the peer and NCCL exchanges of ShardedStep.step_parts() group, pool and reduce: the parts of one table as
  one batch (the mono_pool_part arrays of the forward rows and of the gradients)."""

  def __init__(self, st, fwd, grads, grad_scale):
    self.st, self.fwd, self.grads, self.grad_scale = st, fwd, grads, grad_scale
    self.n_fids, self.device = fwd.n_fids, st.device
    self.bwd = None

  def build(self, N, D):
    return self.st.grouping.build_parts(self.st.table, self.fwd.arr, self.fwd.n, self.n_fids, N, D)

  def pool(self, rows, offs):
    self.st.dops.gather_pool_parts(self.st.table, rows, offs, self.fwd.arr, self.fwd.n, self.fwd.bf16)

  def take_grads(self):
    self.bwd = self.st._grad_parts(self.fwd, self.grads() if callable(self.grads) else self.grads)

  def reduce(self, out_rows):
    self.st.grouping.reduce_parts(self.st.table, self.bwd.arr, self.bwd.n, self.bwd.bf16, out_rows,
                                  grad_scale=self.grad_scale)

  def reduce_push(self, counts, window, region_off, dst_row_off):
    self.st.grouping.reduce_push_parts(self.st.table, self.bwd.arr, self.bwd.n, self.bwd.bf16, counts, window,
                                       region_off, dst_row_off, grad_scale=self.grad_scale)


class _PartsArr:
  """A parts call's mono_pool_part array with the tensors it points at (alive until the kernels have run)."""

  def __init__(self, table, parts, forward: bool):
    self.parts = list(parts)
    self.n = len(self.parts)
    self.arr, self.keep, self.rows = table._parts_arr(self.parts, forward=forward)
    self.bf16 = self.rows[0].dtype == torch.bfloat16
    self.n_fids = sum(int(self.arr[i].n_fids) for i in range(self.n))


class ShardedStep:
  """Sparse train step of ONE table on N GPUs, fast path: the batch is grouped once
  (distribution_ops.Grouping) and that grouping serves both the forward (dedup + bucket by owner + pooling
  offsets) and the backward (deterministic per-FID gradient reduction), around the same 3 + 1 all-to-alls
  as PartitionedHashTable.  Differences from the reference-layout path: the order of the distinct FIDs
  inside a shard bucket is the engine's, and no float atomics are used."""

  def __init__(self, table, name: str, dim: int, world: int, rank: int, device, group=None,
               exchange: Optional[str] = None):
    """exchange: "peer" = NVLink peer windows (fused lookup+send / reduce+send kernels, flag barriers,
    counts through /dev/shm; one node), "nccl" = all_to_all_single.  Default: env MONO_EXCHANGE, else
    "peer" on CUDA devices."""
    from . import distribution_ops
    import os
    self.table, self.name, self.dim, self.N, self.rank, self.group = table, name, dim, world, rank, group
    self.device = torch.device(device)
    self.dops = distribution_ops
    self.grouping = distribution_ops.Grouping(device)
    self.k = table.table_names.index(name)
    self.K = len(table.table_names)
    self.phases = _Phases(os.environ.get("MONO_TIMING", "0") in ("1", "2"))
    # default: the device-driven exchange (validated against ONE global oracle table: tests/test_gpu_distributed.py)
    self.exchange = exchange or os.environ.get("MONO_EXCHANGE", "direct" if torch.device(device).type == "cuda" else "nccl")
    if self.exchange not in ("peer", "nccl", "direct"):
      raise ValueError("exchange must be 'direct', 'peer' or 'nccl'")
    self.xstep = None        # exchange == "direct": the device-driven step (csrc/xstep.cu), two C calls per step
    self.cap_pair = 0
    # bulk rows / gradients: "push" = the producing kernel stores them into the consumer's window (fused
    # lookup+send / reduce+send; default), "pull" = the producer writes its own window and the consumer
    # copies it over with remote loads (one more pass over the rows)
    self.bulk = os.environ.get("MONO_PEER_BULK", "push")
    if self.bulk not in ("pull", "push"):
      raise ValueError("MONO_PEER_BULK must be 'pull' or 'push'")
    self.window = None
    self.hostx = HostCounts(world, rank, world + 1, group) if self.exchange == "peer" else None
    self.direct_steps = 0
    self.cap_rows = self.cap_recv = self._base_m = 0
    self.peer_steps = self.nccl_steps = 0

  # ---- NVLink window sizing: rows_in holds this rank's distinct rows (<= M), ids_in / grads_in what the
  # other ranks send it (about sum_r U_r / N).  A step that does not fit re-creates the window first; every
  # rank takes that decision from the same shared count matrix, so the re-creation is collective.
  def _make_window(self, max_m: int):
    D = self.dim
    if self.window is not None:
      torch.cuda.synchronize(self.device)
      self.window.close(self.group)
    self._base_m = max_m
    self.cap_rows = int(max_m * 1.25) + 1024
    self.cap_recv = int(max_m * 1.5) + 4096
    al = lambda x: (x + 255) & ~255
    self.off_ids = [0, al(self.cap_recv * 8)]
    self.off_rows = self.off_ids[1] + al(self.cap_recv * 8)
    self.off_grads = self.off_rows + al(self.cap_rows * D * 4)
    total = self.off_grads + al(self.cap_recv * D * 4)
    # pull mode: rows_out (owner side, what the requesters read) and grads_out (requester side)
    self.off_rows_out = total
    self.off_grads_out = self.off_rows_out + al(self.cap_recv * D * 4)
    total = self.off_grads_out + al(self.cap_rows * D * 4)
    self.window = self.dops.PeerWindow(self.device, self.N, self.rank, total, self.group)

  def _step_peer(self, src, req_time):
    """src: what is pooled and reduced (_FlatSource for step(), _PartsSource for step_parts())."""
    import numpy as np
    N, D, me, ph = self.N, self.dim, self.rank, self.phases
    ph.mark("start")
    uniq, offs, shard_sizes = src.build(N, D)                                         # 1
    ph.mark("f1_group")
    mat = self.hostx.exchange([src.n_fids] + list(shard_sizes))                       # 2 (host only)
    max_m, cnt = int(mat[:, 0].max()), mat[:, 1:]                                     # cnt[r][o]
    need_recv = int(cnt.sum(axis=0).max())
    if self.window is None or max_m > self.cap_rows or need_recv > self.cap_recv:      # same decision on every rank
      self._make_window(max(max_m, int(need_recv / 1.5) + 1, self._base_m))
    par = self.hostx.epoch & 1
    plan = exchange_plan(cnt, me)
    recv, my_seg, bucket_at = plan["recv"], plan["seg_at"], plan["bucket_at"]
    tot_recv = int(recv.sum())
    self.window.put(self.off_ids[par], my_seg * 8, uniq, bucket_at * 8, cnt[me] * 8)        # 3
    ph.fine("f3a_put_kernel")
    self.window.barrier()
    ph.mark("f3_put_ids")
    ids_in = self.window.view(self.off_ids[par], tot_recv, torch.int64)
    rows_in = self.window.view(self.off_rows, uniq.numel() * D, torch.float32)
    grads_in = self.window.view(self.off_grads, tot_recv * D, torch.float32)
    slot = self._slot(recv)
    if self.bulk == "push":
      self.table.lookup_push(self.name, ids_in, recv, self.window, self.off_rows, plan["rows_dst"])  # 4+5
      ph.fine("f5a_lookup_push_kernel")
      self.window.barrier()
      ph.mark("f5_lookup_push")
    else:
      rows_out = self.window.view(self.off_rows_out, tot_recv * D, torch.float32)     # 4 owner: rows of requester r at col_pre[r][me]
      self.table.fused_lookup(ids_in, slot, N, out=rows_out)
      ph.fine("f5a_owner_lookup")
      self.window.barrier()
      ph.fine("f5b_barrier")
      self.window.get(self.off_rows_out, my_seg * D * 4, rows_in, bucket_at * D * 4, cnt[me] * D * 4)  # 5 pull
      ph.mark("f5_lookup_pull")
    src.pool(rows_in, offs)                                                           # 6
    ph.mark("f6_gather_pool")
    src.take_grads()            # forward enqueued: the caller's dense tower / host round trip goes here
    if self.bulk == "push":
      src.reduce_push(cnt[me], self.window, self.off_grads, my_seg)                   # 7+8
      ph.fine("b8a_reduce_push_kernels")
      self.window.barrier()
      ph.mark("b8_reduce_push")
    else:
      grads_out = self.window.view(self.off_grads_out, uniq.numel() * D, torch.float32)
      src.reduce(grads_out)                                                           # 7 requester: bucketed by owner
      ph.fine("b8a_reduce")
      self.window.barrier()
      ph.fine("b8b_barrier")
      self.window.get(self.off_grads_out, plan["rows_dst"] * D * 4, grads_in, plan["recv_at"] * D * 4, recv * D * 4)  # 8 pull
      ph.mark("b8_reduce_pull")                                                        # 9
    _, _, id_off, emb_off = self.table.fused_offsets(slot, N)
    self.table.fused_apply_gradient(ids_in, ids_in, slot, grads_in, id_off, emb_off, 0, req_time, N)
    ph.mark("b9_owner_apply")
    ph.flush()
    self.peer_steps += 1
    return uniq.numel()

  # ---- exchange == "direct": nothing returns to the host inside a step (csrc/xstep.cu) ----------------------
  def _make_xstep(self, m: int):
    """(Re)create the fixed-capacity window and the step object; collective: the capacity is the largest batch of
    any rank (+ 25 % headroom), so every rank decides the same."""
    import ctypes as C
    lib = _lib.load()
    self.close_direct()
    cap = int(m)
    if self.N > 1:
      t = torch.tensor([cap], dtype=torch.int64, device=self.device)
      dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
      cap = int(t.item())
    cap = int(cap * 1.25) + 1024
    nbytes = lib.mono_xstep_window_bytes(self.N, cap, self.dim)
    if nbytes <= 0:
      raise ValueError("xstep: bad window geometry")
    self.window = self.dops.PeerWindow(self.device, self.N, self.rank, nbytes, self.group)
    h = C.c_void_p()
    _lib.check(lib.mono_xstep_create(self.table.handle, self.k, self.window._h, cap, C.byref(h)))
    self.xstep, self.cap_pair = h, cap

  def prepare(self, fids_next: torch.Tensor):
    """exchange == "direct": build the grouping of the NEXT batch on a side stream while the step in flight runs
    (no table dependency).  Pass the SAME tensor to the next step()."""
    import ctypes as C
    if self.exchange != "direct" or self.xstep is None:
      return
    f = fids_next.reshape(-1)
    if f.dtype != torch.int64 or not f.is_contiguous() or f.numel() > self.cap_pair or f.numel() == 0:
      return
    if getattr(self, "_side", None) is None:
      self._side = torch.cuda.Stream(device=self.device)
    self._side.wait_stream(torch.cuda.current_stream(self.device))   # fids_next may have been produced on the main stream
    _lib.check(_lib.load().mono_xstep_prepare(self.xstep, C.c_void_p(f.data_ptr()), f.numel(),
                                              C.c_void_p(self._side.cuda_stream)))
    self._keep_prep = f

  def close_direct(self):
    if self.xstep is not None:
      torch.cuda.synchronize(self.device)
      _lib.check(_lib.load().mono_xstep_destroy(self.xstep))
      self.xstep = None
    if self.window is not None:
      torch.cuda.synchronize(self.device)
      self.window.close(self.group)
      self.window = None

  def _step_direct(self, fids, pooled_grad, out, req_time, row_offsets, pooling, grad_scale):
    import ctypes as C
    lib = _lib.load()
    fids = fids.reshape(-1)
    if fids.dtype != torch.int64 or not fids.is_contiguous():
      fids = fids.to(torch.int64).contiguous()
    m = fids.numel()
    if self.xstep is None or m > self.cap_pair:
      # NOTE collective: every rank must come here in the same step (constant batch sizes never do after step 1)
      self._make_xstep(m)
    pool = _lib.POOLINGS[pooling]
    row_offsets, n_rows = _lib.row_offsets(row_offsets, m, self.device)
    ro = _lib.ptr(row_offsets)
    _lib.check(lib.mono_xstep_forward(self.xstep, _lib.ptr(fids), m, ro, n_rows, pool, _lib.ptr(out),
                                      out.stride(0) if out.dim() == 2 else self.dim, 0, _lib.stream(self.device)))
    if callable(pooled_grad):   # forward enqueued: the caller's dense tower / host round trip goes here
      pooled_grad = pooled_grad()
    if pooled_grad.dtype != torch.float32 or pooled_grad.stride(-1) != 1:
      pooled_grad = pooled_grad.to(torch.float32).contiguous()
    lr = self.table.configs[self.name].call_learning_rate_fns()
    lr_arr = (C.c_float * len(lr))(*lr)
    _lib.call("mono_xstep_backward", self.xstep, _lib.ptr(pooled_grad),
              pooled_grad.stride(0) if pooled_grad.dim() == 2 else self.dim, 0, ro, pool, lr_arr, int(req_time),
              scale=_lib.ptr(grad_scale), stream=_lib.stream(self.device))
    self._keep = (fids, pooled_grad, row_offsets, grad_scale)   # alive until the kernels have consumed them
    self.direct_steps += 1
    return 0

  # ---- several features of the table in one step (step_parts) ----------------------------------------------------
  def _grad_parts(self, fwd, grads) -> _PartsArr:
    """The gradient rows of step_parts, checked before any device work: one tensor per part, on the step's device with
    unit column stride and at least the part's [n_rows, col + width] (width: dim, max_seq_len * dim for "firstn"), all
    float32 or all bfloat16, with the rows the reduce reads (stride and col multiples of 4, 16-byte aligned float32 or
    8-byte aligned bfloat16 rows).  The forward's array with the gradient rows in place of the output rows."""
    import ctypes as C
    if isinstance(grads, torch.Tensor) or len(grads) != fwd.n:
      raise ValueError("step_parts: grads must be a list with one gradient tensor per part")
    dtypes = {g.dtype for g in grads if isinstance(g, torch.Tensor)}
    if len(dtypes) != 1 or not dtypes <= {torch.float32, torch.bfloat16}:
      raise ValueError("step_parts: the gradients must be tensors, all float32 or all bfloat16")
    gp = _PartsArr.__new__(_PartsArr)
    gp.parts, gp.n, gp.n_fids, gp.rows, gp.keep = fwd.parts, fwd.n, fwd.n_fids, list(grads), fwd.keep
    gp.bf16 = dtypes == {torch.bfloat16}
    gp.arr = (type(fwd.arr[0]) * len(fwd.arr))()
    C.memmove(gp.arr, fwd.arr, C.sizeof(fwd.arr))
    esz = 2 if gp.bf16 else 4
    for i, (p, g) in enumerate(zip(fwd.parts, grads)):
      a = gp.arr[i]
      width = self.dim * (p.max_seq_len if p.pooling == "firstn" else 1)
      if g.dim() != 2 or g.device != self.table.device or g.stride(1) != 1 or g.shape[0] < a.n_rows or \
          g.shape[1] < p.col + width:
        raise ValueError("step_parts: a gradient must be a 2-D tensor on the step's device with unit column stride and "
                         "at least the part's [n_rows, col + width]")
      if g.stride(0) % 4 or p.col % 4 or g.data_ptr() % (4 * esz):
        raise ValueError("step_parts: gradient rows need stride % 4 == 0, col % 4 == 0 and 16-byte (bfloat16: 8-byte) "
                         "aligned rows")
      a.rows_dev, a.stride = g.data_ptr(), g.stride(0)
    return gp

  def step_parts(self, parts, grads, req_time: int, grad_scale: Optional[torch.Tensor] = None):
    """One sparse train step over several features of this table: the many-feature form of step(), with the semantics
    of MultiHashTable.lookup_pool_parts / pool_backward_parts on the global table.

    parts: PoolPart list, every one naming this step's table (ValueError otherwise).  Each part's rows are its forward
    output ("sum", "mean" or "firstn" with max_seq_len, at any column and stride, so several parts may write disjoint
    columns of one tower tensor; a part without rows gets a new tensor), all float32 or all bfloat16.
    grads: one gradient tensor per part, with the part's shape and column, all float32 or all bfloat16 (independent of
    the forward's dtype), or a callable returning that list: it is called once the forward has been enqueued.
    grad_scale: as step()'s.

    The occurrences of all parts are ONE batch, part order then occurrence order, so each distinct FID gets one upsert,
    one timestamp bump, one admission-filter count and one optimizer step with the sum of its terms over all parts (a
    "mean" term divided by its row's n; a "firstn" occurrence at j >= max_seq_len a +0.0 term).  bfloat16 outputs are
    the float32 values rounded once; bfloat16 gradients are widened exactly first.  With one "sum" or "mean" part the
    step is bit for bit step() on that part.  Bad inputs raise before any device work and leave the table unchanged (a
    callable's list is checked when it returns, after the forward).  Returns each part's output rows, in part order."""
    parts = list(parts)
    if not parts:
      raise ValueError("step_parts needs at least one part")
    for p in parts:
      if p.slot != self.name:
        raise ValueError(f"step_parts: part of table {p.slot!r}, the step's table is {self.name!r}")
    scale_ptr(grad_scale, self.device, "grad_scale")
    fwd = _PartsArr(self.table, parts, forward=True)
    # the engine's own checks, here too: the direct exchange may re-create its window before its forward call
    for i in range(fwd.n):
      a = fwd.arr[i]
      if a.pooling == _lib.POOL_FIRSTN and a.n_rows * a.max_seq_len > (1 << 31):
        raise ValueError("step_parts: a 'firstn' part needs n_rows * max_seq_len <= 2^31")
    if fwd.n_fids >= (1 << 29):
      raise ValueError("step_parts: 2^29 occurrences or more in one step")
    bwd = None if callable(grads) else self._grad_parts(fwd, grads)
    if self.exchange == "direct":
      self._step_parts_direct(fwd, bwd, grads, req_time, grad_scale)
    else:
      src = _PartsSource(self, fwd, grads, grad_scale)
      if self.exchange == "peer":
        self._step_peer(src, req_time)
      else:
        self._step_nccl(src, req_time)
    return fwd.rows

  def _step_parts_direct(self, fwd, bwd, grads, req_time, grad_scale):
    import ctypes as C
    if self.xstep is None or fwd.n_fids > self.cap_pair:
      # NOTE collective, as in _step_direct
      self._make_xstep(fwd.n_fids)
    _lib.call("mono_xstep_forward_parts", self.xstep, fwd.arr, fwd.n, bf16=fwd.bf16, stream=_lib.stream(self.device))
    if bwd is None:   # forward enqueued: the caller's dense tower / host round trip goes here
      bwd = self._grad_parts(fwd, grads())
    lr = self.table.configs[self.name].call_learning_rate_fns()
    lr_arr = (C.c_float * len(lr))(*lr)
    _lib.call("mono_xstep_backward_parts", self.xstep, bwd.arr, bwd.n, lr_arr, int(req_time), bf16=bwd.bf16,
              scale=_lib.ptr(grad_scale), stream=_lib.stream(self.device))
    self._keep = (fwd, bwd, grad_scale)   # alive until the kernels have consumed them
    self.direct_steps += 1

  def _slot(self, per_shard):
    """per-(shard, table) sizes with only this table populated."""
    out = [0] * (self.N * self.K)
    for n in range(self.N):
      out[n * self.K + self.k] = int(per_shard[n])
    return out

  def step(self, fids: torch.Tensor, pooled_grad, out: torch.Tensor, req_time: int,
           row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
           grad_scale: Optional[torch.Tensor] = None):
    """One sparse train step.  `pooled_grad` is the gradient w.r.t. the pooled rows written to `out`, or a
    callable returning it: the callable runs once the forward has been enqueued (what produces the gradient —
    the dense tower, or a round trip of `out` to the host — belongs there).

    grad_scale (clip by global norm, ref: the deferred sparse scale of feature_utils.py:245-265): a one-element
    float32 tensor on the step's device.  The step is then bit for bit the step on pooled_grad multiplied by it in
    float32 first, in every exchange: the backward's per-FID reduce multiplies each term where it loads it
    (mono_xstep_backward_scaled, mono_grouping_reduce[_push]_scaled), so the owners apply sums of scaled terms.
    The value is read on the device when that reduce runs, not when step() is entered: a callable `pooled_grad`
    may fill the tensor on the current stream, e.g.
    `scale_buf.copy_(clip_ops.global_norm_scale(dense_grads + [g], clip_norm)[0])` before it returns g."""
    scale_ptr(grad_scale, self.device, "grad_scale")
    if self.exchange == "direct":
      return self._step_direct(fids, pooled_grad, out, req_time, row_offsets, pooling, grad_scale)
    src = _FlatSource(self, fids, pooled_grad, out, row_offsets, pooling, grad_scale)
    if self.exchange == "peer":
      return self._step_peer(src, req_time)
    return self._step_nccl(src, req_time)

  def _step_nccl(self, src, req_time):
    N, D, dev, ph = self.N, self.dim, src.device, self.phases
    self.nccl_steps += 1
    ph.mark("start")
    uniq, offs, shard_sizes = src.build(N, D)                                       # 1
    ph.mark("f1_group")
    send_cnt = torch.tensor(shard_sizes, dtype=torch.int64, device=dev)               # 2
    recv_cnt = torch.empty_like(send_cnt)
    _a2a(recv_cnt, send_cnt, [1] * N, [1] * N, self.group)
    recv_sizes = [int(x) for x in recv_cnt.cpu().tolist()]
    ph.mark("f2_a2a_counts")
    recv_ids = torch.empty(sum(recv_sizes), dtype=torch.int64, device=dev)            # 3
    _a2a(recv_ids, uniq, recv_sizes, shard_sizes, self.group)
    ph.mark("f3_a2a_ids")
    rows = self.table.fused_lookup(recv_ids, self._slot(recv_sizes), N)[0]            # 4
    ph.mark("f4_owner_lookup")
    recv_rows = torch.empty(uniq.numel() * D, dtype=torch.float32, device=dev)        # 5
    _a2a(recv_rows, rows, [s * D for s in shard_sizes], [s * D for s in recv_sizes], self.group)
    ph.mark("f5_a2a_rows")
    src.pool(recv_rows, offs)                                                         # 6
    ph.mark("f6_gather_pool")
    src.take_grads()
    grad_rows = torch.empty(uniq.numel() * D, dtype=torch.float32, device=dev)        # 7
    src.reduce(grad_rows)
    ph.mark("b7_reduce_grads")
    owner_grads = torch.empty(sum(recv_sizes) * D, dtype=torch.float32, device=dev)   # 8
    _a2a(owner_grads, grad_rows, [s * D for s in recv_sizes], [s * D for s in shard_sizes], self.group)
    ph.mark("b8_a2a_grads")
    slot = self._slot(recv_sizes)                                                     # 9
    _, _, id_off, emb_off = self.table.fused_offsets(slot, N)
    self.table.fused_apply_gradient(recv_ids, recv_ids, slot, owner_grads, id_off, emb_off, 0, req_time, N)
    ph.mark("b9_owner_apply")
    ph.flush()
    return uniq.numel()


class DistributedMultiTypeHashTable:
  """The async parameter-server (PS) table on the raw API — ref: DistributedMultiTypeHashTable, NT/distributed_ps.py
  :192-516, the table distributed_ps_factory.create_native_multi_hash_table builds for num_ps > 0.

  table_factory(i, slot_to_config) -> MultiHashTable makes PS i's table; the PS tables may sit on any CUDA devices and
  every table must hold the same tables with the same dims.  A unique key k lives on PS floormod(k, num_ps)
  (tf.math.floormod, so key -1 with 3 PS goes to PS 2).  The worker side runs on the device of PS 0's table: dedup
  of the keys with their occurrence offsets (unique_key_with_value_and_offset), the split by PS
  (ragged_split_by_indices), and the fill of every PS's rows into the occurrences (fill_with_offset_map) or the sum of
  the occurrence gradients per unique key (fill_with_offset_map_gradient).  Ids, rows and gradients cross devices
  with plain torch copies.

  lookup and apply_gradients make one host synchronisation each on the worker side: the split's per-PS row splits,
  which the PS tables' raw calls take on the host.

  transfer_float16 (ref: distributed_ps.py:201,207,392-410,539-549): rows and gradients cross between the servers and
  the worker as fp16.  Each server's lookup writes its rows rounded to fp16 and the worker's fill widens them; the
  worker's gradient sums are rounded to fp16 and each server widens them (exactly) before its apply.  So a looked-up
  value is f32(f16(row)) and a server applies f32(f16(sum)), which is what the reference's per-slot path with the
  casts computes.  assign, assign_add and reinitialize send fp32, as in the reference."""

  def __init__(self, num_ps: int, slot_to_config: Dict, table_factory, transfer_float16: bool = False):
    if num_ps < 1:
      raise ValueError("num_ps must be >= 1")
    self._num_ps = int(num_ps)
    self._transfer_dtype = torch.float16 if transfer_float16 else torch.float32
    self._slot_to_config = slot_to_config
    self._tables = [table_factory(i, slot_to_config) for i in range(self._num_ps)]
    t0 = self._tables[0]
    for t in self._tables[1:]:
      if tuple(t.table_names) != tuple(t0.table_names) or tuple(t.get_table_dim_sizes()) != tuple(
          t0.get_table_dim_sizes()):
        raise ValueError("every PS table must hold the same tables with the same dims")

  @property
  def tables(self):
    return self._tables

  def get_table_dim_sizes(self):
    """ref: distributed_ps.py get_table_dim_sizes: PS 0's table's dims, tables in sorted-name order."""
    return self._tables[0].get_table_dim_sizes()

  @property
  def transfer_float16(self) -> bool:
    return self._transfer_dtype == torch.float16

  def as_op(self, *args, **kwargs):
    return self

  def _unique_split(self, slot_to_id, generate_buffer):
    from . import distribution_ops as dops
    t0 = self._tables[0]
    ids, splits = t0.get_ragged_id(slot_to_id)
    dims = t0.get_table_dim_sizes()
    res = dops.unique_key_with_value_and_offset(ids, splits, dims, generate_buffer, sync=False)
    uniq, uniq_split = res.unique_key
    index = torch.remainder(uniq, self._num_ps)  # tf.math.floormod; the entries past U are ignored by the split
    sp = dops.ragged_split_by_indices(index, uniq, uniq_split, self._num_ps, sync=True)  # the one synchronisation
    U = sum(r[-1] for r in sp.row_splits_host)
    return splits, dims, res, sp, U

  def lookup(self, slot_to_id: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """ref: distributed_ps.py:282-338 (raw API path): every slot's embeddings [n, dim], misses as the tables give them."""
    from . import distribution_ops as dops
    splits, dims, res, sp, U = self._unique_split(slot_to_id, True)
    buf = res.value_buffer
    for i, table in enumerate(self._tables):
      (vals, _), rs = sp.splits[i], sp.row_splits_host[i]
      flat = table.raw_lookup(vals.to(table.device), rs, dtype=self._transfer_dtype)
      dops.fill_with_offset_map(sp.pos[i], rs, flat.to(buf.device), res.value_offset, buf, dims, num_unique=U,
                                sync=False)
    emb = self._tables[0].get_embeddings(splits, buf)
    return {k: v for k, v in emb.items() if k in slot_to_id}

  def apply_gradients(self, slot_to_id_and_grad: Dict[str, Tuple[torch.Tensor, torch.Tensor]], global_step: int = 0,
                      req_time: int = 0) -> "DistributedMultiTypeHashTable":
    """ref: distributed_ps.py:481-514 (raw API path): the occurrence gradients summed per unique key in occurrence
    order, then each PS's raw_apply_gradients on its keys."""
    from . import distribution_ops as dops
    slot_to_id = {k: v[0] for k, v in slot_to_id_and_grad.items()}
    splits, dims, res, sp, U = self._unique_split(slot_to_id, False)
    flat_grad = self._tables[0].get_flat_value({k: v[1] for k, v in slot_to_id_and_grad.items()})
    for i, table in enumerate(self._tables):
      (vals, _), rs = sp.splits[i], sp.row_splits_host[i]
      g = dops.fill_with_offset_map_gradient(sp.pos[i], rs, flat_grad, res.value_offset, dims, num_unique=U,
                                             sync=False, dtype=self._transfer_dtype)
      g = g.to(table.device)
      if self.transfer_float16:
        g = g.float()  # the server's exact widening (the reference's CastToFloat32 on the PS)
      table.raw_apply_gradients(vals.to(table.device), rs, g, global_step=global_step, req_time=req_time)
    return self

  def _update(self, method_name: str, slot_to_id_and_value):
    """ref: distributed_ps.py:430-451: every slot's ids and values split by floormod(id, num_ps)."""
    from . import distribution_ops as dops
    per_ps = [dict() for _ in range(self._num_ps)]
    for slot, (ids, value) in slot_to_id_and_value.items():
      ids = ids.reshape(-1).to(torch.int64)
      index = torch.remainder(ids, self._num_ps)
      split_ids = dops.split_by_indices(index, ids, self._num_ps)
      split_values = dops.split_by_indices(index, value.to(ids.device), self._num_ps)
      for i in range(self._num_ps):
        per_ps[i][slot] = (split_ids[i], split_values[i])
    for i, table in enumerate(self._tables):
      dev = table.device
      getattr(table, method_name)({k: (a.to(dev), b.to(dev)) for k, (a, b) in per_ps[i].items()})
    return self

  def assign(self, slot_to_id_and_value: Dict[str, Tuple[torch.Tensor, torch.Tensor]]):
    """ref: distributed_ps.py:453-456."""
    return self._update("assign", slot_to_id_and_value)

  def assign_add(self, slot_to_id_and_value: Dict[str, Tuple[torch.Tensor, torch.Tensor]]):
    """ref: distributed_ps.py:458-461."""
    return self._update("assign_add", slot_to_id_and_value)

  def reinitialize(self, slot: str, ids: torch.Tensor):
    """ref: distributed_ps.py:463-476: the ids split by PS, each PS's status concatenated in PS order (so the status
    follows the split, not the input order)."""
    from . import distribution_ops as dops
    ids = ids.reshape(-1).to(torch.int64)
    index = torch.remainder(ids, self._num_ps)
    split_ids = dops.split_by_indices(index, ids, self._num_ps)
    status = []
    for i, table in enumerate(self._tables):
      _, st = table.reinitialize(slot, split_ids[i].to(table.device))
      status.append(st.to(ids.device))
    return self, torch.cat(status)


class PSLayoutContext:
  """What PartitionedHashTablePS.apply_gradients needs from its lookup (ref: the `__sharding_sparse_fids__*` entries
  of the auxiliary bundle): the version-5 sharding outputs, every server's ids and host row splits over its tables,
  the float size of every (table, server) list and the batch size."""
  __slots__ = ("sharding", "server_ids", "server_splits", "emb_sizes", "batch_size")


class PartitionedHashTablePS:
  """PartitionedHashTable's parameter-server mode with the fused layout — ref: NT/distributed_ps.py:581-2001 without
  enable_gpu_emb, the table a job with enable_fused_layout=True and num_ps > 0 builds (NT/cpu_training.py:713-741).
  The GPU all-to-all mode is PartitionedHashTable above; the two share no step logic.

  table_factory(i, slot_to_config) -> MultiHashTable makes server i's table (any CUDA device; every server holds the
  same tables, named like the features' tables).  feature_table / feature_dims_sum / shared_features describe the
  features as sharding_sparse_fids takes them, and every feature's dims_sum must be its table's dim.  tasks are
  fused_embedding_to_layout's (nfl_idx = the feature's index in sorted-name order) and out_shapes the layout tensors'
  shapes per sample: each lookup allocates [batch_size, *shape].  Every task's out_row_stride must fit in its tensor's
  per-sample elements.  A FID lives on server (uint64)fid % num_ps, the sharding's shard.

  lookup: sharding_sparse_fids(version=5), one raw_lookup per server over its (table, server) lists, then
  fused_embedding_to_layout over the K*N lists (index table_index * num_ps + server).  apply_gradients: the layout
  gradient into one zeroed buffer laid out server after server, then one raw_apply_gradients per server on its slab.
  Both calls synchronise with the host: lookup reads the sharding's list lengths back (the servers' raw calls take
  them on the host), the layout forward and gradient launchers wait for their staged task tables, and the servers'
  raw table calls may wait as well (e.g. for rounds of duplicate ids in an apply).
  unique: the sharding's (each (feature, server) list keeps its distinct FIDs, or every occurrence).

  transfer_float16 (ref: distributed_ps.py:912-927, 1425-1440): each server's lookup writes its rows rounded to fp16
  and the layout forward reads them as they are, widening where it loads (no cast pass on the worker); the fp32 layout
  gradient is rounded once to fp16 after its atomics have completed, and each server widens its slab exactly before
  its apply.  So a looked-up element is f32(f16(row)) and a server applies f32(f16(sum)).  Rows and gradients cross
  devices with plain torch copies."""

  def __init__(self, num_ps: int, slot_to_config: Dict, table_factory, feature_table: Dict[str, str],
               feature_dims_sum: Dict[str, int], tasks, out_shapes, shared_features: Sequence[str] = (), *,
               unique: bool = True, transfer_float16: bool = False):
    if num_ps < 1:
      raise ValueError("num_ps must be >= 1")
    self._num_ps = int(num_ps)
    self._transfer_dtype = torch.float16 if transfer_float16 else torch.float32
    self._tables = [table_factory(i, slot_to_config) for i in range(self._num_ps)]
    t0 = self._tables[0]
    for t in self._tables[1:]:
      if tuple(t.table_names) != tuple(t0.table_names) or tuple(t.get_table_dim_sizes()) != tuple(
          t0.get_table_dim_sizes()):
        raise ValueError("every PS table must hold the same tables with the same dims")
    dims = dict(zip(t0.table_names, t0.get_table_dim_sizes()))
    for f, t in feature_table.items():
      if t not in dims:
        raise ValueError(f"feature {f}'s table {t} is not a table of the servers")
      if int(feature_dims_sum[f]) != dims[t]:
        raise ValueError(f"feature {f}: dims_sum {feature_dims_sum[f]} is not table {t}'s dim {dims[t]}")
    self._feature_table = dict(feature_table)
    self._dims_sum = {f: int(feature_dims_sum[f]) for f in feature_table}
    self._shared = tuple(shared_features)
    self._tasks = list(tasks)
    self._out_shapes = [tuple(int(x) for x in s) for s in out_shapes]
    for t in self._tasks:
      if not 0 <= t.out_tensor < len(self._out_shapes):
        raise ValueError(f"task out_tensor {t.out_tensor} outside the {len(self._out_shapes)} layout tensors")
      per_sample = 1
      for x in self._out_shapes[t.out_tensor]:
        per_sample *= x
      if t.out_row_stride > per_sample:
        raise ValueError(f"task out_row_stride {t.out_row_stride} exceeds layout tensor {t.out_tensor}'s "
                         f"{per_sample} elements per sample")
    self._unique = bool(unique)
    self._dims = dims

  @property
  def tables(self):
    return self._tables

  @property
  def transfer_float16(self) -> bool:
    return self._transfer_dtype == torch.float16

  def lookup(self, features: Dict[str, Tuple[torch.Tensor, torch.Tensor]], dtype: torch.dtype = torch.float32,
             batch_size: Optional[int] = None):
    """features[name] = (fids int64, row_splits int64[rows + 1]) on the worker's CUDA device, every configured
    feature present.  Returns (the layout tensors, float32 or bfloat16, ctx)."""
    from . import distribution_ops as dops
    if set(features) != set(self._feature_table):
      raise ValueError(f"features must be exactly {sorted(self._feature_table)}, not {sorted(features)}")
    if dtype not in (torch.float32, torch.bfloat16):
      raise ValueError(f"dtype must be torch.float32 or torch.bfloat16, not {dtype}")
    N = self._num_ps
    names = sorted(features)
    B = dops._v5_batch_size(features, names, set(self._shared), batch_size)
    sh = dops.sharding_sparse_fids(features, self._feature_table, self._dims_sum, N, self._shared, unique=self._unique,
                                   sync=True, version=5, batch_size=B)   # the one synchronisation
    dev = sh["fid_offset"].device
    k_of = {t: k for k, t in enumerate(sh["table_names"])}
    lens = [t.numel() for t in sh["fid_list"]]                          # [k * N + i], host ints
    fused = sh["fid_list_fused"]                                         # server-major, table-minor
    embs = [None] * (len(k_of) * N)
    server_ids, server_splits, emb_sizes = [], [], [0] * (len(k_of) * N)
    start = 0
    for i, table in enumerate(self._tables):
      split = [0]
      for name in table.table_names:
        split.append(split[-1] + (lens[k_of[name] * N + i] if name in k_of else 0))
      ids = fused[start:start + split[-1]].to(table.device)
      start += split[-1]
      flat = table.raw_lookup(ids, split, dtype=self._transfer_dtype).to(dev)
      off = 0
      for name in table.table_names:
        if name in k_of:
          k = k_of[name]
          n = lens[k * N + i] * self._dims[name]
          embs[k * N + i], emb_sizes[k * N + i] = flat[off:off + n], n
          off += n
      server_ids.append(ids)
      server_splits.append(split)
    layouts = dops.fused_embedding_to_layout(embs, [1] * len(embs), sh["fid_offset"], sh["feature_offset"],
                                             sh["nfl_offset"], B, self._tasks,
                                             [(B,) + s for s in self._out_shapes], dtype=dtype)
    ctx = PSLayoutContext()
    ctx.sharding, ctx.server_ids, ctx.server_splits, ctx.emb_sizes, ctx.batch_size = (sh, server_ids, server_splits,
                                                                                       emb_sizes, B)
    return layouts, ctx

  def apply_gradients(self, ctx: PSLayoutContext, layout_grads: Sequence[torch.Tensor], global_step: int = 0,
                      req_time: int = 0, layout_tensors_grad_scale: Optional[torch.Tensor] = None):
    """layout_grads: the gradients of lookup's layout tensors (all float32 or all bfloat16).
    layout_tensors_grad_scale: as fused_embedding_to_layout_grad's (e.g. clip_ops.global_norm_scale's scale)."""
    from . import distribution_ops as dops
    sh, N = ctx.sharding, self._num_ps
    dev = sh["fid_offset"].device
    K = len(ctx.emb_sizes) // N
    buf = torch.zeros(sum(ctx.emb_sizes), dtype=torch.float32, device=dev)
    views, bounds, off = [None] * (K * N), [], 0
    for i in range(N):                                                    # server-major: one slab per server
      lo = off
      for k in range(K):
        views[k * N + i] = buf[off:off + ctx.emb_sizes[k * N + i]]
        off += ctx.emb_sizes[k * N + i]
      bounds.append((lo, off))
    dops.fused_embedding_to_layout_grad(ctx.emb_sizes, [1] * (K * N), sh["fid_offset"], sh["feature_offset"],
                                        sh["nfl_offset"], ctx.batch_size, self._tasks, layout_grads,
                                        layout_tensors_grad_scale, out=views)
    send = dops.round_to_f16(buf) if self.transfer_float16 else buf
    for i, table in enumerate(self._tables):
      lo, hi = bounds[i]
      g = send[lo:hi].to(table.device)
      if self.transfer_float16:
        g = g.float()  # the server's exact widening (the reference's CastToFloat32 on the PS)
      table.raw_apply_gradients(ctx.server_ids[i], ctx.server_splits[i], g, global_step=global_step,
                                req_time=req_time)
    return self

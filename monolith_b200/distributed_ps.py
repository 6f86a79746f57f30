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

  def gather_pool_grad_into(self, grad_buf, pooled_grad, offs, dim, row_offsets, pooling):
    """Fills grad_buf (pre-zeroed, shared by all tables of the step).  dim % 4 == 0 and <= 128: the
    deterministic sort-based scatter; otherwise the float-atomic kernel (like the reference GPU path).
    pooled_grad is float32 or bfloat16 (the bf16 kernels widen it exactly); grad_buf is float32."""
    if self.vec_ok and dim <= 128:
      self.dops.scatter_grad_rows(pooled_grad, offs, dim, grad_buf, row_offsets, pooling)
      return
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    n_rows = offs.numel() if row_offsets is None else row_offsets.numel() - 1
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    ro = None if row_offsets is None else C.c_void_p(row_offsets.data_ptr())
    fn = lib.mono_gather_pool_grad_bf16 if pooled_grad.dtype == torch.bfloat16 else lib.mono_gather_pool_grad
    _lib.check(fn(pooled_grad.device.index, C.c_void_p(pooled_grad.data_ptr()), pooled_grad.stride(0), 0,
                  C.c_void_p(offs.data_ptr()), ro, n_rows, dim, pool, C.c_void_p(grad_buf.data_ptr()),
                  C.c_void_p(torch.cuda.current_stream(pooled_grad.device).cuda_stream)))

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

  def apply_gradients(self, ctx: StepContext, pooled_grads: Dict[str, torch.Tensor], req_time: int = 0):
    """Backward steps 7-9.  pooled_grads are float32 or bfloat16; the exchanged row gradients are float32."""
    be, N = self.backend, self.N
    some = next(iter(pooled_grads.values()))
    ph = self.phases
    ph.mark("bwd_start")
    # 7 scatter pooled grads to the unique rows, in the layout of the received row buffer
    grad_rows = be.zeros(sum(ctx.recv_row_splits), some)
    for k, name in enumerate(self.names):
      if name not in pooled_grads:
        continue
      lo, hi = ctx.occ_splits[k]
      be.gather_pool_grad_into(grad_rows, pooled_grads[name], ctx.offs[lo:hi], self.dims[k], ctx.row_offsets.get(name),
                               ctx.poolings.get(name, "sum"))
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

  def _step_peer(self, fids, pooled_grad, out, req_time, row_offsets, pooling):
    import numpy as np
    N, D, me, ph = self.N, self.dim, self.rank, self.phases
    ph.mark("start")
    uniq, offs, shard_sizes = self.grouping.build(fids, N, D)                         # 1
    ph.mark("f1_group")
    mat = self.hostx.exchange([fids.numel()] + list(shard_sizes))                     # 2 (host only)
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
    self.dops.gather_pool(rows_in, offs, D, row_offsets, pooling, out=out)            # 6
    ph.mark("f6_gather_pool")
    if callable(pooled_grad):   # forward enqueued: the caller's dense tower / host round trip goes here
      pooled_grad = pooled_grad()
    if self.bulk == "push":
      self.grouping.reduce_push(pooled_grad, cnt[me], self.window, self.off_grads, my_seg, row_offsets, pooling)  # 7+8
      ph.fine("b8a_reduce_push_kernels")
      self.window.barrier()
      ph.mark("b8_reduce_push")
    else:
      grads_out = self.window.view(self.off_grads_out, uniq.numel() * D, torch.float32)
      self.grouping.reduce(pooled_grad, grads_out, row_offsets, pooling)              # 7 requester: bucketed by owner
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
    from . import _lib
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
    from . import _lib
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
    from . import _lib
    if self.xstep is not None:
      torch.cuda.synchronize(self.device)
      _lib.check(_lib.load().mono_xstep_destroy(self.xstep))
      self.xstep = None
    if self.window is not None:
      torch.cuda.synchronize(self.device)
      self.window.close(self.group)
      self.window = None

  def _step_direct(self, fids, pooled_grad, out, req_time, row_offsets, pooling):
    import ctypes as C
    from . import _lib
    lib = _lib.load()
    fids = fids.reshape(-1)
    if fids.dtype != torch.int64 or not fids.is_contiguous():
      fids = fids.to(torch.int64).contiguous()
    m = fids.numel()
    if self.xstep is None or m > self.cap_pair:
      # NOTE collective: every rank must come here in the same step (constant batch sizes never do after step 1)
      self._make_xstep(m)
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    ro = None
    n_rows = m
    if row_offsets is not None:
      row_offsets = row_offsets.to(device=self.device, dtype=torch.int32).contiguous()
      ro, n_rows = C.c_void_p(row_offsets.data_ptr()), row_offsets.numel() - 1
    stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
    _lib.check(lib.mono_xstep_forward(self.xstep, C.c_void_p(fids.data_ptr()), m, ro, n_rows, pool,
                                      C.c_void_p(out.data_ptr()), out.stride(0) if out.dim() == 2 else self.dim, 0, stream))
    if callable(pooled_grad):   # forward enqueued: the caller's dense tower / host round trip goes here
      pooled_grad = pooled_grad()
    if pooled_grad.dtype != torch.float32 or pooled_grad.stride(-1) != 1:
      pooled_grad = pooled_grad.to(torch.float32).contiguous()
    lr = self.table.configs[self.name].call_learning_rate_fns()
    lr_arr = (C.c_float * len(lr))(*lr)
    stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
    _lib.check(lib.mono_xstep_backward(self.xstep, C.c_void_p(pooled_grad.data_ptr()),
                                       pooled_grad.stride(0) if pooled_grad.dim() == 2 else self.dim, 0, ro, pool, lr_arr,
                                       int(req_time), stream))
    self._keep = (fids, pooled_grad, row_offsets)   # alive until the kernels have consumed them
    self.direct_steps += 1
    return 0

  def _slot(self, per_shard):
    """per-(shard, table) sizes with only this table populated."""
    out = [0] * (self.N * self.K)
    for n in range(self.N):
      out[n * self.K + self.k] = int(per_shard[n])
    return out

  def step(self, fids: torch.Tensor, pooled_grad, out: torch.Tensor, req_time: int,
           row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum"):
    """One sparse train step.  `pooled_grad` is the gradient w.r.t. the pooled rows written to `out`, or a
    callable returning it: the callable runs once the forward has been enqueued (what produces the gradient —
    the dense tower, or a round trip of `out` to the host — belongs there)."""
    if self.exchange == "direct":
      return self._step_direct(fids, pooled_grad, out, req_time, row_offsets, pooling)
    if self.exchange == "peer":
      return self._step_peer(fids, pooled_grad, out, req_time, row_offsets, pooling)
    N, D, dev, ph = self.N, self.dim, fids.device, self.phases
    self.nccl_steps += 1
    ph.mark("start")
    uniq, offs, shard_sizes = self.grouping.build(fids, N, D)                       # 1
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
    self.dops.gather_pool(recv_rows, offs, D, row_offsets, pooling, out=out)          # 6
    ph.mark("f6_gather_pool")
    if callable(pooled_grad):
      pooled_grad = pooled_grad()
    grad_rows = torch.empty(uniq.numel() * D, dtype=torch.float32, device=dev)        # 7
    self.grouping.reduce(pooled_grad, grad_rows, row_offsets, pooling)
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

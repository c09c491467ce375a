"""Work split for multi-GPU runs: windows are independent units, so a ZMW batch is sharded across
ranks with no data-path collective.

Shards are ZMW-granular (all windows of a molecule stay on one rank so `stitch_to_fastq`, which
runs per ZMW after the model -- quick_inference.py:721-736 -- needs no cross-rank merge) and assigned
round-robin in order of first appearance.  Only counters are ever reduced across ranks.
"""
from __future__ import annotations

from typing import Dict, List, Sequence


def shard_by_zmw(molecule_names: Sequence[str], world_size: int) -> List[List[int]]:
  """Window indices per rank; molecules are dealt round-robin in order of first appearance."""
  if world_size <= 0:
    raise ValueError("world_size must be positive")
  owner: Dict[str, int] = {}
  shards: List[List[int]] = [[] for _ in range(world_size)]
  for i, name in enumerate(molecule_names):
    if name not in owner:
      owner[name] = len(owner) % world_size
    shards[owner[name]].append(i)
  return shards


def shard_range(n_items: int, rank: int, world_size: int) -> range:
  """Contiguous, balanced split of n independent items (used for synthetic window batches)."""
  base, rem = divmod(n_items, world_size)
  start = rank * base + min(rank, rem)
  return range(start, start + base + (1 if rank < rem else 0))


def reduce_counters(counters: Dict[str, int], group=None) -> Dict[str, int]:
  """SUM-all-reduce outcome counters across ranks (the only collective on the path)."""
  import torch
  import torch.distributed as dist
  if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
    return dict(counters)
  keys = sorted(counters)
  dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
  t = torch.tensor([counters[k] for k in keys], dtype=torch.int64, device=dev)
  dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
  return {k: int(v) for k, v in zip(keys, t.tolist())}


class ScatterFeeder:
  """BASELINE configs[3]: ONE reader rank holds the packed rows of a whole step and deals one chunk to every rank
  (itself included) -- grouped point-to-point sends / receives, i.e. ncclGroupStart; ncclSend(chunk_r -> r) for all r;
  ncclRecv; ncclGroupEnd -- and collects every rank's base / quality characters the same way.

  Double-buffered: `scatter(step)` posts the transfers of step k+1 asynchronously while the caller scores step k out of
  the other buffer; `wait()` blocks the host until the posted transfers have landed (the engine runs on its own
  stream, so completion is awaited on the host before the buffer's address is handed to dcb_submit_packed).

  Tensors are torch uint8 tensors on the communication device ("cuda" with NCCL, "cpu" with gloo for the tests);
  chunk bytes per rank = chunk_windows * packed_window_bytes, result bytes per rank = 2 * chunk_windows * L.
  """

  def __init__(self, chunk_bytes: int, result_bytes: int, reader: int = 0, device=None, group=None):
    import torch
    import torch.distributed as dist
    self.torch, self.dist, self.group, self.reader = torch, dist, group, reader
    self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
    if device is None:
      device = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    self.device = device
    self.inbox = [torch.empty(chunk_bytes, dtype=torch.uint8, device=device) for _ in range(2)]   # my chunk, 2 buffers
    self.results = torch.empty(result_bytes, dtype=torch.uint8, device=device)                    # my outputs
    self.gathered = (torch.empty((self.world, result_bytes), dtype=torch.uint8, device=device)
                     if self.rank == reader else None)
    self._pending = []

  def scatter(self, buf: int, step_rows=None) -> None:
    """Post the transfer of one step: on the reader, `step_rows` is a uint8 tensor [world, chunk_bytes] (device
    resident); every rank receives its chunk into inbox[buf]."""
    dist, ops = self.dist, []
    if self.rank == self.reader:
      for r in range(self.world):
        if r == self.rank:
          self.inbox[buf].copy_(step_rows[r], non_blocking=True)
        else:
          ops.append(dist.P2POp(dist.isend, step_rows[r], r, self.group))
    else:
      ops.append(dist.P2POp(dist.irecv, self.inbox[buf], self.reader, self.group))
    self._pending += dist.batch_isend_irecv(ops) if ops else []

  def gather(self) -> None:
    """Post the collection of every rank's `results` on the reader (row r of `gathered`)."""
    dist, ops = self.dist, []
    if self.rank == self.reader:
      for r in range(self.world):
        if r == self.rank:
          self.gathered[r].copy_(self.results, non_blocking=True)
        else:
          ops.append(dist.P2POp(dist.irecv, self.gathered[r], r, self.group))
    else:
      ops.append(dist.P2POp(dist.isend, self.results, self.reader, self.group))
    self._pending += dist.batch_isend_irecv(ops) if ops else []

  def wait(self) -> None:
    """Host-blocking: every posted transfer has completed (and, on CUDA, its stream work has finished)."""
    for w in self._pending:
      w.wait()
    self._pending = []
    if str(self.device).startswith("cuda"):
      self.torch.cuda.current_stream().synchronize()

"""Data-parallel plumbing of the hot path (SURVEY.md §8e).

Lists are independent, the scorer parameters are shared: the batch is sharded by
lists across ranks (one process per GPU) and the ONLY data-path collective per
training step is one all-reduce(SUM) of the flat fp32 scorer gradient, with the
1/num_replicas factor of the reference (extension/task.py:256-262) folded into
the optimizer kernel.  Metric means all-reduce their (sum v*w, sum w) state.
Works on any backend: NCCL over NVLink on H100 boxes, gloo in the CPU tests.
"""
import torch
import torch.distributed as dist


def is_distributed():
  return dist.is_available() and dist.is_initialized()


def world_size(group=None):
  return dist.get_world_size(group) if is_distributed() else 1


def rank(group=None):
  return dist.get_rank(group) if is_distributed() else 0


def all_reduce_sum_(tensor, group=None):
  """In-place SUM all-reduce of a flat buffer (no-op for a single process)."""
  if world_size(group) > 1:
    dist.all_reduce(tensor, op=dist.ReduceOp.SUM, group=group)
  return tensor


def broadcast_(tensor, src=0, group=None):
  """Makes every replica start from rank `src`'s parameters."""
  if world_size(group) > 1:
    dist.broadcast(tensor, src=src, group=group)
  return tensor


def replica_grad_scale(group=None):
  """Factor applied to the summed gradient: 1 / num_replicas_in_sync."""
  return 1.0 / world_size(group)


def shard_lists(num_lists, group=None):
  """Contiguous, equal shard of the batch dimension for this rank (the reference
  semantics need equal local batches for SUM_OVER_BATCH_SIZE to equal the global
  loss, SURVEY.md §5)."""
  w, r = world_size(group), rank(group)
  if num_lists % w != 0:
    raise ValueError('batch of %d lists does not split evenly over %d replicas' %
                     (num_lists, w))
  per = num_lists // w
  return slice(r * per, (r + 1) * per)


def cross_replica_list_weights(raw, kind, group=None):
  """Per-list metric weights with the batch-average rule of
  `_per_example_weights_to_per_list_weights` (metrics_impl.py:63-119) taken over the
  GLOBAL batch: lists without relevant items get the average weight of ALL replicas'
  lists, as a single device stepping the concatenated batch would compute it.  (Under
  tf.distribute the reference evaluates the rule per replica — that is what the metric
  kernel's own finalise pass does; this is the opt-in single-device-equivalent form.)

  raw [B, 5] = {sum w, sum w*gain, sum gain, sum w*rel, sum rel} per list, as written by
  tfr_rank_metrics; kind 'ndcg' uses the gain columns, 'mrr' the relevance columns.
  Costs one 2-float all-reduce."""
  m = 0 if kind == 'ndcg' else 1
  sum_w, wr, r = raw[:, 0], raw[:, 1 + 2 * m], raw[:, 2 + 2 * m]
  per = torch.where(r != 0, wr / torch.where(r != 0, r, torch.ones_like(r)),
                    torch.zeros_like(r))
  nz = (sum_w > 0) & (r > 0)
  stats = torch.stack([per.sum(), nz.to(per.dtype).sum()])
  all_reduce_sum_(stats, group)
  avg = torch.where(stats[1] > 0, stats[0] / torch.clamp(stats[1], min=1.0),
                    torch.ones_like(stats[0]))
  return torch.where(sum_w > 0, torch.where(r > 0, per, avg.expand_as(per)),
                     torch.zeros_like(per))


def bind_to_gpu_numa_node(device_index):
  """Pins this process (and therefore the pinned host buffers it allocates afterwards:
  first-touch) to the CPUs of the NUMA node the GPU hangs off.  With 8 ranks on a
  two-socket box, unbound ranks push half of their H2D traffic across the socket link.
  Returns {'node': k, 'cpus': n} or None when the topology cannot be read."""
  import os
  try:
    props = torch.cuda.get_device_properties(device_index)
    bdf = '%04x:%02x:%02x.0' % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
    with open('/sys/bus/pci/devices/%s/numa_node' % bdf) as f:
      node = int(f.read().strip())
    if node < 0:
      return None
    with open('/sys/devices/system/node/node%d/cpulist' % node) as f:
      cpus = set()
      for part in f.read().strip().split(','):
        if '-' in part:
          a, b = part.split('-')
          cpus.update(range(int(a), int(b) + 1))
        elif part:
          cpus.add(int(part))
    allowed = cpus & os.sched_getaffinity(0)
    if not allowed:
      return None
    os.sched_setaffinity(0, allowed)
    return {'node': node, 'cpus': len(allowed)}
  except (OSError, AttributeError, ValueError):
    return None


class _DeviceArray(object):
  """Zero-copy torch view of raw device memory (the `__cuda_array_interface__`)."""

  def __init__(self, ptr, n, typestr):
    self.__cuda_array_interface__ = {'shape': (n,), 'typestr': typestr,
                                     'data': (ptr, False), 'version': 2}


class FusedGradReducer(object):
  """Peer-memory plumbing of the fused all-reduce + optimizer kernel (csrc/dp_fused.cu, K7).

  Owns, per rank: two gradient slots of `n` floats and a flag pad in IPC-shareable device
  memory; maps every peer's slots and pad (CUDA IPC handles exchanged once through the
  process group: torch.distributed is plumbing, the collective itself is our kernel).
  `grads(step)` is the torch view of this step's local slot — the scorer backward writes
  straight into it — and `step(...)` launches the kernel.  One node, <= 16 ranks.
  """

  MAX_RANKS = 16

  def __init__(self, n, device, group=None):
    import ctypes
    from ranking_b200 import _C
    self._C = _C
    self.group = group
    self.world = world_size(group)
    self.rank = rank(group)
    if self.world > self.MAX_RANKS:
      raise ValueError('fused all-reduce supports at most %d ranks' % self.MAX_RANKS)
    self.n = int(n)
    self.device = torch.device(device)
    self.n_pad = (self.n + 63) // 64 * 64
    slot_bytes = self.n_pad * 4
    total = 2 * slot_bytes + 256           # two gradient slots + the flag pad
    self._slot_bytes = slot_bytes
    with torch.cuda.device(self.device):
      ptr = ctypes.c_void_p()
      handle = (ctypes.c_ubyte * 64)()
      _C.check(_C.lib.tfr_dp_alloc(total, ctypes.byref(ptr), handle))
      self._base = ptr.value
      handles = [None] * self.world
      if self.world > 1:
        dist.all_gather_object(handles, bytes(handle), group=group)
      else:
        handles[0] = bytes(handle)
      self._peer_base = []
      for r in range(self.world):
        if r == self.rank:
          self._peer_base.append(self._base)
        else:
          p = ctypes.c_void_p()
          hb = (ctypes.c_ubyte * 64).from_buffer_copy(handles[r])
          _C.check(_C.lib.tfr_dp_open(hb, ctypes.byref(p)))
          self._peer_base.append(p.value)
    self._views = [
        torch.as_tensor(_DeviceArray(self._base + s * slot_bytes, self.n, '<f4'),
                        device=self.device) for s in range(2)]
    ptr_arr = ctypes.c_void_p * self.world
    self._grad_tabs = [ptr_arr(*[b + s * slot_bytes for b in self._peer_base])
                       for s in range(2)]
    self._flag_tab = ptr_arr(*[b + 2 * slot_bytes for b in self._peer_base])
    self.epoch = 0
    if self.world > 1:
      dist.barrier(group=group)      # every mapping exists before the first flag is written

  def grads(self, step=None):
    """Local gradient slot of step `step` (default: the next step)."""
    e = self.epoch + 1 if step is None else step
    return self._views[e % 2]

  def step(self, params, accum, kind, lr, eps, summed_out=None):
    """All ranks: sum the gradient slots over NVLink peer loads, scale by 1 / world and
    apply the optimizer — one kernel."""
    _C = self._C
    self.epoch += 1
    _C.check(_C.lib.tfr_allreduce_optimizer_step(
        self._grad_tabs[self.epoch % 2], self._flag_tab, self.rank, self.world,
        self.epoch & 0xFFFFFFFF, _C.ptr(params), _C.ptr(accum), _C.ptr(summed_out), self.n,
        kind, lr, eps, 1.0 / self.world, _C.stream()))

  def close(self):
    _C = self._C
    if self._base is None:
      return
    torch.cuda.synchronize(self.device)
    if self.world > 1:
      dist.barrier(group=self.group)
    for r, p in enumerate(self._peer_base):
      if r != self.rank:
        _C.lib.tfr_dp_close(p)
    self._views = None
    _C.lib.tfr_dp_free(self._base)
    self._base = None

"""Multi-GPU execution of the EPro-PnP path: objects are independent, so the batch is split into
contiguous shards (one process per GPU) and solved with NO collective inside the solve.  The only
communication is one gather of the small results afterwards (poses, optional covariances / costs and
the (B, M) log-weights); the (B, M, D) pose samples stay sharded unless explicitly requested
(SURVEY.md section 8e).  The Philox noise is keyed by the GLOBAL object index (`obj_offset`), so a sharded
run reproduces the single-GPU run bit for bit.
"""
import functools

import torch
import torch.distributed as dist


def shard_range(num_obj, rank, world_size):
    """Contiguous [begin, end) of `rank`: sizes differ by at most one, earlier ranks take the extra."""
    base, extra = divmod(int(num_obj), int(world_size))
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


def shard_sizes(num_obj, world_size):
    return [shard_range(num_obj, r, world_size)[1] - shard_range(num_obj, r, world_size)[0]
            for r in range(world_size)]


def gather_objects(local, num_obj, group=None):
    """All-gather a per-object tensor (local shard (b_r, ...)) into the full (num_obj, ...) tensor on
    every rank.  Equal shards use all_gather_into_tensor (one NCCL call); ragged shards pad to the
    largest shard."""
    if not (dist.is_available() and dist.is_initialized()):
        return local
    world = dist.get_world_size(group)
    if world == 1:
        return local
    sizes = shard_sizes(num_obj, world)
    tail = tuple(local.shape[1:])
    if len(set(sizes)) == 1:
        out = local.new_empty((num_obj,) + tail)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    biggest = max(sizes)
    padded = local.new_zeros((biggest,) + tail)
    padded[:local.shape[0]] = local
    buf = local.new_empty((world * biggest,) + tail)
    dist.all_gather_into_tensor(buf, padded, group=group)
    return torch.cat([buf[r * biggest:r * biggest + sizes[r]] for r in range(world)], dim=0)


def gather_results(result, num_obj, keys=("pose_opt", "logw", "pose_cov", "cost"), group=None):
    """result: dict of local object-major tensors (as returned by native.lm_amis_fused)."""
    return {k: gather_objects(result[k], num_obj, group) for k in keys if result.get(k) is not None}


class PendingGather:
    """Handle of an asynchronous gather: `.wait()` makes the current stream wait for it and returns the dict."""

    def __init__(self, tensors, works):
        self.tensors, self.works = tensors, works

    def wait(self):
        for w in self.works:
            w.wait()
        self.works = []
        return self.tensors


def gather_results_async(result, num_obj, keys=("pose_opt", "logw"), group=None):
    """Same gather, issued asynchronously (equal shards only): NCCL runs it on its own stream after the work
    already enqueued on the current stream, so the NEXT batch's solve overlaps this batch's exchange.  Objects of
    different batches are independent; nothing inside a solve ever waits for a collective."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return PendingGather({k: result[k] for k in keys if result.get(k) is not None}, [])
    world = dist.get_world_size(group)
    if len(set(shard_sizes(num_obj, world))) != 1:
        return PendingGather(gather_results(result, num_obj, keys, group), [])
    outs, works = {}, []
    present = [k for k in keys if result.get(k) is not None]
    for k in present:
        outs[k] = result[k].new_empty((num_obj,) + tuple(result[k].shape[1:]))
    for k in present:
        works.append(dist.all_gather_into_tensor(outs[k], result[k].contiguous(), group=group, async_op=True))
    return PendingGather(outs, works)


# ---- raw CUDA IPC: a peer's buffer mapped while THIS process's own device is current.  torch's tensor IPC
# (reduce_tensor / rebuild_cuda_tensor) opens the handle under the EXPORTER's device index and relies on torch's lazy
# peer-access switch, which is enough for cross-device copies but not a documented contract for kernels of
# another device dereferencing the pointer; the in-kernel push (PushGather) therefore maps its peers the way NCCL does:
# cudaIpcOpenMemHandle(handle, cudaIpcMemLazyEnablePeerAccess) on the importing device.
_cudart = None


def _runtime():
    global _cudart
    if _cudart is None:
        import ctypes
        for name in ("libcudart.so.12", "libcudart.so"):
            try:
                _cudart = ctypes.CDLL(name)
                break
            except OSError:
                continue
        if _cudart is None:
            raise RuntimeError("libcudart not found")
    return _cudart


def raw_ipc_export(t):
    """Picklable description of a CUDA tensor's memory: the cudaIpcMemHandle_t of the cudaMalloc allocation it lives in
    (cuMemGetAddressRange finds its base; torch's caching allocator sub-allocates segments) + the byte offset of the
    tensor's first element.  The exporter must keep the tensor alive while peers use the mapping."""
    import ctypes

    class _Handle(ctypes.Structure):
        _fields_ = [("reserved", ctypes.c_char * 64)]
    rt = _runtime()
    drv = ctypes.CDLL("libcuda.so.1")
    base, size = ctypes.c_uint64(0), ctypes.c_size_t(0)
    with torch.cuda.device(t.device):
        fn = getattr(drv, "cuMemGetAddressRange_v2", None) or drv.cuMemGetAddressRange
        fn.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_size_t), ctypes.c_uint64]
        fn.restype = ctypes.c_int
        rc = fn(ctypes.byref(base), ctypes.byref(size), ctypes.c_uint64(t.data_ptr()))
        if rc != 0:
            raise RuntimeError(f"cuMemGetAddressRange failed with CUresult {rc}")
        h = _Handle()
        rt.cudaIpcGetMemHandle.argtypes = [ctypes.POINTER(_Handle), ctypes.c_void_p]
        rt.cudaIpcGetMemHandle.restype = ctypes.c_int
        rc = rt.cudaIpcGetMemHandle(ctypes.byref(h), ctypes.c_void_p(base.value))
        if rc != 0:
            raise RuntimeError(f"cudaIpcGetMemHandle failed with cudaError {rc} (expandable segments have no classic IPC "
                               "handle: PushGather needs PYTORCH_CUDA_ALLOC_CONF without expandable_segments)")
    return dict(device=int(t.device.index), handle=bytes(h), offset=int(t.data_ptr() - base.value),
                nbytes=t.numel() * t.element_size())


def raw_ipc_open(desc, device):
    """Map the exported allocation into this process with `device` current; returns the device pointer (int) of the tensor's
    first element, usable by kernels running on `device`."""
    import ctypes

    class _Handle(ctypes.Structure):
        _fields_ = [("reserved", ctypes.c_char * 64)]
    rt = _runtime()
    rt.cudaIpcOpenMemHandle.argtypes = [ctypes.POINTER(ctypes.c_void_p), _Handle, ctypes.c_uint]
    rt.cudaIpcOpenMemHandle.restype = ctypes.c_int
    base = ctypes.c_void_p()
    with torch.cuda.device(device):
        rc = rt.cudaIpcOpenMemHandle(ctypes.byref(base), _Handle.from_buffer_copy(desc["handle"]), 1)   # 1 = lazy peer access
    if rc != 0:
        raise RuntimeError(f"cudaIpcOpenMemHandle failed with cudaError {rc}")
    return int(base.value) + int(desc["offset"])


class _DeviceHooks:
    """The device-specific pieces of the peer-memory gathers (CUDA streams / events, CUDA IPC).  The CPU test-suite
    substitutes host equivalents (inert streams, shared-memory tensors) to exercise the bookkeeping over gloo."""

    def _new_stream(self):
        return torch.cuda.Stream(self.device)

    def _new_event(self):
        return torch.cuda.Event()

    def _current_stream(self):
        return torch.cuda.current_stream(self.device)

    def _on_stream(self, stream):
        return torch.cuda.stream(stream)

    def _device_synchronize(self):
        torch.cuda.synchronize(self.device)

    def _record_stream(self, tensor, stream):
        tensor.record_stream(stream)

    def _export_raw(self, t):
        return raw_ipc_export(t)

    def _import_raw(self, desc):
        return raw_ipc_open(desc, self.device)     # a raw device pointer (int)


@functools.lru_cache(maxsize=None)
def _resident_limit(dof, mc_samples, mc_iter):
    from . import native
    return native.max_points(dof, mc_samples, mc_iter)


def _push_call(prob, params):
    """native.lm_amis_fused_push, or its cluster-split form when the objects' points do not fit one SM."""
    from . import native
    split = prob.N > _resident_limit(params.dof, params.mc_samples, params.mc_iter)
    return native.lm_amis_fused_split_push if split else native.lm_amis_fused_push


class _EventWork:
    def __init__(self, event, cur_stream=None):
        self.event, self.cur_stream = event, cur_stream

    def wait(self):
        (self.cur_stream() if self.cur_stream is not None else torch.cuda.current_stream()).wait_event(self.event)


class PushGather(_DeviceHooks):
    """Fused solve + gather over peer memory (opt-in; equal shards, one NVLink / NVSwitch node, <= 9 ranks).

    There is no gather step at all: every rank keeps a ring of `depth` FULL-batch result buffers (pose_opt
    (num_obj, D), logw (num_obj, M)), exposed to the other ranks through CUDA IPC once, and the solve kernel itself
    (native.lm_amis_fused_push -> the AMIS kernel's push epilogue; for objects above the resident point limit
    native.lm_amis_fused_split_push, whose copy kernel follows the cluster-split solve) stores each finished object's rows into slot t mod depth of EVERY
    rank's ring -- its own slice directly as the kernel's normal output, the peers' with plain stores over NVLink,
    object by object underneath the remaining CTAs' math.  What is left per batch is one 4-byte all-reduce on a side
    stream ("all ranks' kernels for batch t have finished, so every row of my slot t is in place").

    Lifetime of results: the tensors a PendingGather of batch t hands out ARE ring slot t mod depth; they stay valid
    until this rank calls solve() for batch t + valid_for (default: the usual overlapped pattern -- start batch t+1,
    then wait for and read batch t).  Slot reuse is made safe by making the kernel of batch u wait for the rendezvous
    of batch u - (depth - valid_for): every rank has by then started batch u - depth + valid_for, i.e. is past its
    reads of batch u - depth.  depth - valid_for is how many batches the ranks may drift apart (1 = lock step).

    Requires every process to see all GPUs of the node (torchrun's default) with peer access between them.
    """

    def __init__(self, num_obj, mc_samples, pose_dim, device, depth=4, valid_for=2, group=None, copy_out=False):
        """copy_out=True hands out private copies of the full-batch tensors (one device-to-device copy per batch on the
        side stream) instead of views of the ring, for callers that keep results longer than `valid_for` batches."""
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("PushGather needs an initialised process group")
        self.copy_out = bool(copy_out)
        self.group, self.depth, self.valid_for = group, int(depth), int(valid_for)
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if len(set(shard_sizes(num_obj, self.world))) != 1:
            raise ValueError("PushGather handles equal shards only (use gather_results for ragged batches)")
        if self.world - 1 > 8:
            raise ValueError("the kernel pushes to at most 8 peers")
        if self.valid_for < 1 or self.depth - self.valid_for < 1:
            raise ValueError("need valid_for >= 1 and depth > valid_for")
        self.num_obj, self.per_rank = int(num_obj), int(num_obj) // self.world
        self.device = torch.device(device)
        self.comm = self._new_stream()
        self.flag = torch.zeros(1, device=self.device)
        new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=self.device)
        self.ring = [dict(pose_opt=new(self.num_obj, pose_dim), logw=new(self.num_obj, mc_samples))
                     for _ in range(self.depth)]
        mine = dict(ring=[{k: self._export_raw(t) for k, t in slot.items()} for slot in self.ring])
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=group)
        self.peers = []                       # peers[r][slot][key] -> rank r's full-batch buffer, mapped for THIS device's kernels (None = me)
        for r, theirs in enumerate(everyone):
            if r == self.rank:
                self.peers.append(None)
                continue
            self.peers.append([{k: self._import_raw(h) for k, h in slot.items()} for slot in theirs["ring"]])
        # per ring slot: the device arrays of pointers the kernel reads its peers' buffer addresses from (built once)
        from . import native
        others = [r for r in range(self.world) if r != self.rank]
        self.n_peers = len(others)
        self.tables = [(native.peer_table([self.peers[r][s]["logw"] for r in others], self.device),
                        native.peer_table([self.peers[r][s]["pose_opt"] for r in others], self.device))
                       for s in range(self.depth)]
        self._device_synchronize()
        self.met = {}                         # batch index -> event of its rendezvous (last `depth` kept)
        self.step = 0
        dist.barrier(group=group)

    def solve(self, prob, pose_init, params, seed=0, want_cost=False, want_cov=False, init=None):
        """Enqueue batch `step`: fused solve with in-kernel push.  Returns (local result dict, PendingGather of the
        full-batch pose_opt / logw).  pose_init None: `init` (native.rslm_spec / epnp_spec) first computes it on this
        rank's shard, on the current stream, with the RSLM draws keyed by the global object index, so the assembled
        batch equals the single-process run from the same initialiser."""
        t = self.step
        s = t % self.depth
        lo, hi = self.rank * self.per_rank, (self.rank + 1) * self.per_rank
        if init is not None:
            if pose_init is not None:
                raise ValueError("PushGather.solve takes pose_init or an initialiser (init), not both")
            from . import native
            pose_init = native.initial_pose(prob, init, params.dof, obj_offset=lo)
        cur = self._current_stream()
        gate = self.met.get(t - (self.depth - self.valid_for))
        if gate is not None:
            cur.wait_event(gate)              # every rank is past its reads of the slot this batch overwrites
        out = _push_call(prob, params)(prob, pose_init, params, self.ring[s]["pose_opt"][lo:hi],
                                       self.ring[s]["logw"][lo:hi], self.tables[s][0], self.tables[s][1],
                                       seed=seed, obj_offset=lo, want_cost=want_cost, want_cov=want_cov, n_peers=self.n_peers)
        ready = self._new_event()
        ready.record(cur)
        with self._on_stream(self.comm):
            self.comm.wait_event(ready)
            dist.all_reduce(self.flag, group=self.group)          # rendezvous: every rank's kernel of batch t is done
            met = self._new_event()
            met.record(self.comm)
            full, done = dict(self.ring[s]), met
            if self.copy_out:
                full = {k: torch.empty_like(v) for k, v in self.ring[s].items()}
                for k, v in self.ring[s].items():
                    full[k].copy_(v, non_blocking=True)
                    self._record_stream(full[k], self.comm)
                done = self._new_event()
                done.record(self.comm)
        self.met[t] = met
        self.met.pop(t - self.depth, None)
        self.step += 1
        return out, PendingGather(full, [_EventWork(done, cur_stream=self._current_stream)])

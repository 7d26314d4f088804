"""Multi-GPU sharding of the query path (one process per GPU, torch.distributed).

The path is embarrassingly parallel: meshes / BVHs / tables are replicated on every rank and the work is split
into contiguous slabs, so there is no data-path collective inside a query.  The only exchange is the optional
re-assembly of the per-rank result slabs (one all-gather over NCCL / NVLink), used by the RobotSDF and chamfer
sweeps when the caller wants the full result on every rank.

  shard_range           contiguous slab [begin, end) of `n` items for (rank, world)
  sharded_query         ObjectFrameSDF over a shard of the flattened point axis (+ optional all-gather)
  sharded_robot_query   RobotSDF over a shard of the configuration batch (+ optional all-gather)
  sharded_chamfer       chamfer partial means over a shard of the cloud, all-reduced (B floats)
  PeerResult            full-size RobotSDF result buffers mapped into every process of the node, so that
                        sharded_robot_query(gather="peer") re-assembles the result with stores from the kernel
                        epilogue (NVLink traffic under the lookups) instead of a trailing all-gather
"""
import ctypes

import torch
import torch.distributed as dist

from .sdf import _config_count


def shard_range(n, rank, world):
    """Contiguous split of n items; the first n % world ranks take one extra."""
    base, extra = divmod(n, world)
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


def _parse_cpulist(text):
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.update(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_numa_node(device_index):
    """NUMA node the GPU's PCIe root hangs off (sysfs), or None when the platform does not say."""
    try:
        props = torch.cuda.get_device_properties(device_index)
        bus = f"{props.pci_domain_id:04x}:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0"
    except Exception:
        try:
            import pynvml
            pynvml.nvmlInit()
            bus = pynvml.nvmlDeviceGetPciInfo(pynvml.nvmlDeviceGetHandleByIndex(device_index)).busId
            bus = (bus.decode() if isinstance(bus, bytes) else bus).lower()[-12:]
        except Exception:
            return None
    try:
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as fh:
            node = int(fh.read())
        return node if node >= 0 else None
    except (OSError, ValueError):
        return None


def bind_to_gpu_numa_node(device_index):
    """Restrict this process to the CPUs of its GPU's NUMA node, so that the pinned host buffers it allocates from
    now on (first touch) and the threads that fill them sit next to the PCIe root of that GPU.  With eight ranks
    streaming results to host memory on a two-socket box, unbound ranks cross the socket interconnect and the
    end-to-end time per step suffers.  Returns (node, n_cpus, previous
    affinity) or None when nothing was changed; pass the previous affinity to os.sched_setaffinity to undo."""
    import os
    node = gpu_numa_node(device_index)
    if node is None or not hasattr(os, "sched_setaffinity"):
        return None
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as fh:
            cpus = _parse_cpulist(fh.read())
        before = os.sched_getaffinity(0)
        allowed = before & cpus
        if not allowed or allowed == before:
            return None
        os.sched_setaffinity(0, allowed)
        return node, len(allowed), before
    except (OSError, ValueError):
        return None


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def all_gather_slabs(local, counts, group=None):
    """Concatenate per-rank slabs (dim 0, sizes `counts`) on every rank with one all_gather."""
    rank, world = _world(group)
    if world == 1:
        return local
    if len(set(counts)) == 1:
        out = torch.empty((world * counts[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    # ragged shards: pad to the largest slab, gather, strip
    m = max(counts)
    pad = torch.zeros((m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty((world * m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return torch.cat([out[r * m:r * m + counts[r]] for r in range(world)], dim=0)


def sharded_query(sdf, points, gather=True, group=None):
    """Evaluate `sdf` on this rank's slab of the flattened points [..., N, 3].

    Returns (val, grad) for the full batch when gather=True (original leading shape), else the local slab
    (flat) together with its (begin, end)."""
    rank, world = _world(group)
    lead = tuple(points.shape[:-1])
    flat = points.reshape(-1, 3)
    n = flat.shape[0]
    begin, end = shard_range(n, rank, world)
    val, grad = sdf(flat[begin:end])
    if not gather:
        return val, grad, (begin, end)
    counts = [shard_range(n, r, world)[1] - shard_range(n, r, world)[0] for r in range(world)]
    val = all_gather_slabs(val, counts, group)
    grad = all_gather_slabs(grad, counts, group)
    return val.reshape(lead), grad.reshape(*lead, 3)


class _DeviceSpan:
    """Raw device memory exposed through __cuda_array_interface__ so torch can view it without owning it."""

    def __init__(self, address, n_float, owner):
        self.owner = owner      # keeps the allocation alive as long as any tensor view exists
        self.__cuda_array_interface__ = {"shape": (int(n_float),), "typestr": "<f4", "data": (int(address), False),
                                         "version": 3, "strides": None}


class PeerResult:
    """Full-size (n_cfg, n_pts) value / gradient buffers, one pair of SLOTS per rank, each mapped into every process
    of the node.

    Rank r's RobotSDF kernel stores its configuration slab into all `world` buffers (its own and, over NVLink, the
    peers'), so after `publish()` every rank holds the complete result -- the re-assembly SURVEY section 8(e) asks
    for -- without a separate all-gather pass.  Buffers are plain cudaMalloc allocations shared with CUDA IPC
    (pvb_ipc_*); same-node processes only, at most 8 ranks per launch (pvb.h PVB_MAX_TARGETS).

    Ordering.  Two slots alternate per query.  `publish()` (a stream-ordered all-reduce after the kernel) guarantees
    that every rank's kernel k has finished before anyone reads result k.  The write-after-read hazard -- a fast rank's
    NEXT kernel storing into a buffer a slow rank is still reading -- is closed by the alternation: query k+2 reuses
    the slot of query k, and rank A's kernel k+2 follows A's publish k+1, which cannot complete before rank B has
    entered its own publish k+1, which B's stream orders after everything B enqueued to consume result k.  So the
    tensors returned for query k stay valid until the same rank issues query k+2 into this PeerResult, provided the
    consumers are enqueued on the query stream (or synchronised with it) before query k+1 is issued.
    """

    SLOTS = 2

    def __init__(self, n_cfg, n_pts, group=None, backend="auto"):
        """backend: "ipc" = cudaMalloc + CUDA IPC handles (pvb_ipc_*); "symm" = torch symmetric memory (CUDA VMM
        allocations exchanged by torch.distributed), which additionally yields an NVLS MULTICAST mapping of the
        buffers when the NVSwitch fabric supports it (`self.multicast`); "auto" = symm when it works on every rank,
        else ipc."""
        from . import _native as nat
        self.nat = nat
        self.group = group
        self.rank, self.world = _world(group)
        if self.world > nat.MAX_TARGETS:
            raise ValueError(f"PeerResult supports up to {nat.MAX_TARGETS} ranks, got {self.world}")
        if backend not in ("auto", "ipc", "symm"):
            raise ValueError(f"backend must be 'auto', 'ipc' or 'symm', got {backend!r}")
        self.n_cfg, self.n_pts = int(n_cfg), int(n_pts)
        n = self.n_cfg * self.n_pts
        self._grad_offset = (4 * n + 255) // 256 * 256          # value block first, gradient block 256-B aligned
        self._slot_bytes = (self._grad_offset + 12 * n + 255) // 256 * 256
        self.nbytes = self.SLOTS * self._slot_bytes
        self.device = torch.device("cuda", torch.cuda.current_device())
        self._peer_ptrs = {}
        self._local = ctypes.c_void_p()
        self._symm = None               # (tensor, handle) of the symmetric-memory backend
        self._mc_base = 0
        self.backend = None
        self.backend_note = None
        bases = None
        if backend in ("auto", "symm") and self.world > 1:
            bases = self._init_symm(group)
            if bases is None and backend == "symm":
                raise RuntimeError(f"PeerResult(backend='symm'): {self.backend_note}")
        if bases is None:
            bases = self._init_ipc(group)
        self._bases = bases
        # own buffer first, then the peers in ring order: at any moment the ranks target different destinations
        self._order = [(self.rank + k) % self.world for k in range(self.world)]
        self._vals, self._grads, self._targets = [], [], []
        for slot in range(self.SLOTS):
            off = slot * self._slot_bytes
            self._vals.append(torch.as_tensor(_DeviceSpan(bases[self.rank] + off, n, self),
                                              device=self.device).view(self.n_cfg, self.n_pts))
            self._grads.append(torch.as_tensor(_DeviceSpan(bases[self.rank] + off + self._grad_offset, 3 * n, self),
                                               device=self.device).view(self.n_cfg, self.n_pts, 3))
            self._targets.append([(bases[r] + off, bases[r] + off + self._grad_offset) for r in self._order])
        self._slot = self.SLOTS - 1
        self._flag = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._closed = False

    def _init_ipc(self, group):
        nat = self.nat
        with torch.cuda.device(self.device):
            nat.check(nat.lib().pvb_ipc_alloc(self.nbytes, ctypes.byref(self._local)), "pvb_ipc_alloc")
            bases = [None] * self.world
            bases[self.rank] = self._local.value
            if self.world > 1:
                handle = ctypes.create_string_buffer(nat.IPC_HANDLE_BYTES)
                nat.check(nat.lib().pvb_ipc_export(self._local, handle), "pvb_ipc_export")
                handles = [None] * self.world
                dist.all_gather_object(handles, bytes(handle.raw), group=group)
                for r in range(self.world):
                    if r == self.rank:
                        continue
                    mapped = ctypes.c_void_p()
                    nat.check(nat.lib().pvb_ipc_open(handles[r], ctypes.byref(mapped)), "pvb_ipc_open")
                    self._peer_ptrs[r] = mapped.value
                    bases[r] = mapped.value
        self.backend = "ipc"
        return bases

    def _init_symm(self, group):
        """torch symmetric memory: peer-mapped addresses of every rank's buffer and, on an NVSwitch fabric, one
        multicast address that aliases all of them.  Collective; returns None (with the reason in backend_note) when
        any rank cannot set it up."""
        bases, err = None, None
        try:
            import torch.distributed._symmetric_memory as symm_mem
            grp = group if group is not None else dist.group.WORLD
            t = symm_mem.empty(self.nbytes // 4, dtype=torch.float32, device=self.device)
            hdl = symm_mem.rendezvous(t, group=grp)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            # buffer_ptrs address the allocation block; the tensor may sit at an offset inside it (same on every rank)
            off0 = t.data_ptr() - ptrs[self.rank]
            if len(ptrs) != self.world or off0 < 0 or off0 % 256:
                raise RuntimeError("unexpected buffer_ptrs from the symmetric memory handle")
            bases = [p + off0 for p in ptrs]
            self._symm = (t, hdl)
            mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
            self._mc_base = mc + off0 if mc else 0
        except Exception as e:      # noqa: BLE001 -- any failure means "not available here"
            err = f"{type(e).__name__}: {e}"[:300]
            bases = None
        ok = torch.tensor([0.0 if bases is None else 1.0, 1.0 if self._mc_base else 0.0], device=self.device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        if ok[0].item() == 0.0:
            self._symm, self._mc_base = None, 0
            self.backend_note = err or "another rank could not set up symmetric memory"
            return None
        if ok[1].item() == 0.0:
            self._mc_base = 0
        self.backend = "symm"
        return bases

    @property
    def multicast(self):
        """True when one multimem.st per chunk reaches every rank's buffer (NVLS multicast mapping available)."""
        return self._mc_base != 0

    def multicast_target(self):
        """(val, grad) multicast addresses of the slot of the most recent next_slot() call."""
        off = self._slot * self._slot_bytes
        return self._mc_base + off, self._mc_base + off + self._grad_offset

    # the slot of the most recent query
    @property
    def val(self):
        return self._vals[self._slot]

    @property
    def grad(self):
        return self._grads[self._slot]

    @property
    def targets(self):
        return self._targets[self._slot]

    def next_slot(self):
        """Advance to the slot the next query writes into; returns its (val, grad) device-address pairs, own first."""
        self._slot = (self._slot + 1) % self.SLOTS
        return self._targets[self._slot]

    #: gather="dma": configurations per kernel launch / copy batch (0 = the whole slab at once); the pushes of chunk
    #: k run on the copy engines while chunk k + 1 is being evaluated
    dma_chunk_cfgs = 0

    def dma_gather(self, comp, points, begin, end):
        """Copy-engine re-assembly: the slab is evaluated into this rank's own buffer with the ordinary
        single-destination kernel (in `dma_chunk_cfgs`-configuration pieces), and every finished piece is pushed to
        each peer's buffer with cudaMemcpyAsync over the peer mappings, on side streams, while the next piece is being
        evaluated.  The SMs never issue a remote store; NVLink carries large DMA packets."""
        nat = self.nat
        dev = self.device
        P = self.n_pts
        own_val, own_grad = self._targets[self._slot][0]
        cur = torch.cuda.current_stream(dev)
        if not hasattr(self, "_copy_streams"):
            self._copy_streams = [torch.cuda.Stream(dev) for _ in range(max(1, min(self.world - 1, 4)))]
        step = self.dma_chunk_cfgs if self.dma_chunk_cfgs > 0 else max(1, end - begin)
        L = nat.lib()
        with torch.cuda.device(dev):
            for cb in range(begin, end, step):
                cc = min(step, end - cb)
                comp.query_at(points, own_val, own_grad, cfg_begin=cb, cfg_count=cc)
                if self.world == 1:
                    continue
                done = torch.cuda.Event()
                done.record(cur)
                for k in range(1, self.world):                       # peers in ring order
                    peer_val, peer_grad = self._targets[self._slot][k]
                    st = self._copy_streams[(k - 1) % len(self._copy_streams)]
                    st.wait_event(done)
                    nat.check(L.pvb_memcpy_async(peer_val + 4 * cb * P, own_val + 4 * cb * P, 4 * cc * P, st.cuda_stream),
                              "pvb_memcpy_async")
                    nat.check(L.pvb_memcpy_async(peer_grad + 12 * cb * P, own_grad + 12 * cb * P, 12 * cc * P,
                                                 st.cuda_stream), "pvb_memcpy_async")
            if self.world > 1:
                for st in self._copy_streams:
                    cur.wait_stream(st)         # publish() below is ordered after every push of this rank

    def publish(self):
        """Stream-ordered barrier: when it completes on this rank, every rank's kernel (and with it all of its peer
        stores) has finished."""
        if self.world > 1:
            dist.all_reduce(self._flag, group=self.group)

    def close(self):
        """Unmap the peers' buffers and release the local one (collective: every rank must call it)."""
        if self._closed:
            return
        self._closed = True
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        with torch.cuda.device(self.device):
            for mapped in self._peer_ptrs.values():
                self.nat.check(self.nat.lib().pvb_ipc_close(ctypes.c_void_p(mapped)), "pvb_ipc_close")
            self._peer_ptrs = {}
            if self.world > 1:
                dist.barrier(group=self.group)
            self._vals = self._grads = None
            if self._symm is not None:
                self._symm = None           # the symmetric allocation is released with its tensor
            else:
                self.nat.check(self.nat.lib().pvb_ipc_free(self._local), "pvb_ipc_free")


def sharded_robot_query(robot_sdf, points, gather=True, group=None, result=None, paired=False, clearance=False):
    """RobotSDF over this rank's contiguous slab of the (flattened) configuration batch.

    The output slab (cfg_count, P) is a contiguous block of the (|A|, P) result, so re-assembly is a plain
    concatenation on dim 0.  Returns ([A,] *B, N) / (..., 3) when gather=True, else the local slab and its range.
    gather="peer" with a PeerResult: the kernel stores the slab into every rank's buffer directly (no all-gather);
    the returned tensors are views of one of `result`'s two slots and stay valid until the second-next query into
    it (see PeerResult for the cross-rank ordering this relies on).
    paired=True: RobotSDF.paired sharded the same way -- points [*A, *B, N, 3], and this rank evaluates its
    configurations on their own points[begin:end] only; gather must be True or False.
    clearance=True: RobotSDF.clearance sharded the same way -- points [*B, N, 3], this rank's slab is
    (cfg_count, prod(B)) and the re-assembled result ([A,] *B) / (..., 3); gather must be True or False."""
    rank, world = _world(group)
    comp = robot_sdf.sdf
    n_cfg = _config_count(comp.tsf_batch)
    begin, end = shard_range(n_cfg, rank, world)
    batch = tuple(comp.tsf_batch) if comp.tsf_batch is not None else ()
    if paired and clearance:
        raise ValueError("paired and clearance queries cannot be combined")
    if clearance:
        if isinstance(gather, str):
            raise ValueError("clearance queries re-assemble with gather=True or gather=False only")
        n_seg, _ = comp._clearance_segments(tuple(points.shape))
        if end > begin:
            val, grad = comp.query_clearance(points, cfg_begin=begin, cfg_count=end - begin)
        else:                               # more ranks than configurations: this rank's slab is empty
            dev = torch.device("cuda", torch.cuda.current_device())
            val, grad = torch.empty(0, device=dev), torch.empty(0, 3, device=dev)
        return _slab_result(val, grad, begin, end, n_cfg, n_seg, batch, tuple(points.shape[:-2]), gather, group)
    if paired:
        if isinstance(gather, str):
            raise ValueError("paired queries re-assemble with gather=True or gather=False only")
        pts_shape = tuple(points.shape)
        comp._check_leading_batch(pts_shape, "paired query", "..., 3", 1)
        per_cfg = points.reshape(n_cfg, -1, 3)
        P = per_cfg.shape[1]
        val, grad = comp.query_paired(per_cfg[begin:end], cfg_begin=begin, cfg_count=end - begin)
        lead = pts_shape[len(batch):-1]
        return _slab_result(val, grad, begin, end, n_cfg, P, batch, lead, gather, group)
    P = points.reshape(-1, 3).shape[0]
    if isinstance(gather, str):
        if gather not in ("peer", "multicast", "dma") or result is None:
            raise ValueError('gather must be True, False, "peer", "multicast" or "dma" (the latter three with '
                             'result=PeerResult(...))')
        if (result.n_cfg, result.n_pts) != (n_cfg, P):
            raise ValueError(f"PeerResult is ({result.n_cfg}, {result.n_pts}), the query is ({n_cfg}, {P})")
        targets = result.next_slot()
        if gather == "dma":
            result.dma_gather(comp, points, begin, end)
        elif gather == "multicast":
            if not result.multicast:
                raise RuntimeError("this PeerResult has no multicast mapping (needs backend='symm' on an NVSwitch fabric)")
            comp.query_multicast(points, *result.multicast_target(), cfg_begin=begin, cfg_count=end - begin)
        else:
            comp.query_into(points, targets, cfg_begin=begin, cfg_count=end - begin)
        result.publish()
        lead = tuple(points.shape[:-1])
        return result.val.view(*batch, *lead), result.grad.view(*batch, *lead, 3)
    val, grad = comp.query(points, cfg_begin=begin, cfg_count=end - begin)
    return _slab_result(val, grad, begin, end, n_cfg, P, batch, tuple(points.shape[:-1]), gather, group)


def _slab_result(val, grad, begin, end, n_cfg, P, batch, lead, gather, group):
    """This rank's (cfg_count, P) slab, or with gather=True the full result re-assembled by all_gather_slabs and
    shaped (*batch, *lead) / (..., 3)."""
    _, world = _world(group)
    val = val.reshape(end - begin, P)
    grad = grad.reshape(end - begin, P, 3)
    if not gather:
        return val, grad, (begin, end)
    counts = [shard_range(n_cfg, r, world)[1] - shard_range(n_cfg, r, world)[0] for r in range(world)]
    val = all_gather_slabs(val, counts, group)
    grad = all_gather_slabs(grad, counts, group)
    return val.reshape(*batch, *lead), grad.reshape(*batch, *lead, 3)


def sharded_chamfer(world_to_object, points, obj_factory=None, obj_sdf=None, scale=1000., group=None):
    """batch_chamfer_dist with the cloud split over ranks; the B partial sums are all-reduced."""
    from .chamfer import batch_chamfer_dist
    rank, world = _world(group)
    n = points.shape[0]
    begin, end = shard_range(n, rank, world)
    local = batch_chamfer_dist(world_to_object, points[begin:end], obj_factory=obj_factory, obj_sdf=obj_sdf,
                               scale=scale) if end > begin else torch.zeros(world_to_object.shape[0],
                                                                            dtype=world_to_object.dtype,
                                                                            device=world_to_object.device)
    total = local * float(end - begin)
    if world > 1:
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
    return total / float(n)

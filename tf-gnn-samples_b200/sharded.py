"""One large graph over several GPUs: binding of the node-range partition + peer-memory halo exchange of
include/rgnn.h (rgnn_halo_plan_*, rgnn_halo_exchange, rgnn_peer_*).

One process per GPU.  ``torch.distributed`` is used once, to ship the 64-byte CUDA-IPC handles of the peer buffers between
the ranks (and for nothing on the data path): after ``attach`` every layer's halo refresh is ONE kernel of this library that
reads the owners' rows over NVLink and carries its own cross-rank barrier.

    sg = ShardedGraph(adjacency_lists_with_global_ids, cuts, rank, world, device)      # index lists built on the device
    sg.attach(state_dim)                         # two [n_local, d] state buffers + flags in peer-mapped memory
    sg.states(0)[:sg.n_own] = h_own              # this rank's slice of the initial node states
    for t, w in enumerate(layer_weights):
        sg.exchange(t % 2)                       # halo rows of buffer t % 2 <- their owners
        sparse_gnn_film_layer(sg.states(t % 2), sg.plan, cnt_local, d, weights=w, out=sg.states(1 - t % 2))
    result = sg.states(len(layer_weights) % 2)[:sg.n_own]

The reference has no multi-device path (SURVEY.md 2.1); the partition follows SURVEY.md 8(e): targets owned, sources
fetched, weights replicated.
"""
import ctypes
from typing import List, Optional, Sequence

import numpy as np
import torch

from .engine import (GraphPlan, RgnnError, RGNN_E_INVALID, c_int64, c_void_p, check, current_stream_ptr, load_library,
                     ptr_table)

PEER_HANDLE_BYTES = 64


class _CudaView:
    """__cuda_array_interface__ wrapper: lets torch alias device memory that this library allocated (peer buffers)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class PeerBuffer:
    """A zeroed device allocation of ``nbytes`` on every rank of ``group``, each mapped into every other rank's address
    space (rgnn_peer_alloc / rgnn_peer_open).  ``ptrs[r]`` is rank r's allocation as seen from THIS process."""

    def __init__(self, nbytes: int, rank: int, world: int, device: torch.device, group=None):
        import torch.distributed as dist
        lib = load_library()
        self.nbytes, self.rank, self.world, self.device = int(nbytes), rank, world, device
        self._opened: List[int] = []
        self._local = c_void_p()
        handle = (ctypes.c_ubyte * PEER_HANDLE_BYTES)()
        with torch.cuda.device(device):
            check(lib.rgnn_peer_alloc(ctypes.byref(self._local), self.nbytes, handle))
            handles = [bytes(handle)]
            if world > 1:
                handles = [None] * world
                dist.all_gather_object(handles, bytes(handle), group=group)
            self.ptrs: List[int] = []
            for r in range(world):
                if r == rank:
                    self.ptrs.append(int(self._local.value))
                    continue
                p = c_void_p()
                buf = (ctypes.c_ubyte * PEER_HANDLE_BYTES).from_buffer_copy(handles[r])
                check(lib.rgnn_peer_open(buf, ctypes.byref(p)))
                self._opened.append(int(p.value))
                self.ptrs.append(int(p.value))
        if world > 1:
            dist.barrier(group=group)            # nobody frees before everybody has mapped

    def tensor(self, shape, dtype=torch.float32, rank: Optional[int] = None, byte_offset: int = 0) -> torch.Tensor:
        """A torch tensor aliasing (a slice of) rank ``rank``'s allocation (default: this rank's own)."""
        typestr = {torch.float32: "<f4", torch.int32: "<i4", torch.uint8: "|u1"}[dtype]
        ptr = self.ptrs[self.rank if rank is None else rank] + int(byte_offset)
        t = torch.as_tensor(_CudaView(ptr, shape, typestr), device=self.device)
        t._rgnn_keepalive = self                 # the tensor does not own the memory
        return t

    def close(self):
        lib = load_library()
        with torch.cuda.device(self.device):
            for p in self._opened:
                lib.rgnn_peer_close(c_void_p(p))
            self._opened = []
            if self._local is not None and self._local.value:
                lib.rgnn_peer_free(self._local)
                self._local = None


def degree_balanced_cuts(adjacency_lists: Sequence[np.ndarray], num_nodes: int, world: int) -> np.ndarray:
    """Split points [world + 1] with ~equal sum of (in-degree + 1) per rank (SURVEY.md 8e: degree-balanced, not equal
    node counts).  Host-side, O(M) once per batch; every rank computes the same cuts from the same lists."""
    from .partition import balanced_cuts
    indeg = np.zeros(num_nodes, dtype=np.int64)
    for a in adjacency_lists:
        a = np.asarray(a).reshape(-1, 2)
        if a.shape[0]:
            indeg += np.bincount(a[:, 1], minlength=num_nodes)
    return balanced_cuts(indeg + 1, world)


class ShardedGraph:
    """Rank-local structure of a node-range partition, built on the device by rgnn_halo_plan_create.

    ``plan`` carries no adjacency lists, so the layer paths that need them (the differentiable FiLM, RGAT, Edge-MLP,
    RGIN and composed RGCN) refuse it with an RgnnError.  Training on a node-range partition uses a GraphPlan over
    ``NodeRangePartition.local_adjacency_lists`` with ``set_num_targets(n_own)`` and ``NodeRangePartition.exchange``."""

    def __init__(self, adjacency_lists: Sequence, cuts: Sequence[int], rank: int, world: int,
                 device: Optional[torch.device] = None, group=None):
        lib = load_library()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device, self.rank, self.world, self.group = torch.device(device), int(rank), int(world), group
        self.cuts = [int(c) for c in cuts]
        if len(self.cuts) != world + 1:
            raise RgnnError(RGNN_E_INVALID, "cuts must have world + 1 = %d entries, got %d" % (world + 1, len(self.cuts)))
        dev_adj = []
        for a in adjacency_lists:
            if not isinstance(a, torch.Tensor):
                a = torch.as_tensor(np.ascontiguousarray(a))
            dev_adj.append(a.reshape(-1, 2).to(device=self.device, dtype=torch.int32).contiguous())
        self.num_edge_types = len(dev_adj)
        counts = (c_int64 * max(len(dev_adj), 1))(*[int(a.shape[0]) for a in dev_adj])
        ccuts = (c_int64 * (world + 1))(*self.cuts)
        handle = c_void_p()
        with torch.cuda.device(self.device):
            check(lib.rgnn_halo_plan_create(ctypes.byref(handle), self.rank, self.world, ccuts, self.num_edge_types,
                                            ptr_table(dev_adj, weights=False), counts, current_stream_ptr(self.device)))
        self._handle = handle
        self.lo, self.hi = self.cuts[rank], self.cuts[rank + 1]
        self.n_own = int(lib.rgnn_halo_plan_num_own(handle))
        self.n_halo = int(lib.rgnn_halo_plan_num_halo(handle))
        self.n_local = self.n_own + self.n_halo
        self.local_num_edges = [int(lib.rgnn_halo_plan_num_edges(handle, l)) for l in range(self.num_edge_types)]
        self.plan = GraphPlan.from_handle(lib.rgnn_halo_plan_graph(handle), self.n_local, self.num_edge_types,
                                          sum(self.local_num_edges), self.device, num_targets=self.n_own, owner=self)
        self._peer = None
        self.state_dim = None

    @property
    def handle(self):
        if self._handle is None:
            raise RgnnError(RGNN_E_INVALID, "ShardedGraph used after close()")
        return self._handle

    def export(self):
        """Copies of the device-built index lists (tests): halo_global / halo_owner / halo_row [n_halo] and the local
        adjacency lists."""
        lib = load_library()
        n = max(self.n_halo, 1)
        out = {k: torch.empty(n, dtype=torch.int32, device=self.device) for k in ("halo_global", "halo_owner", "halo_row")}
        adj = [torch.empty((max(e, 1), 2), dtype=torch.int32, device=self.device) for e in self.local_num_edges]
        with torch.cuda.device(self.device):
            check(lib.rgnn_halo_plan_export(self.handle, out["halo_global"].data_ptr(), out["halo_owner"].data_ptr(),
                                            out["halo_row"].data_ptr(), ptr_table(adj, weights=False),
                                            current_stream_ptr(self.device)))
        res = {k: v[: self.n_halo] for k, v in out.items()}
        res["local_adjacency_lists"] = [a[:e] for a, e in zip(adj, self.local_num_edges)]
        return res

    def local_num_incoming(self, type_to_num_incoming_edges) -> torch.Tensor:
        """[L, n_local] in-degrees in local numbering: the owned columns of the global table, zeros for halo nodes (they are
        never targets here)."""
        c = torch.as_tensor(type_to_num_incoming_edges)
        out = torch.zeros((c.shape[0], self.n_local), dtype=torch.float32, device=self.device)
        out[:, : self.n_own] = c[:, self.lo:self.hi].to(self.device, dtype=torch.float32)
        return out

    # ---- peer memory -------------------------------------------------------------------------------------------
    def attach(self, state_dim: int):
        """Allocate this rank's two state buffers [n_local, state_dim] and its flag array in peer-mapped memory, exchange
        the IPC handles (the only host-side collective) and hand the mapped pointers to the library."""
        import torch.distributed as dist
        lib = load_library()
        d = int(state_dim)
        if d % 4:
            raise RgnnError(RGNN_E_INVALID, "state_dim %d must be a multiple of 4" % d)
        rows = torch.tensor([self.n_local], dtype=torch.int64, device=self.device)
        if self.world > 1:
            dist.all_reduce(rows, op=dist.ReduceOp.MAX, group=self.group)
        max_rows = int(rows.item())
        self._buf_bytes = (max_rows * d * 4 + 255) // 256 * 256          # same layout on every rank
        nbytes = 2 * self._buf_bytes + 256
        self._peer = PeerBuffer(nbytes, self.rank, self.world, self.device, self.group)
        self.state_dim = d
        s0 = (c_void_p * self.world)(*[p for p in self._peer.ptrs])
        s1 = (c_void_p * self.world)(*[p + self._buf_bytes for p in self._peer.ptrs])
        fl = (c_void_p * self.world)(*[p + 2 * self._buf_bytes for p in self._peer.ptrs])
        check(lib.rgnn_halo_plan_attach(self.handle, s0, s1, fl))
        self._states = [self._peer.tensor((self.n_local, d), byte_offset=b * self._buf_bytes) for b in (0, 1)]
        return self

    @staticmethod
    def attach_in_process(graphs: Sequence["ShardedGraph"], state_dim: int):
        """All ranks of the partition live in THIS process on one GPU ("virtual ranks": single-GPU tests of the exchange
        protocol, SURVEY.md 4.4): plain torch allocations, every rank sees every other rank's pointers directly.  The
        exchanges of the virtual ranks must then be enqueued on DIFFERENT streams (they wait for each other on the device),
        and all of their pull kernels must fit on the GPU at once (a rank's CTAs spin until every other rank's CTA 0 has run:
        small test graphs only -- at most 264 CTAs of 512 threads per rank, 528 fit on an H100)."""
        lib = load_library()
        d = int(state_dim)
        world = len(graphs)
        max_rows = max(g.n_local for g in graphs)
        buf_floats = (max_rows * d + 63) // 64 * 64
        arenas = [torch.zeros(2 * buf_floats + 64, dtype=torch.float32, device=g.device) for g in graphs]
        for g, arena in zip(graphs, arenas):
            base = [a.data_ptr() for a in arenas]
            s0 = (c_void_p * world)(*base)
            s1 = (c_void_p * world)(*[p + buf_floats * 4 for p in base])
            fl = (c_void_p * world)(*[p + 2 * buf_floats * 4 for p in base])
            check(lib.rgnn_halo_plan_attach(g.handle, s0, s1, fl))
            g.state_dim, g._arena, g._peer = d, arenas, "in-process"
            g._states = [arena[b * buf_floats: b * buf_floats + g.n_local * d].view(g.n_local, d) for b in (0, 1)]

    def states(self, buffer: int) -> torch.Tensor:
        """This rank's state buffer 0 / 1 as a [n_local, state_dim] tensor (owned rows first, then the halo rows)."""
        if self._peer is None:
            raise RgnnError(RGNN_E_INVALID, "ShardedGraph.attach(state_dim) has not been called")
        return self._states[buffer]

    def exchange(self, buffer: int, overlap: bool = False):
        """Refresh the halo rows of state buffer ``buffer`` from their owners (rgnn_halo_exchange).  Collective.
        ``overlap=True`` (rgnn_halo_exchange_overlapped): the pull runs on a side stream and is joined by the next layer call
        on ``self.plan`` right before it reads halo rows -- the layer's target-side work overlaps the transfer."""
        lib = load_library()
        fn = lib.rgnn_halo_exchange_overlapped if overlap else lib.rgnn_halo_exchange
        with torch.cuda.device(self.device):
            check(fn(self.handle, int(buffer), int(self.state_dim or 0), current_stream_ptr(self.device)))

    def halo_bytes(self) -> int:
        return self.n_halo * (self.state_dim or 0) * 4

    def close(self):
        if getattr(self, "_handle", None) is not None:
            torch.cuda.synchronize(self.device)
            self._states = None
            if self._peer is not None and not isinstance(self._peer, str):
                if self.world > 1:
                    import torch.distributed as dist
                    dist.barrier(group=self.group)          # no peer is still pulling from this rank's buffers
                self._peer.close()
            self._peer = None
            load_library().rgnn_halo_plan_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._peer is None:
                load_library().rgnn_halo_plan_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

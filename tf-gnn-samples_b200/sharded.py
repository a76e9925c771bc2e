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

Training uses the same plan and buffers in both directions: ``gather`` is differentiable, its backward is the transposed
exchange (rgnn_halo_exchange_backward: the gradients of the halo rows are added into their owners' rows, in peer memory, in
a fixed rank order).  The weight gradients are still summed over the ranks by the caller.

    sg.attach(state_dim, training=True)          # + two gradient buffers, their flags, the published halo list;
                                                 #   builds the reverse index on the device
    plan = sg.training_plan()                    # GraphPlan over the device-built local lists, restricted to n_own
    cnt = sg.local_num_incoming(type_to_num_incoming_edges)
    h = h_own                                    # [n_own, d], e.g. a leaf that requires grad
    for t, w in enumerate(layer_weights):
        h = sparse_gnn_film_layer(sg.gather(h, t % 2), plan, cnt, d, weights=w)[:sg.n_own]
    loss_of(h).backward()                        # every rank: the halo gradients travel back inside the backward pass
    scaffold.all_reduce_gradients_(model)        # the replicated weights' gradients

The reference has no multi-device path (SURVEY.md 2.1); the partition follows SURVEY.md 8(e): targets owned, sources
fetched, weights replicated.
"""
import ctypes
from typing import List, Optional, Sequence

import numpy as np
import torch

from .engine import (GraphPlan, RgnnError, RGNN_E_INVALID, as_f32, c_int64, c_void_p, check, current_stream_ptr,
                     load_library, ptr_table)

PEER_HANDLE_BYTES = 64
HALO_LIST_HEADER = 4          # int32 words before the owners in a published halo list (include/rgnn.h)


class _HaloGather(torch.autograd.Function):
    """ShardedGraph.gather: forward = the owned rows into a state buffer + rgnn_halo_exchange, returned as a fresh
    [n_local, d] tensor; backward = rgnn_halo_exchange_backward on the gradient buffer of the same parity."""

    @staticmethod
    def forward(ctx, h_own, sg, buffer):
        ctx.sg, ctx.buffer = sg, buffer
        st = sg.states(buffer)
        st[: sg.n_own].copy_(h_own)
        sg.exchange(buffer)
        return st.clone()

    @staticmethod
    def backward(ctx, grad_local):
        return ctx.sg.exchange_backward(ctx.buffer, grad_local), None, None


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
    RGIN and composed RGCN) refuse it with an RgnnError.  Training runs on ``training_plan()`` between ``gather`` calls,
    after ``attach(state_dim, training=True)``."""

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
        self._training_plan = None

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
    def attach(self, state_dim: int, training: bool = False):
        """Allocate this rank's two state buffers [n_local, state_dim] and its flag array in peer-mapped memory, exchange
        the IPC handles (the only host-side collective) and hand the mapped pointers to the library.

        ``training=True`` also allocates, in the same peer-mapped allocation, the two gradient buffers, their own flag
        array and this rank's published halo list (rgnn_halo_plan_attach_grad), waits for every rank to publish, and
        builds the reverse index on the device (rgnn_halo_plan_build_reverse): ``gather`` becomes differentiable."""
        import torch.distributed as dist
        lib = load_library()
        d = int(state_dim)
        if d % 4:
            raise RgnnError(RGNN_E_INVALID, "state_dim %d must be a multiple of 4" % d)
        rows = torch.tensor([self.n_local, self.n_halo], dtype=torch.int64, device=self.device)
        if self.world > 1:
            dist.all_reduce(rows, op=dist.ReduceOp.MAX, group=self.group)
        max_rows, max_halo = (int(x) for x in rows.tolist())
        self._buf_bytes = (max_rows * d * 4 + 255) // 256 * 256          # same layout on every rank
        nbytes = 2 * self._buf_bytes + 256
        list_bytes = ((HALO_LIST_HEADER + 2 * max_halo) * 4 + 255) // 256 * 256
        if training:                                   # [g0][g1][gradient flags][halo list] after the forward's layout
            nbytes += 2 * self._buf_bytes + 256 + list_bytes
        self._peer = PeerBuffer(nbytes, self.rank, self.world, self.device, self.group)
        self.state_dim = d
        s0 = (c_void_p * self.world)(*[p for p in self._peer.ptrs])
        s1 = (c_void_p * self.world)(*[p + self._buf_bytes for p in self._peer.ptrs])
        fl = (c_void_p * self.world)(*[p + 2 * self._buf_bytes for p in self._peer.ptrs])
        check(lib.rgnn_halo_plan_attach(self.handle, s0, s1, fl))
        self._states = [self._peer.tensor((self.n_local, d), byte_offset=b * self._buf_bytes) for b in (0, 1)]
        if training:
            g0 = 2 * self._buf_bytes + 256
            self._attach_grad([[p + g0 + b * self._buf_bytes for p in self._peer.ptrs] for b in (0, 1)],
                              [p + g0 + 2 * self._buf_bytes for p in self._peer.ptrs],
                              [p + g0 + 2 * self._buf_bytes + 256 for p in self._peer.ptrs])
            if self.world > 1:
                dist.barrier(group=self.group)        # every rank has published its halo list
            self.build_reverse()
        return self

    def _attach_grad(self, grads, flags, lists):
        """rgnn_halo_plan_attach_grad with per-rank pointer lists (grads: one list per gradient buffer)."""
        w = self.world
        with torch.cuda.device(self.device):
            check(load_library().rgnn_halo_plan_attach_grad(self.handle, (c_void_p * w)(*grads[0]), (c_void_p * w)(*grads[1]),
                                                           (c_void_p * w)(*flags), (c_void_p * w)(*lists)))

    @staticmethod
    def attach_in_process(graphs: Sequence["ShardedGraph"], state_dim: int, training: bool = False):
        """All ranks of the partition live in THIS process on one GPU ("virtual ranks": single-GPU tests of the exchange
        protocol, SURVEY.md 4.4): plain torch allocations, every rank sees every other rank's pointers directly.  The
        exchanges of the virtual ranks must then be enqueued on DIFFERENT streams (they wait for each other on the device),
        and all of their pull kernels must fit on the GPU at once (a rank's CTAs spin until every other rank's CTA 0 has run:
        small test graphs only -- at most 264 CTAs of 512 threads per rank, 528 fit on an H100).  ``training=True``: as in
        ``attach``; a training step must then make no call that waits for the device between two exchanges of a rank (the
        other ranks' work is enqueued by the same host thread), which ``training_plan()`` arranges for the layer paths."""
        lib = load_library()
        d = int(state_dim)
        world = len(graphs)
        max_rows = max(g.n_local for g in graphs)
        buf_floats = (max_rows * d + 63) // 64 * 64
        list_floats = (HALO_LIST_HEADER + 2 * max(g.n_halo for g in graphs) + 63) // 64 * 64
        extra = 2 * buf_floats + 64 + list_floats if training else 0
        arenas = [torch.zeros(2 * buf_floats + 64 + extra, dtype=torch.float32, device=g.device) for g in graphs]
        base = [a.data_ptr() for a in arenas]
        for g, arena in zip(graphs, arenas):
            s0 = (c_void_p * world)(*base)
            s1 = (c_void_p * world)(*[p + buf_floats * 4 for p in base])
            fl = (c_void_p * world)(*[p + 2 * buf_floats * 4 for p in base])
            check(lib.rgnn_halo_plan_attach(g.handle, s0, s1, fl))
            g.state_dim, g._arena, g._peer = d, arenas, "in-process"
            g._states = [arena[b * buf_floats: b * buf_floats + g.n_local * d].view(g.n_local, d) for b in (0, 1)]
        if training:
            for g in graphs:                          # the zeroed arenas are in place before the lists are published
                torch.cuda.current_stream(g.device).synchronize()
            g0 = (2 * buf_floats + 64) * 4
            for g in graphs:
                g._attach_grad([[p + g0 + b * buf_floats * 4 for p in base] for b in (0, 1)],
                               [p + g0 + 2 * buf_floats * 4 for p in base],
                               [p + g0 + (2 * buf_floats + 64) * 4 for p in base])
            for g in graphs:
                g.build_reverse()

    def build_reverse(self):
        """(Re)build the reverse index of the halo lists on the device (rgnn_halo_plan_build_reverse): every rank must have
        published its list (``attach(..., training=True)`` does both).  Synchronises; refused during a CUDA-graph capture."""
        with torch.cuda.device(self.device):
            check(load_library().rgnn_halo_plan_build_reverse(self.handle, current_stream_ptr(self.device)))

    def export_reverse(self):
        """Copy of the reverse index (tests): offsets [n_own + 1] over the owned rows, and per entry the consuming peer and
        the row of that peer's gradient buffer (its n_own + the halo position), sorted by (owned row, peer)."""
        lib = load_library()
        n = int(lib.rgnn_halo_plan_num_reverse(self.handle))
        if n < 0:
            raise RgnnError(RGNN_E_INVALID, "the reverse index has not been built (attach(state_dim, training=True))")
        out = {"offsets": torch.empty(self.n_own + 1, dtype=torch.int32, device=self.device),
               "peer": torch.empty(max(n, 1), dtype=torch.int32, device=self.device),
               "row": torch.empty(max(n, 1), dtype=torch.int32, device=self.device)}
        with torch.cuda.device(self.device):
            check(lib.rgnn_halo_plan_export_reverse(self.handle, out["offsets"].data_ptr(), out["peer"].data_ptr(),
                                                    out["row"].data_ptr(), current_stream_ptr(self.device)))
        out["peer"], out["row"] = out["peer"][:n], out["row"][:n]
        return out

    def training_plan(self) -> GraphPlan:
        """The plan the differentiable layer paths run on between ``gather`` calls: a GraphPlan over this rank's
        device-exported local adjacency lists, restricted to the owned rows.  Built once; its index views and regrouped
        plans are built here, eagerly, so that a training step neither synchronises nor builds plan state inside a
        CUDA-graph capture."""
        if self._training_plan is None:
            lists = self.export()["local_adjacency_lists"]
            plan = GraphPlan(lists, self.n_local, device=self.device).set_num_targets(self.n_own)
            for view in ("message_sources", "message_targets", "message_types", "in_degree"):
                getattr(plan, view)
            for by in ("source", "source_type", "target_type"):
                plan.regrouped(by)
            self._training_plan = plan
        return self._training_plan

    def gather(self, h_own: torch.Tensor, buffer: int) -> torch.Tensor:
        """[n_own, state_dim] owned states -> a fresh [n_local, state_dim] tensor: owned rows, then the halo rows pulled
        from their owners through state buffer ``buffer`` (rgnn_halo_exchange).  Collective.  Differentiable: the backward
        adds the gradients of the halo rows into their owners' rows (rgnn_halo_exchange_backward, gradient buffer
        ``buffer``), which needs ``attach(..., training=True)``.  Consecutive gathers alternate the buffer, and every rank
        runs the backward of each gather (a rank that skips one leaves its peers waiting)."""
        d = self.state_dim or 0
        if not isinstance(h_own, torch.Tensor) or tuple(h_own.shape) != (self.n_own, d):
            raise RgnnError(RGNN_E_INVALID, "gather: h_own must be [n_own, state_dim] = [%d, %d], got %s"
                            % (self.n_own, d, tuple(getattr(h_own, "shape", ()))))
        return _HaloGather.apply(as_f32(h_own, "h_own"), self, int(buffer))

    def exchange_backward(self, buffer: int, grad_local: torch.Tensor) -> torch.Tensor:
        """The transposed exchange (rgnn_halo_exchange_backward): [n_local, state_dim] local gradient -> [n_own,
        state_dim] = its owned rows plus, per row, the gradients the peers hold for it as a halo row, added in ascending
        rank.  Collective."""
        d = self.state_dim or 0
        g = as_f32(grad_local, "grad_local")
        if tuple(g.shape) != (self.n_local, d):
            raise RgnnError(RGNN_E_INVALID, "exchange_backward: grad_local must be [n_local, state_dim] = [%d, %d], got %s"
                            % (self.n_local, d, tuple(g.shape)))
        out = torch.empty((self.n_own, d), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(load_library().rgnn_halo_exchange_backward(self.handle, int(buffer), d, g.data_ptr(), out.data_ptr(),
                                                             current_stream_ptr(self.device)))
        return out

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
            if self._training_plan is not None:
                self._training_plan.close()
                self._training_plan = None
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

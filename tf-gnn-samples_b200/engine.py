"""ctypes binding of librgnn.so (include/rgnn.h) + the per-batch GraphPlan.

This is the thin host layer the north star asks for: Python -> ctypes -> C ABI -> CUDA.  torch is
used for device memory (``Tensor.data_ptr()``) and the stream (``torch.cuda.current_stream()``).
There is no CPU path: if the library cannot be loaded the first call raises RgnnError.
"""
import ctypes
import os
import threading
from typing import Dict, List, Optional, Sequence

import torch

from . import _build

c_void_p, c_int, c_int32, c_int64, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t
c_char_p = ctypes.c_char_p

RGNN_OK, RGNN_E_INVALID, RGNN_E_CUDA, RGNN_E_WORKSPACE, RGNN_E_UNSUPPORTED = 0, -1, -2, -3, -4


class RgnnError(RuntimeError):
    """Raised when a librgnn call returns a negative status (message from rgnn_last_error())."""

    def __init__(self, code: int, message: str):
        super().__init__("librgnn error %d: %s" % (code, message))
        self.code = code
        self.message = message


# every exported symbol of include/rgnn.h: name -> (restype, argtypes)
_PTR = c_void_p
SIGNATURES = {
    "rgnn_version": (c_int, []),
    "rgnn_last_error": (c_char_p, []),
    "rgnn_launch_count": (c_int64, []),
    "rgnn_plan_create": (c_int, [ctypes.POINTER(c_void_p), c_int32, c_int32, _PTR, _PTR, _PTR]),
    "rgnn_plan_create_ex": (c_int, [ctypes.POINTER(c_void_p), c_int32, c_int32, _PTR, _PTR, c_int, _PTR]),
    "rgnn_plan_status": (c_int, [_PTR]),
    "rgnn_plan_destroy": (c_int, [_PTR]),
    "rgnn_plan_num_nodes": (c_int32, [_PTR]),
    "rgnn_plan_num_edge_types": (c_int32, [_PTR]),
    "rgnn_plan_num_edges": (c_int64, [_PTR]),
    "rgnn_plan_export": (c_int, [_PTR, _PTR, _PTR, _PTR, _PTR, _PTR]),
    "rgnn_set_weight_cache": (c_int, [c_int]),
    "rgnn_weight_cache_clear": (c_int, []),
    "rgnn_workspace_bytes": (c_size_t, [_PTR, c_int, c_int32, c_int32, c_int32]),
    "rgnn_rgcn_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, c_int, c_int, c_int, c_int,
                                  _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgcn_backward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, c_int, c_int, _PTR, _PTR, _PTR, _PTR,
                                   _PTR, c_size_t, _PTR]),
    "rgnn_ggnn_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, _PTR, _PTR, c_int, c_int, c_int, c_int,
                                  _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_ggnn_backward": (c_int, [_PTR, _PTR, c_int32, _PTR, _PTR, _PTR, _PTR, c_int, c_int, c_int, _PTR, _PTR, _PTR, _PTR,
                                   _PTR, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgat_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, c_int, c_int,
                                  _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_film_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, _PTR, _PTR, _PTR, c_int, c_int, c_int, c_int,
                                  _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_film_backward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, _PTR, _PTR, _PTR, c_int, c_int, c_int, _PTR, _PTR,
                                   _PTR, _PTR, _PTR, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgat_backward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, c_int, _PTR, _PTR, _PTR, _PTR, _PTR, c_size_t,
                                   _PTR]),
    "rgnn_edge_mlp_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, _PTR, _PTR, _PTR,
                                      c_int, c_int, c_int, c_int, c_int, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgin_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, _PTR, _PTR, c_int, _PTR, _PTR,
                                  c_int, c_int, c_int, c_int, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgin_backward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, _PTR, _PTR, c_int, _PTR, _PTR,
                                   c_int, c_int, c_int, _PTR, _PTR, _PTR, _PTR, _PTR, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_rgdcn_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, c_int, _PTR, c_int, c_int, c_int, c_int, _PTR,
                                   _PTR, c_size_t, _PTR]),
    "rgnn_rgdcn_backward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, c_int, c_int, _PTR, c_int, c_int, c_int, _PTR, _PTR,
                                    _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_plan_set_num_targets": (c_int, [_PTR, c_int32]),
    "rgnn_segment_aggregate": (c_int, [_PTR, _PTR, c_int32, c_int, _PTR, _PTR]),
    "rgnn_edge_aggregate_forward": (c_int, [_PTR, _PTR, c_int32, _PTR, c_int, _PTR, _PTR]),
    "rgnn_edge_aggregate_backward": (c_int, [_PTR, _PTR, c_int32, _PTR, c_int, _PTR, _PTR]),
    "rgnn_dense_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32]),
    "rgnn_dense_forward": (c_int, [_PTR, c_int32, c_int32, _PTR, c_int32, _PTR, c_int, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_dense_backward": (c_int, [_PTR, c_int32, c_int32, _PTR, c_int32, _PTR, _PTR, _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_layer_norm": (c_int, [_PTR, c_int32, c_int32, _PTR, _PTR, _PTR, _PTR]),
    "rgnn_halo_plan_create": (c_int, [ctypes.POINTER(c_void_p), c_int32, c_int32, _PTR, c_int32, _PTR, _PTR, _PTR]),
    "rgnn_halo_plan_destroy": (c_int, [_PTR]),
    "rgnn_halo_plan_num_own": (c_int32, [_PTR]),
    "rgnn_halo_plan_num_halo": (c_int32, [_PTR]),
    "rgnn_halo_plan_num_edges": (c_int64, [_PTR, c_int32]),
    "rgnn_halo_plan_graph": (c_void_p, [_PTR]),
    "rgnn_halo_plan_export": (c_int, [_PTR, _PTR, _PTR, _PTR, _PTR, _PTR]),
    "rgnn_halo_plan_attach": (c_int, [_PTR, _PTR, _PTR, _PTR]),
    "rgnn_halo_exchange": (c_int, [_PTR, c_int, c_int32, _PTR]),
    "rgnn_halo_exchange_overlapped": (c_int, [_PTR, c_int, c_int32, _PTR]),
    "rgnn_halo_plan_attach_grad": (c_int, [_PTR, _PTR, _PTR, _PTR, _PTR]),
    "rgnn_halo_plan_build_reverse": (c_int, [_PTR, _PTR]),
    "rgnn_halo_plan_num_reverse": (c_int64, [_PTR]),
    "rgnn_halo_plan_export_reverse": (c_int, [_PTR, _PTR, _PTR, _PTR, _PTR]),
    "rgnn_halo_exchange_backward": (c_int, [_PTR, c_int, c_int32, _PTR, _PTR, _PTR]),
    "rgnn_peer_alloc": (c_int, [ctypes.POINTER(c_void_p), c_size_t, _PTR]),
    "rgnn_peer_open": (c_int, [_PTR, ctypes.POINTER(c_void_p)]),
    "rgnn_peer_close": (c_int, [_PTR]),
    "rgnn_peer_free": (c_int, [_PTR]),
    "rgnn_rgcn_stack_forward": (c_int, [_PTR, _PTR, c_int32, c_int32, _PTR, _PTR, c_int, c_int, c_int,
                                        _PTR, _PTR, c_size_t, _PTR]),
    "rgnn_pack_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "rgnn_pack_minibatch": (c_int, [c_int64, c_int64, c_int32, _PTR, _PTR, _PTR, _PTR, c_int32, _PTR, _PTR, c_int32, _PTR,
                                    _PTR, _PTR, c_int64, c_int32, c_int32, _PTR, _PTR, _PTR, _PTR, _PTR, _PTR, _PTR, _PTR,
                                    c_size_t, _PTR]),
}
OPTIONAL_SYMBOLS = set()

_lib = None
_lib_lock = threading.Lock()


def library_path() -> str:
    return _build.LIB_PATH


def load_library(build_if_missing: bool = True):
    """dlopen lib/librgnn.so and bind every symbol.  Fails loudly (RgnnError) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        path = _build.LIB_PATH
        if not os.path.exists(path):
            if not build_if_missing:
                raise RgnnError(RGNN_E_INVALID, "librgnn.so not found at %s" % path)
            try:
                _build.build()
            except Exception as exc:   # no nvcc / compile error: there is no fallback path by design
                raise RgnnError(RGNN_E_INVALID, "librgnn.so is missing and could not be built: %s" % exc)
        lib = ctypes.CDLL(path)
        for name, (restype, argtypes) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                if name in OPTIONAL_SYMBOLS:
                    continue
                raise RgnnError(RGNN_E_INVALID, "librgnn.so at %s does not export %s (stale build?)" % (path, name))
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return _lib


def check(code: int):
    if code != RGNN_OK:
        msg = load_library().rgnn_last_error()
        raise RgnnError(code, msg.decode("utf-8", "replace") if msg else "unknown error")


def launch_count() -> int:
    """Kernels launched by librgnn in this process so far (bench.py 'gpu_launches')."""
    return int(load_library().rgnn_launch_count())


_weight_cache_on = False
# data_ptr -> (Tensor._version, weakref to the tensor that owns the memory) of every weight passed down while the cache is on
_weight_versions: Dict[int, tuple] = {}


def refuse_under_capture(what: str):
    """Raise RgnnError if the current stream is capturing a CUDA graph: for the calls that synchronise or free device
    memory, which would otherwise invalidate the capture halfway through."""
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise RgnnError(RGNN_E_INVALID, "%s cannot run during CUDA-graph capture" % what)


def set_weight_cache(enable: bool):
    """Static-weight mode (inference / benchmarking): keep the GEMM's packed weight images across calls
    (rgnn_set_weight_cache in include/rgnn.h).  The library keys the images on device POINTERS; this layer makes that
    safe: an in-place update (``Tensor._version`` changed) or the death of the tensor that owned a cached address
    (its memory may since belong to a different weight) flushes the cache the next time that address is passed down.
    Turning the cache off clears it, and clearing it frees the images that CUDA graphs captured with the cache on read:
    such graphs must not be replayed afterwards."""
    global _weight_cache_on
    refuse_under_capture("set_weight_cache (it clears the weight cache with cudaFree)")
    check(load_library().rgnn_set_weight_cache(1 if enable else 0))
    _weight_cache_on = bool(enable)
    _weight_versions.clear()


def weight_cache_clear():
    refuse_under_capture("weight_cache_clear (cudaFree)")
    check(load_library().rgnn_weight_cache_clear())
    _weight_versions.clear()


def _owner(t: torch.Tensor) -> torch.Tensor:
    """The tensor whose lifetime bounds the memory ``t`` points into (a view's base)."""
    base = t._base
    return base if base is not None else t


def note_weights(tensors):
    """Called by the layer functions with every WEIGHT tensor they are about to pass down (not with adjacency lists or
    gradient buffers)."""
    if not _weight_cache_on:
        return
    import weakref
    stale = False
    for t in tensors:
        old = _weight_versions.get(t.data_ptr())
        if old is not None:
            old_ver, old_ref = old
            owner = old_ref()
            # a dead owner means the address may have been recycled for a different weight; a live but different owner at
            # the same address IS a different allocation (two live tensors cannot overlap unless they share a base)
            if owner is None or old_ver != t._version or owner is not _owner(t):
                stale = True
    dead = [k for k, (_, r) in _weight_versions.items() if r() is None] if len(_weight_versions) > 4096 else []
    if stale or dead:
        # checked before any bookkeeping changes, so that the next eager call still sees the weight as stale
        refuse_under_capture("flushing the weight cache (a weight changed in place or was reallocated since it was "
                             "cached; the flush calls cudaFree)")
    for t in tensors:
        _weight_versions[t.data_ptr()] = (t._version, weakref.ref(_owner(t)))
    for k in dead:                                        # forget addresses whose owners are gone
        del _weight_versions[k]
    if stale or dead:
        check(load_library().rgnn_weight_cache_clear())


def current_stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t: torch.Tensor, what: str):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor, got %r" % (what, type(t)))
    if not t.is_cuda:
        raise RgnnError(RGNN_E_INVALID, "%s lives on %s: this engine has no CPU path -- move it to a CUDA device"
                        % (what, t.device))


def as_f32(t: torch.Tensor, what: str) -> torch.Tensor:
    require_cuda(t, what)
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def ptr_table(tensors: Sequence[torch.Tensor], weights: bool = True):
    """Host array of device pointers (the 'host array of L device pointers' of include/rgnn.h).  ``weights=False`` for
    tables that are not layer weights (adjacency lists, gradient buffers): those never enter the weight-image cache."""
    if weights:
        note_weights(tensors)
    arr = (c_void_p * max(len(tensors), 1))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def workspace(device: torch.device, nbytes: int) -> torch.Tensor:
    """Scratch for one library call, from torch's caching allocator.  One allocation per call (not a grow-only global
    buffer): the allocator is stream-ordered and capture-safe, so a block recorded into a CUDA graph stays owned by that
    graph's private pool and a later, larger request can never hand it to somebody else (ADVICE r1: a replayed graph was
    writing into a freed global workspace); callers on several streams get distinct blocks."""
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def output_rows(plan: "GraphPlan", dim: int, device) -> torch.Tensor:
    """[V, dim] result buffer of a layer call.  Kernels write rows [0, num_targets) only (rgnn_plan_set_num_targets): on a
    restricted plan the remaining (halo) rows are zero-filled so that nothing downstream reads uninitialised memory."""
    if getattr(plan, "num_targets", plan.num_nodes) < plan.num_nodes:
        return torch.zeros((plan.num_nodes, dim), dtype=torch.float32, device=device)
    return torch.empty((plan.num_nodes, dim), dtype=torch.float32, device=device)


class GraphPlan:
    """Device-resident structure of one batch (CSR by target over all edge types).

    Built once per batch from the task batcher's output (tasks/ppi_task.py:197-256: per-type int32
    [E, 2] adjacency lists with node ids already offset per graph) and reused by every layer and
    timestep.  ``adjacency_lists`` may be CUDA tensors, CPU tensors or numpy arrays (host inputs are
    copied to ``device`` like a feed_dict would).
    """

    def __init__(self, adjacency_lists: Sequence, num_nodes: int, device: Optional[torch.device] = None,
                 validate: bool = True):
        """validate=True: synchronise and raise RgnnError if an adjacency list holds a node id outside [0, V)
        (what TF does at sess.run).  validate=False: fully asynchronous build; ``check()`` reports later.

        The plan is built on the current stream and may be used on any stream: the first use on another stream waits for
        the build, and ``close()`` frees the plan after the work queued on every stream it was used on.  Inside a
        CUDA-graph capture only validate=False is allowed (validation synchronises)."""
        if validate:
            refuse_under_capture("GraphPlan(validate=True) (it synchronises the stream; build with validate=False inside "
                                 "a capture)")
        lib = load_library()
        adj: List[torch.Tensor] = []
        for a in adjacency_lists:
            if not isinstance(a, torch.Tensor):
                a = torch.as_tensor(a)
            if device is None and a.is_cuda:
                device = a.device
            adj.append(a)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
        if device is None:
            raise RgnnError(RGNN_E_INVALID, "GraphPlan needs a CUDA device: this engine has no CPU path")
        device = torch.device(device)
        dev_adj = []
        for a in adj:
            a = a.reshape(-1, 2)
            if a.dtype != torch.int32:
                a = a.to(torch.int32)
            a = a.to(device, non_blocking=True).contiguous()
            dev_adj.append(a)
        self.device = device
        self.adjacency_lists = dev_adj            # keep the inputs alive / available to callers
        self.num_nodes = int(num_nodes)
        self.num_edge_types = len(dev_adj)
        counts = (c_int64 * max(len(dev_adj), 1))(*[int(a.shape[0]) for a in dev_adj])
        ptrs = ptr_table(dev_adj, weights=False)
        handle = c_void_p()
        self._stream = torch.cuda.current_stream(device)      # creation stream: the library frees the plan on it
        self._other_streams: Dict[int, torch.cuda.Stream] = {}
        self._built = None
        with torch.cuda.device(device):
            check(lib.rgnn_plan_create_ex(ctypes.byref(handle), self.num_nodes, self.num_edge_types, ptrs, counts,
                                          0 if validate else 1, self._stream.cuda_stream))
            if not validate and not torch.cuda.is_current_stream_capturing():
                # a deferred build is still running on the creation stream: other streams wait for this event first (an
                # event recorded during a capture cannot be waited on eagerly; a captured build is ordered by its graph)
                self._built = torch.cuda.Event()
                self._built.record(self._stream)
        self._handle = handle
        self.num_edges = int(lib.rgnn_plan_num_edges(handle))

    @classmethod
    def from_handle(cls, handle, num_nodes: int, num_edge_types: int, num_edges: int, device, num_targets=None,
                    owner=None, adjacency_lists=None) -> "GraphPlan":
        """Wrap an rgnn_plan_t that somebody else owns (rgnn_halo_plan_graph): usable wherever a GraphPlan is, never
        destroyed by this object; ``owner`` is kept alive with it."""
        self = cls.__new__(cls)
        self.device = torch.device(device)
        self.adjacency_lists = adjacency_lists
        self.num_nodes, self.num_edge_types, self.num_edges = int(num_nodes), int(num_edge_types), int(num_edges)
        self._handle = c_void_p(handle) if not isinstance(handle, c_void_p) else handle
        self._borrowed, self._owner = True, owner
        if num_targets is not None:
            self.num_targets = int(num_targets)
        return self

    @property
    def handle(self):
        if self._handle is None:
            raise RgnnError(RGNN_E_INVALID, "GraphPlan used after close()")
        self._note_stream()
        return self._handle

    def _note_stream(self):
        """Called before work that reads the plan is queued on the current stream.  On a stream other than the creation
        stream, the first use waits for a deferred build and the stream is remembered for close().  Work queued during a
        CUDA-graph capture runs at replay, on the replaying stream: the caller keeps the plan alive while the graph is used."""
        stream = getattr(self, "_stream", None)
        if stream is None:                                     # a borrowed handle: its owner orders its lifetime
            return
        s = torch.cuda.current_stream(self.device)
        if s.cuda_stream == stream.cuda_stream or s.cuda_stream in self._other_streams:
            return
        if torch.cuda.is_current_stream_capturing():
            return
        if self._built is not None:
            s.wait_event(self._built)
        self._other_streams[s.cuda_stream] = s

    # ---- index views used by the differentiable building blocks (ops.py); built lazily, cached ----
    def _cached(self, key, make):
        cache = self.__dict__.setdefault("_derived", {})
        if key not in cache:
            # what make() records in a capture is computed only when the graph replays, but the cache would keep it for
            # every later eager call (and torch.bincount synchronises): build the views eagerly, before capturing
            refuse_under_capture("building the plan's index views / regrouped plans for the training paths on first use "
                                 "(run one forward and backward on this plan eagerly before capturing)")
            cache[key] = make()
        return cache[key]

    def _lists(self) -> List[torch.Tensor]:
        """The adjacency lists the plan was built from; a plan wrapped around a device-built handle has none."""
        if self.adjacency_lists is None:
            raise RgnnError(RGNN_E_INVALID,
                            "this plan wraps a graph built inside the library (ShardedGraph.plan) and has no adjacency lists, "
                            "which the differentiable (training) layer paths need.  To train on a node-range partition, use "
                            "GraphPlan(NodeRangePartition.local_adjacency_lists, n_local).set_num_targets(n_own) with the "
                            "states exchanged by NodeRangePartition.exchange")
        self._note_stream()
        return self.adjacency_lists

    @property
    def message_sources(self) -> torch.Tensor:
        """int64 [M]: source of every message, type-major concatenation order (gnns/rgcn.py:85,108)."""
        return self._cached("src", lambda: torch.cat([a[:, 0] for a in self._lists()]).long())

    @property
    def message_targets(self) -> torch.Tensor:
        """int64 [M]: target of every message (gnns/rgcn.py:78)."""
        return self._cached("tgt", lambda: torch.cat([a[:, 1] for a in self._lists()]).long())

    @property
    def message_types(self) -> torch.Tensor:
        return self._cached("typ", lambda: torch.cat([torch.full((a.shape[0],), l, dtype=torch.long, device=self.device)
                                                      for l, a in enumerate(self._lists())]))

    @property
    def type_offsets(self) -> List[int]:
        off = [0]
        for a in self._lists():
            off.append(off[-1] + int(a.shape[0]))
        return off

    @property
    def in_degree(self) -> torch.Tensor:
        """float32 [V]: incoming messages per node over all types (the segment sizes of tf.unsorted_segment_mean)."""
        return self._cached("indeg", lambda: torch.bincount(self.message_targets, minlength=self.num_nodes).float())

    def regrouped(self, by: str) -> "GraphPlan":
        """A plan over the SAME messages (same type-major row order of per-edge matrices) whose segments are
        'source': the source node; 'source_type': (source, type) -> segment u*L + l; 'target_type': (target, type).
        Segment-summing per-edge gradients with these plans is the (deterministic) backward of the gathers."""
        L = self.num_edge_types

        def make():
            lists = []
            for l, a in enumerate(self._lists()):
                src, tgt = a[:, 0], a[:, 1]
                if by == "source":
                    lists.append(torch.stack([tgt, src], dim=1))
                elif by == "source_type":
                    lists.append(torch.stack([tgt, src * L + l], dim=1))
                elif by == "target_type":
                    lists.append(torch.stack([src, tgt * L + l], dim=1))
                else:
                    raise RgnnError(RGNN_E_INVALID, "unknown regrouping '%s'" % by)
            n = self.num_nodes if by == "source" else self.num_nodes * L
            return GraphPlan(lists, n, device=self.device, validate=False)
        return self._cached("plan_" + by, make)

    def set_num_targets(self, num_targets: int) -> "GraphPlan":
        """Sharded execution: only rows [0, num_targets) are wanted as outputs (owned nodes first, halo nodes after them,
        as NodeRangePartition numbers them).  See rgnn_plan_set_num_targets in include/rgnn.h."""
        check(load_library().rgnn_plan_set_num_targets(self.handle, int(num_targets)))
        self.num_targets = int(num_targets)
        return self

    def check(self):
        """Synchronise the creation stream and raise if the index-range check failed (deferred validation)."""
        check(load_library().rgnn_plan_status(self.handle))

    def export(self) -> Dict[str, torch.Tensor]:
        """Copies of the plan arrays (tests / debugging)."""
        lib = load_library()
        m = max(self.num_edges, 1)
        out = {
            "seg_off": torch.empty(self.num_nodes + 1, dtype=torch.int32, device=self.device),
            "e_src": torch.empty(m, dtype=torch.int32, device=self.device),
            "e_type": torch.empty(m, dtype=torch.int32, device=self.device),
            "e_orig": torch.empty(m, dtype=torch.int32, device=self.device),
        }
        with torch.cuda.device(self.device):
            check(lib.rgnn_plan_export(self.handle, out["seg_off"].data_ptr(), out["e_src"].data_ptr(),
                                       out["e_type"].data_ptr(), out["e_orig"].data_ptr(),
                                       current_stream_ptr(self.device)))
        for k in ("e_src", "e_type", "e_orig"):
            out[k] = out[k][: self.num_edges]
        return out

    def close(self):
        """Free the plan.  The library frees it stream-ordered on the creation stream; that stream first waits for the
        work queued so far on every other stream the plan was used on (else the next allocation on the creation stream,
        typically the next batch's plan, could reuse the memory while that work still reads it)."""
        if getattr(self, "_handle", None) is not None:
            if not getattr(self, "_borrowed", False):
                if torch.cuda.is_current_stream_capturing():
                    # e.g. the previous batch's plan garbage-collected inside a capture: freeing it now would invalidate
                    # the capture, so it is freed by the next close() outside one
                    _capture_pending.append(self._close_args())
                else:
                    for args in _capture_pending + [self._close_args()]:
                        _destroy(*args)
                    _capture_pending.clear()
            self._handle = None

    def _close_args(self):
        return self._handle, getattr(self, "_stream", None), list(getattr(self, "_other_streams", {}).values()), \
            self.adjacency_lists or []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


_capture_pending: List[tuple] = []     # plans closed during a CUDA-graph capture, freed by the next close() outside one


def _destroy(handle, stream, other_streams, adjacency_lists):
    for s in other_streams:
        stream.wait_stream(s)
        for a in adjacency_lists:
            a.record_stream(s)
    load_library().rgnn_plan_destroy(handle)


def resolve_plan(node_embeddings: torch.Tensor, adjacency_lists, plan: Optional[GraphPlan]) -> GraphPlan:
    """Layer functions accept either raw adjacency lists (reference call convention) or a GraphPlan."""
    if plan is not None:
        return plan
    if isinstance(adjacency_lists, GraphPlan):
        return adjacency_lists
    refuse_under_capture("a layer called with raw adjacency lists (it builds and validates a plan, which synchronises; "
                         "pass a GraphPlan built before the capture)")
    return GraphPlan(adjacency_lists, node_embeddings.shape[0], device=node_embeddings.device)

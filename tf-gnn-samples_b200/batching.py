"""Batch construction: the host-side tensor contract the hot path consumes.

Mirrors the reference's task batchers (tasks/ppi_task.py:197-256, tasks/qm9_task.py:200-261,
tasks/varmisuse_task.py:451-538): graphs are packed into one block-diagonal graph by offsetting
node ids, per-type adjacency lists are concatenated, in-degrees are concatenated along axis 1.
The reference's datasets are not shipped (data/ppi, data/varmisuse) or not available on the GPU
box (data/qm9), so the generators below produce seeded, shape-matched synthetic graphs
(SURVEY.md 8d / Appendix B).  Everything here is numpy on the host, like the reference, except DeviceGraphSet at the end:
the same batches packed on the GPU from a data set uploaded once (rgnn_pack_minibatch).
"""
from typing import Dict, Iterator, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np


class GraphSample(NamedTuple):
    """tasks/ppi_task.py:19-23 (without the labels, which belong to the task head, not the hot path)."""
    adjacency_lists: List[np.ndarray]                      # L x int32 [E_l, 2], (src, tgt), node ids local to the graph
    type_to_node_to_num_incoming_edges: np.ndarray         # [L, V_graph]
    node_features: np.ndarray                              # [V_graph, D0] float32


class Batch(NamedTuple):
    """What a reference MinibatchData feed_dict carries for the GNN layers (tasks/sparse_graph_task.py:139-149)."""
    node_features: np.ndarray                              # float32 [V, D0]
    adjacency_lists: List[np.ndarray]                      # L x int32 [E_l, 2]
    type_to_num_incoming_edges: np.ndarray                 # float32 [L, V]
    num_graphs: int
    num_nodes: int
    num_edges: int                                         # sum_l E_l: the reference's edges/sec counter (sparse_graph_model.py:285)
    graph_node_offsets: np.ndarray                         # int64 [num_graphs + 1]


def _in_degrees(adj: Sequence[np.ndarray], num_nodes: int) -> np.ndarray:
    return np.stack([np.bincount(a[:, 1], minlength=num_nodes) if a.shape[0] else np.zeros(num_nodes, np.int64)
                     for a in adj]).astype(np.int32)


def make_ppi_like_graph(num_nodes: int = 2245, num_links: int = 59000, feature_dim: int = 50, seed: int = 0,
                        zipf_targets: bool = False) -> GraphSample:
    """One PPI-shaped graph with the reference's three edge types: 0 = fwd (u,v), 1 = self-loop (i,i),
    2 = bkwd (v,u)  (tasks/ppi_task.py:99-106,125-127,144-148; add_self_loop_edges=True,
    tie_fwd_bkwd_edges=False).  Links are i.i.d. uniform (or Zipf(1.0)-skewed targets)."""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, num_nodes, size=num_links, dtype=np.int64)
    if zipf_targets:
        p = 1.0 / np.arange(1, num_nodes + 1)
        p /= p.sum()
        tgt = rng.choice(num_nodes, size=num_links, p=p).astype(np.int64)
        tgt = rng.permutation(num_nodes)[tgt]          # hubs are not the low ids
    else:
        tgt = rng.integers(0, num_nodes, size=num_links, dtype=np.int64)
    fwd = np.stack([src, tgt], axis=1).astype(np.int32)
    loops = np.stack([np.arange(num_nodes), np.arange(num_nodes)], axis=1).astype(np.int32)
    bkwd = np.stack([tgt, src], axis=1).astype(np.int32)
    adj = [fwd, loops, bkwd]
    feats = rng.standard_normal((num_nodes, feature_dim)).astype(np.float32)
    return GraphSample(adj, _in_degrees(adj, num_nodes), feats)


def make_qm9_like_graph(rng: np.random.Generator, feature_dim: int = 15, add_self_loop_edges: bool = False) -> GraphSample:
    """One molecule-shaped graph (QM9 statistics measured in SURVEY.md Appendix B: 3..29 nodes, mean 18,
    ~1.03 bonds per node, bond types 1-4) laid out like tasks/qm9_task.py:114-147 with
    tie_fwd_bkwd_edges=True: both directions of a bond live in the bond's type, adjacency sorted by (src, dst)."""
    n = int(np.clip(round(rng.normal(18.0, 3.0)), 3, 29))
    edges = []
    for v in range(1, n):                                   # random spanning tree
        edges.append((int(rng.integers(0, v)), v))
    for _ in range(max(0, int(round(0.035 * n + rng.random())))):   # a few ring closures
        a, b = int(rng.integers(0, n)), int(rng.integers(0, n))
        if a != b:
            edges.append((a, b))
    num_types = 4 + (1 if add_self_loop_edges else 0)
    shift = 1 if add_self_loop_edges else 0
    per_type = [[] for _ in range(num_types)]
    if add_self_loop_edges:
        per_type[0] = [(i, i) for i in range(n)]
    for (a, b) in edges:
        t = int(rng.choice(4, p=[0.86, 0.09, 0.03, 0.02])) + shift
        per_type[t].append((a, b))
        per_type[t].append((b, a))
    adj = []
    for lst in per_type:
        arr = np.array(sorted(lst), dtype=np.int32).reshape(-1, 2)
        adj.append(arr)
    feats = rng.standard_normal((n, feature_dim)).astype(np.float32)
    return GraphSample(adj, _in_degrees(adj, n), feats)


def make_qm9_like_graphs(num_graphs: int, seed: int = 0, add_self_loop_edges: bool = False) -> List[GraphSample]:
    rng = np.random.default_rng(seed)
    return [make_qm9_like_graph(rng, add_self_loop_edges=add_self_loop_edges) for _ in range(num_graphs)]


# ---- PPI files (tasks/ppi_task.py:68-160; the dgl "ppi.zip" layout: <fold>_graph.json, _feats.npy, _labels.npy, _graph_id.npy) ----
def load_ppi_fold(data_dir: str, fold: str = "train", add_self_loop_edges: bool = True, tie_fwd_bkwd_edges: bool = False):
    """Read one PPI data fold the way PPI_Task.__load_data does and return (graphs, labels): one GraphSample per graph id in
    order of first appearance, node ids shifted so every graph starts at 0 (:115-121,136-141), edge types in the reference's
    order -- 0 = forward links in file order, then the self-loop type if enabled (one (i, i) per node, in-degree 1), then the
    backward type (tgt, src) unless directions are tied (:99-106).  ``labels``: per graph a float32 [V_g, num_labels] array.
    (The data set itself is not shipped with the reference; the format is the public dgl download named at :69.)"""
    import json
    import os
    if fold not in ("train", "valid", "test"):
        raise ValueError("Unknown data fold '%s'" % str(fold))
    with open(os.path.join(data_dir, "%s_graph.json" % fold)) as f:
        links = json.load(f)["links"]
    feats = np.load(os.path.join(data_dir, "%s_feats.npy" % fold))
    labels = np.load(os.path.join(data_dir, "%s_labels.npy" % fold))
    graph_id = np.load(os.path.join(data_dir, "%s_graph_id.npy" % fold))
    num_types = 1 + (1 if add_self_loop_edges else 0) + (0 if tie_fwd_bkwd_edges else 1)
    self_type = 1 if add_self_loop_edges else None
    bkwd_type = None if tie_fwd_bkwd_edges else num_types - 1
    # graphs in order of first appearance; offset = id of the first node of the graph
    order, first = [], {}
    for node, g in enumerate(graph_id.tolist()):
        if g not in first:
            first[g] = node
            order.append(g)
    nodes_of = {g: np.nonzero(graph_id == g)[0] for g in order}
    src = np.asarray([e["source"] for e in links], dtype=np.int64)
    tgt = np.asarray([e["target"] for e in links], dtype=np.int64)
    link_graph = graph_id[src] if len(links) else np.zeros(0, dtype=graph_id.dtype)
    graphs, graph_labels = [], []
    for g in order:
        ids = nodes_of[g]
        n, off = int(ids.shape[0]), first[g]
        sel = link_graph == g                                   # links are assigned to the graph of their SOURCE (:137)
        fwd = np.stack([src[sel] - off, tgt[sel] - off], axis=1).astype(np.int32).reshape(-1, 2)
        adj = [None] * num_types
        adj[0] = fwd
        if self_type is not None:
            adj[self_type] = np.stack([np.arange(n), np.arange(n)], axis=1).astype(np.int32)
        if bkwd_type is not None:
            adj[bkwd_type] = fwd[:, ::-1].copy()
        graphs.append(GraphSample(adj, _in_degrees(adj, n), feats[ids].astype(np.float32)))
        graph_labels.append(labels[ids].astype(np.float32))
    return graphs, graph_labels


# ---- real QM9 records (data/qm9/*.jsonl.gz of the reference; tasks/qm9_task.py:85-147) ----
def qm9_num_edge_types(raw_graphs: Sequence[Dict], add_self_loop_edges: bool = True, tie_fwd_bkwd_edges: bool = True) -> int:
    """tasks/qm9_task.py:89-96: max bond type (+1 for the self-loop type 0), doubled when directions are untied."""
    num_fwd = max(max(e[1] for e in g["graph"]) for g in raw_graphs if len(g["graph"]))
    if add_self_loop_edges:
        num_fwd += 1
    return num_fwd * (1 if tie_fwd_bkwd_edges else 2)


def qm9_graph_to_sample(raw: Dict, num_edge_types: int, add_self_loop_edges: bool = True,
                        tie_fwd_bkwd_edges: bool = True) -> GraphSample:
    """One record {"graph": [(src, bond, dst)...], "node_features": [[15 floats]...]} -> per-type adjacency lists and
    in-degrees exactly as __graph_to_adjacency_lists builds them (tasks/qm9_task.py:114-147): bond types start at 1
    (0 is the self-loop type when enabled, else types are shifted down by one); tied directions put (dst, src) in the
    same type; each list is sorted by (src, dst); untied directions append the reversed lists as extra types.
    (tie_fwd_bkwd_edges=False cannot actually run in the reference: :139-145 appends to the list it enumerates and raises
    IndexError on the first molecule -- tests/test_reference_batcher_pin.py.  What is built here is what that loop evidently
    means, in-degree quirk included; every configuration the reference CAN run is pinned bit-exact by the same test.)"""
    num_nodes = len(raw["node_features"])
    lists: List[List] = [[] for _ in range(num_edge_types)]
    indeg = np.zeros((num_edge_types, num_nodes), dtype=np.float64)
    for src, e, dst in raw["graph"]:
        t = e if add_self_loop_edges else e - 1
        lists[t].append((src, dst))
        indeg[t, dst] += 1
        if tie_fwd_bkwd_edges:
            lists[t].append((dst, src))
            indeg[t, src] += 1
    if add_self_loop_edges:
        for v in range(num_nodes):
            indeg[0, v] = 1
            lists[0].append((v, v))
    adj = [np.array(sorted(l), dtype=np.int32).reshape(-1, 2) for l in lists]
    if not tie_fwd_bkwd_edges:
        half = num_edge_types // 2
        adj = adj[:half]
        for t in range(half):
            adj.append(np.array(sorted((y, x) for (x, y) in adj[t]), dtype=np.int32).reshape(-1, 2))
            for (x, y) in adj[t]:
                indeg[half + t][y] += 1      # as the reference counts it (:143-144): at the forward edge's target y,
                                             # although the reversed edge (y, x) arrives at x -- kept for identical feeds
    return GraphSample(adj, indeg.astype(np.float32), np.asarray(raw["node_features"], dtype=np.float32))


def load_qm9_jsonl(path: str, limit: Optional[int] = None) -> List[Dict]:
    """Read records of a reference data/qm9/*.jsonl.gz file (dpu_utils RichPath.read_by_file_suffix in the reference)."""
    import gzip
    import json
    out = []
    with gzip.open(path, "rt") as f:
        for line in f:
            out.append(json.loads(line))
            if limit is not None and len(out) >= limit:
                break
    return out


def qm9_records_from_structure(path: str, feature_dim: int = 15, seed: int = 0, num_targets: int = 13) -> List[Dict]:
    """Records in the layout of data/qm9/*.jsonl.gz rebuilt from a structure-only archive (tests/golden/make_qm9_structure.py:
    atoms per molecule + bonds of the reference's 10,000 validation molecules).  The graph structure is the real one; node
    features are seeded random numbers and targets are zero -- for timing the real batch shape, not for accuracy work."""
    z = np.load(path)
    sizes, nbonds, bonds = z["num_atoms"].astype(np.int64), z["num_bonds"].astype(np.int64), z["bonds"].astype(np.int64)
    rng = np.random.default_rng(seed)
    recs, b0 = [], 0
    for i in range(sizes.shape[0]):
        n, nb = int(sizes[i]), int(nbonds[i])
        recs.append({"id": "qm9-structure:%d" % i, "graph": bonds[b0:b0 + nb].tolist(),
                     "node_features": rng.standard_normal((n, feature_dim)).astype(np.float32),
                     "targets": [[0.0]] * num_targets})
        b0 += nb
    return recs


def qm9_batch(raw_graphs: Sequence[Dict], add_self_loop_edges: bool = True, tie_fwd_bkwd_edges: bool = True,
              task_ids: Sequence[int] = (0,), max_nodes_per_batch: Optional[int] = None):
    """Records -> (Batch, graph_nodes_list int32 [V], target_values float32 [len(task_ids), G]): the feed_dict of
    tasks/qm9_task.py:200-261 for one minibatch."""
    L = qm9_num_edge_types(raw_graphs, add_self_loop_edges, tie_fwd_bkwd_edges)
    samples = [qm9_graph_to_sample(g, L, add_self_loop_edges, tie_fwd_bkwd_edges) for g in raw_graphs]
    batch = pack_batch(samples, max_nodes_per_batch)
    G = batch.num_graphs
    sizes = np.diff(batch.graph_node_offsets)
    graph_nodes_list = np.repeat(np.arange(G, dtype=np.int32), sizes)
    targets = np.array([[raw_graphs[g]["targets"][t][0] for g in range(G)] for t in task_ids], dtype=np.float32)
    return batch, graph_nodes_list, targets


def make_typed_random_graph(num_nodes: int, num_edges: int, type_fractions: Sequence[float], feature_dim: int,
                            seed: int = 0) -> GraphSample:
    """Uniform random multigraph with the edges split over L types in the given proportions
    (VarMisuse-shaped config: SURVEY.md 8d config 5)."""
    rng = np.random.default_rng(seed)
    fr = np.asarray(type_fractions, dtype=np.float64)
    counts = np.floor(fr / fr.sum() * num_edges).astype(np.int64)
    counts[0] += num_edges - counts.sum()
    adj = []
    for c in counts:
        a = np.stack([rng.integers(0, num_nodes, size=int(c)), rng.integers(0, num_nodes, size=int(c))], axis=1)
        adj.append(a.astype(np.int32))
    feats = rng.standard_normal((num_nodes, feature_dim)).astype(np.float32)
    return GraphSample(adj, _in_degrees(adj, num_nodes), feats)


def pack_batch(graphs: Sequence[GraphSample], max_nodes_per_batch: Optional[int] = None) -> Batch:
    """The packing loop of tasks/ppi_task.py:213-251: add graphs while node_offset + |graph| <
    max_nodes_per_batch, shift node ids by the running offset, concatenate per type; an edge type with no
    edge in the batch becomes np.zeros((0, 2)) (:246-249)."""
    num_types = len(graphs[0].adjacency_lists)
    feats, indeg, offsets = [], [], [0]
    adj: List[List[np.ndarray]] = [[] for _ in range(num_types)]
    node_offset = 0
    for g in graphs:
        n = g.node_features.shape[0]
        if max_nodes_per_batch is not None and not (node_offset + n < max_nodes_per_batch):
            break
        feats.append(g.node_features)
        for i in range(num_types):
            adj[i].append(g.adjacency_lists[i].reshape(-1, 2) + node_offset)
        indeg.append(g.type_to_node_to_num_incoming_edges)
        node_offset += n
        offsets.append(node_offset)
    merged, num_edges = [], 0
    for i in range(num_types):
        a = np.concatenate(adj[i]).astype(np.int32) if len(adj[i]) > 0 else np.zeros((0, 2), dtype=np.int32)
        num_edges += a.shape[0]
        merged.append(a)
    return Batch(node_features=np.concatenate(feats, axis=0).astype(np.float32),
                 adjacency_lists=merged,
                 type_to_num_incoming_edges=np.concatenate(indeg, axis=1).astype(np.float32),
                 num_graphs=len(feats), num_nodes=node_offset, num_edges=num_edges,
                 graph_node_offsets=np.asarray(offsets, dtype=np.int64))


def batch_bounds(num_nodes: Sequence[int], max_nodes_per_batch: int) -> Iterator[Tuple[int, int]]:
    """The minibatch boundaries of tasks/ppi_task.py:211-256 (same in qm9_task.py:212-261) from the graphs' node counts alone:
    add graphs in order while node_offset + |graph| < max_nodes_per_batch, emit, continue with the graph that did not fit.
    Yields (index of the first graph, number of graphs).  A graph with >= max_nodes_per_batch nodes can never be packed --
    the reference then spins on an empty batch (np.concatenate of an empty list raises); here it is a ValueError when the
    loop reaches it."""
    start, count = 0, len(num_nodes)
    while start < count:
        n = int(num_nodes[start])
        if not (n < max_nodes_per_batch):
            raise ValueError("graph %d has %d nodes: does not fit max_nodes_per_batch=%d" % (start, n, max_nodes_per_batch))
        end, offset = start, 0
        while end < count and offset + int(num_nodes[end]) < max_nodes_per_batch:
            offset += int(num_nodes[end])
            end += 1
        yield start, end - start
        start = end


def minibatches(graphs: Sequence[GraphSample], max_nodes_per_batch: int) -> Iterator[Tuple[Batch, int]]:
    """One epoch of minibatches, the outer loop of tasks/ppi_task.py:211-256 (same in qm9_task.py:212-261), with the
    boundaries of ``batch_bounds``.  Yields (batch, index of its first graph)."""
    for start, count in batch_bounds([g.node_features.shape[0] for g in graphs], max_nodes_per_batch):
        yield pack_batch(graphs[start:start + count]), start


def ppi_like_batch(num_graphs: int = 1, num_nodes: int = 2245, num_links: int = 59000, seed: int = 0,
                   zipf_targets: bool = False) -> Batch:
    """BASELINE config 2: one PPI-shaped graph -> V=2,245, M = 2*59,000 + 2,245 = 120,245, L=3."""
    return pack_batch([make_ppi_like_graph(num_nodes, num_links, seed=seed + i, zipf_targets=zipf_targets)
                       for i in range(num_graphs)])


def qm9_like_batch(num_graphs: int = 10000, seed: int = 0, add_self_loop_edges: bool = False) -> Batch:
    """BASELINE config 3 shape: 10k molecule graphs, ~18 nodes each, 4 bond types (5 with self loops)."""
    return pack_batch(make_qm9_like_graphs(num_graphs, seed, add_self_loop_edges))


VARMISUSE_TYPE_FRACTIONS = (0.30, 0.30, 0.15, 0.15, 0.05, 0.05)


def varmisuse_like_batch(num_nodes: int = 50000, num_edges: int = 1000000, packed_graphs: int = 0, seed: int = 0,
                         feature_dim: int = 64) -> Batch:
    """BASELINE config 5 shape: V=50k, M=1M, L=6.  packed_graphs=0 -> one random graph (worst-case halo);
    packed_graphs=g -> g equal graphs packed block-diagonally (zero-halo partition possible)."""
    if packed_graphs <= 0:
        return pack_batch([make_typed_random_graph(num_nodes, num_edges, VARMISUSE_TYPE_FRACTIONS, feature_dim, seed)])
    n, e = num_nodes // packed_graphs, num_edges // packed_graphs
    return pack_batch([make_typed_random_graph(n, e, VARMISUSE_TYPE_FRACTIONS, feature_dim, seed + i)
                       for i in range(packed_graphs)])


# ---- minibatches packed on the GPU from a device-resident graph set (rgnn_pack_minibatch in include/rgnn.h) ----
class DeviceBatch:
    """One minibatch packed on the device: the tensors of a reference feed (tasks/sparse_graph_task.py:139-149) plus the
    counters ``training.run_epoch`` reads.  ``args()`` returns what ``training.device_args`` returns for the same batch, so
    ``run_epoch(..., batches=graph_set.minibatches(budget, order), to_device=lambda b: b.args())`` trains on it unchanged."""

    def __init__(self, graph_set, num_graphs, num_nodes, num_edges, node_tensors, adjacency_lists, num_incoming,
                 graph_nodes_list, graph_tensors, status):
        self.graph_set = graph_set
        self.num_graphs, self.num_nodes, self.num_edges = num_graphs, num_nodes, num_edges
        self.node_features = node_tensors[0]                # float32 [V, D0]
        self.node_tensors = node_tensors                    # [0] = features, then the set's extra per-node tensors
        self.adjacency_lists = adjacency_lists              # L x int32 [E_l, 2]; a type without edges is [0, 2]
        self.type_to_num_incoming_edges = num_incoming      # float32 [L, V]
        self.graph_nodes_list = graph_nodes_list            # int32 [V]
        self.graph_tensors = graph_tensors                  # float32 [T_k, num_graphs] each
        self.status = status                                # int32 [1]: RGNN_PACK_* bits, 0 = consistent

    @property
    def batch(self) -> "DeviceBatch":
        """The counters live on the batch itself (run_epoch reads ``tb.batch.num_graphs`` of a TaskBatch)."""
        return self

    @property
    def targets(self):
        """PPI: the node labels [V, num_labels]; QM9: the target values [len(task_ids), num_graphs]."""
        kind = self.graph_set.targets_kind
        if kind == "graph":
            return self.graph_tensors[0]
        return self.node_tensors[1] if kind == "node" else None

    def args(self) -> Tuple:
        """(features, plan, num_incoming, targets[, graph_nodes_list, num_graphs]), like training.device_args.  The plan is
        built without validation (no synchronisation): the graph set checked every node id when it was uploaded."""
        from .engine import GraphPlan
        plan = GraphPlan(self.adjacency_lists, self.num_nodes, device=self.node_features.device, validate=False)
        args = (self.node_features, plan, self.type_to_num_incoming_edges, self.targets)
        if self.graph_set.targets_kind == "graph":
            args += (self.graph_nodes_list, self.num_graphs)
        return args

    def check(self):
        """Synchronise and raise RgnnError if the device-computed totals disagreed with the host's or ``order`` held an id
        outside the set (the status word of rgnn_pack_minibatch)."""
        from .engine import RGNN_E_INVALID, RgnnError
        st = int(self.status.item())
        if st != 0:
            raise RgnnError(RGNN_E_INVALID, "pack_minibatch: status %d (1 = node total, 2 = edge total differs from the "
                                            "host's; 4 = order entry outside the graph set)" % st)


class DeviceGraphSet:
    """A whole data set uploaded once, packed into minibatches on the GPU (one rgnn_pack_minibatch per batch: no per-batch
    host-to-device copy, no Python loop over graphs, no synchronisation).  Feed for feed the batches equal ``minibatches``
    over ``[graphs[i] for i in order]``, bit for bit.

    Layout (CSR over graphs, data-set order, graph-local node ids): node offsets int64 [G + 1]; per edge type edge offsets
    int64 [G + 1] and edges int32 [E_l, 2]; in-degrees float32 [L, N]; per-node tensors float32 [N, w] (``node_tensors[0]``
    is the node features; ``node_tensors`` adds more, each a per-graph sequence of [V_g, w] arrays, e.g. PPI labels);
    per-graph tensors float32 [T, G] (``graph_tensors``: one [T, G] array or a sequence of them, e.g. QM9 targets).
    ``targets`` of a batch: the first per-graph tensor if there is one (and ``args()`` then carries graph_nodes_list and
    num_graphs like a QM9 feed), else the first extra per-node tensor (a PPI feed).

    Every node id is checked against its graph's size once, here on the host (RgnnError on a violation), so the per-batch
    GraphPlan needs no validation."""

    def __init__(self, graphs: Sequence[GraphSample], device=None, node_tensors: Sequence[Sequence[np.ndarray]] = (),
                 graph_tensors=None):
        import torch
        from .engine import RGNN_E_INVALID, RgnnError
        graphs = list(graphs)
        if not graphs:
            raise ValueError("DeviceGraphSet needs at least one graph")
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        G, L = len(graphs), len(graphs[0].adjacency_lists)
        if any(len(g.adjacency_lists) != L for g in graphs):
            raise ValueError("every graph needs the same number of edge types (%d)" % L)
        sizes = np.array([g.node_features.shape[0] for g in graphs], dtype=np.int64)
        node_off = np.zeros(G + 1, dtype=np.int64)
        np.cumsum(sizes, out=node_off[1:])
        edge_counts = np.zeros((L, G), dtype=np.int64)
        edge_off, edges = [], []
        for l in range(L):
            lists = [np.asarray(g.adjacency_lists[l]).reshape(-1, 2) for g in graphs]
            edge_counts[l] = [a.shape[0] for a in lists]
            off = np.zeros(G + 1, dtype=np.int64)
            np.cumsum(edge_counts[l], out=off[1:])
            cat = np.concatenate(lists).astype(np.int64) if off[-1] > 0 else np.zeros((0, 2), dtype=np.int64)
            bad = ((cat < 0) | (cat >= np.repeat(sizes, edge_counts[l])[:, None])).any(axis=1)
            if bad.any():
                e = int(np.argmax(bad))
                g = int(np.searchsorted(off, e, side="right") - 1)
                raise RgnnError(RGNN_E_INVALID, "graph %d, edge type %d: edge %s holds a node index outside [0, %d)"
                                % (g, l, tuple(int(x) for x in cat[e]), sizes[g]))
            edge_off.append(off)
            edges.append(cat.astype(np.int32))
        indeg = [np.asarray(g.type_to_node_to_num_incoming_edges) for g in graphs]
        if any(d.shape != (L, n) for d, n in zip(indeg, sizes)):
            raise ValueError("in-degrees must be [L, V_g] for every graph")
        indeg = np.concatenate(indeg, axis=1)
        per_node = [[g.node_features for g in graphs]] + [list(t) for t in node_tensors]
        node_arrays = []
        for k, parts in enumerate(per_node):
            parts = [np.asarray(p, dtype=np.float32) for p in parts]
            if len(parts) != G or any(p.ndim != 2 or p.shape != (n, parts[0].shape[1]) for p, n in zip(parts, sizes)):
                raise ValueError("per-node tensor %d must hold one [V_g, w] array per graph, w the same for all" % k)
            node_arrays.append(np.concatenate(parts, axis=0))
        if graph_tensors is None:
            graph_tensors = []
        elif isinstance(graph_tensors, np.ndarray):
            graph_tensors = [graph_tensors]
        graph_arrays = [np.asarray(t, dtype=np.float32).reshape(-1, G) for t in graph_tensors]
        if len(node_arrays) > 8 or len(graph_arrays) > 8:       # RGNN_PACK_MAX_TENSORS
            raise ValueError("at most 8 per-node tensors (features included) and 8 per-graph tensors")

        def up(a):
            return torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        self.num_graphs, self.num_nodes, self.num_edge_types = G, int(node_off[-1]), L
        self.graph_sizes, self.edge_counts = sizes, edge_counts          # host-side counts: batch boundaries and totals
        self.node_offsets = up(node_off)
        self.edge_offsets = [up(o) for o in edge_off]
        self.adjacency_lists = [up(e) for e in edges]
        self.num_incoming = up(indeg.astype(np.float32))
        self.node_tensors = [up(a) for a in node_arrays]
        self.graph_tensors = [up(a) for a in graph_arrays]
        self.targets_kind = "graph" if graph_arrays else ("node" if len(node_arrays) > 1 else None)

    @classmethod
    def from_qm9_records(cls, records: Sequence[Dict], add_self_loop_edges: bool = True, tie_fwd_bkwd_edges: bool = True,
                         task_ids: Sequence[int] = (0,), device=None) -> "DeviceGraphSet":
        """QM9 records (load_qm9_jsonl) converted once, as qm9_batch converts them per batch; targets [len(task_ids), G]."""
        L = qm9_num_edge_types(records, add_self_loop_edges, tie_fwd_bkwd_edges)
        samples = [qm9_graph_to_sample(r, L, add_self_loop_edges, tie_fwd_bkwd_edges) for r in records]
        targets = np.array([[r["targets"][t][0] for r in records] for t in task_ids], dtype=np.float32).reshape(-1, len(records))
        return cls(samples, device, graph_tensors=targets)

    @classmethod
    def from_ppi_fold(cls, graphs: Sequence[GraphSample], labels: Sequence[np.ndarray], device=None) -> "DeviceGraphSet":
        """A PPI fold as load_ppi_fold returns it; the per-node labels [V_g, num_labels] become the batches' targets."""
        return cls(graphs, device, node_tensors=(labels,))

    def _host_order(self, order) -> np.ndarray:
        if order is None:
            return np.arange(self.num_graphs, dtype=np.int32)
        order = np.asarray(order).reshape(-1)
        if order.size and (order.min() < 0 or order.max() >= self.num_graphs):
            raise ValueError("order holds a graph index outside [0, %d)" % self.num_graphs)
        return order.astype(np.int32)

    def upload_order(self, order=None):
        """(host int32 order, device int32 copy): the epoch's graph order, checked on the host, copied once from pinned
        memory without synchronising.  None = data-set order."""
        import torch
        order = self._host_order(order)
        return order, torch.from_numpy(order).pin_memory().to(self.device, non_blocking=True)

    def pack(self, order: np.ndarray, order_dev, start: int, count: int) -> DeviceBatch:
        """Pack the graphs order[start : start + count] on the current stream.  ``order`` is the host copy of ``order_dev``
        (the totals come from it); the kernel reads ``order_dev``, so a CUDA graph that captured this call packs whatever
        order_dev holds when it is replayed."""
        import ctypes
        import torch
        from .engine import check, current_stream_ptr, load_library, ptr_table, workspace
        lib = load_library()
        L, dev = self.num_edge_types, self.device
        sel = order[start:start + count]
        V = int(self.graph_sizes[sel].sum())
        E = [int(x) for x in self.edge_counts[:, sel].sum(axis=1)]
        nodes = [torch.empty((V, t.shape[1]), dtype=torch.float32, device=dev) for t in self.node_tensors]
        adj = [torch.empty((e, 2), dtype=torch.int32, device=dev) for e in E]
        indeg = torch.empty((L, V), dtype=torch.float32, device=dev)
        gnl = torch.empty(V, dtype=torch.int32, device=dev)
        per_graph = [torch.empty((t.shape[0], count), dtype=torch.float32, device=dev) for t in self.graph_tensors]
        status = torch.empty(1, dtype=torch.int32, device=dev)
        ws_bytes = int(lib.rgnn_pack_workspace_bytes(count, L))
        ws = workspace(dev, ws_bytes)
        widths = (ctypes.c_int32 * 8)(*[t.shape[1] for t in self.node_tensors])
        rows = (ctypes.c_int32 * 8)(*[t.shape[0] for t in self.graph_tensors])
        with torch.cuda.device(dev):
            check(lib.rgnn_pack_minibatch(
                self.num_graphs, self.num_nodes, L, self.node_offsets.data_ptr(),
                ptr_table(self.edge_offsets, weights=False), ptr_table(self.adjacency_lists, weights=False),
                self.num_incoming.data_ptr(),
                len(self.node_tensors), ptr_table(self.node_tensors, weights=False), widths,
                len(self.graph_tensors), ptr_table(self.graph_tensors, weights=False), rows,
                order_dev.data_ptr(), int(start), int(count), V, (ctypes.c_int64 * L)(*E),
                ptr_table(nodes, weights=False), ptr_table(adj, weights=False), indeg.data_ptr(), gnl.data_ptr(),
                ptr_table(per_graph, weights=False), status.data_ptr(), ws.data_ptr(), ws.numel(),
                current_stream_ptr(dev)))
        return DeviceBatch(self, int(count), V, int(sum(E)), nodes, adj, indeg, gnl, per_graph, status)

    def minibatches(self, max_nodes_per_batch: int, order=None) -> Iterator[DeviceBatch]:
        """One epoch: the batches ``minibatches([graphs[i] for i in order], max_nodes_per_batch)`` yields, packed on the
        device.  ``order`` is the caller's shuffle (the reference shuffles the training fold every epoch); it is uploaded
        once.  Every boundary is computed, and a graph that can never fit raises ValueError, before anything is launched."""
        order_host = self._host_order(order)
        bounds = list(batch_bounds(self.graph_sizes[order_host], max_nodes_per_batch))
        order_host, order_dev = self.upload_order(order_host)
        for start, count in bounds:
            yield self.pack(order_host, order_dev, start, count)

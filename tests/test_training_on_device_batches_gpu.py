"""Minibatches packed on the GPU from a device-resident graph set (batching.DeviceGraphSet, rgnn_pack_minibatch) against the
host batcher, feed for feed:

* the committed feeds of the REFERENCE's own batchers (tests/golden/ref_batcher_feeds.npz, every case of batcher_cases.py);
* pack_batch under a seeded shuffle, on QM9-shaped molecules and Zipf PPI graphs, with budgets that a graph's end hits
  exactly;
* edge cases, the C ABI's refusals and its bounded writes under wrong totals, a plan and two layers on the packed lists;
* no synchronisation (one CUDA graph holds pack + plan; torch's sync debug mode stays silent) and the epoch loop.
The boundary helper shared with the host batcher is tested without a GPU.

The module's name sorts it after every module that asserts launched kernels from torch.profiler traces.  With lazy module
loading (CUDA's default), a kernel first loaded between two profiler sessions of one process was missing from the later
session's trace on the H100: run between test_buffer_contract_gpu.py and test_large_batch_training_gpu.py, this module made
three cases of the latter miss seg_reduce_kernel in their traces (they pass with CUDA_MODULE_LOADING=EAGER, and when this
module runs before any profiler session or after them)."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC      # noqa: E402

from tf_gnn_samples_b200 import batching, engine, training   # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "ref_batcher_feeds.npz")
gpu = pytest.mark.gpu


# ---- host part -------------------------------------------------------------------------------------------------------
def old_minibatch_loop(sizes, budget):
    """The loop minibatches ran before the boundary rule became batch_bounds: pack while offset + n < budget."""
    out, start = [], 0
    while start < len(sizes):
        if not (sizes[start] < budget):
            out.append(("raise", start))
            return out
        offset, end = 0, start
        for n in sizes[start:]:
            if not (offset + n < budget):
                break
            offset += n
            end += 1
        out.append((start, end - start))
        start = end
    return out


def bounds_or_raise(sizes, budget):
    out = []
    try:
        for b in batching.batch_bounds(sizes, budget):
            out.append(b)
    except ValueError as exc:
        assert "does not fit max_nodes_per_batch=%d" % budget in str(exc)
        out.append(("raise", int(str(exc).split()[1])))
    return out


def test_batch_bounds_equal_the_old_loop_on_random_sizes():
    rng = np.random.default_rng(3)
    for trial in range(300):
        sizes = [int(x) for x in rng.integers(0 if trial % 7 == 0 else 1, 40, size=int(rng.integers(0, 60)))]
        for budget in (1, 2, 17, 40, 41, 97, int(sum(sizes[:5])) if sizes else 5, 10 ** 6):
            assert bounds_or_raise(sizes, budget) == old_minibatch_loop(sizes, budget), (sizes, budget)


def test_minibatches_raise_where_the_old_loop_raised():
    graphs = batching.make_qm9_like_graphs(6, seed=2)
    sizes = [g.node_features.shape[0] for g in graphs]
    budget = max(sizes)                                 # the largest graph can never fit; batches before it are packed
    it = batching.minibatches(graphs, budget)
    seen = []
    with pytest.raises(ValueError, match="graph %d has %d nodes" % (sizes.index(budget), budget)):
        for b, first in it:
            seen.append(first)
    assert [s for s, _ in old_minibatch_loop(sizes, budget) if s != "raise"] == seen


def test_an_out_of_range_local_id_is_refused_at_upload():
    graphs = batching.make_qm9_like_graphs(5, seed=4, add_self_loop_edges=True)
    adj = [a.copy() for a in graphs[3].adjacency_lists]
    adj[1][0, 1] = graphs[3].node_features.shape[0]       # one past the graph's last node
    graphs[3] = graphs[3]._replace(adjacency_lists=adj)
    with pytest.raises(engine.RgnnError, match="graph 3, edge type 1"):
        batching.DeviceGraphSet(graphs, device="cuda")    # checked on the host before anything is uploaded
    adj[1][0, 1] = -1
    with pytest.raises(engine.RgnnError, match="outside"):
        batching.DeviceGraphSet(graphs, device="cuda")


# ---- helpers ---------------------------------------------------------------------------------------------------------
def to_np(t):
    return t.detach().cpu().numpy()


def device_feed(b, target_name):
    feed = {"initial_node_features": to_np(b.node_features), "type_to_num_incoming_edges": to_np(b.type_to_num_incoming_edges),
            "graph_nodes_list": to_np(b.graph_nodes_list), "num_graphs": np.int64(b.num_graphs),
            "num_nodes": np.int64(b.num_nodes), "num_edges": np.int64(b.num_edges), target_name: to_np(b.targets)}
    for i, a in enumerate(b.adjacency_lists):
        feed["adjacency_e%d" % i] = to_np(a)
    return feed


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def assert_batches_equal(dev, host, what=""):
    """bit-identical: features, every adjacency list (shape and edge order), in-degrees, graph ids, counters."""
    assert (dev.num_graphs, dev.num_nodes, dev.num_edges) == (host.num_graphs, host.num_nodes, host.num_edges), what
    assert np.array_equal(bits(to_np(dev.node_features)), bits(host.node_features.astype(np.float32))), what
    assert np.array_equal(bits(to_np(dev.type_to_num_incoming_edges)), bits(host.type_to_num_incoming_edges)), what
    assert len(dev.adjacency_lists) == len(host.adjacency_lists)
    for l, (a, b) in enumerate(zip(dev.adjacency_lists, host.adjacency_lists)):
        assert a.dtype == engine.torch.int32 and tuple(a.shape) == b.shape, (what, l, tuple(a.shape), b.shape)
        assert np.array_equal(to_np(a), b), (what, l)
    want_gnl = np.repeat(np.arange(host.num_graphs, dtype=np.int32), np.diff(host.graph_node_offsets))
    assert np.array_equal(to_np(dev.graph_nodes_list), want_gnl), what


def zipf_ppi_graphs(count, seed):
    rng = np.random.default_rng(seed)
    return [batching.make_ppi_like_graph(int(rng.integers(40, 2245)), int(rng.integers(0, 6000)), feature_dim=50,
                                         seed=seed + i, zipf_targets=True) for i in range(count)]


# ---- 1. pinned to the reference's own batcher ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fixture():
    return np.load(FIXTURE)


@pytest.fixture(scope="module")
def ppi_dir(tmp_path_factory):
    return BC.write_ppi_dir(str(tmp_path_factory.mktemp("ppi")), "test")


@gpu
@pytest.mark.parametrize("case", sorted(BC.QM9_CASES))
def test_qm9_device_feeds_equal_the_reference_feeds(case, fixture, cuda_device):
    params, budget = BC.QM9_CASES[case]
    recs = batching.load_qm9_jsonl(BC.QM9_SUBSET)
    gs = batching.DeviceGraphSet.from_qm9_records(recs, params.get("add_self_loop_edges", True),
                                                  params.get("tie_fwd_bkwd_edges", True), params.get("task_ids", [0]),
                                                  device=cuda_device)
    assert gs.num_edge_types == int(fixture[case + "/num_edge_types"])
    got = [device_feed(b, "target_values") for b in gs.minibatches(budget)]
    BC.compare_feeds(got, BC.unpack_feeds(fixture, case), case)


@gpu
@pytest.mark.parametrize("case", sorted(BC.PPI_CASES))
def test_ppi_device_feeds_equal_the_reference_feeds(case, fixture, ppi_dir, cuda_device):
    params, budget = BC.PPI_CASES[case]
    graphs, labels = batching.load_ppi_fold(ppi_dir, "test", params.get("add_self_loop_edges", True),
                                            params.get("tie_fwd_bkwd_edges", False))
    gs = batching.DeviceGraphSet.from_ppi_fold(graphs, labels, device=cuda_device)
    assert gs.num_edge_types == int(fixture[case + "/num_edge_types"])
    got = [device_feed(b, "target_labels") for b in gs.minibatches(budget)]
    BC.compare_feeds(got, BC.unpack_feeds(fixture, case), case)


# ---- 2. equal to the host packer under shuffling ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def qm9_like():
    return batching.make_qm9_like_graphs(20000, seed=11, add_self_loop_edges=True)


def exact_hit_budget(sizes, order, k):
    """A budget that the end of the k-th graph of the order reaches exactly: offset + n == budget, so it is excluded."""
    return int(np.sum(sizes[order[:k]]))


def check_shuffled(graphs, gs, order, budgets):
    shuffled = [graphs[i] for i in order]
    for budget in budgets:
        dev = list(gs.minibatches(budget, order))
        host = list(batching.minibatches(shuffled, budget))
        assert len(dev) == len(host), budget
        for i, (d, (h, _)) in enumerate(zip(dev, host)):
            assert_batches_equal(d, h, "budget %d batch %d" % (budget, i))
            assert int(d.status.item()) == 0


@gpu
def test_shuffled_qm9_shaped_batches_equal_pack_batch(qm9_like, cuda_device):
    gs = batching.DeviceGraphSet(qm9_like, cuda_device)
    assert gs.num_edge_types == 5 and gs.node_tensors[0].shape[1] == 15
    order = np.random.default_rng(0).permutation(len(qm9_like))
    hit = exact_hit_budget(gs.graph_sizes, order, 700)
    first = next(iter(batching.batch_bounds(gs.graph_sizes[order], hit)))
    assert first == (0, 699)                            # the 700th graph ends exactly at the budget: excluded
    check_shuffled(qm9_like, gs, order, [hit, 50000, 200000, 400000])


@gpu
def test_shuffled_zipf_ppi_batches_equal_pack_batch(cuda_device):
    graphs = zipf_ppi_graphs(14, seed=21)
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    order = np.random.default_rng(1).permutation(len(graphs))
    ends = np.cumsum(gs.graph_sizes[order])
    k = int(np.argmax(ends > gs.graph_sizes.max())) + 1         # the first budget end that every graph fits under
    hit = exact_hit_budget(gs.graph_sizes, order, max(k, 2))
    assert next(iter(batching.batch_bounds(gs.graph_sizes[order], hit))) == (0, max(k, 2) - 1)
    check_shuffled(graphs, gs, order, [hit, 2246, 5000, 12000, 10 ** 6])


# ---- 3. edge cases ---------------------------------------------------------------------------------------------------
def tiny_graph(n, lists, width=15, seed=0):
    rng = np.random.default_rng(seed)
    adj = [np.asarray(a, dtype=np.int32).reshape(-1, 2) for a in lists]
    return batching.GraphSample(adj, batching._in_degrees(adj, n), rng.standard_normal((n, width)).astype(np.float32))


@gpu
def test_empty_types_edgeless_graphs_and_single_graph_batches(cuda_device):
    graphs = [tiny_graph(4, [[(0, 1), (1, 2)], [], [(3, 0)]], seed=1),
              tiny_graph(3, [[], [], []], seed=2),                        # a graph with no edge at all
              tiny_graph(5, [[(4, 4)], [], []], seed=3),
              tiny_graph(2, [[], [], [(1, 0), (0, 1)]], seed=4)]
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    for order, budget in [([1, 2, 0, 3], 100), ([1, 3], 6), ([2, 1], 100), ([0], 5), ([1], 4), ([3, 1, 0, 2], 6)]:
        order = np.asarray(order)
        dev = list(gs.minibatches(budget, order))
        host = list(batching.minibatches([graphs[i] for i in order], budget))
        assert len(dev) == len(host)
        for d, (h, _) in zip(dev, host):
            assert_batches_equal(d, h, str((order.tolist(), budget)))
            assert tuple(d.adjacency_lists[1].shape) == (0, 2)            # type 1 has no edge anywhere
            assert d.node_features.shape[1] == 15
    one = list(gs.minibatches(5, [0]))                                     # a single-graph batch
    assert len(one) == 1 and one[0].num_graphs == 1 and one[0].num_nodes == 4
    only_edgeless = list(gs.minibatches(100, [1]))[0]
    assert only_edgeless.num_edges == 0 and all(tuple(a.shape) == (0, 2) for a in only_edgeless.adjacency_lists)


@gpu
def test_a_graph_at_the_budget_raises_before_any_launch(cuda_device):
    graphs = batching.make_qm9_like_graphs(40, seed=9)
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    order = np.random.default_rng(2).permutation(40)
    big = int(np.argmax(gs.graph_sizes[order]))
    budget = int(gs.graph_sizes[order][big])
    with pytest.raises(ValueError) as host_exc:
        list(batching.minibatches([graphs[i] for i in order], budget))
    before = engine.launch_count()
    with pytest.raises(ValueError) as dev_exc:
        next(gs.minibatches(budget, order))
    assert str(dev_exc.value) == str(host_exc.value)
    assert engine.launch_count() == before


# ---- the C ABI directly: refusals, workspace, wrong totals ------------------------------------------------------------
POISON = -2.0 ** 100                                    # exact in float32


def raw_pack(gs, order_dev, start, count, V, E, nodes, adj, indeg, gnl, per_graph, status, ws, ws_bytes, L=None,
             node_offsets=None):
    """rgnn_pack_minibatch with every argument under the caller's control; returns the status code."""
    lib = engine.load_library()
    L = gs.num_edge_types if L is None else L
    widths = (ctypes.c_int32 * 8)(*[t.shape[1] for t in gs.node_tensors])
    rows = (ctypes.c_int32 * 8)(*[t.shape[0] for t in gs.graph_tensors])
    E_arr = (ctypes.c_int64 * len(E))(*E)
    pt = lambda ts: engine.ptr_table(ts, weights=False)    # noqa: E731
    return lib.rgnn_pack_minibatch(
        gs.num_graphs, gs.num_nodes, L, gs.node_offsets.data_ptr() if node_offsets is None else node_offsets,
        pt(gs.edge_offsets), pt(gs.adjacency_lists), gs.num_incoming.data_ptr(),
        len(gs.node_tensors), pt(gs.node_tensors), widths, len(gs.graph_tensors), pt(gs.graph_tensors), rows,
        order_dev.data_ptr(), start, count, V, E_arr, pt(nodes), pt(adj), indeg.data_ptr(), gnl.data_ptr(), pt(per_graph),
        status.data_ptr(), ws, ws_bytes, engine.current_stream_ptr(order_dev.device))


class Poisoned:
    """Output buffers of (V, E) rows inside poison-filled allocations that extend `guard` rows past them."""

    def __init__(self, gs, count, V, E, guard=64):
        import torch
        dev = gs.device
        self.V, self.E, self.L = V, E, gs.num_edge_types
        self.node_bufs = [torch.full(((V + guard) * t.shape[1],), POISON, device=dev) for t in gs.node_tensors]
        self.nodes = [b[: V * t.shape[1]].view(V, t.shape[1]) for b, t in zip(self.node_bufs, gs.node_tensors)]
        self.adj_bufs = [torch.full(((e + guard) * 2,), -123456, dtype=torch.int32, device=dev) for e in E]
        self.adj = [b[: 2 * e].view(e, 2) for b, e in zip(self.adj_bufs, E)]
        self.indeg_buf = torch.full((self.L * V + guard,), POISON, device=dev)
        self.indeg = self.indeg_buf[: self.L * V].view(self.L, V)
        self.gnl_buf = torch.full((V + guard,), -123456, dtype=torch.int32, device=dev)
        self.gnl = self.gnl_buf[:V]
        self.pg_bufs = [torch.full((t.shape[0] * count + guard,), POISON, device=dev) for t in gs.graph_tensors]
        self.per_graph = [b[: t.shape[0] * count].view(t.shape[0], count) for b, t in zip(self.pg_bufs, gs.graph_tensors)]
        self.status = torch.full((1,), -99, dtype=torch.int32, device=dev)

    def args(self):
        return self.nodes, self.adj, self.indeg, self.gnl, self.per_graph, self.status

    def untouched(self):
        """every buffer, payload and guard, still holds its poison"""
        fills = [(b, POISON) for b in self.node_bufs + [self.indeg_buf] + self.pg_bufs]
        fills += [(b, -123456) for b in self.adj_bufs + [self.gnl_buf]] + [(self.status, -99)]
        return all(bool((b == v).all()) for b, v in fills)

    def guards_intact(self, V, E):
        ok = all(bool((b[V * t.shape[1]:] == POISON).all()) for b, t in zip(self.node_bufs, self.nodes))
        ok &= all(bool((b[2 * e:] == -123456).all()) for b, e in zip(self.adj_bufs, E))
        ok &= bool((self.indeg_buf[self.L * self.V:] == POISON).all()) and bool((self.gnl_buf[V:] == -123456).all())
        return ok


@pytest.fixture(scope="module")
def small_qm9_set(cuda_device):
    recs = batching.load_qm9_jsonl(BC.QM9_SUBSET)
    return batching.DeviceGraphSet.from_qm9_records(recs, task_ids=(0, 4), device=cuda_device)


def batch_totals(gs, order, start, count):
    sel = order[start:start + count]
    return int(gs.graph_sizes[sel].sum()), [int(x) for x in gs.edge_counts[:, sel].sum(axis=1)]


@gpu
def test_refusals_and_a_short_workspace_write_nothing(small_qm9_set):
    import torch
    gs = small_qm9_set
    lib = engine.load_library()
    order, order_dev = gs.upload_order(np.random.default_rng(5).permutation(gs.num_graphs))
    start, count = 20, 60
    V, E = batch_totals(gs, order, start, count)
    need = int(lib.rgnn_pack_workspace_bytes(count, gs.num_edge_types))
    assert need > 0 and int(lib.rgnn_pack_workspace_bytes(-1, 5)) == 0 and int(lib.rgnn_pack_workspace_bytes(4, 65)) == 0
    ws = torch.empty(need + 64, dtype=torch.uint8, device=gs.device)
    out = Poisoned(gs, count, V, E)
    torch.cuda.synchronize()
    for nbytes, ptr in [(need - 16, ws.data_ptr()), (0, ws.data_ptr()), (need, 0)]:
        assert raw_pack(gs, order_dev, start, count, V, E, *out.args(), ptr, nbytes) == engine.RGNN_E_WORKSPACE
    assert raw_pack(gs, order_dev, start, count, V, E, *out.args(), ws.data_ptr() + 8, need) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, start, -1, V, E, *out.args(), ws.data_ptr(), need) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, -1, count, V, E, *out.args(), ws.data_ptr(), need) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, start, count, -V, E, *out.args(), ws.data_ptr(), need) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, start, count, V, [-1] + E[1:], *out.args(), ws.data_ptr(), need) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, start, count, V, E + [0] * 60, *out.args(), ws.data_ptr(), need, L=65) == engine.RGNN_E_INVALID
    assert raw_pack(gs, order_dev, start, count, V, E, *out.args(), ws.data_ptr(), need, node_offsets=0) == engine.RGNN_E_INVALID
    torch.cuda.synchronize()
    assert out.untouched()
    # the same call with a sufficient workspace packs the batch (the refusals above were not about anything else)
    assert raw_pack(gs, order_dev, start, count, V, E, *out.args(), ws.data_ptr(), need) == engine.RGNN_OK
    want = gs.pack(order, order_dev, start, count)
    torch.cuda.synchronize()
    assert int(out.status.item()) == 0 and torch.equal(out.nodes[0], want.node_features) and torch.equal(out.indeg, want.type_to_num_incoming_edges)
    assert all(torch.equal(a, b) for a, b in zip(out.adj, want.adjacency_lists)) and torch.equal(out.per_graph[0], want.targets)
    assert out.guards_intact(V, E)


@gpu
def test_wrong_totals_set_the_status_word_and_write_nothing_past_the_given_sizes(small_qm9_set):
    import torch
    gs = small_qm9_set
    lib = engine.load_library()
    order, order_dev = gs.upload_order(np.random.default_rng(6).permutation(gs.num_graphs))
    start, count = 7, 50
    V, E = batch_totals(gs, order, start, count)
    want = gs.pack(order, order_dev, start, count)
    need = int(lib.rgnn_pack_workspace_bytes(count, gs.num_edge_types))
    ws = torch.empty(need, dtype=torch.uint8, device=gs.device)
    for V_given, E_given, bit in [(V - 5, E, 1), (V, [E[0] - 3] + E[1:], 2), (V + 6, E, 1), (V, [e + 9 for e in E], 2),
                                  (V - 1, [max(e - 1, 0) for e in E], 3)]:
        out = Poisoned(gs, count, V_given, E_given)
        assert raw_pack(gs, order_dev, start, count, V_given, E_given, *out.args(), ws.data_ptr(), need) == engine.RGNN_OK
        torch.cuda.synchronize()
        assert int(out.status.item()) == bit, (V_given, E_given)
        assert out.guards_intact(V_given, E_given)
        v = min(V, V_given)                                  # rows both totals cover hold the batch; the rest is untouched
        assert torch.equal(out.nodes[0][:v], want.node_features[:v]) and bool((out.nodes[0][v:] == POISON).all())
        assert torch.equal(out.gnl[:v], want.graph_nodes_list[:v]) and bool((out.gnl[v:] == -123456).all())
        for a, b, e in zip(out.adj, want.adjacency_lists, E_given):
            k = min(e, b.shape[0])
            assert torch.equal(a[:k], b[:k]) and bool((a[k:] == -123456).all())
    # an order entry outside the set: the graph is skipped, the status says so
    bad = order.copy()
    bad[start + 3] = gs.num_graphs + 5
    bad_dev = torch.from_numpy(bad).to(gs.device)
    out = Poisoned(gs, count, V, E)
    assert raw_pack(gs, bad_dev, start, count, V, E, *out.args(), ws.data_ptr(), need) == engine.RGNN_OK
    torch.cuda.synchronize()
    assert int(out.status.item()) == 1 | 2 | 4 and out.guards_intact(V, E)
    with pytest.raises(engine.RgnnError, match="status 7"):
        batching.DeviceBatch(gs, count, V, 0, out.nodes, out.adj, out.indeg, out.gnl, out.per_graph, out.status).check()


# ---- 4. plan and layers on the packed lists --------------------------------------------------------------------------
@gpu
def test_plan_and_layers_on_packed_lists_equal_the_host_route(qm9_like, cuda_device):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    graphs = qm9_like[:3000]
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    order = np.random.default_rng(7).permutation(len(graphs))
    dev = next(gs.minibatches(20000, order))
    host, _ = next(batching.minibatches([graphs[i] for i in order], 20000))
    _, dplan, dcnt, _ = dev.args()
    hplan = G.GraphPlan(host.adjacency_lists, host.num_nodes, device=cuda_device)
    ed, eh = dplan.export(), hplan.export()
    for k in eh:
        assert torch.equal(ed[k], eh[k]), k
    D = 64
    rng = np.random.default_rng(8)
    h = torch.as_tensor(np.tanh(rng.standard_normal((host.num_nodes, D))).astype(np.float32)).to(cuda_device)
    proj = torch.as_tensor(rng.standard_normal((15, D)).astype(np.float32) * 0.3).to(cuda_device)
    hd = dev.node_features @ proj                             # both routes start from their own packed features
    hh = torch.as_tensor(host.node_features).to(cuda_device) @ proj
    assert torch.equal(hd, hh)
    hcnt = torch.as_tensor(host.type_to_num_incoming_edges).to(cuda_device)
    wr = W.to_torch(W.rgcn_weights(5, D, D, seed=3), cuda_device)
    wg = W.to_torch(W.ggnn_weights(5, D, seed=4), cuda_device)
    for x in (h, hd):
        a = G.sparse_rgcn_layer(x, dplan, dcnt, D, activation_function="ReLU", weights=wr)
        b = G.sparse_rgcn_layer(x, hplan, hcnt, D, activation_function="ReLU", weights=wr)
        assert torch.equal(a, b)
        a = G.sparse_ggnn_layer(x, dplan, D, num_timesteps=2, weights=wg)
        b = G.sparse_ggnn_layer(x, hplan, D, num_timesteps=2, weights=wg)
        assert torch.equal(a, b)
    dplan.check()                                              # the deferred range check agrees: every id in range


# ---- 5. no synchronisation; capturable -------------------------------------------------------------------------------
@gpu
def test_pack_and_plan_run_under_sync_debug_error_mode(qm9_like, cuda_device):
    import torch
    graphs = qm9_like[:2000]
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    order = np.random.default_rng(12).permutation(len(graphs))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        packed = []
        for b in gs.minibatches(6000, order):
            packed.append((b, b.args()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    host = list(batching.minibatches([graphs[i] for i in order], 6000))
    assert len(packed) == len(host) > 1
    for (d, args), (h, _) in zip(packed, host):
        assert_batches_equal(d, h)
        args[1].check()


@gpu
def test_pack_and_plan_capture_into_one_cuda_graph_and_replay_a_new_order(qm9_like, cuda_device):
    import torch
    from tf_gnn_samples_b200.engine import GraphPlan
    graphs = qm9_like[:1500]
    gs = batching.DeviceGraphSet(graphs, cuda_device)
    order_a = np.random.default_rng(13).permutation(len(graphs)).astype(np.int32)
    order_host, order_dev = gs.upload_order(order_a)
    start, count = 200, 400
    warm = gs.pack(order_host, order_dev, start, count)          # eager once (module load) before capturing
    GraphPlan(warm.adjacency_lists, warm.num_nodes, device=cuda_device, validate=False)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream(cuda_device)
    s.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b = gs.pack(order_host, order_dev, start, count)
            plan = GraphPlan(b.adjacency_lists, b.num_nodes, device=cuda_device, validate=False)
    torch.cuda.current_stream(cuda_device).wait_stream(s)
    # the same graphs in a different order: the totals are unchanged, every output moves
    order_b = order_a.copy()
    order_b[start:start + count] = np.random.default_rng(14).permutation(order_a[start:start + count])
    assert not np.array_equal(order_b, order_a)
    order_dev.copy_(torch.from_numpy(order_b))
    g.replay()
    torch.cuda.synchronize()
    want = gs.pack(order_b, gs.upload_order(order_b)[1], start, count)
    want_plan = GraphPlan(want.adjacency_lists, want.num_nodes, device=cuda_device)
    host, _ = next(batching.minibatches([graphs[i] for i in order_b[start:start + count]], 10 ** 9))
    assert_batches_equal(b, host, "replay")
    assert_batches_equal(want, host, "eager")
    assert int(b.status.item()) == 0
    ep, ew = plan.export(), want_plan.export()
    for k in ew:
        assert torch.equal(ep[k], ew[k]), k
    plan.close()


# ---- 6. the epoch loop -----------------------------------------------------------------------------------------------
def run_losses(model_fn, batches, to_device, seed):
    import torch
    torch.manual_seed(seed)
    model = model_fn()
    opt = model.make_optimizer()
    torch.manual_seed(seed + 1)
    _, metrics, graphs, _, _, _ = training.run_epoch(model, opt, batches, True, to_device)
    return [m["loss"] for m in metrics], graphs


@gpu
def test_run_epoch_on_device_batches_equals_host_batches_rgcn_ppi(cuda_device):
    from tf_gnn_samples_b200.scaffold import RGCNPPIModel
    graphs = [batching.make_ppi_like_graph(150 + 17 * i, 1500 + 90 * i, feature_dim=50, seed=40 + i, zipf_targets=i % 2 == 0)
              for i in range(9)]
    label_map = np.random.default_rng(5).standard_normal((50, 121)).astype(np.float32)
    labels = [(g.node_features @ label_map > 0).astype(np.float32) for g in graphs]
    gs = batching.DeviceGraphSet.from_ppi_fold(graphs, labels, device=cuda_device)
    order = np.random.default_rng(3).permutation(len(graphs))
    budget = 700
    host = [training.TaskBatch(b, np.concatenate([labels[i] for i in order[first:first + b.num_graphs]]))
            for b, first in batching.minibatches([graphs[i] for i in order], budget)]
    make = lambda: RGCNPPIModel(device=cuda_device, params={"hidden_size": 64, "learning_rate": 0.005})   # noqa: E731
    want, wg = run_losses(make, host, lambda tb: training.device_args(tb, cuda_device), 0)
    got, gg = run_losses(make, gs.minibatches(budget, order), lambda b: b.args(), 0)
    assert len(host) > 2 and gg == wg == len(graphs)
    assert got == want, (got, want)


@gpu
def test_run_epoch_on_device_batches_equals_host_batches_ggnn_qm9(cuda_device):
    from tf_gnn_samples_b200.scaffold import SparseGraphModel
    recs = batching.load_qm9_jsonl(BC.QM9_SUBSET)
    gs = batching.DeviceGraphSet.from_qm9_records(recs, task_ids=(0,), device=cuda_device)
    L = batching.qm9_num_edge_types(recs)
    samples = [batching.qm9_graph_to_sample(r, L) for r in recs]
    order = np.random.default_rng(4).permutation(len(recs))
    budget = 600
    host = []
    for b, first in batching.minibatches([samples[i] for i in order], budget):
        idx = order[first:first + b.num_graphs]
        gnl = np.repeat(np.arange(b.num_graphs, dtype=np.int32), np.diff(b.graph_node_offsets))
        host.append(training.TaskBatch(b, np.array([[recs[i]["targets"][0][0] for i in idx]], dtype=np.float32), gnl))
    params = {"graph_num_layers": 2, "hidden_size": 64, "graph_num_timesteps_per_layer": 2, "graph_rnn_cell": "GRU",
              "graph_layer_input_dropout_keep_prob": 1.0, "learning_rate": 0.003}
    make = lambda: SparseGraphModel("ggnn", "qm9", num_edge_types=L, feature_size=15, params=params, task_ids=(0,),   # noqa: E731
                                    device=cuda_device)
    want, wg = run_losses(make, host, lambda tb: training.device_args(tb, cuda_device), 1)
    got, gg = run_losses(make, gs.minibatches(budget, order), lambda b: b.args(), 1)
    assert len(host) > 2 and gg == wg == len(recs)
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)

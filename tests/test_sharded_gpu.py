"""GPU (one device): the node-range partition of include/rgnn.h's rgnn_halo_* entry points.

* the device-built index lists (order-preserving select, sort + unique, renumbering) equal the host construction of
  partition.NodeRangePartition for every rank;
* "virtual ranks" (SURVEY.md 4.4): all ranks of a partition live in this process on ONE GPU, each with its own stream; the
  pull exchange -- including its device-side cross-rank barrier and the epoch counter that makes it replayable -- runs for
  real, and a multi-layer sharded GNN-FiLM stack reproduces the numpy oracle on the whole graph at 1e-4.
The same code on 2-8 real GPUs (CUDA-IPC peer memory over NVLink) is exercised by bench.py --gpus N.
"""
import numpy as np
import pytest

from oracle import ref_layers as R
from tf_gnn_samples_b200 import ShardedGraph, batching, degree_balanced_cuts, sparse_gnn_film_layer, weights as W
from tf_gnn_samples_b200.partition import NodeRangePartition

from helpers import assert_parity, node_states

pytestmark = pytest.mark.gpu


def small_graph(seed=0, V=900, M=12000, L=4):
    g = batching.make_typed_random_graph(V, M, (0.4, 0.3, 0.2, 0.1)[:L], 8, seed=seed)
    return g.adjacency_lists, g.type_to_node_to_num_incoming_edges, V


@pytest.mark.parametrize("world", [1, 2, 5])
def test_device_built_partition_matches_host_construction(cuda_device, world):
    adj, indeg, V = small_graph()
    cuts = degree_balanced_cuts(adj, V, world)
    for rank in range(world):
        sg = ShardedGraph(adj, cuts, rank, world, device=cuda_device)
        host = NodeRangePartition(adj, indeg, V, rank, world)
        assert list(host.cuts) == list(cuts)
        assert (sg.n_own, sg.n_halo) == (host.n_own, host.n_halo)
        ex = sg.export()
        np.testing.assert_array_equal(ex["halo_global"].cpu().numpy(), host.halo_global)
        owner = np.searchsorted(cuts, host.halo_global, side="right") - 1
        np.testing.assert_array_equal(ex["halo_owner"].cpu().numpy(), owner)
        np.testing.assert_array_equal(ex["halo_row"].cpu().numpy(), host.halo_global - cuts[owner])
        for got, want in zip(ex["local_adjacency_lists"], host.local_adjacency_lists):
            np.testing.assert_array_equal(got.cpu().numpy(), want)
        np.testing.assert_array_equal(sg.local_num_incoming(indeg).cpu().numpy(), host.local_num_incoming)
        sg.close()


def test_edges_of_other_ranks_and_bad_ids(cuda_device):
    from tf_gnn_samples_b200 import RgnnError
    adj, _, V = small_graph(seed=3)
    cuts = degree_balanced_cuts(adj, V, 3)
    only_mine = [a[(a[:, 1] >= cuts[1]) & (a[:, 1] < cuts[2])] for a in adj]       # a shard and the full lists give the same plan
    a, b = ShardedGraph(adj, cuts, 1, 3, device=cuda_device), ShardedGraph(only_mine, cuts, 1, 3, device=cuda_device)
    ea, eb = a.export(), b.export()
    np.testing.assert_array_equal(ea["halo_global"].cpu().numpy(), eb["halo_global"].cpu().numpy())
    for x, y in zip(ea["local_adjacency_lists"], eb["local_adjacency_lists"]):
        np.testing.assert_array_equal(x.cpu().numpy(), y.cpu().numpy())
    bad = [x.copy() for x in adj]
    bad[0][5, 0] = V + 7
    with pytest.raises(RgnnError):
        ShardedGraph(bad, cuts, int(np.searchsorted(cuts, bad[0][5, 1], side="right") - 1), 3, device=cuda_device)
    with pytest.raises(RgnnError):
        a.exchange(0)                                                              # not attached
    a.close(); b.close()


@pytest.mark.parametrize("world,layers,overlap", [(2, 3, False), (4, 2, False), (3, 4, True)])
def test_virtual_ranks_film_stack_matches_oracle(cuda_device, world, layers, overlap):
    """world ranks on one GPU, one stream each: exchange (pull + device barrier) -> FiLM layer -> ... ; the reassembled
    result equals the float64 oracle on the unpartitioned graph, and a second pass (epochs continue) repeats it bit for bit."""
    import torch
    adj, indeg, V = small_graph(seed=5, V=700, M=9000)
    D = 64
    h = node_states(V, D, seed=2)
    ws = [W.film_weights(len(adj), D, D, seed=11 + i, random_ln=True) for i in range(layers)]
    want = h
    for w in ws:
        want = R.sparse_gnn_film_layer(want, adj, indeg, D, activation_function="ReLU", normalize_by_num_incoming=True, weights=w)
    cuts = degree_balanced_cuts(adj, V, world)
    graphs = [ShardedGraph(adj, cuts, r, world, device=cuda_device) for r in range(world)]
    ShardedGraph.attach_in_process(graphs, D)
    streams = [torch.cuda.Stream(device=cuda_device) for _ in range(world)]
    wts = [W.to_torch(w, cuda_device) for w in ws]
    cnts = [g.local_num_incoming(indeg) for g in graphs]
    torch.cuda.synchronize()

    def run_once():
        for g in graphs:
            g.states(0)[: g.n_own] = torch.as_tensor(h[g.lo:g.hi]).to(cuda_device)
        torch.cuda.synchronize()
        for t in range(layers):
            for g, s, c in zip(graphs, streams, cnts):                 # the ranks' work is enqueued round-robin, runs concurrently
                with torch.cuda.stream(s):
                    g.exchange(t % 2, overlap=overlap)   # overlap: pull on a side stream, joined inside the layer call
                    sparse_gnn_film_layer(g.states(t % 2), g.plan, c, D, activation_function="ReLU",
                                          normalize_by_num_incoming=True, weights=wts[t], out=g.states(1 - t % 2))
        torch.cuda.synchronize()
        return np.concatenate([g.states(layers % 2)[: g.n_own].cpu().numpy() for g in graphs])

    got = run_once()
    assert_parity(got, want, "sharded FiLM x%d on %d virtual ranks" % (layers, world), tol=1e-4)
    again = run_once()
    np.testing.assert_array_equal(got, again)
    for g in graphs:
        g.close()


def test_overlapped_exchange_captured_into_cuda_graphs(cuda_device):
    """The K-layer sharded sequence with the overlapped exchange (fork onto the plan's side stream, join inside the layer) is
    recorded into ONE CUDA graph per virtual rank and replayed: the device-side epochs continue across replays, the result
    equals the float64 oracle every time."""
    import torch
    world, layers, D = 2, 2, 64
    adj, indeg, V = small_graph(seed=9, V=640, M=8000)
    h = node_states(V, D, seed=4)
    ws = [W.film_weights(len(adj), D, D, seed=21 + i, random_ln=True) for i in range(layers)]
    want = h
    for w in ws:
        want = R.sparse_gnn_film_layer(want, adj, indeg, D, activation_function="ReLU", normalize_by_num_incoming=False, weights=w)
    cuts = degree_balanced_cuts(adj, V, world)
    graphs = [ShardedGraph(adj, cuts, r, world, device=cuda_device) for r in range(world)]
    ShardedGraph.attach_in_process(graphs, D)
    streams = [torch.cuda.Stream(device=cuda_device) for _ in range(world)]
    wts = [W.to_torch(w, cuda_device) for w in ws]
    cnts = [g.local_num_incoming(indeg) for g in graphs]

    def stack(g, c):
        for t in range(layers):
            g.exchange(t % 2, overlap=True)
            sparse_gnn_film_layer(g.states(t % 2), g.plan, c, D, activation_function="ReLU", weights=wts[t], out=g.states(1 - t % 2))

    def load_inputs():
        for g in graphs:
            g.states(0)[: g.n_own] = torch.as_tensor(h[g.lo:g.hi]).to(cuda_device)
        torch.cuda.synchronize()

    load_inputs()
    for g, s, c in zip(graphs, streams, cnts):            # eager warm-up (creates the side streams / events, fills caches)
        with torch.cuda.stream(s):
            stack(g, c)
    torch.cuda.synchronize()
    captured = []
    for g, s, c in zip(graphs, streams, cnts):            # capture does not execute: the ranks can be recorded one after the other
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            stack(g, c)
        captured.append(cg)
    for _ in range(2):
        load_inputs()
        for cg, s in zip(captured, streams):
            with torch.cuda.stream(s):
                cg.replay()
        torch.cuda.synchronize()
        got = np.concatenate([g.states(0)[: g.n_own].cpu().numpy() for g in graphs])   # an even number of layers ends in buffer 0
        assert_parity(got, want, "overlapped exchange, CUDA-graph replay", tol=1e-4)
    for g in graphs:
        g.close()

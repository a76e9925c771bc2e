"""GPU: gradients of every layer function under autograd (training-mode paths, gnns/_train.py + the engine's differentiable
building blocks) against torch float64 autograd over the reference op order (oracle/ref_autograd.py, pinned on the CPU in
tests/test_oracle_autograd.py).  Smooth activations are used where a gradient is compared element by element: with ReLU a
single fp32/fp64 sign disagreement at a ~1e-6 pre-activation flips a whole gradient path (see test_scaffold_gpu.py)."""
import numpy as np
import pytest

from oracle import ref_autograd as A
from tf_gnn_samples_b200 import (GraphPlan, batching, ops, sparse_ggnn_layer, sparse_gnn_edge_mlp_layer, sparse_gnn_film_layer,
                                 sparse_rgat_layer, sparse_rgcn_layer, sparse_rgin_layer, weights as W)

from helpers import compare, node_states, rel, tiny_graph, to_dev

pytestmark = pytest.mark.gpu

V, L, D = 61, 4, 32


def graph(seed=71):
    return tiny_graph(V, (170, 61, 0, 95), seed=seed)


def test_building_blocks(cuda_device):
    """edge_aggregate / segment_aggregate / gather_rows / gather_table_rows: values and gradients, all aggregations."""
    import torch
    adj, indeg = graph()
    plan = GraphPlan(adj, V, device=cuda_device)
    rng = np.random.default_rng(1)
    table = rng.standard_normal((V, L, D)).astype(np.float32)
    M = plan.num_edges
    data = rng.standard_normal((M, D)).astype(np.float32)
    src = np.concatenate([a[:, 0] for a in adj]).astype(np.int64); tgt = np.concatenate([a[:, 1] for a in adj]).astype(np.int64)
    # a tie for the max gradient: a copy of row i inside its own segment, the maximum of that segment in some columns
    i = 4
    j = int(np.flatnonzero(tgt == tgt[i])[-1])
    assert j != i and tgt[j] == tgt[i]
    data[j] = data[i]
    assert (data[i] == data[tgt == tgt[i]].max(axis=0)).any(), "row %d is the segment maximum in no column" % i
    typ = np.concatenate([np.full(a.shape[0], l, dtype=np.int64) for l, a in enumerate(adj)])
    cnt64 = torch.as_tensor(indeg, dtype=torch.float64)
    for agg in ["sum", "mean", "sqrt_n", "max"]:
        proj = rng.standard_normal((V, D))
        # segment_aggregate
        d_dev = torch.as_tensor(data).to(cuda_device).requires_grad_(True)
        out = ops.segment_aggregate(plan, d_dev, agg)
        (out * torch.as_tensor(proj, dtype=torch.float32).to(cuda_device)).sum().backward()
        d64 = torch.as_tensor(data, dtype=torch.float64).requires_grad_(True)
        o64 = A.segment_reduce(d64, torch.as_tensor(tgt), V, agg)
        (o64 * torch.as_tensor(proj)).sum().backward()
        assert rel(out.detach().cpu().numpy(), o64.detach().numpy()) < 1e-5
        assert rel(d_dev.grad.cpu().numpy(), d64.grad.numpy()) < 1e-5, agg
        if agg == "max":
            continue
        # edge_aggregate with and without in-degree scaling
        for use_cnt in (False, True):
            t_dev = torch.as_tensor(table).to(cuda_device).requires_grad_(True)
            out = ops.edge_aggregate(t_dev, plan, torch.as_tensor(indeg).to(cuda_device) if use_cnt else None, agg)
            (out * torch.as_tensor(proj, dtype=torch.float32).to(cuda_device)).sum().backward()
            t64 = torch.as_tensor(table, dtype=torch.float64).requires_grad_(True)
            rows = t64[torch.as_tensor(src), torch.as_tensor(typ)]
            if use_cnt:
                rows = rows * (1.0 / (cnt64[torch.as_tensor(typ), torch.as_tensor(tgt)] + 1e-7)).unsqueeze(1)
            o64 = A.segment_reduce(rows, torch.as_tensor(tgt), V, agg)
            (o64 * torch.as_tensor(proj)).sum().backward()
            assert rel(out.detach().cpu().numpy(), o64.detach().numpy()) < 1e-5
            assert rel(t_dev.grad.cpu().numpy(), t64.grad.numpy()) < 1e-5, (agg, use_cnt)
    # gathers
    x = rng.standard_normal((V, D)).astype(np.float32)
    g = rng.standard_normal((M, D)).astype(np.float32)
    for side, idx in (("source", src), ("target", tgt)):
        xd = torch.as_tensor(x).to(cuda_device).requires_grad_(True)
        rows = ops.gather_rows(xd, plan, side)
        assert np.array_equal(rows.detach().cpu().numpy(), x[idx])
        (rows * torch.as_tensor(g).to(cuda_device)).sum().backward()
        want = np.zeros((V, D)); np.add.at(want, idx, g.astype(np.float64))
        assert rel(xd.grad.cpu().numpy(), want) < 1e-5
        td = torch.as_tensor(table).to(cuda_device).requires_grad_(True)
        rows = ops.gather_table_rows(td, plan, side)
        assert np.array_equal(rows.detach().cpu().numpy(), table[idx, typ])
        (rows * torch.as_tensor(g).to(cuda_device)).sum().backward()
        want = np.zeros((V, L, D)); np.add.at(want, (idx, typ), g.astype(np.float64))
        assert rel(td.grad.cpu().numpy(), want) < 1e-5


@pytest.mark.parametrize("cell,agg,T", [("gru", "sum", 2), ("rnn", "mean", 1), ("gru", "max", 1)])
def test_ggnn_grads(cuda_device, cell, agg, T):
    import torch
    adj, _ = graph()
    h = node_states(V, D, seed=72)
    w = W.ggnn_weights(L, D, seed=73, cell=cell, random_bias=True)
    compare(lambda hd, wd: sparse_ggnn_layer(hd, adj, D, num_timesteps=T, gated_unit_type=cell, message_aggregation_function=agg, weights=wd),
            lambda h64, w64: A.sparse_ggnn_layer(h64, adj, num_timesteps=T, gated_unit_type=cell, message_aggregation_function=agg, weights=w64),
            h, w)


@pytest.mark.parametrize("heads,T", [(4, 1), (8, 2)])
def test_rgat_grads(cuda_device, heads, T):
    adj, _ = graph()
    h = node_states(V, D, seed=74)
    w = W.rgat_weights(L, D, D, seed=75)
    compare(lambda hd, wd: sparse_rgat_layer(hd, adj, D, num_timesteps=T, num_heads=heads, weights=wd),
            lambda h64, w64: A.sparse_rgat_layer(h64, adj, num_timesteps=T, num_heads=heads, weights=w64), h, w)


@pytest.mark.parametrize("act,agg,normalize,T", [("tanh", "sum", False, 1), ("gelu", "mean", True, 2), ("elu", "sqrt_n", True, 1)])
def test_film_grads(cuda_device, act, agg, normalize, T):
    import torch
    adj, indeg = graph()
    h = node_states(V, D, seed=76)
    w = W.film_weights(L, D, D, seed=77, num_timesteps=T, random_ln=True)
    compare(lambda hd, wd: sparse_gnn_film_layer(hd, adj, torch.as_tensor(indeg).to(hd.device), D, num_timesteps=T, activation_function=act,
                                                 message_aggregation_function=agg, normalize_by_num_incoming=normalize, weights=wd),
            lambda h64, w64: A.sparse_gnn_film_layer(h64, adj, torch.as_tensor(indeg, dtype=torch.float64), num_timesteps=T, activation_function=act,
                                                     message_aggregation_function=agg, normalize_by_num_incoming=normalize, weights=w64),
            h, w)


@pytest.mark.parametrize("hidden,use_target,agg", [(1, True, "sum"), (0, True, "mean"), (1, False, "sum")])
def test_edge_mlp_grads(cuda_device, hidden, use_target, agg):
    import torch
    adj, indeg = graph()
    h = node_states(V, D, seed=78)
    w = W.edge_mlp_weights(L, D, D, hidden, use_target, seed=79, random_ln=True)
    compare(lambda hd, wd: sparse_gnn_edge_mlp_layer(hd, adj, torch.as_tensor(indeg).to(hd.device), D, activation_function="tanh",
                                                     message_aggregation_function=agg, use_target_state_as_input=use_target,
                                                     num_edge_hidden_layers=hidden, weights=wd),
            lambda h64, w64: A.sparse_gnn_edge_mlp_layer(h64, adj, None, activation_function="tanh", message_aggregation_function=agg,
                                                         use_target_state_as_input=use_target, weights=w64),
            h, w)


@pytest.mark.parametrize("edge_hidden,aggr_hidden,use_target", [(1, None, False), (1, 1, False), (0, 0, True), (None, 1, False)])
def test_rgin_grads(cuda_device, edge_hidden, aggr_hidden, use_target):
    adj, _ = graph()
    h = node_states(V, D, seed=80)
    w = W.rgin_weights(L, D, D, edge_hidden, aggr_hidden, use_target, seed=81, random_ln=True)
    compare(lambda hd, wd: sparse_rgin_layer(hd, adj, D, activation_function="tanh", use_target_state_as_input=use_target,
                                             num_edge_MLP_hidden_layers=edge_hidden, num_aggr_MLP_hidden_layers=aggr_hidden, weights=wd),
            lambda h64, w64: A.sparse_rgin_layer(h64, adj, activation_function="tanh", use_target_state_as_input=use_target, weights=w64),
            h, w)


@pytest.mark.parametrize("both,agg", [(True, "sum"), (False, "max"), (True, "max")])
def test_rgcn_grads_outside_the_fused_backward(cuda_device, both, agg):
    """[h_u | h_v] messages and max aggregation take the composed path."""
    import torch
    adj, indeg = graph()
    h = node_states(V, D, seed=82)
    w = W.rgcn_weights(L, D, D, seed=83, use_both_source_and_target=both)
    compare(lambda hd, wd: sparse_rgcn_layer(hd, adj, torch.as_tensor(indeg).to(hd.device), D, activation_function="tanh",
                                             message_aggregation_function=agg, use_both_source_and_target=both, weights=wd),
            lambda h64, w64: A.sparse_rgcn_layer(h64, adj, torch.as_tensor(indeg, dtype=torch.float64), activation_function="tanh",
                                                 message_aggregation_function=agg, use_both_source_and_target=both, weights=w64),
            h, w)


def test_training_mode_matches_inference_kernels(cuda_device):
    """The composed training forward and the fused inference kernels are the same function (PPI-shaped, hidden 128)."""
    import torch
    b = batching.ppi_like_batch(num_nodes=700, num_links=12000, seed=90)
    plan = GraphPlan(b.adjacency_lists, b.num_nodes, device=cuda_device)
    cnt = torch.as_tensor(b.type_to_num_incoming_edges).to(cuda_device)
    d = 128
    h = torch.as_tensor(node_states(b.num_nodes, d, seed=91)).to(cuda_device)
    cases = [
        (sparse_ggnn_layer, W.ggnn_weights(3, d, seed=92), dict(state_dim=d, num_timesteps=2), False),
        (sparse_rgat_layer, W.rgat_weights(3, d, d, seed=93), dict(state_dim=d, num_heads=8), False),
        (sparse_gnn_film_layer, W.film_weights(3, d, d, seed=94), dict(state_dim=d), True),
        (sparse_gnn_edge_mlp_layer, W.edge_mlp_weights(3, d, d, 1, True, seed=95), dict(state_dim=d), True),
        (sparse_rgin_layer, W.rgin_weights(3, d, d, 1, 1, False, seed=96), dict(state_dim=d, num_aggr_MLP_hidden_layers=1), False),
    ]
    for fn, w, kw, takes_cnt in cases:
        wi = W.to_torch(w, cuda_device)
        args = (h, plan, cnt) if takes_cnt else (h, plan)
        with torch.no_grad():
            fused = fn(*args, weights=wi, **kw)
        composed = fn(h.clone().requires_grad_(True), *args[1:], weights=wi, **kw)
        assert composed.requires_grad
        assert rel(composed.detach().cpu().numpy(), fused.cpu().numpy()) < 2e-5, fn.__name__


def test_empty_and_degenerate_inputs(cuda_device):
    """No edges at all, a single node, zero rows: the differentiable building blocks and RGDCN return the reference's
    values (sums over nothing = 0, act(0)) and zero gradients instead of faulting."""
    import torch
    from tf_gnn_samples_b200 import sparse_rgdcn_layer
    empty = [np.zeros((0, 2), np.int32) for _ in range(3)]
    Vn, Dn = 7, 16
    plan = GraphPlan(empty, Vn, device=cuda_device)
    assert plan.num_edges == 0
    table = torch.randn(Vn, 3, Dn, device=cuda_device, requires_grad=True)
    out = ops.edge_aggregate(table, plan, None, "sum")
    assert torch.count_nonzero(out) == 0
    out.sum().backward()
    assert torch.count_nonzero(table.grad) == 0
    data = torch.zeros((0, Dn), device=cuda_device, requires_grad=True)
    assert torch.count_nonzero(ops.segment_aggregate(plan, data, "mean")) == 0
    assert float(ops.segment_aggregate(plan, data, "max").max()) < -3e38          # tf.unsorted_segment_max of empty segments
    x = torch.randn(Vn, Dn, device=cuda_device, requires_grad=True)
    assert ops.gather_rows(x, plan, "source").shape == (0, Dn)
    # dense gradients with zero rows: grad_W is exactly zero, grad_x is empty
    gx, gw = ops.dense_backward(torch.zeros((0, 8), device=cuda_device), torch.randn(8, 12, device=cuda_device),
                                torch.zeros((0, 12), device=cuda_device))
    assert gx.shape == (0, 8) and torch.count_nonzero(gw) == 0
    # RGDCN without edges: act(0) = 0 for tanh
    w = W.to_torch(W.rgdcn_weights(3, 4, 4, stddev=0.3), cuda_device)
    cnt = torch.zeros((3, Vn), device=cuda_device)
    got = sparse_rgdcn_layer(torch.randn(Vn, Dn, device=cuda_device), plan, cnt, 4, 4, weights=w)
    assert torch.count_nonzero(got) == 0
    # one node, one self loop, training path of GGNN
    one = GraphPlan([np.array([[0, 0]], np.int32)], 1, device=cuda_device)
    wg = to_dev(W.ggnn_weights(1, Dn, seed=3), torch.device(cuda_device))
    h1 = torch.randn(1, Dn, device=cuda_device, requires_grad=True)
    sparse_ggnn_layer(h1, one, Dn, weights=wg).sum().backward()
    assert torch.isfinite(h1.grad).all()

"""GPU: the exported building blocks against numpy (float64): wgmma 3xTF32 Dense at awkward shapes,
segment aggregation in all four modes, layer norm."""
import numpy as np
import pytest

from oracle import ref_layers as R
from tf_gnn_samples_b200 import GraphPlan, ops

from helpers import assert_parity, tiny_graph

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m,k,n", [(1, 4, 4), (129, 36, 52), (300, 64, 96), (2245, 256, 768), (511, 320, 1280),
                                   (64, 512, 16), (1000, 8, 264), (4100, 128, 384)])
def test_dense_matches_fp64(cuda_device, m, k, n):
    import torch
    rng = np.random.default_rng(m * 7 + n)
    a = rng.standard_normal((m, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    got = ops.dense(torch.as_tensor(a).to(cuda_device), torch.as_tensor(w).to(cuda_device)).cpu().numpy()
    want = a.astype(np.float64) @ w.astype(np.float64)
    err = assert_parity(got, want, "dense %dx%dx%d" % (m, k, n), tol=1e-5)   # 3xTF32: fp32-level accuracy (measured ~3e-6 at K=256)
    print("dense %dx%dx%d max-norm rel err %.2e" % (m, k, n, err))


def test_dense_bias_activation(cuda_device):
    import torch
    rng = np.random.default_rng(3)
    a = rng.standard_normal((77, 48)).astype(np.float32)
    w = rng.standard_normal((48, 40)).astype(np.float32) / 7
    b = rng.standard_normal(40).astype(np.float32)
    for act in ["tanh", "relu", "gelu", None]:
        got = ops.dense(torch.as_tensor(a).to(cuda_device), torch.as_tensor(w).to(cuda_device),
                        torch.as_tensor(b).to(cuda_device), act).cpu().numpy()
        want = a.astype(np.float64) @ w.astype(np.float64) + b
        fn = R.get_activation(act)
        want = want if fn is None else fn(want)
        assert_parity(got, want, "dense+bias+%s" % act, tol=1e-5)


# (rows m = the long contraction axis of the weight gradient, k = in, n = out)
@pytest.mark.parametrize("m,k,n", [(1, 4, 4), (31, 8, 12), (33, 132, 260), (2245, 256, 768), (11225, 256, 256),
                                   (5000, 52, 124), (70000, 128, 128), (97, 512, 36)])
def test_dense_backward_matches_fp64(cuda_device, m, k, n):
    """grad_x = g . W^T (transposed-weight wgmma GEMM) and grad_W = x^T . g (split-K TN kernel) against float64."""
    import torch
    rng = np.random.default_rng(m + 3 * k + n)
    x = rng.standard_normal((m, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    g = rng.standard_normal((m, n)).astype(np.float32)
    gx, gw = ops.dense_backward(torch.as_tensor(x).to(cuda_device), torch.as_tensor(w).to(cuda_device),
                                torch.as_tensor(g).to(cuda_device))
    assert_parity(gx.cpu().numpy(), g.astype(np.float64) @ w.astype(np.float64).T, "dense grad_x %dx%dx%d" % (m, k, n), tol=1e-5)
    err = assert_parity(gw.cpu().numpy(), x.astype(np.float64).T @ g.astype(np.float64), "dense grad_w %dx%dx%d" % (m, k, n), tol=1e-5)
    print("dense grad_w %dx%dx%d max-norm rel err %.2e" % (m, k, n, err))
    # deterministic: the split-K partial sums are combined in a fixed order
    _, gw2 = ops.dense_backward(torch.as_tensor(x).to(cuda_device), torch.as_tensor(w).to(cuda_device),
                                torch.as_tensor(g).to(cuda_device), need_x=False)
    assert torch.equal(gw, gw2)


def test_dense_autograd(cuda_device):
    """ops.dense under autograd: tanh(x W + b) gradients against torch float64 on the CPU."""
    import torch
    rng = np.random.default_rng(11)
    x = rng.standard_normal((301, 48)).astype(np.float32)
    w = (rng.standard_normal((48, 40)) / 7).astype(np.float32)
    b = rng.standard_normal(40).astype(np.float32)
    c = rng.standard_normal((301, 40)).astype(np.float32)
    td = [torch.as_tensor(a).to(cuda_device).requires_grad_(True) for a in (x, w, b)]
    (ops.dense(td[0], td[1], td[2], "tanh") * torch.as_tensor(c).to(cuda_device)).sum().backward()
    t64 = [torch.as_tensor(a, dtype=torch.float64).requires_grad_(True) for a in (x, w, b)]
    (torch.tanh(t64[0] @ t64[1] + t64[2]) * torch.as_tensor(c, dtype=torch.float64)).sum().backward()
    for got, want, name in zip(td, t64, ["x", "kernel", "bias"]):
        assert_parity(got.grad.cpu().numpy(), want.grad.numpy(), "dense autograd d%s" % name, tol=2e-5)


@pytest.mark.parametrize("agg", ["sum", "max", "mean", "sqrt_n"])
def test_segment_aggregate(cuda_device, agg):
    import torch
    adj, _ = tiny_graph(40, (90, 0, 33), seed=5, with_isolated=False)
    adj[1] = np.zeros((0, 2), np.int32)
    adj.append(np.stack([np.arange(40), np.arange(40)], axis=1).astype(np.int32))   # every node has a message
    plan = GraphPlan(adj, 40, device=cuda_device)
    tgt = np.concatenate([a[:, 1] for a in adj])
    data = np.random.default_rng(1).standard_normal((tgt.size, 20)).astype(np.float32)
    got = ops.segment_aggregate(plan, torch.as_tensor(data).to(cuda_device), agg).cpu().numpy()
    want = R.get_aggregation_function(agg)(data.astype(np.float64), tgt, 40)
    assert_parity(got, want, "segment %s" % agg, tol=1e-6)


def test_layer_norm(cuda_device):
    import torch
    rng = np.random.default_rng(2)
    for d in (8, 128, 300, 512):
        x = rng.standard_normal((33, d)).astype(np.float32) * 3 + 1
        x[5] = 0.0                                                              # zero-variance row -> beta
        g, b = rng.standard_normal(d).astype(np.float32), rng.standard_normal(d).astype(np.float32)
        got = ops.layer_norm(*(torch.as_tensor(t).to(cuda_device) for t in (x, g, b))).cpu().numpy()
        assert_parity(got, R.layer_norm(x.astype(np.float64), g, b), "layer_norm d=%d" % d, tol=1e-5)


def test_restricted_target_rows_sharded_execution(cuda_device):
    """rgnn_plan_set_num_targets: on a rank-local graph of a node-range partition (owned rows first, halo rows after)
    restricting the target rows leaves the owned outputs bit-identical, for FiLM (gamma/beta GEMM on owned rows only),
    GGNN (cell on owned rows only) and RGCN (edge stage only)."""
    import torch
    from tf_gnn_samples_b200 import (RgnnError, batching, sparse_ggnn_layer, sparse_gnn_film_layer, sparse_rgcn_layer, weights as W)
    from tf_gnn_samples_b200.partition import NodeRangePartition
    b = batching.varmisuse_like_batch(num_nodes=900, num_edges=14000, seed=5, feature_dim=8)
    part = NodeRangePartition(b.adjacency_lists, b.type_to_num_incoming_edges, b.num_nodes, rank=1, world_size=3)
    assert 0 < part.n_own < part.n_local
    D, L = 64, len(b.adjacency_lists)
    h = torch.as_tensor(np.tanh(np.random.default_rng(2).standard_normal((part.n_local, D))).astype(np.float32)).to(cuda_device)
    cnt = torch.as_tensor(part.local_num_incoming).to(cuda_device)
    full = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device)
    own = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device).set_num_targets(part.n_own)
    wf = W.to_torch(W.film_weights(L, D, D, random_ln=True), cuda_device)
    wg = W.to_torch(W.ggnn_weights(L, D, random_bias=True), cuda_device)
    wr = W.to_torch(W.rgcn_weights(L, D, D), cuda_device)
    n = part.n_own
    assert torch.equal(sparse_gnn_film_layer(h, full, cnt, D, weights=wf)[:n], sparse_gnn_film_layer(h, own, cnt, D, weights=wf)[:n])
    assert torch.equal(sparse_ggnn_layer(h, full, D, weights=wg)[:n], sparse_ggnn_layer(h, own, D, weights=wg)[:n])
    assert torch.equal(sparse_rgcn_layer(h, full, cnt, D, weights=wr)[:n], sparse_rgcn_layer(h, own, cnt, D, weights=wr)[:n])
    with pytest.raises(RgnnError):                       # halo rows are not updated inside the call
        sparse_ggnn_layer(h, own, D, num_timesteps=2, weights=wg)
    with pytest.raises(RgnnError):
        own.set_num_targets(part.n_local + 1)


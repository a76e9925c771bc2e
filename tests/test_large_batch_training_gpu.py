"""GPU: the training-mode gradients at production batch sizes, each compared element by element with float64.

The 61-node graph of test_train_layers_gpu.py reaches none of the gradient paths a QM9 or PPI batch takes: no segment of any
plan is heavy there, D = 32 is a single 128-column slice, and every weight-gradient contraction has at most 326 rows.  Here
the same gradients run on batches of 6,000 - 20,000 nodes with hubs of thousands of edges:

  * the gathers' backward segment-sums per-edge gradients over GraphPlan.regrouped(...) plans, which are built without
    reading back their heavy count, so the one-CTA-per-segment heavy kernel walks the heavy list on the device;
  * ops.segment_aggregate attaches no heavy scratch: hub targets go to the one-CTA heavy kernel (also its max variant);
  * the max gradient splits evenly among exactly tied maxima inside hub segments;
  * the edge-aggregate backward reduces over the (source, type) reverse index, scaled or not, after the mean / sqrt_n divisor;
  * the fused RGCN backward with gelu (recomputed pre-activation), sqrt_n, no normalisation and d_in != d_out;
  * dense gradients over per-type row slices of [M, 2D] per-edge tensors (tens of thousands of rows per type).

Each case's regime is restated from the dispatch code and checked without a GPU (test_case_regimes); the kernels that regime
implies must appear among the kernels the backward pass launched (the forward runs outside the profiler, except for the
segment-aggregate block, whose heavy kernels run in its forward).  Activations are smooth (tanh, gelu, elu): at the kink of
ReLU-like activations one float32/float64 sign disagreement moves a whole gradient path (DESIGN.md 5.5)."""
import zlib

import numpy as np
import pytest

from oracle import ref_autograd as A
from oracle import ref_grads as RG
from oracle import ref_layers as R
from tf_gnn_samples_b200 import weights as W

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, QM9_20K, SMALL_BATCH, TILE_M, graph, pick_bn, segment_sizes
from helpers import compare, launched_kernels, node_states, rel

BLOCK_TOL = 1e-5     # the building blocks: one gather / reduction, float32 accumulation
LAYER_TOL = 1e-4     # whole layers: max-norm relative error of the output, d_h and every weight gradient

CASES = [
    # building blocks on the Zipf-skewed PPI batch (4 heavy targets, sources, (source, type) and (target, type) pairs)
    dict(id="blocks_gather", kind="gather", graph=PPI6K_ZIPF, D=256),
    dict(id="blocks_segment_aggregate", kind="segment", graph=PPI6K_ZIPF, D=256),
    dict(id="blocks_edge_aggregate", kind="edge_aggregate", graph=PPI6K_ZIPF, D=256),
    # layers: GGNN on a QM9-like batch (V * L = 80,000 reverse segments, no hub), the rest on the Zipf-skewed PPI batch
    # GRU gates are hard sigmoids, kinked at +-2.5: with the default cell weights, 2 of the 5.1M gate pre-activations lie
    # within 1e-5 of a kink, where the engine measured a d_h error of 7e-3 on an H100 80GB HBM3 (700 W) and reference-order
    # float32 3e-7 (one gate on the other side of a kink moves a whole gradient element).  Halving the cell weights keeps
    # every pre-activation >= 1e-4 from the kinks (test_case_regimes checks it), 100x the float32 error of the engine's
    # pre-activations.
    dict(id="ggnn_gru_d64_sum_t2", kind="ggnn", graph=QM9_20K, D=64, cell="gru", agg="sum", T=2, cell_scale=0.5),
    dict(id="ggnn_rnn_d128_mean", kind="ggnn", graph=QM9_20K, D=128, cell="rnn", agg="mean", T=1),
    dict(id="rgat_d128_to_256_k8", kind="rgat", graph=PPI6K_ZIPF, d_in=128, D=256, K=8, T=1),
    dict(id="film_gelu_mean_normalized", kind="film", graph=PPI6K_ZIPF, D=256, act="gelu", agg="mean", normalize=True, T=1),
    dict(id="film_tanh_sum_t2", kind="film", graph=PPI6K_ZIPF, D=256, act="tanh", agg="sum", normalize=False, T=2),
    dict(id="edge_mlp_hidden1_target", kind="edge_mlp", graph=PPI6K_ZIPF, D=256, hidden=1, use_target=True, normalize=True),
    dict(id="edge_mlp_hidden0_source", kind="edge_mlp", graph=PPI6K_ZIPF, D=256, hidden=0, use_target=False, normalize=False),
    # mean, not sum: summed over a hub's 2,517 edges the messages drive the aggregation MLP's tanh into saturation, where
    # reference-order float32 itself is 1.9e-4 (d_h) and 2.8e-4 (d_aggr_mlp.0) off float64; the engine measured 2.4e-4 and
    # 3.0e-4 on an H100 80GB HBM3 (700 W)
    dict(id="rgin_target_edge1_aggr1_mean", kind="rgin", graph=PPI6K_ZIPF, D=256, edge_hidden=1, aggr_hidden=1, use_target=True,
         agg="mean"),
    dict(id="rgin_source_edge1", kind="rgin", graph=PPI6K_ZIPF, D=256, edge_hidden=1, aggr_hidden=None, use_target=False),
    # [h_u | h_v] messages: ZIPF6K draws its sources uniformly, so its (source, type) regrouping has no hub; on the
    # Zipf-skewed PPI batch both gathers regroup onto heavy segments
    dict(id="rgcn_both_sum", kind="rgcn", graph=PPI6K_ZIPF, D=256),
    # the fused RGCN backward (rgnn_rgcn_backward), against the analytic gradients of oracle/ref_grads.py
    dict(id="rgcn_fused_gelu_sqrt_n_d128_to_256", kind="rgcn_fused", graph=PPI6K_ZIPF, d_in=128, D=256, act="gelu", agg="sqrt_n",
         normalize=True),
    dict(id="rgcn_fused_linear_sum_unnormalized", kind="rgcn_fused", graph=PPI6K_ZIPF, d_in=256, D=256, act=None, agg="sum",
         normalize=False),
]

GATHER = ["seg_reduce_kernel<1, 0, false, false, false>", "seg_reduce_heavy_kernel<1, 0, false, false, false>"]
DENSE_GRAD = ["gemm_tn_wgmma_kernel", "gemm_tn_reduce_kernel"]


def _b(x):
    return "true" if x else "false"


def edge_backward_kernels(agg, scaled):
    """The reverse-index reduction of rgnn_edge_aggregate_backward (heavy count never read back: the one-CTA heavy kernel
    always runs) and, for mean / sqrt_n, the divisor pass in front of it."""
    names = ["seg_reduce_kernel<1, 0, false, %s, false>" % _b(scaled), "seg_reduce_heavy_kernel<1, 0, false, %s, false>" % _b(scaled)]
    return names + (["act_backward_kernel"] if agg in ("mean", "sqrt_n") else [])


def segment_forward_kernels(agg):
    """rgnn_segment_aggregate on a validated plan with heavy targets and no heavy scratch: the one-CTA heavy kernel."""
    mx = agg == "max"
    return ["seg_reduce_kernel<1, 0, %s, false, false>" % _b(mx), "seg_reduce_heavy_kernel<1, 0, %s, false, false>" % _b(mx)]


def grad_x_kernel(rows, k_in):
    """dx = g . W^T of ops.dense: the wgmma GEMM with N = k_in and the BN pick_bn gives it."""
    return "gemm_wgmma_kernel<0, %d, false>" % pick_bn(-(-rows // TILE_M), k_in)


def _uses(case, adj, V):
    """(plans, per-edge dense rows, grad_x GEMM): the (regrouping, row width) pairs whose segment kernels the backward runs,
    the rows of the largest per-type slice a per-edge dense gradient contracts (0: none), and (rows, k_in) of one dense
    whose input gradient the case computes."""
    k, D = case["kind"], case["D"]
    per_type = max(a.shape[0] for a in adj)
    if k == "gather":
        return [("target", D), ("source", D), ("source_type", D), ("target_type", 2 * D)], 0, None
    if k == "segment":
        return [("target", D)], 0, None
    if k in ("edge_aggregate", "ggnn"):
        return [("source_type", D)], 0, ((V, D) if k == "ggnn" else None)
    if k == "rgat":
        return [("source_type", D)], 0, (V, case["d_in"])
    if k == "film":
        return [("source_type", D), ("target_type", 2 * D)], 0, (V, D)
    if k in ("edge_mlp", "rgin") and case["use_target"]:
        return [("source", D), ("target", D)], per_type, (per_type, 2 * D)
    if k == "edge_mlp":
        return [("source", D)], per_type, (per_type, D)
    if k == "rgin":
        return [("source_type", D)], 0, (V, D)
    if k == "rgcn":
        return [("source_type", D), ("target_type", D)], 0, (V, D)
    plans = [("source_type", D)] + ([("target", D)] if case["act"] == "gelu" else [])
    return plans, 0, (V, case["d_in"])


def ggnn_weights(case, L):
    w = W.ggnn_weights(L, case["D"], seed=zlib.crc32(case["id"].encode()) % 10000, cell=case["cell"], random_bias=True)
    w["cell"] = {k: v * np.float32(case.get("cell_scale", 1.0)) for k, v in w["cell"].items()}
    return w


def gru_kink_distance(case):
    """Smallest distance of a float64 GRU gate pre-activation (z, r; every timestep) from the hard-sigmoid kinks at +-2.5."""
    import torch
    adj, _, V = graph(case["graph"])
    D = case["D"]
    w = ggnn_weights(case, len(adj))
    K, R, B = (torch.as_tensor(w["cell"][k], dtype=torch.float64) for k in ("kernel", "recurrent_kernel", "bias"))
    ws = [torch.as_tensor(x, dtype=torch.float64) for x in w["edge_weights"]]
    tgt = torch.cat([torch.as_tensor(a[:, 1]).long() for a in adj])
    cur = torch.as_tensor(node_states(V, D, seed=zlib.crc32(case["id"].encode()) % 1000), dtype=torch.float64)
    dist = float("inf")
    for _ in range(case["T"]):             # oracle/ref_autograd.py sparse_ggnn_layer, GRU cell
        m = torch.zeros(V, D, dtype=torch.float64).index_add(0, tgt, torch.cat([cur[torch.as_tensor(a[:, 0]).long()] @ ws[l] for l, a in enumerate(adj)]))
        zr = m @ K[:, :2 * D] + B[:2 * D] + cur @ R[:, :2 * D]
        dist = min(dist, float(((zr.abs() - 2.5).abs()).min()))
        z, r = A.hard_sigmoid(zr[:, :D]), A.hard_sigmoid(zr[:, D:])
        cur = z * cur + (1.0 - z) * torch.tanh(m @ K[:, 2 * D:] + B[2 * D:] + (r * cur) @ R[:, 2 * D:])
    return dist


def regime(case):
    """(claims, kernels): the inequalities that put the case in its regime as (text, holds) pairs, and the kernel-name
    substrings that regime implies in the backward pass (in the forward for the segment-aggregate block)."""
    adj, _, V = graph(case["graph"])
    L, D, k = len(adj), case["D"], case["kind"]
    plans, edge_rows, gx = _uses(case, adj, V)
    claims, kernels = [], []
    for by, width in plans:
        sizes = segment_sizes(adj, V, by)
        warps = sizes.size * -(-width // 128)
        claims.append(("%s plan: %d segments x %d slices = %d warps >= %d (not the half-warp kernel)"
                       % (by, sizes.size, -(-width // 128), warps, SMALL_BATCH), warps >= SMALL_BATCH))
        heavy = int((sizes > HEAVY_SEGMENT).sum())
        if case["graph"] == QM9_20K:      # molecules have no hub: the heavy kernel walks an empty list
            claims.append(("%s plan: no segment above %d edges (largest %d)" % (by, HEAVY_SEGMENT, sizes.max()), heavy == 0))
        else:
            claims.append(("%s plan: %d segments above %d edges (largest %d)" % (by, heavy, HEAVY_SEGMENT, sizes.max()), heavy > 0))
    if case["graph"] != QM9_20K:
        claims.append(("D = %d > 128: gridDim.y = %d" % (D, -(-D // 128)), D > 128))
    if k == "ggnn" and case["cell"] == "gru":
        dist = gru_kink_distance(case)
        claims.append(("GRU gate pre-activations >= 1e-4 from the hard-sigmoid kinks (closest %.1e)" % dist, dist >= 1e-4))
    if edge_rows:
        claims.append(("per-edge dense gradient over %d rows of one type >= 20000" % edge_rows, edge_rows >= 20000))
    if k == "gather":
        kernels += GATHER
    elif k == "segment":
        kernels += segment_forward_kernels("max")
    elif k == "edge_aggregate":
        kernels += edge_backward_kernels("mean", True)
    elif k == "ggnn":
        kernels += edge_backward_kernels(case["agg"], False)
    elif k == "rgin" and not case["use_target"]:
        kernels += edge_backward_kernels("sum", False)
    elif k == "rgcn_fused":
        kernels += edge_backward_kernels("mean", case["normalize"])        # act_backward_kernel runs for every aggregation
    else:
        kernels += GATHER
    if gx is not None:
        kernels += DENSE_GRAD + [grad_x_kernel(*gx)]
    return claims, kernels


def test_case_regimes():
    """Every case is sized into the regime it is meant to test (no GPU needed)."""
    for case in CASES:
        claims, kernels = regime(case)
        assert kernels, case["id"]
        for text, holds in claims:
            print("%-36s %s" % (case["id"], text))
            assert holds, "%s: %s" % (case["id"], text)


def test_oracle_splits_tied_maxima_evenly():
    """The known answer of the max-gradient check holds for the float64 oracle too: k tied maxima get g / k each."""
    import torch
    data = torch.tensor([[1.0], [3.0], [3.0], [3.0], [2.0], [2.0], [0.5]], dtype=torch.float64, requires_grad=True)
    out = A.segment_reduce(data, torch.tensor([0, 0, 0, 0, 1, 1, 1]), 2, "max")
    out.backward(torch.tensor([[0.75], [0.5]], dtype=torch.float64))
    assert data.grad.flatten().tolist() == [0.0, 0.25, 0.25, 0.25, 0.25, 0.25, 0.0]


def test_planted_ties_are_the_maxima():
    """tied_segment_data: every planted (segment, column) has exactly its k in {2, 3} planted rows at the maximum."""
    adj, _, V = graph(PPI6K_ZIPF)
    _, tgt, _ = _messages(adj)
    data, planted = tied_segment_data(tgt, V, 16, np.random.default_rng(0))
    assert len(planted) == 16 * int((np.bincount(tgt, minlength=V) > HEAVY_SEGMENT).sum()) > 0
    for (v, c), rows in planted.items():
        col = data[tgt == v, c]
        assert col.max() == 3.75 and np.count_nonzero(col == 3.75) == rows.size and rows.size in (2, 3)
    assert np.abs(data).max() < 4 and np.all(data * 256 == np.round(data * 256))


def _assert_launched(what, names, kernels):
    for want in kernels:
        matched = sorted(n for n in names if want in n)
        assert matched, "%s: no launched kernel matches %r; launched: %s" % (what, want, sorted(names))
        print("%s: launched %s" % (what, matched[0]))


def _messages(adj):
    src = np.concatenate([a[:, 0] for a in adj]).astype(np.int64)
    tgt = np.concatenate([a[:, 1] for a in adj]).astype(np.int64)
    typ = np.concatenate([np.full(a.shape[0], l, dtype=np.int64) for l, a in enumerate(adj)])
    return src, tgt, typ


def _backward_twice(what, inp, out, grad, kernels):
    """Profile out.backward(grad) (the backward only), then run it again: the gradient must be bit-identical."""
    def step():
        inp.grad = None
        out.backward(grad, retain_graph=True)
    names = launched_kernels(step, kernels)
    _assert_launched(what, names, kernels)
    first = inp.grad.clone()
    step()
    assert bool((first == inp.grad).all()), "%s: the gradient differs between two runs" % what
    return first.cpu().numpy()


# ------------------------------------------------------------------ building blocks ---------------------------------
def run_gather(case, dev, _kernels):
    """(a) gather_rows and gather_table_rows, source and target; the target table is FiLM's [V, L, 2D] gamma | beta."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan, ops
    adj, _, V = graph(case["graph"])
    L, D = len(adj), case["D"]
    plan = GraphPlan(adj, V, device=dev)
    src, tgt, typ = _messages(adj)
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    x = rng.standard_normal((V, D)).astype(np.float32)
    steps = [("gather_rows source", ops.gather_rows, x, "source", src),
             ("gather_rows target", ops.gather_rows, x, "target", tgt),
             ("gather_table_rows source", ops.gather_table_rows, rng.standard_normal((V, L, D)).astype(np.float32), "source", src * L + typ),
             ("gather_table_rows target", ops.gather_table_rows, rng.standard_normal((V, L, 2 * D)).astype(np.float32), "target", tgt * L + typ)]
    for what, fn, table, side, idx in steps:
        flat = table.reshape(-1, table.shape[-1])
        inp = torch.as_tensor(table).to(dev).requires_grad_(True)
        rows = fn(inp, plan, side)
        assert np.array_equal(rows.detach().cpu().numpy(), flat[idx]), what
        g = rng.standard_normal(tuple(rows.shape)).astype(np.float32)
        got = _backward_twice(what, inp, rows, torch.as_tensor(g).to(dev), GATHER).reshape(flat.shape)
        want = torch.zeros(flat.shape, dtype=torch.float64).index_add_(0, torch.as_tensor(idx), torch.as_tensor(g, dtype=torch.float64))
        err = rel(got, want.numpy())
        print("%s %s: max-norm relative error %.2e" % (case["id"], what, err))
        assert err <= BLOCK_TOL, (what, err)


def tied_segment_data(tgt, V, D, rng, heavy=HEAVY_SEGMENT):
    """[M, D] on the grid of multiples of 2^-8 within +-3.5 (float32-exact sums of a few thousand terms), with exact ties
    planted at the maximum of hub segments: in every column of every segment above `heavy` edges, k in {2, 3} entries are set
    to 3.75, above everything else.  Returns (data, planted) with planted[(v, c)] = the tied rows."""
    data = (rng.integers(-896, 897, size=(tgt.size, D)) / 256.0).astype(np.float32)
    planted = {}
    for v in np.flatnonzero(np.bincount(tgt, minlength=V) > heavy):
        rows = np.flatnonzero(tgt == v)
        for c in range(D):
            pick = rng.choice(rows, size=int(rng.integers(2, 4)), replace=False)
            data[pick, c] = 3.75
            planted[(int(v), c)] = pick
    return data, planted


def run_segment(case, dev, _kernels):
    """(b) segment_aggregate sum / mean / sqrt_n / max over hub targets; ties of the max gradient planted exactly."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan, ops
    adj, _, V = graph(case["graph"])
    D = case["D"]
    plan = GraphPlan(adj, V, device=dev)
    _, tgt, _ = _messages(adj)
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    data, planted = tied_segment_data(tgt, V, D, rng)
    d64 = torch.as_tensor(data, dtype=torch.float64)
    mx = A.segment_reduce(d64, torch.as_tensor(tgt), V, "max")
    ties = torch.zeros((V, D), dtype=torch.float64).index_add_(0, torch.as_tensor(tgt), (d64 == mx[torch.as_tensor(tgt)]).double())
    print("%s: %d tied (segment, column) maxima, %d of them planted" % (case["id"], int((ties > 1).sum()), len(planted)))
    assert int((ties > 1).sum()) >= 300 and len(planted) >= 300
    proj = rng.standard_normal((V, D)).astype(np.float32)
    for agg in ("sum", "mean", "sqrt_n", "max"):
        what = "%s %s" % (case["id"], agg)
        dd = torch.as_tensor(data).to(dev).requires_grad_(True)
        kernels = segment_forward_kernels(agg)
        got_out = {}
        names = launched_kernels(lambda: got_out.update(out=ops.segment_aggregate(plan, dd, agg)), kernels)
        _assert_launched(what + " forward", names, kernels)
        out = got_out["out"]
        got = _backward_twice(what, dd, out, torch.as_tensor(proj).to(dev), [])
        x64 = d64.clone().requires_grad_(True)
        o64 = A.segment_reduce(x64, torch.as_tensor(tgt), V, agg)
        (o64 * torch.as_tensor(proj, dtype=torch.float64)).sum().backward()
        e_out, e_grad = rel(out.detach().cpu().numpy(), o64.detach().numpy()), rel(got, x64.grad.numpy())
        print("%s: max-norm relative error out %.2e, d_data %.2e" % (what, e_out, e_grad))
        assert e_out <= BLOCK_TOL and e_grad <= BLOCK_TOL, (what, e_out, e_grad)
        if agg == "max":                  # known answer: k tied maxima receive g / k each, the other entries nothing
            for (v, c), rows in planted.items():
                share = np.float32(proj[v, c]) / np.float32(rows.size)
                assert np.all(got[rows, c] == share), (v, c, got[rows, c], share)
                assert np.count_nonzero(got[tgt == v, c]) == rows.size, (v, c)
            for k in (2, 3):
                assert sum(r.size == k for r in planted.values()) > 0, "no segment with %d tied maxima" % k


def run_edge_aggregate(case, dev, _kernels):
    """(c) edge_aggregate sum / mean / sqrt_n, with and without in-degree scaling: the reverse (source, type) index."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan, ops
    adj, indeg, V = graph(case["graph"])
    L, D = len(adj), case["D"]
    plan = GraphPlan(adj, V, device=dev)
    src, tgt, typ = _messages(adj)
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    table = rng.standard_normal((V, L, D)).astype(np.float32)
    proj = rng.standard_normal((V, D)).astype(np.float32)
    cnt64 = torch.as_tensor(indeg, dtype=torch.float64)
    for agg in ("sum", "mean", "sqrt_n"):
        for scaled in (False, True):
            what = "%s %s%s" % (case["id"], agg, " scaled" if scaled else "")
            td = torch.as_tensor(table).to(dev).requires_grad_(True)
            out = ops.edge_aggregate(td, plan, torch.as_tensor(indeg).to(dev) if scaled else None, agg)
            got = _backward_twice(what, td, out, torch.as_tensor(proj).to(dev), edge_backward_kernels(agg, scaled))
            t64 = torch.as_tensor(table, dtype=torch.float64).requires_grad_(True)
            rows = t64[torch.as_tensor(src), torch.as_tensor(typ)]
            if scaled:
                rows = rows * (1.0 / (cnt64[torch.as_tensor(typ), torch.as_tensor(tgt)] + 1e-7)).unsqueeze(1)
            o64 = A.segment_reduce(rows, torch.as_tensor(tgt), V, agg)
            (o64 * torch.as_tensor(proj, dtype=torch.float64)).sum().backward()
            e_out, e_grad = rel(out.detach().cpu().numpy(), o64.detach().numpy()), rel(got, t64.grad.numpy())
            print("%s: max-norm relative error out %.2e, d_table %.2e" % (what, e_out, e_grad))
            assert e_out <= BLOCK_TOL and e_grad <= BLOCK_TOL, (what, e_out, e_grad)


# ------------------------------------------------------------------ layers ------------------------------------------
def _layer_fns(case, plan, adj, indeg, dev):
    """(engine_fn(h, w), oracle_fn(h64, w64), numpy weights, d_in) of a layer case."""
    import torch
    import tf_gnn_samples_b200 as G
    k, D = case["kind"], case["D"]
    L = len(adj)
    cnt, cnt64 = torch.as_tensor(indeg).to(dev), torch.as_tensor(indeg, dtype=torch.float64)
    seed = zlib.crc32(case["id"].encode()) % 10000
    if k == "ggnn":
        kw = dict(num_timesteps=case["T"], gated_unit_type=case["cell"], activation_function="tanh", message_aggregation_function=case["agg"])
        return (lambda h, w: G.sparse_ggnn_layer(h, plan, D, **kw, weights=w),
                lambda h, w: A.sparse_ggnn_layer(h, adj, **kw, weights=w), ggnn_weights(case, L), D)
    if k == "rgat":
        kw = dict(num_timesteps=case["T"], num_heads=case["K"], activation_function="tanh")
        return (lambda h, w: G.sparse_rgat_layer(h, plan, D, **kw, weights=w),
                lambda h, w: A.sparse_rgat_layer(h, adj, **kw, weights=w),
                W.rgat_weights(L, case["d_in"], D, seed=seed), case["d_in"])
    if k == "film":
        kw = dict(num_timesteps=case["T"], activation_function=case["act"], message_aggregation_function=case["agg"],
                  normalize_by_num_incoming=case["normalize"])
        return (lambda h, w: G.sparse_gnn_film_layer(h, plan, cnt, D, **kw, weights=w),
                lambda h, w: A.sparse_gnn_film_layer(h, adj, cnt64, **kw, weights=w),
                W.film_weights(L, D, D, seed=seed, num_timesteps=case["T"], random_ln=True), D)
    if k == "edge_mlp":
        kw = dict(activation_function="tanh", message_aggregation_function="sum", normalize_by_num_incoming=case["normalize"],
                  use_target_state_as_input=case["use_target"])
        return (lambda h, w: G.sparse_gnn_edge_mlp_layer(h, plan, cnt, D, **kw, num_edge_hidden_layers=case["hidden"], weights=w),
                lambda h, w: A.sparse_gnn_edge_mlp_layer(h, adj, cnt64, **kw, weights=w),
                W.edge_mlp_weights(L, D, D, case["hidden"], case["use_target"], seed=seed, random_ln=True), D)
    if k == "rgin":
        kw = dict(activation_function="tanh", message_aggregation_function=case.get("agg", "sum"), use_target_state_as_input=case["use_target"])
        return (lambda h, w: G.sparse_rgin_layer(h, plan, D, **kw, num_edge_MLP_hidden_layers=case["edge_hidden"],
                                                 num_aggr_MLP_hidden_layers=case["aggr_hidden"], weights=w),
                lambda h, w: A.sparse_rgin_layer(h, adj, **kw, weights=w),
                W.rgin_weights(L, D, D, case["edge_hidden"], case["aggr_hidden"], case["use_target"], seed=seed, random_ln=True), D)
    kw = dict(activation_function="tanh", message_aggregation_function="sum", use_both_source_and_target=True)
    return (lambda h, w: G.sparse_rgcn_layer(h, plan, cnt, D, **kw, weights=w),
            lambda h, w: A.sparse_rgcn_layer(h, adj, cnt64, **kw, weights=w),
            W.rgcn_weights(L, D, D, seed=seed, use_both_source_and_target=True), D)


def run_layer(case, dev, kernels):
    """Output, d_h and every weight gradient against torch float64 autograd (oracle/ref_autograd.py); backward profiled."""
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(case["graph"])
    plan = GraphPlan(adj, V, device=dev)
    engine_fn, oracle_fn, w, d_in = _layer_fns(case, plan, adj, indeg, dev)
    h = node_states(V, d_in, seed=zlib.crc32(case["id"].encode()) % 1000)
    errs, names = compare(engine_fn, oracle_fn, h, w, tol=LAYER_TOL, expect=kernels)
    _assert_launched(case["id"], names, kernels)
    worst = max(errs, key=errs.get)
    print("%s: largest max-norm relative error %.2e (%s)" % (case["id"], errs[worst], worst))


def run_rgcn_fused(case, dev, kernels):
    """One timestep through rgnn_rgcn_backward against the analytic gradients of oracle/ref_grads.py."""
    import torch
    import tf_gnn_samples_b200 as G
    adj, indeg, V = graph(case["graph"])
    L, D, d_in = len(adj), case["D"], case["d_in"]
    seed = zlib.crc32(case["id"].encode())
    plan = G.GraphPlan(adj, V, device=dev)
    h = node_states(V, d_in, seed=seed % 1000)
    w = W.rgcn_weights(L, d_in, D, seed=seed % 10000)
    g = np.random.default_rng(seed).standard_normal((V, D)).astype(np.float32)
    kw = dict(activation_function=case["act"], message_aggregation_function=case["agg"], normalize_by_num_incoming=case["normalize"])
    hg = torch.as_tensor(h).to(dev).requires_grad_(True)
    wg = [torch.as_tensor(a).to(dev).requires_grad_(True) for a in w["edge_weights"]]
    out = G.sparse_rgcn_layer(hg, plan, torch.as_tensor(indeg).to(dev), D, **kw, weights={"edge_weights": wg})
    loss = (out * torch.as_tensor(g).to(dev)).sum()

    def backward():
        for t in [hg] + wg:
            t.grad = None
        loss.backward(retain_graph=True)
    names = launched_kernels(backward, kernels)
    _assert_launched(case["id"], names, kernels)
    want_out = R.sparse_rgcn_layer(h, adj, indeg, D, weights=w, **kw)
    want_h, want_w = RG.rgcn_layer_grads(h, adj, indeg, g, case["act"], case["agg"], case["normalize"], weights=w)
    errs = {"out": rel(out.detach().cpu().numpy(), want_out), "d_h": rel(hg.grad.cpu().numpy(), want_h)}
    for l in range(L):
        errs["d_W%d" % l] = rel(wg[l].grad.cpu().numpy(), want_w[l])
    print("%s: %s" % (case["id"], {k: "%.1e" % v for k, v in errs.items()}))
    bad = {k: v for k, v in errs.items() if not v <= LAYER_TOL}
    assert not bad, bad


RUNNERS = {"gather": run_gather, "segment": run_segment, "edge_aggregate": run_edge_aggregate, "rgcn_fused": run_rgcn_fused}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_large_batch_gradient(cuda_device, case):
    _, kernels = regime(case)
    RUNNERS.get(case["kind"], run_layer)(case, cuda_device, kernels)

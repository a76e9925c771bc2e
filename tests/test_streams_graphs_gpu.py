"""GPU: CUDA-graph replay and cross-stream use of every layer family, forward and training, against the float64 oracle.

include/rgnn.h promises that all work goes on the caller's stream, that forwards make no hidden synchronisation and are
CUDA-graph capturable, and that calls are re-entrant on distinct plans and streams.  The bench's headline numbers are graph
replays, so this module checks the promise itself:

  A. forward capture and replay of every family: each of three rounds writes new node states (and, with the weight cache
     off, new weights) into the captured buffers in place, replays, and compares with the float64 oracle on that round's
     inputs and bit for bit with an eager call on the same plan -- a graph that baked in a host value or kept a stale
     pointer fails here;
  B. a plan built INSIDE the graph (deferred check) from adjacency copied in by the graph, replayed on three structures of
     one shape, each checked against the oracle and by plan.check(); one replay with a bad id makes check() raise;
  C. training under capture (forward + loss.backward(), torch's whole-network recipe) after one eager step, replayed with
     new states and weights, against float64 autograd; and the calls that cannot be captured (the first backward on a
     plan, a validated plan build, raw adjacency lists, a weight-cache flush) raise RgnnError up front;
  D. streams: every kernel of a call issued on stream s runs on s; a plan built on stream A (validated or deferred) is used
     on stream B with no host synchronisation; closing a plan while another stream still uses it;
  E. threads: two threads with their own plans and streams are bit-identical to the same calls made one after the other,
     while a third thread's invalid calls get their own error text.

test_case_regimes checks, without a GPU, the regime each case claims (hubs, pair table, whole-row layer norm, equal shapes)."""
import functools
import json
import threading
import time

import numpy as np
import pytest

from oracle import ref_autograd as A
from oracle import ref_layers as R
from tf_gnn_samples_b200 import weights as W

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, QM9_20K, SMALL_BATCH, graph, in_degrees
from helpers import assert_parity, assert_parity_8c, launched_kernels, node_states, rel, to_dev
from test_large_batch_training_gpu import tied_segment_data
from test_sharded_layers_gpu import autograd_oracle, engine_layer, make_weights, oracle_layer

TOL = 1e-4
ROUNDS = 3
PPI_BENCH = ("ppi", 2245, 59000, 0, False)          # bench.py's RGCN workload: V = 2,245, M = 120,245, L = 3
TRAIN_ZIPF = ("zipf", 2000, 3000, 3, 100, 48)      # 9,000 edges, hubs above the heavy threshold
SMALL_ZIPF = ("zipf", 600, 1000, 3, 30, 47)        # RGDCN's oracle holds a [E, K, K] tensor per type
LN_FAMILIES = ("film", "edge_mlp", "rgin")
HEAVY_PART = ["seg_reduce_heavy_part_kernel", "seg_reduce_heavy_finish_kernel"]


def max_in_degree(key):
    adj, _, V = graph(key)
    return int(in_degrees(adj, V).max())


def wants_pairs(key):
    adj, _, V = graph(key)
    return sum(a.shape[0] for a in adj) < 0.75 * V * len(adj)


# ---------------------------------------------------------------- helpers ------------------------------------------------
def layer(c, h, plan, cnt, w):
    """engine_layer of test_sharded_layers_gpu, plus the RGCN stack of bench.py and GGNN with T timesteps."""
    import tf_gnn_samples_b200 as G
    if c["kind"] == "stack3":
        return G.rgcn_layer_stack(h, plan, cnt, w, activation_function="ReLU", message_aggregation_function="sum",
                                  normalize_by_num_incoming=True)
    if c["kind"] == "ggnn":
        return G.sparse_ggnn_layer(h, plan, c["D"], num_timesteps=c.get("T", 1), gated_unit_type=c["cell"],
                                   activation_function=c.get("act", "tanh"), weights=w)
    return engine_layer(c, h, plan, cnt, w)


def oracle(c, h, adj, indeg, w, dtype=np.float64):
    if c["kind"] == "stack3":
        cur = h
        for wl in w:
            cur = R.sparse_rgcn_layer(cur, adj, indeg, c["D"], activation_function="ReLU", message_aggregation_function="sum",
                                      normalize_by_num_incoming=True, weights=wl, dtype=dtype)
        return cur
    if c["kind"] == "ggnn":
        return R.sparse_ggnn_layer(h, adj, c["D"], num_timesteps=c.get("T", 1), gated_unit_type=c["cell"],
                                   activation_function=c.get("act", "tanh"), weights=w, dtype=dtype)
    return oracle_layer(c, h, adj, indeg, w, dtype)


def weights_np(c, L, seed):
    if c["kind"] == "stack3":
        return [W.rgcn_weights(L, c["D"], c["D"], seed=seed + 10 * i) for i in range(3)]
    return make_weights(c, L, seed=seed)


def assign(dst, src):
    """Write the numpy weight container `src` into the torch container `dst` in place (same shapes)."""
    import torch
    if isinstance(dst, dict):
        for k in dst:
            assign(dst[k], src[k])
    elif isinstance(dst, (list, tuple)):
        for d, s in zip(dst, src):
            assign(d, s)
    elif dst is not None:
        with torch.no_grad():
            dst.copy_(torch.as_tensor(np.ascontiguousarray(src), dtype=torch.float32))


def check_parity(c, got, h, adj, indeg, w, what):
    want = oracle(c, h, adj, indeg, w)
    if c["kind"] in LN_FAMILIES:
        return assert_parity_8c(got, want, oracle(c, h, adj, indeg, w, np.float32), what)[0]
    return assert_parity(got, want, what, tol=TOL)


def capture(fn, device):
    """bench.py's recipe: two eager warm-up calls on a side stream, then torch.cuda.graph (global capture mode)."""
    import torch
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


@pytest.fixture
def weight_cache():
    """Sets the weight-cache mode for one test and restores the default (off) afterwards."""
    from tf_gnn_samples_b200.engine import set_weight_cache
    yield set_weight_cache
    set_weight_cache(False)


# ---------------------------------------------------------------- A. forward capture and replay --------------------------
# regime words (test_case_regimes): hub = a target above 512 incoming edges; pair = M < 0.75 V L (the compact pair table);
# ln_row = D > 128 and V >= 132 * 40 (the whole-row layer-norm epilogue); deferred = validate=False, never checked
FORWARD = [
    dict(id="rgcn_stack3_ppi_bench_cached", kind="stack3", graph=PPI_BENCH, D=256, cache=True),
    dict(id="rgcn_stack3_ppi_bench_uncached", kind="stack3", graph=PPI_BENCH, D=256),
    dict(id="rgcn_mean_both_zipf_hub_d128", kind="rgcn", graph=PPI6K_ZIPF, D=128, agg="mean", both=True, regime=["hub"],
         expect=HEAVY_PART),
    dict(id="ggnn_gru_t2_qm9_d64", kind="ggnn", graph=QM9_20K, D=64, cell="gru", T=2, regime=["pair"]),
    dict(id="rgat_k8_ppi_bench_d256", kind="rgat", graph=PPI_BENCH, D=256, heads=8),
    dict(id="rgat_half_zipf_d128_k4", kind="rgat", graph=PPI6K_ZIPF, D=128, heads=4),
    dict(id="film_ln_row_zipf_hub_d256", kind="film", graph=PPI6K_ZIPF, D=256, act="relu", normalize=True,
         regime=["hub", "ln_row"], expect=HEAVY_PART),
    dict(id="film_deferred_zipf_hub_d128", kind="film", graph=PPI6K_ZIPF, D=128, act="relu", validate=False,
         regime=["hub", "deferred"], expect=["seg_reduce_heavy_kernel<"]),
    dict(id="edge_mlp_h1_target_zipf_d128", kind="edge_mlp", graph=PPI6K_ZIPF, D=128, hidden=1, use_target=True,
         act="relu", normalize=True, regime=["hub"]),
    dict(id="rgin_target_aggr1_zipf_d128", kind="rgin", graph=PPI6K_ZIPF, D=128, edge_hidden=1, aggr_hidden=1,
         use_target=True, agg="mean", regime=["hub"]),
    dict(id="rgdcn_channel_k16_max", kind="rgdcn", graph=SMALL_ZIPF, D=64, K=16, full=False, tied=False, agg="max"),
    dict(id="rgdcn_full_k4_sum_norm", kind="rgdcn", graph=PPI6K_ZIPF, D=64, K=4, full=True, tied=False, normalize=True),
]


def regime_holds(word, c):
    adj, _, V = graph(c["graph"])
    if word == "hub":
        return max_in_degree(c["graph"]) > HEAVY_SEGMENT
    if word == "pair":
        return wants_pairs(c["graph"])
    if word == "ln_row":
        return c["D"] > 128 and V >= SMALL_BATCH
    if word == "deferred":
        return c.get("validate", True) is False
    raise ValueError(word)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FORWARD, ids=[c["id"] for c in FORWARD])
def test_forward_graph_replay_matches_oracle(cuda_device, weight_cache, case):
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(case["graph"])
    L, D, cached = len(adj), case["D"], case.get("cache", False)
    weight_cache(cached)
    plan = GraphPlan(adj, V, device=cuda_device, validate=case.get("validate", True))
    cnt = torch.as_tensor(indeg).to(cuda_device)
    h = torch.as_tensor(node_states(V, D, seed=90)).to(cuda_device)
    w_np = weights_np(case, L, seed=7)
    w = W.to_torch(w_np, cuda_device)
    fn = lambda: layer(case, h, plan, cnt, w)
    if case.get("expect"):
        names = launched_kernels(fn, case["expect"])
        missing = [s for s in case["expect"] if not any(s in n for n in names)]
        assert not missing, "%s: kernels %s not launched" % (case["id"], missing)
    g, out = capture(fn, cuda_device)
    errs = []
    for r in range(ROUNDS):
        h_np = node_states(V, D, seed=100 + r)
        h.copy_(torch.as_tensor(h_np))
        if not cached:
            w_np = weights_np(case, L, seed=20 + r)
            assign(w, w_np)
        g.replay()
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert torch.equal(out, fn()), "%s round %d: replay differs from an eager call" % (case["id"], r)
        errs.append(check_parity(case, got, h_np, adj, indeg, w_np, "%s round %d" % (case["id"], r)))
    print("%s: largest max-norm relative error over %d replays %.2e" % (case["id"], ROUNDS, max(errs)))


@pytest.mark.gpu
def test_building_blocks_graph_replay(cuda_device):
    """dense, segment_aggregate (max), edge_aggregate forward and backward and layer_norm in one graph, three rounds."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan, ops
    adj, indeg, V = graph(TRAIN_ZIPF)
    L, D = len(adj), 128
    M = sum(a.shape[0] for a in adj)
    src = np.concatenate([a[:, 0] for a in adj]).astype(np.int64)
    tgt = np.concatenate([a[:, 1] for a in adj]).astype(np.int64)
    typ = np.concatenate([np.full(a.shape[0], l) for l, a in enumerate(adj)])
    plan = GraphPlan(adj, V, device=cuda_device)
    cnt = torch.as_tensor(indeg).to(cuda_device)
    x, k, data = (torch.zeros(s, device=cuda_device) for s in ((V, D), (D, D), (M, D)))
    table, gout = torch.zeros((V, L, D), device=cuda_device), torch.zeros((V, D), device=cuda_device)
    gamma, beta = torch.zeros(D, device=cuda_device), torch.zeros(D, device=cuda_device)
    dtab = torch.empty((V, L, D), device=cuda_device)

    def fn():
        y = ops.dense(x, k, activation="tanh")
        s = ops.segment_aggregate(plan, data, "max")
        t = table.clone().requires_grad_(True)
        e = ops.edge_aggregate(t, plan, cnt, "sum")
        e.backward(gout)
        dtab.copy_(t.grad)
        return y, s, e, ops.layer_norm(y, gamma, beta)

    # the first backward on the plan builds its reverse index: eagerly, before the capture
    fn()
    g, outs = capture(fn, cuda_device)
    scale = 1.0 / (indeg[typ, tgt].astype(np.float64) + 1e-7)
    for r in range(ROUNDS):
        rng = np.random.default_rng(300 + r)
        vals = dict(x=node_states(V, D, seed=310 + r), k=(rng.standard_normal((D, D)) / np.sqrt(D)).astype(np.float32),
                    data=node_states(M, D, seed=320 + r), table=node_states(V * L, D, seed=330 + r).reshape(V, L, D),
                    gout=node_states(V, D, seed=340 + r), gamma=(1 + 0.1 * rng.standard_normal(D)).astype(np.float32),
                    beta=(0.1 * rng.standard_normal(D)).astype(np.float32))
        for t, v in ((x, "x"), (k, "k"), (data, "data"), (table, "table"), (gout, "gout"), (gamma, "gamma"), (beta, "beta")):
            t.copy_(torch.as_tensor(vals[v]))
        g.replay()
        torch.cuda.synchronize()
        eager = fn()
        for a, b in zip(outs, eager):
            assert torch.equal(a, b), "round %d: replay differs from an eager call" % r
        y64 = np.tanh(R.dense(vals["x"].astype(np.float64), vals["k"].astype(np.float64)))
        assert_parity(outs[0].detach().cpu().numpy(), y64, "dense round %d" % r)
        got_max, has_in = outs[1].detach().cpu().numpy(), in_degrees(adj, V) > 0
        assert_parity(got_max[has_in], R.unsorted_segment_max(vals["data"].astype(np.float64), tgt, V)[has_in],
                      "segment max round %d" % r)
        assert np.all(got_max[~has_in] == np.finfo(np.float32).min), "segment max of an empty segment"
        msg = vals["table"].astype(np.float64)[src, typ] * scale[:, None]
        assert_parity(outs[2].detach().cpu().numpy(), R.unsorted_segment_sum(msg, tgt, V), "edge_aggregate round %d" % r)
        d64 = np.zeros((V * L, D))
        np.add.at(d64, src * L + typ, vals["gout"].astype(np.float64)[tgt] * scale[:, None])
        assert_parity(dtab.cpu().numpy(), d64.reshape(V, L, D), "edge_aggregate backward round %d" % r)
        ln = R.layer_norm(y64, vals["gamma"].astype(np.float64), vals["beta"].astype(np.float64))
        assert_parity(outs[3].detach().cpu().numpy(), ln, "layer_norm round %d" % r)


@pytest.mark.gpu
def test_restricted_film_out_graph_replay(cuda_device):
    """A plan restricted to its first num_targets rows, FiLM writing into the caller's buffer (out=): the wanted rows follow
    the oracle on every replay, the rows at and beyond num_targets keep their NaN contents bit for bit."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(PPI6K_ZIPF)
    L, D, n = len(adj), 128, 4000
    plan = GraphPlan(adj, V, device=cuda_device).set_num_targets(n)
    cnt = torch.as_tensor(indeg).to(cuda_device)
    h = torch.zeros((V, D), device=cuda_device)
    w_np = W.film_weights(L, D, D, 13, random_ln=True)
    w = W.to_torch(w_np, cuda_device)
    out = torch.full((V, D), float("nan"), device=cuda_device)
    fn = lambda: G.sparse_gnn_film_layer(h, plan, cnt, D, normalize_by_num_incoming=True, weights=w, out=out)
    g, _ = capture(fn, cuda_device)
    c = dict(kind="film", D=D, act="relu", normalize=True)
    for r in range(ROUNDS):
        h_np = node_states(V, D, seed=400 + r)
        h.copy_(torch.as_tensor(h_np))
        w_np = W.film_weights(L, D, D, 14 + r, random_ln=True)
        assign(w, w_np)
        g.replay()
        torch.cuda.synchronize()
        bits = out[n:].contiguous().view(torch.int32)
        assert bool(torch.all(bits == 0x7FC00000).item()), "round %d: rows >= num_targets were written" % r
        got = out[:n].cpu().numpy()
        assert_parity_8c(got, oracle_layer(c, h_np, adj, indeg, w_np)[:n],
                         oracle_layer(c, h_np, adj, indeg, w_np, np.float32)[:n], "restricted FiLM out= round %d" % r)
        eager = torch.full((V, D), float("nan"), device=cuda_device)
        G.sparse_gnn_film_layer(h, plan, cnt, D, normalize_by_num_incoming=True, weights=w, out=eager)
        assert torch.equal(eager[:n], out[:n])


# ---------------------------------------------------------------- B. plan built inside the graph -------------------------
PLAN_V, PLAN_E, PLAN_L = 6000, 3000, 3


@functools.lru_cache(maxsize=None)
def structure(kind, seed):
    """Graphs of ONE shape (V = 6,000, 3 types of 3,000 edges): Zipf-skewed targets (hubs) or uniform ones."""
    from dispatch import zipf_isolated_graph
    if kind == "zipf":
        return zipf_isolated_graph(PLAN_V, PLAN_E, PLAN_L, 300, seed)
    rng = np.random.default_rng(seed)
    adj = [rng.integers(0, PLAN_V, size=(PLAN_E, 2)).astype(np.int32) for _ in range(PLAN_L)]
    return adj, np.stack([np.bincount(a[:, 1], minlength=PLAN_V) for a in adj]).astype(np.float32)


STRUCTURES = [("zipf", 61), ("uniform", 62), ("zipf", 63)]


@pytest.mark.gpu
def test_plan_built_inside_graph(cuda_device, weight_cache):
    """bench.py's e2e pattern: the graph copies the adjacency lists and in-degrees from pinned host buffers, builds the plan
    (validate=False) and runs the RGCN stack and a GGNN layer; the warm-up's last plan is garbage-collected during the
    capture, which must not invalidate it (GraphPlan.close defers the free).  Each replay on a new structure of the same shape equals the
    oracle on that structure and passes plan.check(); a replay with one out-of-range id makes check() raise."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan, RgnnError
    weight_cache(False)
    D = 64
    adj_host = [torch.empty((PLAN_E, 2), dtype=torch.int32).pin_memory() for _ in range(PLAN_L)]
    cnt_host = torch.empty((PLAN_L, PLAN_V), dtype=torch.float32).pin_memory()
    adj_dev = [torch.empty((PLAN_E, 2), dtype=torch.int32, device=cuda_device) for _ in range(PLAN_L)]
    cnt_dev = torch.empty((PLAN_L, PLAN_V), device=cuda_device)
    h = torch.as_tensor(node_states(PLAN_V, D, seed=70)).to(cuda_device)
    stack = dict(kind="stack3", D=D)
    ggnn = dict(kind="ggnn", D=D, cell="gru")
    ws_np, wg_np = weights_np(stack, PLAN_L, 71), make_weights(ggnn, PLAN_L, seed=72)
    ws, wg = W.to_torch(ws_np, cuda_device), W.to_torch(wg_np, cuda_device)
    holder = {}

    def load(adj, indeg):
        for t, a in zip(adj_host, adj):
            t.copy_(torch.as_tensor(a))
        cnt_host.copy_(torch.as_tensor(indeg))

    def step():
        for d, s in zip(adj_dev, adj_host):
            d.copy_(s, non_blocking=True)
        cnt_dev.copy_(cnt_host, non_blocking=True)
        p = GraphPlan(adj_dev, PLAN_V, device=cuda_device, validate=False)
        holder["plan"] = p
        return layer(stack, h, p, cnt_dev, ws), layer(ggnn, h, p, None, wg)

    load(*structure(*STRUCTURES[0]))
    g, (out_s, out_g) = capture(step, cuda_device)
    plan = holder["plan"]
    for kind, seed in STRUCTURES:
        adj, indeg = structure(kind, seed)
        load(adj, indeg)
        g.replay()
        torch.cuda.synchronize()
        plan.check()
        what = "%s graph %d" % (kind, seed)
        e1 = assert_parity(out_s.cpu().numpy(), oracle(stack, node_states(PLAN_V, D, seed=70), adj, indeg, ws_np),
                           "RGCN stack, " + what)
        e2 = assert_parity(out_g.cpu().numpy(), oracle(ggnn, node_states(PLAN_V, D, seed=70), adj, None, wg_np), "GGNN, " + what)
        print("%s: max in-degree %d, errors %.2e %.2e" % (what, in_degrees(adj, PLAN_V).max(), e1, e2))
    bad = [a.copy() for a in structure(*STRUCTURES[0])[0]]
    bad[1][17, 0] = PLAN_V                                  # one source id out of range
    load(bad, structure(*STRUCTURES[0])[1])
    g.replay()
    torch.cuda.synchronize()
    with pytest.raises(RgnnError, match="outside"):
        plan.check()


# ---------------------------------------------------------------- C. training under capture ------------------------------
TRAIN = [
    dict(id="ggnn_gru", kind="ggnn", D=64, cell="gru", cell_scale=0.5),
    dict(id="rgat_k4", kind="rgat", D=64, heads=4),
    dict(id="film_gelu_mean", kind="film", D=64, act="gelu", agg="mean", normalize=True),
    dict(id="edge_mlp_h1_target", kind="edge_mlp", D=64, hidden=1, use_target=True, normalize=True),
    dict(id="rgin_target_aggr1_mean", kind="rgin", D=64, edge_hidden=1, aggr_hidden=1, use_target=True, agg="mean"),
    dict(id="rgcn_composed_both", kind="rgcn", D=64, both=True, normalize=True),
    dict(id="rgcn_fused_gelu_sqrt_n", kind="rgcn", D=64, act="gelu", agg="sqrt_n", normalize=True),
    dict(id="rgcn_fused_tanh_sum", kind="rgcn", D=64, act="tanh", agg="sum", normalize=False),
]


def train_oracle(c, adj, indeg):
    import torch
    if c["kind"] == "segment_max":
        tgt = torch_cat_targets(adj)
        return lambda x, w: A.segment_reduce(x, tgt, int(indeg.shape[1]), "max")
    return autograd_oracle(c, adj, torch.as_tensor(indeg, dtype=torch.float64))


def torch_cat_targets(adj):
    import torch
    return torch.cat([torch.as_tensor(a[:, 1]).long() for a in adj])


def captured_training(c, device, fresh_plan=False):
    """(graph, out, leaves, set_inputs): forward + backward of case c captured after one eager step (torch's whole-network
    recipe: grads set to None before the capture, left in place between replays)."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan, ops
    adj, indeg, V = graph(TRAIN_ZIPF)
    L, D = len(adj), c["D"]
    plan = GraphPlan(adj, V, device=device)
    cnt = torch.as_tensor(indeg).to(device)
    if c["kind"] == "segment_max":
        M = sum(a.shape[0] for a in adj)
        hd = torch.zeros((M, D), device=device, requires_grad=True)
        wd = {}
        engine = lambda x, w: ops.segment_aggregate(plan, x, "max")
    else:
        hd = torch.zeros((V, D), device=device, requires_grad=True)
        wd = to_dev(make_weights(c, L, seed=5), device)
        engine = lambda x, w: layer(c, x, plan, cnt, w)
    proj = torch.as_tensor(np.random.default_rng(6).standard_normal((V, D)).astype(np.float32)).to(device)
    leaves = [hd] + list(A.flatten(wd).values())

    def step():
        out = engine(hd, wd)
        (out * proj).sum().backward()
        return out

    if not fresh_plan:
        step()
    for t in leaves:
        t.grad = None
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        if not fresh_plan:
            step()
            for t in leaves:
                t.grad = None
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    return g, out, hd, wd, proj


def train_inputs(c, r):
    adj, _, V = graph(TRAIN_ZIPF)
    if c["kind"] == "segment_max":
        data, _ = tied_segment_data(torch_cat_targets(adj).numpy(), V, c["D"], np.random.default_rng(500 + r))
        return data, {}
    return node_states(V, c["D"], seed=500 + r), make_weights(c, len(adj), seed=510 + r)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRAIN + [dict(id="segment_max_tied", kind="segment_max", D=32)],
                         ids=[c["id"] for c in TRAIN] + ["segment_max_tied"])
def test_training_graph_replay_matches_float64_autograd(cuda_device, weight_cache, case):
    """Forward + loss.backward() captured after one eager step and replayed with new node states and weights copied in
    place: the output, d_h and every weight gradient equal float64 autograd (hubs in the graph: the one-CTA heavy kernels
    of the regrouped plans walk their lists on the device inside the graph)."""
    import torch
    weight_cache(False)
    adj, indeg, V = graph(TRAIN_ZIPF)
    g, out, hd, wd, proj = captured_training(case, cuda_device)
    fo = train_oracle(case, adj, indeg)
    worst = {}
    for r in range(2):
        h_np, w_np = train_inputs(case, r)
        with torch.no_grad():
            hd.copy_(torch.as_tensor(h_np))
        assign(wd, w_np)
        g.replay()
        torch.cuda.synchronize()
        h64 = torch.as_tensor(h_np, dtype=torch.float64).requires_grad_(True)
        w64 = A.to_torch64(w_np)
        out64 = fo(h64, w64)
        (out64 * proj.cpu().double()).sum().backward()
        rows = in_degrees(adj, V) > 0 if case["kind"] == "segment_max" else slice(None)   # empty segments: float32 lowest
        errs = {"out": rel(out.detach().cpu().numpy()[rows], out64.detach().numpy()[rows]),
                "d_h": rel(hd.grad.cpu().numpy(), h64.grad.numpy())}
        fd, f64 = A.flatten(wd), A.flatten(w64)
        for k in fd:
            if f64[k].grad is None:
                continue
            assert fd[k].grad is not None, "no gradient reached %s" % k
            errs["d_" + k] = rel(fd[k].grad.cpu().numpy(), f64[k].grad.numpy())
        bad = {k: v for k, v in errs.items() if not v <= TOL}
        assert not bad, "%s round %d: %s" % (case["id"], r, bad)
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("%s: %s" % (case["id"], {k: "%.1e" % v for k, v in worst.items()}))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["rgcn_fused", "film"])
def test_first_backward_on_fresh_plan_refused_under_capture(cuda_device, weight_cache, kind):
    """The first backward on a plan builds lazy state (the library's reverse index; the Python index views and regrouped
    plans): inside a capture that state would be an unfilled graph allocation kept by the plan.  It raises RgnnError naming
    the eager warm-up before anything is recorded; after one eager step the same capture works (the replay test above)."""
    import torch
    from tf_gnn_samples_b200 import RgnnError
    weight_cache(False)
    c = dict(id=kind, kind="rgcn", D=64, act="tanh") if kind == "rgcn_fused" else dict(id=kind, kind="film", D=64)
    with pytest.raises(RgnnError, match="eagerly"):
        captured_training(c, cuda_device, fresh_plan=True)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_synchronising_calls_refused_under_capture(cuda_device, weight_cache):
    """A validated plan build, a layer called with raw adjacency lists and a weight-cache flush (a cached weight changed in
    place) synchronise or free memory: under capture each raises RgnnError up front, and the capture is still usable."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan, RgnnError
    adj, indeg, V = graph(TRAIN_ZIPF)
    D, L = 64, len(adj)
    adj_dev = [torch.as_tensor(a).to(cuda_device) for a in adj]
    h = torch.as_tensor(node_states(V, D, seed=8)).to(cuda_device)
    weight_cache(True)
    w = W.to_torch(W.rgcn_weights(L, D, D, seed=9), cuda_device)
    plan = GraphPlan(adj_dev, V, device=cuda_device)
    fn = lambda: G.sparse_rgcn_layer(h, plan, None, D, normalize_by_num_incoming=False, weights=w)
    fn()
    torch.cuda.synchronize()
    calls = [("validate=True", lambda: GraphPlan(adj_dev, V, device=cuda_device)),
             ("raw adjacency lists", lambda: G.sparse_rgcn_layer(h, adj_dev, None, D, normalize_by_num_incoming=False,
                                                                 weights=w))]
    for what, call in calls:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
            with pytest.raises(RgnnError, match="capture"):
                call()
            out = fn()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, fn()), what
    with torch.no_grad():
        w["edge_weights"][0].mul_(0.5)                       # the cached images are stale now
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(RgnnError, match="capture"):
            fn()
    out = fn()                                                # eagerly: flushes and repacks
    want = R.sparse_rgcn_layer(node_states(V, D, seed=8), adj, None, D, normalize_by_num_incoming=False,
                               weights={"edge_weights": [t.cpu().numpy() for t in w["edge_weights"]]})
    assert_parity(out.cpu().numpy(), want, "after the refused flush")


# ---------------------------------------------------------------- D. streams ---------------------------------------------
@pytest.mark.gpu
def test_kernels_run_on_the_callers_stream(cuda_device, tmp_path):
    """Plan creation and one call of every family under torch.cuda.stream(s), on a plan built on the default stream: every
    kernel in the profiler trace of that window, torch's included, runs on one stream (a launch onto the plan's creation
    stream would add a second)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(TRAIN_ZIPF)
    L = len(adj)
    cnt = torch.as_tensor(indeg).to(cuda_device)
    h = torch.as_tensor(node_states(V, 64, seed=3)).to(cuda_device)
    base = GraphPlan(adj, V, device=cuda_device)             # built on the default stream
    fams = [c for c in FORWARD if c["kind"] not in ("stack3",)]
    calls = [(c, W.to_torch(weights_np(dict(c, D=64), L, 1), cuda_device)) for c in fams]
    s = torch.cuda.Stream(device=cuda_device)
    # the device trace has been seen to come back without some kernels (helpers.launched_kernels): the window is padded
    # and profiled again, at most three times, while the plan build is missing from it
    for attempt in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.05)
            with torch.cuda.stream(s):
                marker = torch.ones(1 << 16, device=cuda_device)
                marker.mul_(3.0)
                GraphPlan(adj, V, device=cuda_device)
                GraphPlan(adj, V, device=cuda_device, validate=False)
                for c, w in calls:
                    layer(dict(c, D=64), h, base, cnt, w)
            torch.cuda.synchronize()
            time.sleep(0.05)
        path = tmp_path / ("trace%d.json" % attempt)
        prof.export_chrome_trace(str(path))
        events = [e for e in json.loads(path.read_text())["traceEvents"] if e.get("cat") == "kernel"]
        if any("plan_concat_kernel" in e["name"] for e in events):
            break
    # every kernel in the window -- the torch marker, both plan builds, every layer on `base` -- runs on ONE stream; a
    # library launch onto `base`'s creation stream would add a second one
    streams = {e["args"]["stream"] for e in events}
    assert any("plan_concat_kernel" in e["name"] for e in events) and len(events) > 50, len(events)
    assert len(streams) == 1, "kernels on %d streams: %s" % (len(streams), sorted({(e["args"]["stream"], e["name"][:60])
                                                                                   for e in events})[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("validate", [True, False], ids=["validated", "deferred"])
def test_plan_used_on_another_stream(cuda_device, weight_cache, validate):
    """Build the plan on stream A and, with no host synchronisation, run a forward and a training step of every family on
    stream B: each equals the oracle.  A deferred build is still running on A when B starts: the first use of the plan on
    B waits for it."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    weight_cache(False)
    adj, indeg, V = graph(TRAIN_ZIPF)
    L, D = len(adj), 64
    a, b = torch.cuda.Stream(device=cuda_device), torch.cuda.Stream(device=cuda_device)
    h_np = node_states(V, D, seed=33)
    cases = [c for c in FORWARD if c["kind"] not in ("stack3",)]
    w_np = [weights_np(dict(c, D=D), L, 34) for c in cases]
    h = torch.as_tensor(h_np).to(cuda_device)
    cnt = torch.as_tensor(indeg).to(cuda_device)
    ws = [W.to_torch(w, cuda_device) for w in w_np]
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(20_000_000)                        # the build queues behind ~10 ms of work on A
        plan = GraphPlan(adj, V, device=cuda_device, validate=validate)
    outs = []
    with torch.cuda.stream(b):
        for c, w in zip(cases, ws):
            outs.append(layer(dict(c, D=D), h, plan, cnt, w))
    torch.cuda.synchronize()
    for c, o, w in zip(cases, outs, w_np):
        check_parity(dict(c, D=D), o.cpu().numpy(), h_np, adj, indeg, w, "%s on stream B" % c["id"])
    with torch.cuda.stream(a):
        torch.cuda._sleep(20_000_000)
        plan2 = GraphPlan(adj, V, device=cuda_device, validate=validate)
    c = TRAIN[-2]                                             # the fused RGCN backward: builds the reverse index on B
    with torch.cuda.stream(b):
        hd = torch.as_tensor(h_np).to(cuda_device).requires_grad_(True)
        wd = to_dev(make_weights(c, L, seed=35), cuda_device)
        out = layer(c, hd, plan2, cnt, wd)
        out.sum().backward()
    torch.cuda.synchronize()
    h64 = torch.as_tensor(h_np, dtype=torch.float64).requires_grad_(True)
    out64 = train_oracle(c, adj, indeg)(h64, A.to_torch64(make_weights(c, L, seed=35)))
    out64.sum().backward()
    assert rel(out.detach().cpu().numpy(), out64.detach().numpy()) <= TOL
    assert rel(hd.grad.cpu().numpy(), h64.grad.numpy()) <= TOL


def same_shape_graph(seed):
    """TRAIN_ZIPF's shape (V, L, every E_l) with other edges: a plan of it takes the same pool blocks as one of TRAIN_ZIPF."""
    from dispatch import zipf_isolated_graph
    return zipf_isolated_graph(2000, 3000, 3, 100, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("backward", [False, True], ids=["forward", "backward"])
def test_close_while_another_stream_uses_the_plan(cuda_device, weight_cache, backward):
    """Stream B sleeps ~100 ms, then runs a layer (and its backward: the reverse index is built on B) with plan P1 built on
    A.  Without synchronising, P1 is closed, P2 of the same shape is built on A and used on A.  B's result equals the oracle
    on P1's graph: close() orders the free on A after B's queued work."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    weight_cache(False)
    adj1, indeg1, V = graph(TRAIN_ZIPF)
    adj2, indeg2 = same_shape_graph(49)
    L, D = len(adj1), 64
    c = dict(id="rgcn", kind="rgcn", D=D, act="tanh", normalize=True)
    a, b = torch.cuda.Stream(device=cuda_device), torch.cuda.Stream(device=cuda_device)
    h_np = node_states(V, D, seed=44)
    w_np = make_weights(c, L, seed=45)
    with torch.cuda.stream(a):
        p1 = GraphPlan(adj1, V, device=cuda_device)
    h = torch.as_tensor(h_np).to(cuda_device).requires_grad_(backward)
    wd = to_dev(w_np, cuda_device) if backward else W.to_torch(w_np, cuda_device)
    cnt1 = torch.as_tensor(indeg1).to(cuda_device)
    cnt2 = torch.as_tensor(indeg2).to(cuda_device)
    torch.cuda.synchronize()
    with torch.cuda.stream(b):
        torch.cuda._sleep(200_000_000)                       # ~100 ms at H100 clocks
        out = layer(c, h, p1, cnt1, wd)
        if backward:
            out.sum().backward()
    with torch.cuda.stream(a):
        p1.close()
        p2 = GraphPlan(adj2, V, device=cuda_device)
        with torch.no_grad():
            other = layer(c, h.detach(), p2, cnt2, W.to_torch(w_np, cuda_device))
    torch.cuda.synchronize()
    assert_parity(out.detach().cpu().numpy(), oracle_layer(c, h_np, adj1, indeg1, w_np), "B's layer on P1")
    assert_parity(other.cpu().numpy(), oracle_layer(c, h_np, adj2, indeg2, w_np), "A's layer on P2")
    if backward:
        h64 = torch.as_tensor(h_np, dtype=torch.float64).requires_grad_(True)
        out64 = train_oracle(c, adj1, indeg1)(h64, A.to_torch64(w_np))
        out64.sum().backward()
        assert rel(h.grad.cpu().numpy(), h64.grad.numpy()) <= TOL


# ---------------------------------------------------------------- E. threads ---------------------------------------------
@pytest.mark.gpu
def test_threads_with_own_plans_and_streams(cuda_device, weight_cache):
    """Two threads, each with its own plan and stream (GGNN with the weight cache on; FiLM), 20 iterations each: bit-identical
    to the same calls made one after the other.  A third thread's invalid calls meanwhile get their own error text."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan, RgnnError
    from tf_gnn_samples_b200.engine import check, load_library
    weight_cache(True)
    adj, indeg, V = graph(TRAIN_ZIPF)
    L, D, iters = len(adj), 64, 20
    cnt = torch.as_tensor(indeg).to(cuda_device)
    jobs = [(dict(kind="ggnn", D=D, cell="gru"), make_weights(dict(kind="ggnn", D=D, cell="gru"), L, seed=51)),
            (dict(kind="film", D=D, act="relu", normalize=True), make_weights(dict(kind="film", D=D), L, seed=52))]
    plans = [GraphPlan(adj, V, device=cuda_device) for _ in jobs]
    ws = [W.to_torch(w, cuda_device) for _, w in jobs]
    hs = [[torch.as_tensor(node_states(V, D, seed=600 + 100 * j + i)).to(cuda_device) for i in range(iters)]
          for j in range(len(jobs))]
    serial = [[layer(c, x, p, cnt, w) for x in xs] for (c, _), p, w, xs in zip(jobs, plans, ws, hs)]
    torch.cuda.synchronize()
    results, errors, bad_msgs = [[None] * iters for _ in jobs], [], []
    start = threading.Barrier(3)

    def worker(j):
        try:
            s = torch.cuda.Stream(device=cuda_device)
            start.wait()
            with torch.cuda.stream(s):
                for i in range(iters):
                    results[j][i] = layer(jobs[j][0], hs[j][i], plans[j], cnt, ws[j])
            s.synchronize()
        except Exception as exc:                              # surfaced in the main thread
            errors.append(repr(exc))

    x6 = torch.zeros((V, 6), device=cuda_device)
    w6 = W.to_torch(W.rgcn_weights(L, 6, 6), cuda_device)     # one set: a new address per call would flush the weight cache
    other = GraphPlan(adj, V, device=cuda_device)

    def invalid():
        lib = load_library()
        start.wait()
        for _ in range(iters):
            try:
                G.sparse_rgcn_layer(x6, other, None, 6, normalize_by_num_incoming=False, weights=w6)
            except RgnnError as exc:
                bad_msgs.append(exc.message)
            rc = lib.rgnn_plan_set_num_targets(other.handle, V + 1)
            bad_msgs.append(lib.rgnn_last_error().decode())
            if rc == 0:
                errors.append("set_num_targets(V + 1) was accepted")

    threads = [threading.Thread(target=worker, args=(j,)) for j in range(len(jobs))] + [threading.Thread(target=invalid)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for j in range(len(jobs)):
        for i in range(iters):
            assert torch.equal(results[j][i], serial[j][i]), "thread %d iteration %d differs from the serial call" % (j, i)
    assert len(bad_msgs) == 2 * iters
    assert all("multiple" in m and "4" in m for m in bad_msgs[0::2]), set(bad_msgs[0::2])
    assert all("outside [0, V=%d]" % V in m for m in bad_msgs[1::2]), set(bad_msgs[1::2])


# ---------------------------------------------------------------- F. without a GPU ---------------------------------------
def test_case_regimes():
    """The regime every case claims holds, and the shapes the scheduling tests rely on are as stated."""
    for c in FORWARD:
        for word in c.get("regime", []):
            assert regime_holds(word, c), "%s: regime '%s' does not hold" % (c["id"], word)
    # the bench's RGCN shape
    adj, _, V = graph(PPI_BENCH)
    assert (V, sum(a.shape[0] for a in adj), len(adj)) == (2245, 120245, 3)
    # B: three structures of one shape; hubs in the Zipf ones; M < 0.75 V L, so the pair table is built inside the graph
    for kind, seed in STRUCTURES:
        a, indeg = structure(kind, seed)
        assert [x.shape for x in a] == [(PLAN_E, 2)] * PLAN_L
        assert (in_degrees(a, PLAN_V).max() > HEAVY_SEGMENT) == (kind == "zipf")
        assert PLAN_E * PLAN_L < 0.75 * PLAN_V * PLAN_L
    # C and D: the training graph has hubs; D3's two graphs have equal V, L, every E_l and pair-table regime
    assert max_in_degree(TRAIN_ZIPF) > HEAVY_SEGMENT
    adj1, _, V1 = graph(TRAIN_ZIPF)
    adj2, _ = same_shape_graph(49)
    assert [x.shape for x in adj1] == [x.shape for x in adj2] and V1 == 2000
    m = sum(x.shape[0] for x in adj1)
    assert (m < 0.75 * V1 * 3) == (sum(x.shape[0] for x in adj2) < 0.75 * V1 * 3)
    assert {"stack3", "rgcn", "ggnn", "rgat", "film", "edge_mlp", "rgin", "rgdcn"} == {c["kind"] for c in FORWARD}

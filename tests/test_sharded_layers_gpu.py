"""GPU: restricted-target (sharded) execution of every layer family against the float64 oracle.

One rank of a node-range partition runs a layer on its local graph (owned nodes first, halo nodes after them) through a
plan restricted to its owned rows (GraphPlan.set_num_targets / rgnn_plan_set_num_targets).  Every family honours that
restriction in its own way (the segment reduce, the GGNN cell, FiLM's gamma / beta GEMM, RGIN's aggregation MLP, the RGAT
softmax, RGDCN's dynamic kernels), so every family is checked here:

  * forward: the owned rows of every rank, reassembled, equal the oracle on the WHOLE graph (1e-4; assert_parity_8c for
    the layer-norm layers), in the regimes the restricted plan changes -- compact pair table or not, a hub inside the owned
    range (heavy part / finish kernels with V = num_targets), deferred validation, the layer-norm epilogue with NV > 1 and
    the split layer norm, a packed graph without halo, BASELINE config-5 size;
  * the halo-row contract of include/rgnn.h: rows >= num_targets are left untouched (a NaN-filled output buffer keeps its
    NaNs bit for bit) and, through the Python API, are zero; also with num_targets = 0 and with a hub that is not wanted;
  * multi-layer stacks on "virtual ranks" (ShardedGraph exchange on one GPU) for every family, overlapped or not;
  * training on rank-local plans: autograd through the per-rank gathers of a global leaf is the all-to-all return of the
    halo gradients, so d_h and the rank-summed weight gradients must equal float64 autograd on the whole graph;
  * the restricted calls that must be refused.

Each forward case states its regime; test_case_regimes checks those statements without a GPU."""
import functools
import importlib

import numpy as np
import pytest

from oracle import ref_autograd as A
from oracle import ref_layers as R
from tf_gnn_samples_b200 import batching, weights as W
from tf_gnn_samples_b200.partition import NodeRangePartition

from dispatch import HEAVY_SEGMENT, PPI6K_DENSE, PPI6K_ZIPF, QM9_20K, SMALL_BATCH, graph as dispatch_graph
from helpers import assert_parity, assert_parity_8c, compare, launched_kernels, node_states

TOL = 1e-4
SMALL_ZIPF = ("zipf", 600, 1000, 3, 30, 47)        # 3,000 edges: RGDCN's K = 128 oracle holds a [E, K, K] tensor per type
TRAIN_ZIPF = ("zipf", 2000, 3000, 3, 100, 48)      # 9,000 edges, hubs above the heavy threshold
CONFIG5 = ("varmisuse", 0)                         # BASELINE config 5: V = 50,000, M = 1,000,000, L = 6
PACKED = ("varmisuse", 4)                          # the same size, 4 graphs packed block-diagonally
LN_FAMILIES = ("film", "edge_mlp", "rgin")


@functools.lru_cache(maxsize=None)
def graph(key):
    if key[0] == "varmisuse":
        b = batching.varmisuse_like_batch(packed_graphs=key[1], seed=0)
        return b.adjacency_lists, b.type_to_num_incoming_edges, b.num_nodes
    return dispatch_graph(key)


@functools.lru_cache(maxsize=None)
def partition(key, world):
    adj, indeg, V = graph(key)
    return tuple(NodeRangePartition(adj, indeg, V, r, world) for r in range(world))


def local_ids(part):
    """Global id of every local row: the owned range, then the halo (what the exchange delivers)."""
    return np.concatenate([np.arange(part.lo, part.hi), part.halo_global]).astype(np.int64)


def local_in_degree(part):
    return np.bincount(np.concatenate([a[:, 1] for a in part.local_adjacency_lists]), minlength=part.n_local)


# ---------------------------------------------------------------- the families ------------------------------------------
def make_weights(c, L, seed=7):
    k, D = c["kind"], c["D"]
    if k in ("rgcn", "rgcn_stack"):
        return W.rgcn_weights(L, D, D, seed, use_both_source_and_target=c.get("both", False))
    if k == "ggnn":
        w = W.ggnn_weights(L, D, seed, cell=c["cell"], random_bias=True)
        w["cell"] = {n: v * np.float32(c.get("cell_scale", 1.0)) for n, v in w["cell"].items()}
        return w
    if k == "rgat":
        return W.rgat_weights(L, D, D, seed)
    if k == "film":
        return W.film_weights(L, D, D, seed, random_ln=True)
    if k == "edge_mlp":
        return W.edge_mlp_weights(L, D, D, c["hidden"], c["use_target"], seed, random_ln=True)
    if k == "rgin":
        return W.rgin_weights(L, D, D, c["edge_hidden"], c["aggr_hidden"], c["use_target"], seed, random_ln=True)
    return W.rgdcn_weights(L, D // c["K"], c["K"], c["full"], c["tied"], seed, stddev=c.get("stddev", 0.5 / c["K"]))


def engine_layer(c, h, plan, cnt, w):
    """The engine's layer function of case c on node states h (torch) and plan; cnt: [L, V] in-degrees (torch)."""
    import tf_gnn_samples_b200 as G
    k, D, act, agg, norm = c["kind"], c["D"], c.get("act", "tanh"), c.get("agg", "sum"), c.get("normalize", False)
    if k == "rgcn":
        return G.sparse_rgcn_layer(h, plan, cnt, D, activation_function=act, message_aggregation_function=agg,
                                   normalize_by_num_incoming=norm, use_both_source_and_target=c.get("both", False), weights=w)
    if k == "rgcn_stack":
        return G.rgcn_layer_stack(h, plan, cnt, [w], activation_function=act, message_aggregation_function=agg,
                                  normalize_by_num_incoming=norm)
    if k == "ggnn":
        return G.sparse_ggnn_layer(h, plan, D, gated_unit_type=c["cell"], activation_function=act,
                                   message_aggregation_function=agg, weights=w)
    if k == "rgat":
        return G.sparse_rgat_layer(h, plan, D, num_heads=c["heads"], activation_function=act, weights=w)
    if k == "film":
        return G.sparse_gnn_film_layer(h, plan, cnt, D, activation_function=act, message_aggregation_function=agg,
                                       normalize_by_num_incoming=norm, weights=w)
    if k == "edge_mlp":
        return G.sparse_gnn_edge_mlp_layer(h, plan, cnt, D, activation_function=act, message_aggregation_function=agg,
                                           normalize_by_num_incoming=norm, use_target_state_as_input=c["use_target"],
                                           num_edge_hidden_layers=c["hidden"], weights=w)
    if k == "rgin":
        return G.sparse_rgin_layer(h, plan, D, activation_function=act, message_aggregation_function=agg,
                                   use_target_state_as_input=c["use_target"], num_edge_MLP_hidden_layers=c["edge_hidden"],
                                   num_aggr_MLP_hidden_layers=c["aggr_hidden"], weights=w)
    return G.sparse_rgdcn_layer(h, plan, cnt, num_channels=D // c["K"], channel_dim=c["K"],
                                use_full_state_for_channel_weights=c["full"], tie_channel_weights=c["tied"],
                                activation_function=act, message_aggregation_function=agg, normalize_by_num_incoming=norm,
                                weights=w)


def oracle_layer(c, h, adj, indeg, w, dtype=np.float64):
    """oracle/ref_layers.py on the whole graph."""
    k, D, act, agg, norm = c["kind"], c["D"], c.get("act", "tanh"), c.get("agg", "sum"), c.get("normalize", False)
    if k in ("rgcn", "rgcn_stack"):
        return R.sparse_rgcn_layer(h, adj, indeg, D, activation_function=act, message_aggregation_function=agg,
                                   normalize_by_num_incoming=norm, use_both_source_and_target=c.get("both", False),
                                   weights=w, dtype=dtype)
    if k == "ggnn":
        return R.sparse_ggnn_layer(h, adj, D, gated_unit_type=c["cell"], activation_function=act,
                                   message_aggregation_function=agg, weights=w, dtype=dtype)
    if k == "rgat":
        return R.sparse_rgat_layer(h, adj, D, num_heads=c["heads"], activation_function=act, weights=w, dtype=dtype)
    if k == "film":
        return R.sparse_gnn_film_layer(h, adj, indeg, D, activation_function=act, message_aggregation_function=agg,
                                       normalize_by_num_incoming=norm, weights=w, dtype=dtype)
    if k == "edge_mlp":
        return R.sparse_gnn_edge_mlp_layer(h, adj, indeg, D, activation_function=act, message_aggregation_function=agg,
                                           normalize_by_num_incoming=norm, use_target_state_as_input=c["use_target"],
                                           num_edge_hidden_layers=c["hidden"], weights=w, dtype=dtype)
    if k == "rgin":
        return R.sparse_rgin_layer(h, adj, D, activation_function=act, message_aggregation_function=agg,
                                   use_target_state_as_input=c["use_target"], num_edge_MLP_hidden_layers=c["edge_hidden"],
                                   num_aggr_MLP_hidden_layers=c["aggr_hidden"], weights=w, dtype=dtype)
    return R.sparse_rgdcn_layer(h, adj, indeg, num_channels=D // c["K"], channel_dim=c["K"],
                                use_full_state_for_channel_weights=c["full"], tie_channel_weights=c["tied"],
                                activation_function=act, message_aggregation_function=agg, normalize_by_num_incoming=norm,
                                weights=w, dtype=dtype)


# ---------------------------------------------------------------- A. restricted forward ---------------------------------
# regime words (checked by test_case_regimes, every word below is reached by at least one case):
#   pair      every rank's local plan builds the compact pair table: M_local < 0.75 * n_local * L
#   no_pair   no rank's does: M_local >= 0.75 * n_local * L
#   hub       every rank owns a target with more than 512 incoming edges (heavy part / finish kernels with V = num_targets)
#   deferred  plans built with validate=False: the heavy count is never read back, the one-CTA heavy kernel walks the list
#   ln_split  D > 128 and n_own < 132 * 40 on every rank: reduce per 128-column slice, then the layer-norm kernel
#   ln_nv     D > 128 and n_own >= 132 * 40 on every rank: the whole-row layer-norm epilogue with NV = D / 128 > 1
#   no_halo   some rank has no halo row
#   config5   BASELINE config-5 size: V = 50,000, M = 1,000,000, world 4
HEAVY_PART = ["seg_reduce_heavy_part_kernel", "seg_reduce_heavy_finish_kernel"]
CASES = [
    dict(id="rgcn_sum_norm_qm9_d64", kind="rgcn", graph=QM9_20K, world=3, D=64, agg="sum", normalize=True, regime=["pair"]),
    dict(id="rgcn_mean_zipf_hub_d128", kind="rgcn", graph=PPI6K_ZIPF, world=3, D=128, agg="mean", regime=["hub"],
         expect=HEAVY_PART),
    dict(id="rgcn_max_dense_d64", kind="rgcn", graph=PPI6K_DENSE, world=2, D=64, agg="max", act="relu", regime=["no_pair"]),
    dict(id="rgcn_both_zipf_deferred_d256", kind="rgcn", graph=PPI6K_ZIPF, world=3, D=256, both=True, normalize=True,
         validate=False, regime=["hub", "deferred"], expect=["seg_reduce_heavy_kernel<"]),
    dict(id="rgcn_stack1_packed_d64", kind="rgcn_stack", graph=PACKED, world=4, D=64, act="relu", normalize=True,
         regime=["no_halo"]),
    dict(id="rgcn_sum_config5_d32", kind="rgcn", graph=CONFIG5, world=4, D=32, normalize=True, regime=["config5"]),
    dict(id="ggnn_gru_qm9_d64", kind="ggnn", graph=QM9_20K, world=2, D=64, cell="gru", regime=["pair"]),
    dict(id="ggnn_rnn_zipf_hub_d128", kind="ggnn", graph=PPI6K_ZIPF, world=3, D=128, cell="rnn", agg="mean", regime=["hub"],
         expect=HEAVY_PART),
    dict(id="rgat_half_zipf_d128_k4", kind="rgat", graph=PPI6K_ZIPF, world=3, D=128, heads=4, expect=["seg_rgat_half_kernel"]),
    dict(id="rgat_fused_zipf_d128_k1", kind="rgat", graph=PPI6K_ZIPF, world=2, D=128, heads=1, expect=["seg_rgat_kernel<1, true>"]),
    dict(id="rgat_unfused_zipf_d96_k2", kind="rgat", graph=PPI6K_ZIPF, world=3, D=96, heads=2,
         expect=["rgat_scores_kernel", "seg_rgat_kernel<1, false>"]),
    dict(id="film_zipf_hub_d256", kind="film", graph=PPI6K_ZIPF, world=3, D=256, act="relu", normalize=True,
         regime=["hub", "ln_split"], expect=HEAVY_PART + ["layer_norm_kernel"]),
    dict(id="film_qm9_d256", kind="film", graph=QM9_20K, world=2, D=256, act="relu", agg="mean", regime=["pair", "ln_nv"],
         expect=["seg_reduce_kernel<2, 1,"]),
    dict(id="film_zipf_hub_d512", kind="film", graph=PPI6K_ZIPF, world=3, D=512, act="relu",
         regime=["no_pair", "hub", "ln_split"], expect=HEAVY_PART + ["layer_norm_kernel"]),
    dict(id="film_config5_d32", kind="film", graph=CONFIG5, world=4, D=32, act="relu", normalize=True, regime=["config5"]),
    dict(id="edge_mlp_h1_target_zipf_d128", kind="edge_mlp", graph=PPI6K_ZIPF, world=3, D=128, hidden=1, use_target=True,
         act="relu", normalize=True, regime=["hub"], expect=["edge_build_kernel"]),
    dict(id="edge_mlp_h0_source_qm9_d512", kind="edge_mlp", graph=QM9_20K, world=2, D=512, hidden=0, use_target=False,
         regime=["ln_nv"], expect=["seg_reduce_kernel<4, 0,"]),
    dict(id="rgin_source_edge1_zipf_d128", kind="rgin", graph=PPI6K_ZIPF, world=3, D=128, edge_hidden=1, aggr_hidden=None,
         use_target=False, regime=["hub"]),
    dict(id="rgin_target_edge1_aggr1_zipf_d128", kind="rgin", graph=PPI6K_ZIPF, world=3, D=128, edge_hidden=1, aggr_hidden=1,
         use_target=True, agg="mean", regime=["hub"], expect=["layer_norm_kernel"]),
    dict(id="rgin_source_raw_aggr1_zipf_deferred_d64", kind="rgin", graph=PPI6K_ZIPF, world=2, D=64, edge_hidden=None,
         aggr_hidden=1, use_target=False, agg="mean", validate=False, regime=["hub", "deferred"],
         expect=["seg_reduce_heavy_kernel<", "layer_norm_kernel"]),
    dict(id="rgdcn_full_untied_k4_norm_zipf", kind="rgdcn", graph=PPI6K_ZIPF, world=3, D=64, K=4, full=True, tied=False,
         normalize=True, expect=["rgdcn_edge_kernel<1, false>"]),
    dict(id="rgdcn_channel_tied_k128_mean_norm", kind="rgdcn", graph=SMALL_ZIPF, world=2, D=128, K=128, full=False, tied=True,
         agg="mean", normalize=True, stddev=0.01, expect=["rgdcn_edge_kernel<1, false>"]),
    dict(id="rgdcn_channel_untied_k16_max", kind="rgdcn", graph=SMALL_ZIPF, world=2, D=64, K=16, full=False, tied=False,
         agg="max", expect=["rgdcn_edge_kernel<1, true>"]),
    dict(id="rgdcn_full_tied_k32_sqrt_n_norm_d256", kind="rgdcn", graph=SMALL_ZIPF, world=3, D=256, K=32, full=True, tied=True,
         agg="sqrt_n", normalize=True, stddev=0.01, expect=["rgdcn_edge_kernel<2, false>"]),
]
REGIMES = {"pair", "no_pair", "hub", "deferred", "ln_split", "ln_nv", "no_halo", "config5"}


def regime_holds(word, c):
    adj, _, V = graph(c["graph"])
    parts = partition(c["graph"], c["world"])
    L, D = len(adj), c["D"]
    if word == "pair":
        return all(p.num_local_edges < 0.75 * p.n_local * L for p in parts)
    if word == "no_pair":
        return all(p.num_local_edges >= 0.75 * p.n_local * L for p in parts)
    if word == "hub":
        return all(local_in_degree(p)[: p.n_own].max() > HEAVY_SEGMENT for p in parts)
    if word == "deferred":
        return c.get("validate", True) is False
    if word == "ln_split":
        return D > 128 and all(p.n_own < SMALL_BATCH for p in parts)
    if word == "ln_nv":
        return D > 128 and all(p.n_own >= SMALL_BATCH for p in parts)
    if word == "no_halo":
        return any(p.n_halo == 0 for p in parts)
    if word == "config5":
        return (V, sum(a.shape[0] for a in adj), c["world"]) == (50000, 1000000, 4)
    raise ValueError(word)


def test_case_regimes():
    """Every forward case is in the regime it claims, and every regime and D in {64, 128, 256, 512} is reached."""
    reached = set()
    for c in CASES:
        for word in c.get("regime", []):
            assert regime_holds(word, c), "%s: regime '%s' does not hold" % (c["id"], word)
            reached.add(word)
        parts = partition(c["graph"], c["world"])
        assert all(p.n_own > 0 for p in parts), c["id"]
        assert sum(p.n_own for p in parts) == graph(c["graph"])[2], c["id"]
        assert "hub" in c.get("regime", []) or c["kind"] in ("rgat", "rgdcn") or not regime_holds("hub", c), c["id"]
    assert reached == REGIMES, REGIMES - reached
    assert {64, 128, 256, 512} <= {c["D"] for c in CASES}
    assert {"rgcn", "rgcn_stack", "ggnn", "rgat", "film", "edge_mlp", "rgin", "rgdcn"} == {c["kind"] for c in CASES}
    # RGDCN: K from 4 to 128, full and channel state, tied and untied, normalised and not
    rg = [c for c in CASES if c["kind"] == "rgdcn"]
    assert {4, 128} <= {c["K"] for c in rg} and {True, False} == {c["full"] for c in rg} == {c["tied"] for c in rg}
    assert {True, False} == {c.get("normalize", False) for c in rg}
    # the halo-contract families reach each restricted code path that writes output rows
    assert {s["kind"] for s in SENTINEL_CASES} == {"rgcn", "rgcn_stack", "ggnn", "rgat", "film", "edge_mlp", "rgin", "rgdcn"}
    # the halo-contract rank owns a hub and has halo rows
    part = partition(PPI6K_ZIPF, 3)[2]
    assert part.n_halo > 0 and local_in_degree(part)[: part.n_own].max() > HEAVY_SEGMENT
    # training cases: a hub in some owned range, world 2 and 3
    for world in (2, 3):
        assert any(local_in_degree(p)[: p.n_own].max() > HEAVY_SEGMENT for p in partition(TRAIN_ZIPF, world))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_restricted_forward_matches_oracle(cuda_device, case):
    """Every rank of the partition runs the layer on its exchanged local states with a plan restricted to its owned rows;
    the owned rows, reassembled, equal the float64 oracle on the whole graph."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(case["graph"])
    L = len(adj)
    h = node_states(V, case["D"], seed=3)
    w = make_weights(case, L)
    parts = partition(case["graph"], case["world"])
    plans = [GraphPlan(p.local_adjacency_lists, p.n_local, device=cuda_device, validate=case.get("validate", True))
             .set_num_targets(p.n_own) for p in parts]
    hs = [torch.as_tensor(h[local_ids(p)]).to(cuda_device) for p in parts]
    cnts = [torch.as_tensor(p.local_num_incoming).to(cuda_device) for p in parts]
    wt = W.to_torch(w, cuda_device)
    outs = []

    def run():
        outs.clear()
        outs.extend(engine_layer(case, x, pl, c, wt) for x, pl, c in zip(hs, plans, cnts))
        torch.cuda.synchronize()

    names = launched_kernels(run, case.get("expect", ()))
    got = np.concatenate([o[: p.n_own].cpu().numpy() for o, p in zip(outs, parts)])
    for o, p in zip(outs, parts):
        assert not torch.any(o[p.n_own:]).item(), "%s: halo rows are not zero" % case["id"]
    want = oracle_layer(case, h, adj, indeg, w)
    if case["kind"] in LN_FAMILIES:
        err, _ = assert_parity_8c(got, want, oracle_layer(case, h, adj, indeg, w, np.float32), case["id"])
    else:
        err = assert_parity(got, want, case["id"], tol=TOL)
    missing = [s for s in case.get("expect", ()) if not any(s in n for n in names)]
    assert not missing, "%s: kernels %s not launched (got %s)" % (case["id"], missing, sorted(names))
    print("%s: max-norm relative error %.2e, kernels %s" % (case["id"], err,
                                                             sorted({n for n in names for s in case.get("expect", ()) if s in n})))


# ---------------------------------------------------------------- B. the halo-row contract ------------------------------
SENTINEL_CASES = [
    dict(id="rgcn_sum_hub", kind="rgcn", D=128, normalize=True),
    dict(id="rgcn_both_max", kind="rgcn", D=64, both=True, agg="max"),
    dict(id="rgcn_stack1", kind="rgcn_stack", D=64),
    dict(id="ggnn_gru", kind="ggnn", D=64, cell="gru"),
    dict(id="ggnn_rnn", kind="ggnn", D=64, cell="rnn"),
    dict(id="rgat_fused", kind="rgat", D=128, heads=4),
    dict(id="rgat_unfused", kind="rgat", D=96, heads=2),
    dict(id="film_d256", kind="film", D=256, normalize=True),
    dict(id="edge_mlp_h1_target", kind="edge_mlp", D=128, hidden=1, use_target=True),
    dict(id="rgin_source_edge1", kind="rgin", D=128, edge_hidden=1, aggr_hidden=None, use_target=False),
    dict(id="rgin_target_aggr1", kind="rgin", D=128, edge_hidden=1, aggr_hidden=1, use_target=True, agg="mean"),
    dict(id="rgin_source_raw_aggr1", kind="rgin", D=64, edge_hidden=None, aggr_hidden=1, use_target=False),
    dict(id="rgdcn_full_k4_norm", kind="rgdcn", D=64, K=4, full=True, tied=False, normalize=True),
    dict(id="rgdcn_channel_k16_max", kind="rgdcn", D=64, K=16, full=False, tied=True, agg="max"),
]
MODULE = {"rgcn": "rgcn", "rgcn_stack": "rgcn", "ggnn": "ggnn", "rgat": "rgat", "film": "gnn_film", "edge_mlp": "gnn_edge_mlp",
          "rgin": "rgin", "rgdcn": "rgdcn"}
NAN_BITS = 0x7FC00000


def nan_output_rows(plan, dim, device):
    import torch
    return torch.full((plan.num_nodes, dim), float("nan"), dtype=torch.float32, device=device)


def assert_sentinel(t, what):
    """Every element of t still holds the NaN the buffer was filled with, bit for bit."""
    import torch
    bits = t.contiguous().view(torch.int32)
    assert bool(torch.all(bits == NAN_BITS).item()), "%s: %d of %d sentinel elements were written" % (
        what, int((bits != NAN_BITS).sum().item()), bits.numel())


@pytest.mark.gpu
@pytest.mark.parametrize("case", SENTINEL_CASES, ids=[c["id"] for c in SENTINEL_CASES])
def test_halo_rows_left_untouched(cuda_device, monkeypatch, case):
    """include/rgnn.h: output rows >= num_targets are left untouched.  With the output buffer NaN-filled, the halo rows of a
    rank that owns a hub are still NaN after the call and the owned rows are finite and correct; with num_targets = 0 every
    row is still NaN.  Through the unpatched Python API the halo rows are exactly zero."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    key, world, rank = PPI6K_ZIPF, 3, 2
    adj, indeg, V = graph(key)
    part = partition(key, world)[rank]
    assert part.n_halo > 0 and local_in_degree(part).max() > HEAVY_SEGMENT
    h = node_states(V, case["D"], seed=5)
    w = make_weights(case, len(adj), seed=9)
    wt = W.to_torch(w, cuda_device)
    x = torch.as_tensor(h[local_ids(part)]).to(cuda_device)
    cnt = torch.as_tensor(part.local_num_incoming).to(cuda_device)
    own = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device).set_num_targets(part.n_own)
    none = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device).set_num_targets(0)
    want = oracle_layer(case, h, adj, indeg, w)[part.lo:part.hi]

    zero = engine_layer(case, x, own, cnt, wt)
    assert not bool(torch.any(zero[part.n_own:]).item()), "%s: halo rows are not zero" % case["id"]
    mod = importlib.import_module("tf_gnn_samples_b200.gnns." + MODULE[case["kind"]])
    monkeypatch.setattr(mod, "output_rows", nan_output_rows)
    got = engine_layer(case, x, own, cnt, wt)
    torch.cuda.synchronize()
    assert_sentinel(got[part.n_own:], case["id"] + " halo rows")
    assert torch.equal(got[: part.n_own], zero[: part.n_own]), case["id"]
    assert_parity(got[: part.n_own].cpu().numpy(), want, case["id"], tol=TOL)
    assert_sentinel(engine_layer(case, x, none, cnt, wt), case["id"] + " with num_targets = 0")


@pytest.mark.gpu
def test_film_out_argument_halo_rows_left_untouched(cuda_device):
    """sparse_gnn_film_layer(out=...) writes the owned rows of a caller's buffer and nothing else (the sharded data path)."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan
    key, world = PPI6K_ZIPF, 3
    adj, indeg, V = graph(key)
    D = 128
    h = node_states(V, D, seed=6)
    w = W.film_weights(len(adj), D, D, 13, random_ln=True)
    wt = W.to_torch(w, cuda_device)
    want = R.sparse_gnn_film_layer(h, adj, indeg, D, normalize_by_num_incoming=True, weights=w)
    for part in partition(key, world):
        x = torch.as_tensor(h[local_ids(part)]).to(cuda_device)
        cnt = torch.as_tensor(part.local_num_incoming).to(cuda_device)
        for n in (part.n_own, 0):
            plan = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device).set_num_targets(n)
            out = torch.full((part.n_local, D), float("nan"), dtype=torch.float32, device=cuda_device)
            assert G.sparse_gnn_film_layer(x, plan, cnt, D, normalize_by_num_incoming=True, weights=wt, out=out) is out
            torch.cuda.synchronize()
            assert_sentinel(out[n:], "FiLM out= rows >= %d" % n)
            if n:
                assert_parity_8c(out[:n].cpu().numpy(), want[part.lo:part.hi],
                                 R.sparse_gnn_film_layer(h, adj, indeg, D, normalize_by_num_incoming=True, weights=w,
                                                         dtype=np.float32)[part.lo:part.hi], "FiLM out= rank %d" % part.rank)


@pytest.mark.gpu
@pytest.mark.parametrize("validate", [True, False], ids=["heavy_part_finish", "heavy_one_cta"])
def test_hub_outside_wanted_rows_left_untouched(cuda_device, monkeypatch, validate):
    """set_num_targets on a plan whose heavy targets are not all wanted: the heavy kernels walk the plan's whole heavy list,
    and must skip the targets >= num_targets as the warp-per-target kernels do."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    import tf_gnn_samples_b200.gnns.rgcn as mod
    adj, indeg, V = graph(PPI6K_ZIPF)
    deg = np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)
    heavy = np.flatnonzero(deg > HEAVY_SEGMENT)
    k = int(heavy[len(heavy) // 2])                        # hubs on both sides of the cut
    assert heavy.min() < k <= heavy.max()
    case = dict(kind="rgcn", D=128, normalize=True, agg="sum")
    h = node_states(V, 128, seed=8)
    w = make_weights(case, len(adj), seed=17)
    plan = GraphPlan(adj, V, device=cuda_device, validate=validate).set_num_targets(k)
    monkeypatch.setattr(mod, "output_rows", nan_output_rows)
    expect = HEAVY_PART if validate else ["seg_reduce_heavy_kernel<"]
    outs = []
    names = launched_kernels(lambda: outs.append(engine_layer(case, torch.as_tensor(h).to(cuda_device), plan,
                                                              torch.as_tensor(indeg).to(cuda_device),
                                                              W.to_torch(w, cuda_device))), expect)
    assert all(any(s in n for n in names) for s in expect), sorted(names)
    got = outs[-1]
    torch.cuda.synchronize()
    assert_sentinel(got[k:], "rows >= num_targets = %d" % k)
    assert_parity(got[:k].cpu().numpy(), oracle_layer(case, h, adj, indeg, w)[:k], "wanted rows", tol=TOL)


# ---------------------------------------------------------------- C. virtual-rank stacks ---------------------------------
STACKS = [
    dict(id="rgcn", kind="rgcn", D=64, agg="mean", normalize=True, world=2, layers=3),
    dict(id="ggnn_gru", kind="ggnn", D=64, cell="gru", world=3, layers=2),
    dict(id="rgat", kind="rgat", D=64, heads=4, world=2, layers=2),
    dict(id="edge_mlp", kind="edge_mlp", D=64, hidden=1, use_target=True, normalize=True, world=3, layers=3),
    dict(id="rgin", kind="rgin", D=64, edge_hidden=1, aggr_hidden=1, use_target=False, world=2, layers=2),
    dict(id="rgdcn", kind="rgdcn", D=64, K=16, full=True, tied=False, normalize=True, world=3, layers=2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [False, True], ids=["blocking", "overlapped"])
@pytest.mark.parametrize("case", STACKS, ids=[c["id"] for c in STACKS])
def test_virtual_ranks_stack_matches_oracle(cuda_device, case, overlap):
    """Every rank of the partition on one GPU with its own stream (ShardedGraph.attach_in_process): exchange into one state
    buffer, run the layer on ShardedGraph.plan, copy the owned rows into the other buffer.  The layers other than FiLM join
    a pending overlapped exchange at their entry.  The stack equals the float64 oracle on the whole graph, and a second pass
    repeats it bit for bit.  The graph keeps every rank's pull kernel resident at once (attach_in_process)."""
    import torch
    from tf_gnn_samples_b200 import ShardedGraph, degree_balanced_cuts
    g0 = batching.make_typed_random_graph(700, 9000, (0.4, 0.3, 0.2, 0.1), 8, seed=5)
    adj, indeg, V = g0.adjacency_lists, g0.type_to_node_to_num_incoming_edges, 700
    D, world, layers = case["D"], case["world"], case["layers"]
    h = node_states(V, D, seed=2)
    ws = [make_weights(case, len(adj), seed=11 + 3 * i) for i in range(layers)]
    want = h
    for w in ws:
        want = oracle_layer(case, want, adj, indeg, w)
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
            for g, s, c in zip(graphs, streams, cnts):
                with torch.cuda.stream(s):
                    g.exchange(t % 2, overlap=overlap)
                    out = engine_layer(case, g.states(t % 2), g.plan, c, wts[t])
                    g.states(1 - t % 2)[: g.n_own].copy_(out[: g.n_own])
        torch.cuda.synchronize()
        return np.concatenate([g.states(layers % 2)[: g.n_own].cpu().numpy() for g in graphs])

    got = run_once()
    if case["kind"] in LN_FAMILIES:
        want32 = h
        for w in ws:
            want32 = oracle_layer(case, want32, adj, indeg, w, np.float32)
        assert_parity_8c(got, want, want32, "%s x%d on %d virtual ranks" % (case["id"], layers, world))
    else:
        assert_parity(got, want, "%s x%d on %d virtual ranks" % (case["id"], layers, world), tol=TOL)
    np.testing.assert_array_equal(got, run_once())
    for g in graphs:
        g.close()


# ---------------------------------------------------------------- D. sharded training ------------------------------------
TRAIN = [
    dict(id="rgcn_fused_tanh_sum_norm", kind="rgcn", D=64, normalize=True, world=2),
    dict(id="rgcn_composed_both", kind="rgcn", D=64, both=True, normalize=True, world=3),
    dict(id="ggnn_gru", kind="ggnn", D=64, cell="gru", cell_scale=0.5, world=3),
    dict(id="rgat", kind="rgat", D=64, heads=4, world=2),
    dict(id="film_gelu_mean", kind="film", D=64, act="gelu", agg="mean", normalize=True, world=3),
    dict(id="edge_mlp_h1_target", kind="edge_mlp", D=64, hidden=1, use_target=True, normalize=True, world=2),
    dict(id="rgin_target_aggr1_mean", kind="rgin", D=64, edge_hidden=1, aggr_hidden=1, use_target=True, agg="mean", world=3),
    dict(id="rgin_source_edge1", kind="rgin", D=64, edge_hidden=1, aggr_hidden=None, use_target=False, world=2),
]


def autograd_oracle(c, adj, indeg):
    """oracle/ref_autograd.py layer of case c on the whole graph: (h64, w64) -> out64."""
    k, act, agg, norm = c["kind"], c.get("act", "tanh"), c.get("agg", "sum"), c.get("normalize", False)
    if k == "rgcn":
        return lambda h, w: A.sparse_rgcn_layer(h, adj, indeg, activation_function=act, message_aggregation_function=agg,
                                                normalize_by_num_incoming=norm, use_both_source_and_target=c.get("both", False),
                                                weights=w)
    if k == "ggnn":
        return lambda h, w: A.sparse_ggnn_layer(h, adj, gated_unit_type=c["cell"], activation_function=act,
                                                message_aggregation_function=agg, weights=w)
    if k == "rgat":
        return lambda h, w: A.sparse_rgat_layer(h, adj, num_heads=c["heads"], activation_function=act, weights=w)
    if k == "film":
        return lambda h, w: A.sparse_gnn_film_layer(h, adj, indeg, activation_function=act, message_aggregation_function=agg,
                                                    normalize_by_num_incoming=norm, weights=w)
    if k == "edge_mlp":
        return lambda h, w: A.sparse_gnn_edge_mlp_layer(h, adj, indeg, activation_function=act,
                                                        message_aggregation_function=agg, normalize_by_num_incoming=norm,
                                                        use_target_state_as_input=c["use_target"], weights=w)
    return lambda h, w: A.sparse_rgin_layer(h, adj, activation_function=act, message_aggregation_function=agg,
                                            use_target_state_as_input=c["use_target"], weights=w)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRAIN, ids=[c["id"] for c in TRAIN])
def test_sharded_training_matches_float64_autograd(cuda_device, case):
    """Each rank gathers its local states from the global leaf h (autograd's transpose of that gather is the all-to-all
    return of the halo gradients, NodeRangePartition.exchange) and runs the engine layer on its restricted plan; the owned
    rows of all ranks, concatenated, and d_h and the weight gradients summed over the ranks (all_reduce_gradients_) equal
    float64 autograd on the whole graph."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    adj, indeg, V = graph(TRAIN_ZIPF)
    parts = partition(TRAIN_ZIPF, case["world"])
    plans = [GraphPlan(p.local_adjacency_lists, p.n_local, device=cuda_device).set_num_targets(p.n_own) for p in parts]
    ids = [torch.as_tensor(local_ids(p)).to(cuda_device) for p in parts]
    cnts = [torch.as_tensor(p.local_num_incoming).to(cuda_device) for p in parts]
    h = node_states(V, case["D"], seed=12)
    w = make_weights(case, len(adj), seed=23)

    def engine(hd, wd):
        outs = [engine_layer(case, hd.index_select(0, i), pl, c, wd)[: p.n_own]
                for i, pl, c, p in zip(ids, plans, cnts, parts)]
        return torch.cat(outs, dim=0)

    errs, _ = compare(engine, autograd_oracle(case, adj, torch.as_tensor(indeg, dtype=torch.float64)), h, w, tol=TOL)
    print("%s (world %d): %s" % (case["id"], case["world"], {k: "%.1e" % v for k, v in errs.items()}))


# ---------------------------------------------------------------- E. refused calls ---------------------------------------
@pytest.mark.gpu
def test_restricted_rgcn_stack_rejects_two_layers(cuda_device):
    """A second stacked layer would gather halo rows of the intermediate buffer, which the call never writes: refused, like
    num_timesteps > 1 on a restricted plan (which stays refused)."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import GraphPlan, RgnnError
    adj, indeg, V = graph(PPI6K_ZIPF)
    part = partition(PPI6K_ZIPF, 3)[1]
    D, L = 64, len(adj)
    x = torch.as_tensor(node_states(part.n_local, D, seed=4)).to(cuda_device)
    cnt = torch.as_tensor(part.local_num_incoming).to(cuda_device)
    plan = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device).set_num_targets(part.n_own)
    ws = [W.to_torch(W.rgcn_weights(L, D, D, seed=s), cuda_device) for s in (1, 2)]
    with pytest.raises(RgnnError, match="num_layers == 1"):
        G.rgcn_layer_stack(x, plan, cnt, ws, normalize_by_num_incoming=True)
    with pytest.raises(RgnnError, match="num_timesteps == 1"):
        G.sparse_rgcn_layer(x, plan, cnt, D, num_timesteps=2, weights=ws[0])
    full = GraphPlan(part.local_adjacency_lists, part.n_local, device=cuda_device)
    got = G.rgcn_layer_stack(x, full, cnt, ws, normalize_by_num_incoming=True)      # unrestricted: two layers are fine
    want = x
    for w in ws:
        want = G.sparse_rgcn_layer(want, full, cnt, D, activation_function="ReLU", weights=w)
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_sharded_graph_plan_under_autograd_raises(cuda_device):
    """ShardedGraph.plan wraps the device-built rank-local graph and has no adjacency lists: the training paths that need
    them refuse it with an RgnnError that names the supported route, instead of failing with a TypeError inside the index
    views.  (GGNN and the fused RGCN backward work on the plan arrays alone and need no lists.)"""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import RgnnError, ShardedGraph, degree_balanced_cuts
    adj, indeg, V = graph(TRAIN_ZIPF)
    D, L = 64, len(adj)
    sg = ShardedGraph(adj, degree_balanced_cuts(adj, V, 2), 0, 2, device=cuda_device)
    x = torch.as_tensor(node_states(sg.n_local, D, seed=4)).to(cuda_device).requires_grad_(True)
    cnt = sg.local_num_incoming(indeg)
    for kind, w in (("film", W.film_weights(L, D, D)), ("rgat", W.rgat_weights(L, D, D)),
                    ("edge_mlp", W.edge_mlp_weights(L, D, D, 1, True))):
        c = dict(kind=kind, D=D, heads=4, hidden=1, use_target=True)
        with pytest.raises(RgnnError, match="local_adjacency_lists"):
            engine_layer(c, x, sg.plan, cnt, W.to_torch(w, cuda_device))
    with torch.no_grad():                                  # inference on the same plan is the supported use
        out = engine_layer(dict(kind="film", D=D), x, sg.plan, cnt, W.to_torch(W.film_weights(L, D, D), cuda_device))
    assert bool(torch.isfinite(out[: sg.n_own]).all().item())
    sg.close()

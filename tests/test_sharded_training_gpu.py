"""GPU: training a graph sharded over ranks on the device-built halo plan (ShardedGraph.attach(..., training=True),
ShardedGraph.gather, rgnn_halo_exchange_backward).

Every rank of the partition runs on one H100 ("virtual ranks", one stream each), so the forward pull and its transpose, the
halo-gradient return, both run in peer memory exactly as they would over NVLink:

  * 2-3-layer stacks of every trainable family, world 2, 3 and 4, on a Zipf graph with hubs inside the owned ranges: the
    owned outputs of all ranks, d_h and the rank-summed weight gradients equal float64 autograd on the whole graph (1e-4;
    assert_parity_8c for the layer-norm outputs), agree with the existing torch route (NodeRangePartition lists + a
    GraphPlan, halo gradients returned by the transposed gather) to float32 rounding, and repeat bit for bit (except RGAT,
    whose training layer adds with atomics);
  * known answers for the reverse index and the summation order: the device-built index equals a numpy construction from
    every rank's export(), every owned row is the local gradient plus its consumers' rows added in ascending rank (bit for
    bit), a row without remote consumers is copied bit for bit; a rank without halo rows and a rank whose rows nobody
    consumes;
  * one CUDA graph per rank holding its forward + backward step, replayed with new states and weights written in place;
  * the refused calls.

The cases keep every rank's exchange kernels co-resident (include/rgnn.h: virtual ranks); test_case_regimes checks that
and the other properties the cases rely on without a GPU."""
import numpy as np
import pytest

from oracle import ref_autograd as A
from tf_gnn_samples_b200.partition import NodeRangePartition
from tf_gnn_samples_b200.sharded import degree_balanced_cuts

from dispatch import HEAVY_SEGMENT
from helpers import assert_parity_8c, node_states, rel, to_dev
from test_sharded_layers_gpu import (LN_FAMILIES, TRAIN_ZIPF, autograd_oracle, engine_layer, graph, local_ids, make_weights,
                                     oracle_layer)

TOL = 1e-4
ROUTE_TOL = 1e-5             # the existing torch route differs only in the order its halo gradients are added
HALO_THREADS_ROWS = 128      # halo.cu: 16 warps x 8 rows per CTA of the pull kernels
MAX_CTAS_PER_RANK = 264      # halo.cu: 2 x RGNN_WAVE_SMS
CO_RESIDENT_CTAS = 528       # 512-thread CTAs an H100 holds at once (132 SMs x 4)

STACKS = [
    dict(id="rgcn_fused_sum_norm_w2", kind="rgcn", D=64, normalize=True, world=2, layers=3),
    dict(id="rgcn_composed_max_w3", kind="rgcn", D=64, agg="max", world=3, layers=2),
    dict(id="rgcn_composed_both_w4", kind="rgcn", D=64, both=True, normalize=True, world=4, layers=2),
    dict(id="ggnn_gru_w3", kind="ggnn", D=64, cell="gru", cell_scale=0.5, world=3, layers=2),
    dict(id="film_gelu_mean_w4", kind="film", D=64, act="gelu", agg="mean", normalize=True, world=4, layers=2),
    # the RGAT training path adds its softmax denominators with torch's index_add (atomics): no bitwise repeat
    dict(id="rgat_k4_w2", kind="rgat", D=64, heads=4, world=2, layers=2, repeatable=False),
    dict(id="edge_mlp_h1_target_w3", kind="edge_mlp", D=64, hidden=1, use_target=True, normalize=True, world=3, layers=3),
    dict(id="rgin_target_aggr1_mean_w4", kind="rgin", D=64, edge_hidden=1, aggr_hidden=1, use_target=True, agg="mean",
         world=4, layers=2),
]
GRAPH_CASES = [c for c in STACKS if c["id"] in ("rgcn_fused_sum_norm_w2", "film_gelu_mean_w4", "rgin_target_aggr1_mean_w4")]


# ---------------------------------------------------------------- host constructions -------------------------------------
def host_halo(adj, cuts, r):
    """Sorted global ids of rank r's halo: the remote sources of the edges whose target r owns."""
    lo, hi = int(cuts[r]), int(cuts[r + 1])
    src = np.concatenate([a[(a[:, 1] >= lo) & (a[:, 1] < hi), 0] for a in adj]).astype(np.int64)
    return np.unique(src[(src < lo) | (src >= hi)])


def host_reverse(adj, cuts, p):
    """Rank p's reverse index: offsets [n_own + 1] and, sorted by (owned row, peer), the consuming peer q and the row of q's
    gradient buffer (n_own of q + position in q's halo)."""
    world = len(cuts) - 1
    rows, peers, qrows = [], [], []
    for q in range(world):
        if q == p:
            continue
        halo = host_halo(adj, cuts, q)
        i = np.flatnonzero((halo >= cuts[p]) & (halo < cuts[p + 1]))
        rows.append(halo[i] - cuts[p])
        peers.append(np.full(i.size, q))
        qrows.append(int(cuts[q + 1] - cuts[q]) + i)
    rows, peers, qrows = (np.concatenate(x).astype(np.int64) if x else np.zeros(0, np.int64) for x in (rows, peers, qrows))
    order = np.lexsort((peers, rows))
    n_own = int(cuts[p + 1] - cuts[p])
    return np.searchsorted(rows[order], np.arange(n_own + 1)), peers[order], qrows[order]


def consumers(adj, cuts):
    """Global id -> number of peers holding it as a halo row."""
    count = np.zeros(int(cuts[-1]), np.int64)
    for q in range(len(cuts) - 1):
        count[host_halo(adj, cuts, q)] += 1
    return count


def pull_ctas(rows):
    return min(max(-(-rows // HALO_THREADS_ROWS), 1), MAX_CTAS_PER_RANK)


def layered_graph():
    """600 nodes over 3 ranks of 200: rank 0's targets read only rank 0 (no halo), rank 1's read ranks 0-1, rank 2's read
    ranks 0-1 (nobody reads rank 2's rows, every peer reads some of rank 0's)."""
    rng = np.random.default_rng(31)
    cuts = np.array([0, 200, 400, 600], np.int64)
    adj = []
    for _ in range(2):
        parts = [np.stack([rng.integers(0, 200, 700), rng.integers(0, 200, 700)], 1),
                 np.stack([rng.integers(0, 400, 900), rng.integers(200, 400, 900)], 1),
                 np.stack([rng.integers(0, 400, 900), rng.integers(400, 600, 900)], 1)]
        adj.append(np.concatenate(parts).astype(np.int32))
    return adj, cuts


def test_case_regimes():
    """Each stack has a hub in some owned range and halo rows consumed by >= 2 peers (world >= 3; world 2: both ranks have
    halo rows), and every rank's forward and backward pull kernels stay co-resident; the hand-built graph has a rank
    without halo rows, a rank whose rows nobody consumes and rows consumed by every peer."""
    adj, _, V = graph(TRAIN_ZIPF)
    assert {c["world"] for c in STACKS} == {2, 3, 4}
    assert {"rgcn", "ggnn", "film", "rgat", "edge_mlp", "rgin"} == {c["kind"] for c in STACKS}
    for world in sorted({c["world"] for c in STACKS}):
        cuts = degree_balanced_cuts(adj, V, world)
        parts = [NodeRangePartition(adj, None, V, r, world) for r in range(world)]
        assert all(np.array_equal(p.cuts, cuts) for p in parts)
        indeg = [np.bincount(np.concatenate([a[:, 1] for a in p.local_adjacency_lists]), minlength=p.n_local)
                 for p in parts]
        assert any(d[: p.n_own].max() > HEAVY_SEGMENT for d, p in zip(indeg, parts)), world
        if world >= 3:
            assert consumers(adj, cuts).max() >= 2, world
        else:
            assert all(p.n_halo > 0 for p in parts)
        fwd = [pull_ctas(p.n_halo) for p in parts]
        bwd = [pull_ctas(p.n_own) for p in parts]
        assert max(fwd + bwd) < MAX_CTAS_PER_RANK and sum(fwd) <= CO_RESIDENT_CTAS and sum(bwd) <= CO_RESIDENT_CTAS
    adj, cuts = layered_graph()
    assert host_halo(adj, cuts, 0).size == 0
    assert consumers(adj, cuts)[400:].max() == 0
    assert consumers(adj, cuts)[:200].max() == 2


# ---------------------------------------------------------------- virtual ranks ------------------------------------------
def virtual_ranks(adj, cuts, D, device, training=True):
    import torch
    from tf_gnn_samples_b200 import ShardedGraph
    world = len(cuts) - 1
    sgs = [ShardedGraph(adj, cuts, r, world, device=device) for r in range(world)]
    ShardedGraph.attach_in_process(sgs, D, training=training)
    streams = [torch.cuda.Stream(device=device) for _ in range(world)]
    torch.cuda.synchronize()
    return sgs, streams


def rank_step(case, sg, plan, cnt, h_own, ws, proj):
    """One rank's forward through the stack (a gather before every layer) and its backward; returns the owned output.
    For CUDA-graph capture, which records without executing."""
    x = h_own
    for t, w in enumerate(ws):
        x = engine_layer(case, sg.gather(x, t % 2), plan, cnt, w)[: sg.n_own]
    (x * proj).sum().backward()
    return x


def training_step(case, sgs, streams, plans, cnts, hs, wds, projs, exchange=True):
    """Forward + backward of every rank, each on its own stream, enqueued phase by phase: every rank's gather before any
    rank's next layer, and one backward call over all ranks' losses (autograd runs ready nodes in reverse creation order,
    so every rank's halo-gradient exchange of a layer is enqueued before any rank's backward of the layer below).  A kernel
    loaded lazily at its first launch then never waits for an exchange whose peers are not enqueued yet (include/rgnn.h,
    virtual ranks).  exchange=False: the halo rows are zeros instead of gathered (the warm-up, which loads the layers'
    kernels).  Returns the owned outputs."""
    import torch
    xs = list(hs)
    for t in range(case["layers"]):
        local = []
        for r, (sg, s) in enumerate(zip(sgs, streams)):
            with torch.cuda.stream(s):
                local.append(sg.gather(xs[r], t % 2) if exchange else
                             torch.cat([xs[r], xs[r].new_zeros((sg.n_halo, xs[r].shape[1]))]))
        for r, (sg, s) in enumerate(zip(sgs, streams)):
            with torch.cuda.stream(s):
                xs[r] = engine_layer(case, local[r], plans[r], cnts[r], wds[r][t])[: sg.n_own]
    losses = []
    for x, p, s in zip(xs, projs, streams):
        with torch.cuda.stream(s):
            losses.append((x * p).sum())
    torch.autograd.backward(losses)
    return xs


def warm_up(case, sgs, streams, device):
    """Run every layer kernel of the step once, forward and backward, with no exchange in flight."""
    import torch
    adj, indeg, V = graph(TRAIN_ZIPF)
    h, ws, proj = make_inputs(case, 1)
    hs, wds, projs = rank_inputs(sgs, h, ws, proj, device)
    plans = [sg.training_plan() for sg in sgs]
    cnts = [sg.local_num_incoming(indeg) for sg in sgs]
    torch.cuda.synchronize()
    training_step(case, sgs, streams, plans, cnts, hs, wds, projs, exchange=False)
    torch.cuda.synchronize()


def rank_inputs(sgs, h, ws, proj, device):
    import torch
    hs = [torch.as_tensor(h[sg.lo:sg.hi]).to(device).requires_grad_(True) for sg in sgs]
    wds = [to_dev(ws, device) for _ in sgs]                  # replicated weights: one copy per rank
    projs = [torch.as_tensor(proj[sg.lo:sg.hi]).to(device) for sg in sgs]
    return hs, wds, projs


def collect(outs, hs, wds):
    """Concatenated owned outputs and d_h, weight gradients summed over the ranks (what all_reduce_gradients_ does)."""
    res = {"out": np.concatenate([o.detach().cpu().numpy() for o in outs]),
           "d_h": np.concatenate([x.grad.cpu().numpy() for x in hs])}
    for k in A.flatten(wds[0]):
        gs = [A.flatten(w)[k].grad for w in wds]
        if any(g is not None for g in gs):
            res["d_" + k] = sum(g.cpu().numpy().astype(np.float64) for g in gs if g is not None).astype(np.float32)
    return res


def sharded_training(case, sgs, streams, h, ws, proj, device):
    """One training step of all ranks (training_step) from numpy inputs: the collected results."""
    import torch
    hs, wds, projs = rank_inputs(sgs, h, ws, proj, device)
    plans = [sg.training_plan() for sg in sgs]
    adj, indeg, _ = graph(TRAIN_ZIPF)
    cnts = [sg.local_num_incoming(indeg) for sg in sgs]
    torch.cuda.synchronize()
    outs = training_step(case, sgs, streams, plans, cnts, hs, wds, projs)
    torch.cuda.synchronize()
    return collect(outs, hs, wds)


def existing_route(case, parts, h, ws, proj, device):
    """The torch route: GraphPlans over NodeRangePartition's lists; every layer's local states are gathered from the
    concatenated owned rows, whose autograd transpose returns the halo gradients to their owners (the all-to-all of
    NodeRangePartition.exchange, on one device)."""
    import torch
    from tf_gnn_samples_b200 import GraphPlan
    plans = [GraphPlan(p.local_adjacency_lists, p.n_local, device=device).set_num_targets(p.n_own) for p in parts]
    ids = [torch.as_tensor(local_ids(p)).to(device) for p in parts]
    cnts = [torch.as_tensor(p.local_num_incoming).to(device) for p in parts]
    hd = torch.as_tensor(h).to(device).requires_grad_(True)
    wds = [to_dev(ws, device) for _ in parts]
    x = hd
    for t in range(len(ws)):
        x = torch.cat([engine_layer(case, x.index_select(0, i), pl, c, wd[t])[: p.n_own]
                       for i, pl, c, wd, p in zip(ids, plans, cnts, wds, parts)])
    (x * torch.as_tensor(proj).to(device)).sum().backward()
    torch.cuda.synchronize()
    res = collect([x], [hd], wds)
    for pl in plans:
        pl.close()
    return res


def float64_truth(case, h, ws, proj):
    import torch
    adj, indeg, _ = graph(TRAIN_ZIPF)
    f = autograd_oracle(case, adj, torch.as_tensor(indeg, dtype=torch.float64))
    h64 = torch.as_tensor(h, dtype=torch.float64).requires_grad_(True)
    w64 = [A.to_torch64(w) for w in ws]
    x = h64
    for w in w64:
        x = f(x, w)
    (x * torch.as_tensor(proj, dtype=torch.float64)).sum().backward()
    res = {"out": x.detach().numpy(), "d_h": h64.grad.numpy()}
    for k, t in A.flatten(w64).items():
        res["d_" + k] = None if t.grad is None else t.grad.numpy()
    return res


def assert_matches_truth(case, got, want, h, ws, what):
    """Output: 1e-4 (assert_parity_8c for the layer-norm families), every gradient: 1e-4.  Returns the errors."""
    adj, indeg, _ = graph(TRAIN_ZIPF)
    errs = {}
    if case["kind"] in LN_FAMILIES:
        want32 = h
        for w in ws:
            want32 = oracle_layer(case, want32, adj, indeg, w, np.float32)
        errs["out"], _ = assert_parity_8c(got["out"], want["out"], want32, what)
    else:
        errs["out"] = rel(got["out"], want["out"])
    for k, v in want.items():
        if k == "out":
            continue
        if v is None or not np.any(v):
            assert k not in got or not np.any(got[k]), "%s: %s should be zero" % (what, k)
            continue
        assert k in got, "%s: no gradient reached %s" % (what, k)
        errs[k] = rel(got[k], v)
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, "%s: %s" % (what, bad)
    return errs


def make_inputs(case, seed):
    adj, _, V = graph(TRAIN_ZIPF)
    h = node_states(V, case["D"], seed=seed)
    ws = [make_weights(case, len(adj), seed=seed + 11 + 7 * t) for t in range(case["layers"])]
    proj = np.random.default_rng(seed + 1).standard_normal((V, case["D"])).astype(np.float32)
    return h, ws, proj


@pytest.mark.gpu
@pytest.mark.parametrize("case", STACKS, ids=[c["id"] for c in STACKS])
def test_sharded_stack_training_matches_float64_autograd(cuda_device, case):
    """The stack trained over virtual ranks through ShardedGraph.gather on training_plan(): output, d_h and the
    rank-summed weight gradients equal float64 autograd on the whole graph, agree with the existing torch route to float32
    rounding, and a second pass repeats every number bit for bit (unless the layer itself does not)."""
    adj, indeg, V = graph(TRAIN_ZIPF)
    world = case["world"]
    cuts = degree_balanced_cuts(adj, V, world)
    sgs, streams = virtual_ranks(adj, cuts, case["D"], cuda_device)
    warm_up(case, sgs, streams, cuda_device)
    h, ws, proj = make_inputs(case, 40)
    got = sharded_training(case, sgs, streams, h, ws, proj, cuda_device)
    again = sharded_training(case, sgs, streams, h, ws, proj, cuda_device)
    assert got.keys() == again.keys()
    for k in got:
        same = np.array_equal(got[k].view(np.int32), again[k].view(np.int32))
        assert same or not case.get("repeatable", True), "%s: %s not repeatable" % (case["id"], k)
    errs = assert_matches_truth(case, got, float64_truth(case, h, ws, proj), h, ws, case["id"])
    parts = [NodeRangePartition(adj, indeg, V, r, world) for r in range(world)]
    old = existing_route(case, parts, h, ws, proj, cuda_device)
    assert old.keys() == got.keys()
    diff = {k: rel(got[k], old[k]) for k in got}
    print("%s (world %d): vs float64 %s | vs the torch route %s" % (
        case["id"], world, {k: "%.1e" % v for k, v in errs.items()}, {k: "%.1e" % v for k, v in diff.items()}))
    assert max(diff.values()) <= ROUTE_TOL, diff
    for sg in sgs:
        sg.close()


# ---------------------------------------------------------------- reverse index: known answers ---------------------------
def assert_sums_in_rank_order(sgs, streams, adj, cuts, D, device, seed):
    """Every rank calls exchange_backward on a local gradient with values of very different magnitudes (so that the order
    of the additions shows in the bits); rows without remote consumers hold -0.0, a NaN payload, a denormal and inf.
    Every owned row must equal, bit for bit, its local row followed by its consumers' rows added one at a time in
    ascending rank, in float32.  Returns the number of rows consumed by every peer."""
    import torch
    rng = np.random.default_rng(seed)
    world = len(sgs)
    g = []
    for sg in sgs:
        x = (rng.standard_normal((sg.n_local, D)) * 10.0 ** rng.integers(-3, 4, (sg.n_local, 1))).astype(np.float32)
        g.append(x)
    revs = [host_reverse(adj, cuts, p) for p in range(world)]
    for p, (off, _, _) in enumerate(revs):
        lonely = np.flatnonzero(np.diff(off) == 0)
        if lonely.size:
            special = np.array([0x80000000, 0x7FC00123, 0x00000005, 0x7F800000], np.uint32).view(np.float32)
            g[p][lonely[:, None], np.arange(4)[None, :] % D] = special[None, :]
    every = sum(int(np.sum(np.diff(off) == world - 1)) for off, _, _ in revs)
    for buffer in (0, 1, 0):
        gd = [torch.as_tensor(x).to(device) for x in g]
        torch.cuda.synchronize()
        outs = []
        for sg, s, x in zip(sgs, streams, gd):
            with torch.cuda.stream(s):
                outs.append(sg.exchange_backward(buffer, x))
        torch.cuda.synchronize()
        for p, (sg, out) in enumerate(zip(sgs, outs)):
            off, peer, qrow = revs[p]
            want = g[p][: sg.n_own].copy()
            for r in range(sg.n_own):
                for j in range(off[r], off[r + 1]):
                    want[r] = want[r] + g[peer[j]][qrow[j]]          # float32 + float32, one addition at a time
            got = out.cpu().numpy()
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), "rank %d, buffer %d: %d rows differ" % (
                p, buffer, int(np.any(got.view(np.int32) != want.view(np.int32), axis=1).sum()))
    return every


@pytest.mark.gpu
@pytest.mark.parametrize("world", [3, 4])
def test_reverse_index_matches_host_construction(cuda_device, world):
    """The device-built reverse index of every rank equals a numpy construction from every rank's export(); the device-built
    local numbering equals NodeRangePartition's; the backward exchange adds each owned row's consumers in rank order."""
    adj, _, V = graph(TRAIN_ZIPF)
    cuts = degree_balanced_cuts(adj, V, world)
    sgs, streams = virtual_ranks(adj, cuts, 16, cuda_device)
    exports = [sg.export() for sg in sgs]
    for p, (sg, ex) in enumerate(zip(sgs, exports)):
        part = NodeRangePartition(adj, None, V, p, world)
        assert np.array_equal(ex["halo_global"].cpu().numpy(), part.halo_global)
        for a, b in zip(ex["local_adjacency_lists"], part.local_adjacency_lists):
            assert np.array_equal(a.cpu().numpy(), b)
    owner_row = [(ex["halo_owner"].cpu().numpy(), ex["halo_row"].cpu().numpy()) for ex in exports]
    for p, sg in enumerate(sgs):
        rows, peers, qrows = [], [], []                          # from the exported halo lists alone
        for q, (owner, row) in enumerate(owner_row):
            if q != p:
                i = np.flatnonzero(owner == p)
                rows.append(row[i])
                peers.append(np.full(i.size, q))
                qrows.append(sgs[q].n_own + i)
        rows, peers, qrows = (np.concatenate(x) for x in (rows, peers, qrows))
        order = np.lexsort((peers, rows))
        rev = sg.export_reverse()
        assert np.array_equal(rev["offsets"].cpu().numpy(), np.searchsorted(rows[order], np.arange(sg.n_own + 1)))
        assert np.array_equal(rev["peer"].cpu().numpy(), peers[order])
        assert np.array_equal(rev["row"].cpu().numpy(), qrows[order])
        off, hp, hr = host_reverse(adj, cuts, p)
        assert np.array_equal(rev["offsets"].cpu().numpy(), off) and np.array_equal(rev["peer"].cpu().numpy(), hp)
        assert np.array_equal(rev["row"].cpu().numpy(), hr)
    every = assert_sums_in_rank_order(sgs, streams, adj, cuts, 16, cuda_device, seed=world)
    print("world %d: %d rows consumed by every peer" % (world, every))
    for sg in sgs:
        sg.close()


@pytest.mark.gpu
def test_rank_without_halo_and_rank_nobody_reads(cuda_device):
    """Rank 0 has no halo rows (its backward has nothing to send), nobody consumes rank 2's rows (its gradient comes back
    bit for bit, NaN payloads and denormals included), and some of rank 0's rows are consumed by every peer."""
    adj, cuts = layered_graph()
    sgs, streams = virtual_ranks(adj, cuts, 8, cuda_device)
    assert sgs[0].n_halo == 0 and sgs[0].export_reverse()["peer"].numel() > 0
    assert sgs[2].export_reverse()["peer"].numel() == 0 and sgs[2].n_halo > 0
    every = assert_sums_in_rank_order(sgs, streams, adj, cuts, 8, cuda_device, seed=5)
    assert every > 0
    for sg in sgs:
        sg.close()


# ---------------------------------------------------------------- CUDA graphs ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GRAPH_CASES, ids=[c["id"] for c in GRAPH_CASES])
def test_training_step_captured_per_rank(cuda_device, case):
    """Each rank's forward + backward step is captured into one CUDA graph (after an eager step), then replayed on the
    ranks' streams with new node states and weights copied in place: the replay equals float64 autograd and, bit for bit,
    the same step run eagerly.  The device-side epochs of both exchange directions continue across replays."""
    import torch
    adj, indeg, V = graph(TRAIN_ZIPF)
    world = case["world"]
    cuts = degree_balanced_cuts(adj, V, world)
    sgs, streams = virtual_ranks(adj, cuts, case["D"], cuda_device)
    warm_up(case, sgs, streams, cuda_device)
    plans = [sg.training_plan() for sg in sgs]
    cnts = [sg.local_num_incoming(indeg) for sg in sgs]
    h, ws, proj = make_inputs(case, 60)
    hs, wds, projs = rank_inputs(sgs, h, ws, proj, cuda_device)
    leaves = [[x] + list(A.flatten(w).values()) for x, w in zip(hs, wds)]
    torch.cuda.synchronize()
    training_step(case, sgs, streams, plans, cnts, hs, wds, projs)      # one eager step before capturing
    torch.cuda.synchronize()
    for ls in leaves:
        for t in ls:
            t.grad = None
    graphs, outs = [], []
    for r in range(world):                                 # capturing does not execute: the ranks are recorded in turn
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=streams[r]):
            outs.append(rank_step(case, sgs[r], plans[r], cnts[r], hs[r], wds[r], projs[r]))
        graphs.append(g)
    worst = {}
    for rnd in range(2):
        h, ws, proj = make_inputs(case, 70 + rnd)
        with torch.no_grad():
            for sg, x, w, p in zip(sgs, hs, wds, projs):
                x.copy_(torch.as_tensor(h[sg.lo:sg.hi]))
                p.copy_(torch.as_tensor(proj[sg.lo:sg.hi]))
                for t, v in zip(A.flatten(w).values(), A.flatten(ws).values()):
                    t.copy_(torch.as_tensor(v))
        torch.cuda.synchronize()
        for g, s in zip(graphs, streams):
            with torch.cuda.stream(s):
                g.replay()
        torch.cuda.synchronize()
        got = collect(outs, hs, wds)
        errs = assert_matches_truth(case, got, float64_truth(case, h, ws, proj), h, ws, "%s replay %d" % (case["id"], rnd))
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        eager = sharded_training(case, sgs, streams, h, ws, proj, cuda_device)
        assert eager.keys() == got.keys()
        for k in got:
            assert np.array_equal(got[k].view(np.int32), eager[k].view(np.int32)), "%s: replay %s != eager" % (case["id"], k)
    print("%s (world %d) replays: %s" % (case["id"], world, {k: "%.1e" % v for k, v in worst.items()}))
    del graphs
    torch.cuda.synchronize()
    for sg in sgs:
        sg.close()


# ---------------------------------------------------------------- refused calls -------------------------------------------
@pytest.mark.gpu
def test_refused_calls_record_nothing(cuda_device):
    """The backward of a gather attached without training=True, the reverse-index build during a capture, and a gradient
    of the wrong width raise RgnnError before anything is enqueued; the next backward exchange still gives the known
    answer (no epoch moved).  ShardedGraph.plan keeps refusing autograd with its message."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import RgnnError, launch_count, weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    adj, indeg, V = graph(TRAIN_ZIPF)
    cuts = degree_balanced_cuts(adj, V, 2)
    D, L = 16, len(adj)

    plain, pstreams = virtual_ranks(adj, cuts, D, cuda_device, training=False)
    before = launch_count()
    with pytest.raises(RgnnError, match="attach_grad"):
        plain[0].exchange_backward(0, torch.zeros((plain[0].n_local, D), device=cuda_device))
    assert launch_count() == before
    xs = [torch.ones((sg.n_own, D), device=cuda_device, requires_grad=True) for sg in plain]
    torch.cuda.synchronize()
    outs = []
    for sg, s, x in zip(plain, pstreams, xs):
        with torch.cuda.stream(s):
            outs.append(sg.gather(x, 0))
    torch.cuda.synchronize()
    with pytest.raises(RgnnError, match="attach_grad"):
        outs[0].sum().backward()
    for sg in plain:
        sg.close()

    sgs, streams = virtual_ranks(adj, cuts, D, cuda_device)
    before = launch_count()
    rev = sgs[0].export_reverse()["row"].cpu().numpy()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=streams[0]):
        with pytest.raises(RgnnError, match="capturing"):
            sgs[0].build_reverse()
    del g
    with pytest.raises(RgnnError, match="state_dim"):
        sgs[1].exchange_backward(1, torch.zeros((sgs[1].n_local, D + 4), device=cuda_device))
    bad = torch.zeros((sgs[1].n_local, 8), device=cuda_device)
    own = torch.empty((sgs[1].n_own, 8), device=cuda_device)
    with pytest.raises(RgnnError, match="multiple of 4"):
        check(load_library().rgnn_halo_exchange_backward(sgs[1].handle, 0, 6, bad.data_ptr(), own.data_ptr(),
                                                         streams[1].cuda_stream))
    with pytest.raises(RgnnError, match="buffer 2"):
        sgs[1].exchange_backward(2, torch.zeros((sgs[1].n_local, D), device=cuda_device))
    assert launch_count() == before
    assert np.array_equal(sgs[0].export_reverse()["row"].cpu().numpy(), rev)
    assert_sums_in_rank_order(sgs, streams, adj, cuts, D, cuda_device, seed=9)

    x = torch.as_tensor(node_states(sgs[0].n_local, 64, seed=4)).to(cuda_device).requires_grad_(True)
    with pytest.raises(RgnnError, match="local_adjacency_lists"):
        G.sparse_gnn_film_layer(x, sgs[0].plan, sgs[0].local_num_incoming(indeg), 64,
                                weights=W.to_torch(W.film_weights(L, 64, 64), cuda_device))
    for sg in sgs:
        sg.close()

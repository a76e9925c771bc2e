"""GPU: the kernel variants that only production-size batches select, each compared element by element with the float64
oracle.

The engine picks a kernel from the problem size: half-warp edge kernels and a split layer norm for small batches, one warp
per 128 columns (or per whole row under a layer-norm epilogue) above V * ceil(D / 128) = 132 * 40 warps; BN in {32, 64, 128}
for the persistent wgmma GEMM, whose CTAs walk several tiles once there are more than 132; GRU row slabs of 132 * 128 rows;
a single split of the TN weight-gradient GEMM at >= 132 output tiles.  Each case below is sized just past the threshold it
targets.  Its regime is restated from the case parameters (checked without a GPU by test_case_regimes) and the kernel the
regime implies must appear among the launched kernels, so a changed heuristic fails here instead of silently testing the
small-batch path again."""
import zlib

import numpy as np
import pytest

from oracle import ref_grads as RG
from oracle import ref_layers as R
from tf_gnn_samples_b200 import weights as W

from dispatch import (GRU_SLAB, HEAVY_SEGMENT, PPI6K, PPI6K_DENSE, PPI6K_ZIPF, QM9_20K, SMALL_BATCH, SMS, TILE_K, TILE_M, ZIPF6K,
                      gemm_shape, graph, in_degrees, pair_rows_per_type, ring_stages, runs_crossing_chunks)
from helpers import assert_parity, assert_parity_8c, launched_kernels, node_states

# ------------------------------------------------------------------ cases -----------------------------------------
CASES = [
    # RGAT, fused scores: one warp per 128 columns (never the half-warp kernel).  `scale` multiplies the attention vectors:
    # at 100 the logits have a standard deviation of ~20, the running maximum is rescaled many times per target and exp
    # underflows for ~4 % of the edges.  Two timesteps at that scale are too ill-conditioned for float32 itself (the
    # reference-order float32 path is 7e-5 off float64 there); 50 keeps them at 1.5e-5.
    dict(id="rgat_v6k_d128_k4", kind="rgat", graph=PPI6K_DENSE, D=128, K=4, T=1, scale=100.0),
    dict(id="rgat_v6k_d256_k8", kind="rgat", graph=PPI6K_DENSE, D=256, K=8, T=1, scale=100.0),
    dict(id="rgat_v6k_d256_k8_t2", kind="rgat", graph=PPI6K_DENSE, D=256, K=8, T=2, scale=50.0),
    dict(id="rgat_v800_d128_k1", kind="rgat", graph=("ppi", 800, 16000, 43, False), D=128, K=1, T=1, scale=100.0),
    # whole-row layer-norm epilogue, NV = D / 128 float4 per lane
    dict(id="film_d256_sum_t2", kind="film", graph=PPI6K, D=256, agg="sum", act="ReLU", normalize=False, T=2),
    dict(id="film_d384_max", kind="film", graph=PPI6K, D=384, agg="max", act="elu", normalize=False, T=1),
    dict(id="film_d512_sum", kind="film", graph=PPI6K, D=512, agg="sum", act="gelu", normalize=True, T=1),
    dict(id="film_d256_zipf_heavy", kind="film", graph=PPI6K_ZIPF, D=256, agg="sum", act="tanh", normalize=True, T=1),
    dict(id="edge_mlp_d256_target", kind="edge_mlp", graph=PPI6K, D=256, act="gelu", normalize=True),
    dict(id="rgin_d256", kind="rgin", graph=PPI6K, D=256, act="ReLU"),
    # persistent wgmma GEMM with more tiles than SMs
    dict(id="dense_bn32_k100", kind="dense", M=40000, K=100, N=32, act="tanh"),
    dict(id="dense_bn32_k300", kind="dense", M=40000, K=300, N=32, act="relu"),
    dict(id="dense_bn64_k100", kind="dense", M=40000, K=100, N=64, act="leaky_relu"),
    dict(id="dense_bn64_k300", kind="dense", M=40000, K=300, N=64, act="elu"),
    dict(id="dense_bn128_n96_k100", kind="dense", M=40000, K=100, N=96, act="selu"),
    dict(id="dense_bn128_n96_k300", kind="dense", M=40000, K=300, N=96, act="gelu"),
    dict(id="dense_bn32_k300_linear", kind="dense", M=40000, K=300, N=32, act=None),
    dict(id="dense_grad_x_bn32", kind="dense_backward", M=40000, K=32, N=100),
    # grad_x here contracts 1,536 terms: the 3xTF32 GEMM measured 1.1e-5 on an H100 80GB HBM3 (700 W), a plain float32
    # GEMM 6e-7; grad_x is held to the 1e-4 north star, grad_w (the single-split TN kernel this case is for) to 1e-5
    dict(id="dense_grad_w_one_split", kind="dense_backward", M=300, K=1536, N=1536, grad_x_tol=1e-4),
    # GGNN on a QM9-like batch: two GRU slabs, the RNN cell's second K segment, the gathered (source, type) transform
    dict(id="ggnn_gru_d64_t2", kind="ggnn", graph=QM9_20K, D=64, cell="gru", T=2),
    dict(id="ggnn_rnn_d64", kind="ggnn", graph=QM9_20K, D=64, cell="rnn", T=1),
    dict(id="ggnn_rnn_d100", kind="ggnn", graph=QM9_20K, D=100, cell="rnn", T=1),
    # plain edge stage: RGCN with target-side messages, heavy and isolated targets
    dict(id="rgcn_both_sum", kind="rgcn", graph=ZIPF6K, D=256, agg="sum"),
    dict(id="rgcn_both_mean", kind="rgcn", graph=ZIPF6K, D=256, agg="mean"),
    dict(id="rgcn_both_max", kind="rgcn", graph=ZIPF6K, D=256, agg="max"),
    dict(id="rgcn_backward_sum", kind="rgcn_backward", graph=ZIPF6K, D=256, agg="sum"),
    dict(id="rgcn_backward_mean", kind="rgcn_backward", graph=ZIPF6K, D=256, agg="mean"),
]


def _b(x):
    return "true" if x else "false"


def _act_msg(act):
    return act is not None and act.lower() != "linear"


def regime(case):
    """(claims, kernels): the inequalities that put the case in its regime as (text, holds) pairs, and the kernel-name
    substrings that regime implies."""
    k = case["kind"]
    claims, kernels = [], []
    if k in ("dense", "dense_backward"):
        M, K, N = case["M"], case["K"], case["N"]
        if k == "dense":
            bn, tiles, chunks = gemm_shape(M, N, K)
            claims.append(("%d x %d tiles at BN %d = %d > %d SMs" % (-(-M // TILE_M), -(-N // bn), bn, tiles, SMS), tiles > SMS))
            claims.append(("K = %d is not a multiple of %d" % (K, TILE_K), K % TILE_K != 0))
            claims.append(("%d K chunks vs %d ring stages" % (chunks, ring_stages(bn)), True))
            if N == 96:
                claims.append(("N = 96 < BN = %d: partial n-tile" % bn, N % bn != 0))
            kernels.append("gemm_wgmma_kernel<0, %d, false>" % bn)
        else:
            bn, tiles, _ = gemm_shape(M, K, N)                      # grad_x = g . W^T: [M, N] x [N, K]
            kernels.append("gemm_wgmma_kernel<0, %d, false>" % bn)
            tn_tiles = -(-K // 128) * -(-N // 128)                  # grad_w = x^T . g: [K, N] output tiles of 128 x 128
            steps = -(-M // TILE_K)                                 # gemm_tn_wgmma.cu tn_shape: split K over about one wave
            per_split = -(-steps // max(1, min(SMS // tn_tiles, steps)))
            splits = -(-steps // per_split)
            if K == 32:
                claims.append(("grad_x: %d tiles at BN %d > %d SMs" % (tiles, bn, SMS), tiles > SMS and bn == 32))
                claims.append(("grad_x: K = %d is not a multiple of %d" % (N, TILE_K), N % TILE_K != 0))
            else:
                claims.append(("grad_w: %d x %d = %d output tiles >= %d SMs -> %d split" % (-(-K // 128), -(-N // 128), tn_tiles, SMS, splits),
                               tn_tiles >= SMS and splits == 1))
            kernels.append("gemm_tn_wgmma_kernel")
        return claims, kernels

    adj, indeg, V = graph(case["graph"])
    L, D = len(adj), case["D"]
    deg = in_degrees(adj, V)
    nv = -(-D // 128)
    warps = V * nv
    if k == "rgat":
        lph = D // case["K"] // 4
        claims.append(("per-head width %d: %d lanes per head, a power of two <= 32 (fused scores)" % (D // case["K"], lph),
                       lph <= 32 and lph & (lph - 1) == 0))
        claims.append(("V*ceil(D/128) = %d >= %d or %d lanes per head > 16 (not the half-warp kernel)" % (warps, SMALL_BATCH, lph),
                       warps >= SMALL_BATCH or lph > 16))
        claims.append(("%d targets with a (target, type) run crossing a 32-edge chunk" % runs_crossing_chunks(adj, V),
                       runs_crossing_chunks(adj, V) > 0))
        claims.append(("gridDim.y = %d" % nv, True))
        kernels.append("seg_rgat_kernel<1, true>")
    elif k in ("film", "edge_mlp", "rgin"):
        claims.append(("V = %d >= %d: whole-row layer norm (no split pass)" % (V, SMALL_BATCH), V >= SMALL_BATCH))
        claims.append(("NV = ceil(%d/128) = %d in {2, 3, 4}" % (D, nv), 2 <= nv <= 4))
        heavy = int((deg > HEAVY_SEGMENT).sum())
        mode, scaled, act_msg = {"film": (1, case.get("normalize"), _act_msg(case.get("act"))),
                                 "edge_mlp": (2, case.get("normalize"), _act_msg(case.get("act"))),
                                 "rgin": (0, False, _act_msg(case.get("act")))}[k]
        mx = case.get("agg") == "max"
        kernels.append("seg_reduce_kernel<%d, %d, %s, %s, %s>" % (nv, mode, _b(mx), _b(scaled), _b(act_msg)))
        if mx:
            claims.append(("every target has an incoming edge (no lowest() rows into the layer norm)", deg.min() >= 1))
        if case["id"].endswith("heavy"):
            claims.append(("%d targets above %d edges (max %d): split part / finish kernels" % (heavy, HEAVY_SEGMENT, deg.max()), heavy > 0))
            kernels += ["seg_reduce_heavy_part_kernel<%d, %d, %s, %s, %s>" % (nv, mode, _b(mx), _b(scaled), _b(act_msg)),
                        "seg_reduce_heavy_finish_kernel<%d, %s>" % (nv, _b(mx))]
    elif k == "ggnn":
        M = sum(a.shape[0] for a in adj)
        slabs = -(-V // GRU_SLAB)
        pairs = pair_rows_per_type(adj)
        claims.append(("M = %d < 0.75 * V * L = %d: compact pair table" % (M, int(0.75 * V * L)), M < 0.75 * V * L))
        bn, tiles, _ = gemm_shape(max(pairs), D, D, gz=L, row_counts=pairs)
        claims.append(("gathered transform: per-type rows %s -> %d tiles at BN %d > %d SMs" % (pairs, tiles, bn, SMS), tiles > SMS))
        kernels.append("gemm_wgmma_kernel<0, %d, true>" % bn)
        if case["cell"] == "gru":
            last = V - (slabs - 1) * GRU_SLAB
            claims.append(("%d rows = %d slabs of %d, the last one %d rows" % (V, slabs, GRU_SLAB, last), slabs == 2 and 0 < last < GRU_SLAB))
            for rows in (GRU_SLAB, last):
                kernels.append("gemm_wgmma_kernel<1, %d, false>" % gemm_shape(rows, 2 * D, D, D)[0])
                kernels.append("gemm_wgmma_kernel<2, %d, false>" % gemm_shape(rows, D, D, D)[0])
        else:
            bn, tiles, chunks = gemm_shape(V, D, D, D)
            claims.append(("RNN cell: [m | h] . [W; U], %d tiles at BN %d > %d SMs, %d K chunks over two segments" % (tiles, bn, SMS, chunks),
                           tiles > SMS))
            if D % TILE_K:
                claims.append(("K1 = K2 = %d is not a multiple of %d" % (D, TILE_K), True))
            kernels.append("gemm_wgmma_kernel<0, %d, false>" % bn)
    elif k in ("rgcn", "rgcn_backward"):
        heavy = int((deg > HEAVY_SEGMENT).sum())
        claims.append(("V*ceil(D/128) = %d >= %d: one warp per 128 columns, gridDim.y = %d" % (warps, SMALL_BATCH, nv),
                       warps >= SMALL_BATCH and nv == 2))
        claims.append(("%d targets above %d edges (max %d)" % (heavy, HEAVY_SEGMENT, deg.max()), heavy > 0))
        claims.append(("%d targets without an incoming edge" % int((deg == 0).sum()), (deg == 0).sum() > 0))
        if k == "rgcn":
            mx = case["agg"] == "max"
            bn, tiles, _ = gemm_shape(V, 2 * L * D, D)
            claims.append(("transform [h_u | h_v]: %d tiles at BN %d > %d SMs" % (tiles, bn, SMS), tiles > SMS))
            kernels += ["seg_reduce_kernel<1, 2, %s, true, false>" % _b(mx),
                        "seg_reduce_heavy_part_kernel<1, 2, %s, true, false>" % _b(mx),
                        "gemm_wgmma_kernel<0, %d, false>" % bn]
        else:
            claims.append(("reverse index: V*L*ceil(D/128) = %d >= %d segments' warps" % (V * L * nv, SMALL_BATCH), V * L * nv >= SMALL_BATCH))
            bn, tiles, _ = gemm_shape(V, D, L * D)
            kernels += ["seg_reduce_kernel<1, 0, false, true, false>", "seg_reduce_heavy_part_kernel<1, 0, false, true, false>",
                        "seg_reduce_heavy_kernel<1, 0, false, true, false>", "act_backward_kernel",
                        "gemm_wgmma_kernel<0, %d, false>" % bn, "gemm_tn_wgmma_kernel"]
    return claims, kernels


def test_case_regimes():
    """Every case is sized into the regime it is meant to test (no GPU needed)."""
    for case in CASES:
        claims, kernels = regime(case)
        assert kernels, case["id"]
        for text, holds in claims:
            print("%-24s %s" % (case["id"], text))
            assert holds, "%s: %s" % (case["id"], text)


# ------------------------------------------------------------------ oracle and engine ------------------------------
def _weights(case, L):
    k, D = case["kind"], case["D"]
    if k == "rgat":
        w = W.rgat_weights(L, D, D, seed=5)
        w["attention"] = [a * np.float32(case["scale"]) for a in w["attention"]]
        return w
    if k == "film":
        return W.film_weights(L, D, D, seed=6, num_timesteps=case["T"], random_ln=True)
    if k == "edge_mlp":
        return W.edge_mlp_weights(L, D, D, num_edge_hidden_layers=0, use_target_state_as_input=True, seed=7, random_ln=True)
    if k == "rgin":
        return W.rgin_weights(L, D, D, num_edge_MLP_hidden_layers=1, num_aggr_MLP_hidden_layers=None, seed=8, random_ln=True)
    if k == "ggnn":
        return W.ggnn_weights(L, D, seed=9, cell=case["cell"], random_bias=True)
    return W.rgcn_weights(L, D, D, seed=10, use_both_source_and_target=(k == "rgcn"))


def _layer_kwargs(case):
    k = case["kind"]
    if k == "rgat":
        return dict(state_dim=case["D"], num_heads=case["K"], num_timesteps=case["T"], activation_function="tanh")
    if k == "film":
        return dict(state_dim=case["D"], num_timesteps=case["T"], activation_function=case["act"],
                    message_aggregation_function=case["agg"], normalize_by_num_incoming=case["normalize"])
    if k == "edge_mlp":
        return dict(state_dim=case["D"], activation_function=case["act"], normalize_by_num_incoming=case["normalize"],
                    use_target_state_as_input=True, num_edge_hidden_layers=0)
    if k == "rgin":
        return dict(state_dim=case["D"], activation_function=case["act"], num_edge_MLP_hidden_layers=1, num_aggr_MLP_hidden_layers=None)
    if k == "ggnn":
        return dict(state_dim=case["D"], num_timesteps=case["T"], gated_unit_type=case["cell"], activation_function="tanh")
    if k == "rgcn":
        return dict(state_dim=case["D"], activation_function=None if case["agg"] == "max" else "tanh",
                    message_aggregation_function=case["agg"], normalize_by_num_incoming=True, use_both_source_and_target=True)
    return dict(activation_function="tanh", message_aggregation_function=case["agg"], normalize_by_num_incoming=True)


ORACLES = {"rgat": (R.sparse_rgat_layer, False), "film": (R.sparse_gnn_film_layer, True),
           "edge_mlp": (R.sparse_gnn_edge_mlp_layer, True), "rgin": (R.sparse_rgin_layer, False),
           "ggnn": (R.sparse_ggnn_layer, False), "rgcn": (R.sparse_rgcn_layer, True)}
LAYER_NORM_KINDS = ("film", "edge_mlp", "rgin")


def inputs(case):
    """Seeded inputs of a case: (h, adj, indeg, weights, grad_out or None) for layer cases, (x, w, bias, g) for GEMMs."""
    rng = np.random.default_rng(zlib.crc32(case["id"].encode()))
    if case["kind"] in ("dense", "dense_backward"):
        M, K, N = case["M"], case["K"], case["N"]
        x = rng.standard_normal((M, K)).astype(np.float32)
        w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
        b = rng.standard_normal(N).astype(np.float32)
        g = rng.standard_normal((M, N)).astype(np.float32)
        return x, w, b, g
    adj, indeg, V = graph(case["graph"])
    h = node_states(V, case["D"], seed=11)
    g = rng.standard_normal((V, case["D"])).astype(np.float32) if case["kind"] == "rgcn_backward" else None
    return h, adj, indeg, _weights(case, len(adj)), g


def oracle(case, data):
    """float64 truth of the case (and the reference-order float32 result for the layer-norm layers)."""
    k = case["kind"]
    if k == "dense":
        x, w, b, _ = data
        fn = R.get_activation(case["act"])
        y = x.astype(np.float64) @ w.astype(np.float64) + b
        return {"out": y if fn is None else fn(y)}
    if k == "dense_backward":
        x, w, _, g = data
        return {"grad_x": g.astype(np.float64) @ w.astype(np.float64).T, "grad_w": x.astype(np.float64).T @ g.astype(np.float64)}
    h, adj, indeg, w, g = data
    kw = _layer_kwargs(case)
    if k == "rgcn_backward":
        want = {"out": R.sparse_rgcn_layer(h, adj, indeg, case["D"], weights=w, **kw)}
        want["d_h"], want["d_w"] = RG.rgcn_layer_grads(h, adj, indeg, g, kw["activation_function"], case["agg"], True, weights=w)
        return want
    fn, with_indeg = ORACLES[k]
    args = (h, adj, indeg) if with_indeg else (h, adj)
    want = {"out": fn(*args, **kw, weights=w)}
    if k in LAYER_NORM_KINDS:
        want["out32"] = fn(*args, **kw, weights=w, dtype=np.float32)
    return want


def engine(case, data, device, expect):
    """The engine's result of the case on `device` and the set of kernels it launched (`expect`: see launched_kernels)."""
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import ops
    k = case["kind"]
    got = {}
    if k in ("dense", "dense_backward"):
        x, w, b, g = (torch.as_tensor(a).to(device) for a in data)
        if k == "dense":
            names = launched_kernels(lambda: got.update(out=ops.dense(x, w, b, case["act"])), expect)
        else:
            names = launched_kernels(lambda: got.update(zip(("grad_x", "grad_w"), ops.dense_backward(x, w, g))), expect)
        return {n: t.cpu().numpy() for n, t in got.items()}, names
    h, adj, indeg, w, g = data
    plan = G.GraphPlan(adj, h.shape[0], device=device)
    ht = torch.as_tensor(h).to(device)
    ct = torch.as_tensor(indeg).to(device)
    kw = _layer_kwargs(case)
    if k == "rgcn_backward":
        hg = ht.clone().requires_grad_(True)
        wg = [torch.as_tensor(a).to(device).requires_grad_(True) for a in w["edge_weights"]]

        def step():
            for t in [hg] + wg:                  # gradients accumulate: a second profiled run must start from none
                t.grad = None
            out = G.sparse_rgcn_layer(hg, plan, ct, case["D"], weights={"edge_weights": wg}, **kw)
            (out * torch.as_tensor(g).to(device)).sum().backward()
            got["out"] = out.detach()
        names = launched_kernels(step, expect)
        got["d_h"] = hg.grad
        got["d_w"] = [a.grad for a in wg]
        return {n: ([a.cpu().numpy() for a in t] if isinstance(t, list) else t.cpu().numpy()) for n, t in got.items()}, names
    layer = {"rgat": G.sparse_rgat_layer, "film": G.sparse_gnn_film_layer, "edge_mlp": G.sparse_gnn_edge_mlp_layer,
             "rgin": G.sparse_rgin_layer, "ggnn": G.sparse_ggnn_layer, "rgcn": G.sparse_rgcn_layer}[k]
    wt = W.to_torch(w, device)
    args = (ht, plan, ct) if ORACLES[k][1] else (ht, plan)
    names = launched_kernels(lambda: got.update(out=layer(*args, **kw, weights=wt)), expect)
    return {"out": got["out"].cpu().numpy()}, names


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_large_batch_variant(cuda_device, case):
    _, kernels = regime(case)
    data = inputs(case)
    got, names = engine(case, data, cuda_device, kernels)
    for want_kernel in kernels:
        matched = sorted(n for n in names if want_kernel in n)
        assert matched, "%s: no launched kernel matches %r; launched: %s" % (case["id"], want_kernel, sorted(names))
        print("%s: launched %s" % (case["id"], matched[0]))
    want = oracle(case, data)
    what = case["id"]
    if case["kind"] == "dense":
        print("%s: max-norm relative error %.2e" % (what, assert_parity(got["out"], want["out"], what, tol=1e-5)))
    elif case["kind"] == "dense_backward":
        for n in ("grad_x", "grad_w"):
            tol = case.get(n + "_tol", 1e-5)
            print("%s %s: max-norm relative error %.2e" % (what, n, assert_parity(got[n], want[n], "%s %s" % (what, n), tol=tol)))
    elif case["kind"] in LAYER_NORM_KINDS:
        assert_parity_8c(got["out"], want["out"], want["out32"], what)
    elif case["kind"] == "rgcn" and case["agg"] == "max":
        # targets without a message hold float32 lowest() (linear activation keeps it): same rows, finite part compared
        mask = np.abs(want["out"]) < 1e30
        assert np.array_equal(mask, np.abs(got["out"]) < 1e30), "%s: lowest() rows differ" % what
        assert (~mask).any()
        err = assert_parity(np.where(mask, got["out"], 0), np.where(mask, want["out"], 0), what)
        print("%s: max-norm relative error %.2e (%d lowest() rows)" % (what, err, int((~mask).all(axis=1).sum())))
    else:
        print("%s: max-norm relative error %.2e" % (what, assert_parity(got["out"], want["out"], what)))
        if case["kind"] == "rgcn_backward":
            print("%s d_h: max-norm relative error %.2e" % (what, assert_parity(got["d_h"], want["d_h"], what + " d_h")))
            for l, (gw, ww) in enumerate(zip(got["d_w"], want["d_w"])):
                print("%s d_W[%d]: max-norm relative error %.2e" % (what, l, assert_parity(gw, ww, "%s d_W[%d]" % (what, l))))

"""GPU: the C ABI's buffer contract (include/rgnn.h), for every layer and building block, through the ABI itself.

Every buffer a call touches -- inputs, outputs, workspace and the adjacency lists its plan is built from -- is a guarded
buffer: one allocation with a 64 KiB guard band on each side of the payload, the payload starting at 16 mod 512 (the
16-byte alignment the header promises, not the 512 bytes torch happens to give) and the trailing guard starting right at
the payload's last byte.  Per case:

  (a) the minimum accepted workspace S_min is found by bisection on RGNN_E_WORKSPACE and must not exceed the documented
      bound; every run below uses exactly S_min bytes, so the trailing guard sits where the last carve-out ends;
  (b) the workspace is poisoned with NaN, +FLT_MAX and -FLT_MAX, the outputs with NaN and +FLT_MAX: every run must be bit
      identical to the same call through the Python API (which allocates its buffers from torch);
  (c) that Python-path result must match the float64 oracle, so both paths cannot be wrong together;
  (d) every input is byte-identical after the call; (e) every guard band is intact;
  (f) on a restricted plan, output rows >= num_targets keep their poison bits;
  (g) S_min - 256 bytes, 0 bytes and a NULL workspace return RGNN_E_WORKSPACE, write no output and touch no guard.

One case per family also runs with the weight cache on, which moves the weight images into library memory: S_min shrinks
and the result is bit-identical.  Wider-than-supported MLP layers are refused with RGNN_E_UNSUPPORTED.  Each case states
its regime; test_case_regimes checks those statements without a GPU."""
import ctypes
import functools

import numpy as np
import pytest

from oracle import ref_autograd as A
from oracle import ref_layers as R
from tf_gnn_samples_b200 import weights as W
from tf_gnn_samples_b200.utils import (LAYER_EDGE_MLP, LAYER_FILM, LAYER_GGNN, LAYER_RGAT, LAYER_RGCN, LAYER_RGCN_BACKWARD,
                                       LAYER_RGDCN, LAYER_RGIN, get_activation, get_aggregation_function, get_gated_unit)

from dispatch import (GRU_SLAB, HEAVY_SEGMENT, PPI6K, PPI6K_ZIPF, QM9_20K, SMALL_BATCH, SMS, ZIPF6K, graph as dispatch_graph,
                      in_degrees, segment_sizes)
from helpers import assert_parity, assert_parity_8c, launched_kernels, node_states, rel, tiny_graph

TOL = 1e-4
GUARD = 64 * 1024               # guard band on each side of a payload
SHIFT = 16                      # payload at 16 mod 512: the alignment include/rgnn.h promises, and no more
GUARD_BYTE = 0xA5
WS_POISON = (0xFFFFFFFF, 0x7F7FFFFF, 0xFF7FFFFF)     # NaN, +FLT_MAX, -FLT_MAX
OUT_POISON = (0x7FC00000, 0x7F7FFFFF)                 # NaN, +FLT_MAX
E_WORKSPACE, E_UNSUPPORTED = -3, -4

TINY = ("tiny",)                                      # helpers.tiny_graph: empty type, isolated targets, duplicates
PPI2K = ("ppi", 2000, 6000, 49, False)                # below the 132 * 40-warp small-batch threshold at D <= 128
BENCH = ("ppi", 2245, 59000, 0, False)                # bench.py's RGCN stack batch
SMALL_ZIPF = ("zipf", 600, 1000, 3, 30, 47)           # RGDCN's oracle holds a [E, K, K] tensor per type
ZIPF_SRC = ("zipf_src",)                              # ZIPF6K with sources and targets swapped: hub SOURCES


@functools.lru_cache(maxsize=None)
def graph(key):
    if key == TINY:
        adj, indeg = tiny_graph()
        return adj, indeg, 37
    if key == BENCH:
        from tf_gnn_samples_b200 import batching
        b = batching.ppi_like_batch(num_graphs=1, num_nodes=2245, num_links=59000, seed=0)
        return b.adjacency_lists, b.type_to_num_incoming_edges, b.num_nodes
    if key == ZIPF_SRC:
        adj, _, V = dispatch_graph(ZIPF6K)
        adj = [np.ascontiguousarray(a[:, ::-1]) for a in adj]
        return adj, np.stack([np.bincount(a[:, 1], minlength=V) for a in adj]).astype(np.float32), V
    return dispatch_graph(key)


# ---------------------------------------------------------------- guarded buffers ----------------------------------------
class Guarded:
    """One CUDA uint8 allocation: [GUARD + SHIFT bytes of guard | payload | GUARD bytes of guard]."""

    def __init__(self, name, nbytes, device):
        import torch
        self.name, self.nbytes = name, int(nbytes)
        self.raw = torch.full((GUARD + SHIFT + self.nbytes + GUARD,), GUARD_BYTE, dtype=torch.uint8, device=device)
        assert self.raw.data_ptr() % 512 == 0
        self.payload = self.raw[GUARD + SHIFT: GUARD + SHIFT + self.nbytes]
        assert self.ptr % 512 == SHIFT

    @classmethod
    def copy_of(cls, name, t):
        g = cls(name, t.numel() * t.element_size(), t.device)
        g.payload.copy_(t.contiguous().view(-1).view(__import__("torch").uint8))
        return g

    @property
    def ptr(self):
        return self.raw.data_ptr() + GUARD + SHIFT

    def f32(self, shape):
        import torch
        return self.payload.view(torch.float32).view(shape)

    def fill(self, bits):
        import torch
        self.payload.view(torch.int32).fill_(int(np.uint32(bits).view(np.int32)))

    def check_guards(self):
        import torch
        for part, base, where in ((self.raw[: GUARD + SHIFT], -(GUARD + SHIFT), "start"),
                                  (self.raw[GUARD + SHIFT + self.nbytes:], 0, "end")):
            bad = torch.nonzero(part != GUARD_BYTE)
            if bad.numel():
                raise AssertionError("guard of '%s' hit: %d bytes, the first at offset %+d from the payload's %s"
                                     % (self.name, bad.numel(), int(bad[0, 0]) + base, where))


def poison_bits(t, bits):
    """True where float32 tensor t still holds the bit pattern `bits`."""
    import torch
    return t.contiguous().view(torch.int32) == int(np.uint32(bits).view(np.int32))


# ---------------------------------------------------------------- the cases ----------------------------------------------
class Setup:
    """ins: name -> device tensor; outs: name -> shape; call(lib, plan, p, tab, ws, nbytes, stream) -> rc with p: name ->
    pointer and tab(names) -> pointer table; python(plan) -> {name: tensor}; oracle(py) asserts the Python result against
    float64; bound(lib, plan) -> documented workspace bytes (None: the call takes no workspace)."""
    graph = None
    num_targets = None
    bound = None


def t(x, dev):
    import torch
    return torch.as_tensor(np.ascontiguousarray(x)).to(dev)


def ln_rows(w, T, D):
    return np.stack(w["ln_gamma"]).reshape(T, D), np.stack(w["ln_beta"]).reshape(T, D)


def named(prefix, arrays):
    return {"%s%d" % (prefix, i): a for i, a in enumerate(arrays)}


def layer_setup(c, dev):
    import torch
    import tf_gnn_samples_b200 as G
    k = c["kind"]
    adj, indeg, V = graph(c["graph"])
    L, D, T = len(adj), c["D"], c.get("T", 1)
    di = c.get("din", D)
    act_name, agg_name, norm = c.get("act", "tanh"), c.get("agg", "sum"), c.get("normalize", False)
    act, agg = get_activation(act_name), get_aggregation_function(agg_name)
    h = node_states(V, di, seed=3)
    s = Setup()
    s.graph, s.num_targets = (adj, V), c.get("num_targets")
    s.outs = {"out": (V, D)}
    ins = {"h": h, "cnt": indeg}
    cnt = lambda p: p["cnt"] if norm else None
    tcnt = t(indeg, dev)
    if k == "rgcn":
        both = c.get("both", False)
        w = W.rgcn_weights(L, di, D, 7, use_both_source_and_target=both)
        ins.update(named("w", w["edge_weights"]))
        wn = ["w%d" % l for l in range(L)]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgcn_forward(
            plan, p["h"], di, D, tab(wn), cnt(p), act, agg, int(norm), int(both), T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_rgcn_layer(t(h, dev), pl, tcnt, D, T, act_name, agg_name, norm, both,
                                                          weights=W.to_torch(w, dev))}
        want = lambda: R.sparse_rgcn_layer(h, adj, indeg, D, T, act_name, agg_name, norm, both, weights=w)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGCN, di, D, 0)
    elif k == "rgcn_stack":
        ws3 = [W.rgcn_weights(L, D, D, 7 + 3 * i) for i in range(c["layers"])]
        for i, w in enumerate(ws3):
            ins.update(named("w%d_" % i, w["edge_weights"]))
        wn = ["w%d_%d" % (i, l) for i in range(len(ws3)) for l in range(L)]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgcn_stack_forward(
            plan, p["h"], D, len(ws3), tab(wn), cnt(p), act, agg, int(norm), p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.rgcn_layer_stack(t(h, dev), pl, tcnt, [W.to_torch(w, dev) for w in ws3],
                                                         act_name, agg_name, norm)}

        def want():
            x = h
            for w in ws3:
                x = R.sparse_rgcn_layer(x, adj, indeg, D, 1, act_name, agg_name, norm, weights=w)
            return x
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGCN, D, D, 0) + 2 * (V * D * 4 + 256)
    elif k == "ggnn":
        w = W.ggnn_weights(L, D, 7, cell=c["cell"], random_bias=True)
        ins.update(named("w", w["edge_weights"]))
        ins.update(ck=w["cell"]["kernel"], rk=w["cell"]["recurrent_kernel"], cb=w["cell"]["bias"])
        wn = ["w%d" % l for l in range(L)]
        cell, gact = get_gated_unit(D, c["cell"], act_name)
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_ggnn_forward(
            plan, p["h"], D, D, tab(wn), p["ck"], p["rk"], p["cb"], cell, gact, agg, T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_ggnn_layer(t(h, dev), pl, D, T, c["cell"], act_name, agg_name,
                                                          weights=W.to_torch(w, dev))}
        want = lambda: R.sparse_ggnn_layer(h, adj, D, T, c["cell"], act_name, agg_name, weights=w)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_GGNN, D, D, 0)
    elif k == "rgat":
        w = W.rgat_weights(L, D, D, 7)
        ins.update(named("w", w["edge_weights"]))
        ins.update(named("att", w["attention"]))
        wn, an = ["w%d" % l for l in range(L)], ["att%d" % l for l in range(L)]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgat_forward(
            plan, p["h"], D, D, tab(wn), tab(an), c["heads"], act, T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_rgat_layer(t(h, dev), pl, D, c["heads"], T, act_name, weights=W.to_torch(w, dev))}
        want = lambda: R.sparse_rgat_layer(h, adj, D, c["heads"], T, act_name, weights=w)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGAT, D, D, 0)
    elif k == "film":
        w = W.film_weights(L, D, D, 7, num_timesteps=T, random_ln=True)
        ins.update(named("w", w["edge_weights"]))
        ins.update(named("fw", w["film_weights"]))
        ins["lng"], ins["lnb"] = ln_rows(w, T, D)
        wn, fn = ["w%d" % l for l in range(L)], ["fw%d" % l for l in range(L)]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_film_forward(
            plan, p["h"], D, D, tab(wn), tab(fn), cnt(p), p["lng"], p["lnb"], act, agg, int(norm), T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_gnn_film_layer(t(h, dev), pl, tcnt, D, T, act_name, agg_name, norm,
                                                              weights=W.to_torch(w, dev))}
        want = lambda dt=np.float64: R.sparse_gnn_film_layer(h, adj, indeg, D, T, act_name, agg_name, norm, weights=w, dtype=dt)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_FILM, D, D, 0)
    elif k == "edge_mlp":
        hid, tgt = c["hidden"], c["use_target"]
        w = W.edge_mlp_weights(L, D, D, hid, tgt, 7, num_timesteps=T, random_ln=True)
        if c.get("width"):                                   # hidden layers wider than the workspace bound assumes
            rng = np.random.default_rng(5)
            dims = [D * (1 + tgt)] + [c["width"]] * hid + [D]
            w["edge_mlps"] = [[W.glorot_uniform(rng, dims[j], dims[j + 1]) for j in range(hid + 1)] for _ in range(L)]
        flat = [x for ks in w["edge_mlps"] for x in ks]
        dims = [int(w["edge_mlps"][0][0].shape[0])] + [int(x.shape[1]) for x in w["edge_mlps"][0]]
        ins.update(named("m", flat))
        ins["lng"], ins["lnb"] = ln_rows(w, T, D)
        mn = ["m%d" % i for i in range(len(flat))]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_edge_mlp_forward(
            plan, p["h"], D, D, tab(mn), (ctypes.c_int32 * len(dims))(*dims), hid, cnt(p), p["lng"], p["lnb"], act, agg,
            int(norm), int(tgt), T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_gnn_edge_mlp_layer(t(h, dev), pl, tcnt, D, T, act_name, agg_name, norm, tgt, hid,
                                                                  weights=W.to_torch(w, dev))}
        want = lambda dt=np.float64: R.sparse_gnn_edge_mlp_layer(h, adj, indeg, D, T, act_name, agg_name, norm, tgt, hid,
                                                                 weights=w, dtype=dt)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_EDGE_MLP, D, D, hid + 1)
    elif k == "rgin":
        eh, ah, tgt = c["edge_hidden"], c["aggr_hidden"], c["use_target"]
        w = W.rgin_weights(L, D, D, eh, ah, tgt, 7, num_timesteps=T, random_ln=True)
        if c.get("width"):
            rng = np.random.default_rng(5)
            dims = [D * (1 + tgt)] + [c["width"]] * eh + [D]
            w["edge_mlps"] = [[W.glorot_uniform(rng, dims[j], dims[j + 1]) for j in range(eh + 1)] for _ in range(L)]
        ins["lng"], ins["lnb"] = ln_rows(w, T, D)
        en, an, ed, ad = [], [], None, None
        if eh is not None:
            flat = [x for ks in w["edge_mlps"] for x in ks]
            ins.update(named("m", flat))
            en = ["m%d" % i for i in range(len(flat))]
            ed = [int(w["edge_mlps"][0][0].shape[0])] + [int(x.shape[1]) for x in w["edge_mlps"][0]]
        if ah is not None:
            ins.update(named("a", w["aggr_mlp"]))
            an = ["a%d" % i for i in range(len(w["aggr_mlp"]))]
            ad = [int(w["aggr_mlp"][0].shape[0])] + [int(x.shape[1]) for x in w["aggr_mlp"]]
        i32 = lambda d: (ctypes.c_int32 * len(d))(*d) if d else None
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgin_forward(
            plan, p["h"], D, D, tab(en) if en else None, i32(ed), -1 if eh is None else eh, tab(an) if an else None, i32(ad),
            -1 if ah is None else ah, p["lng"], p["lnb"], act, agg, int(tgt), T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_rgin_layer(t(h, dev), pl, D, T, act_name, agg_name, tgt, eh, ah,
                                                          weights=W.to_torch(w, dev))}
        want = lambda dt=np.float64: R.sparse_rgin_layer(h, adj, D, T, act_name, agg_name, tgt, eh, ah, weights=w, dtype=dt)
        nl = max(0 if eh is None else eh + 1, 0 if ah is None else ah + 1)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGIN, D, D, nl)
    else:                                                    # rgdcn
        K, full, tied = c["K"], c["full"], c.get("tied", False)
        C = D // K
        w = W.rgdcn_weights(L, C, K, full, tied, 7, stddev=c.get("stddev", 0.5 / K))
        ins.update(named("cw", [x for ks in w["channel_weights"] for x in ks]))
        per = 1 if tied else C
        cn = ["cw%d" % (l * per + (0 if tied else ch)) for l in range(L) for ch in range(C)]
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgdcn_forward(
            plan, p["h"], D, C, tab(cn), int(full), cnt(p), act, agg, int(norm), T, p["out"], ws, nb, st)
        s.python = lambda pl: {"out": G.sparse_rgdcn_layer(t(h, dev), pl, tcnt, C, K, T, full, tied, act_name, agg_name, norm,
                                                           weights=W.to_torch(w, dev))}
        want = lambda: R.sparse_rgdcn_layer(h, adj, indeg, C, K, T, full, tied, act_name, agg_name, norm, weights=w)
        s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGDCN, D, D, K)
    s.ins = {n: t(v, dev) for n, v in ins.items()}
    nt = s.num_targets if s.num_targets is not None else V

    def oracle(py):
        got = py["out"][:nt].cpu().numpy()
        if k in ("film", "edge_mlp", "rgin"):
            return assert_parity_8c(got, want()[:nt], want(np.float32)[:nt], c["id"])[0]
        return assert_parity(got, want()[:nt], c["id"], tol=TOL)
    s.oracle = oracle
    return s


def rgcn_backward_setup(c, dev):
    import torch
    import tf_gnn_samples_b200 as G
    adj, indeg, V = graph(c["graph"])
    L, D, di = len(adj), c["D"], c.get("din", c["D"])
    act_name, agg_name, norm = c.get("act", "tanh"), c.get("agg", "sum"), c.get("normalize", True)
    act, agg = get_activation(act_name), get_aggregation_function(agg_name)
    h = node_states(V, di, seed=3)
    w = W.rgcn_weights(L, di, D, 7)
    g = np.random.default_rng(0).standard_normal((V, D)).astype(np.float32)
    with torch.no_grad():
        from tf_gnn_samples_b200 import GraphPlan
        out = G.sparse_rgcn_layer(t(h, dev), GraphPlan(adj, V, device=dev), t(indeg, dev), D, 1, act_name, agg_name, norm,
                                  weights=W.to_torch(w, dev))
    s = Setup()
    s.graph = (adj, V)
    s.ins = {"h": t(h, dev), "cnt": t(indeg, dev), "out": out, "g": t(g, dev), **{n: t(x, dev) for n, x in named("w", w["edge_weights"]).items()}}
    s.outs = {"gh": (V, di), **{"gw%d" % l: (di, D) for l in range(L)}}
    wn, gn = ["w%d" % l for l in range(L)], ["gw%d" % l for l in range(L)]
    s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_rgcn_backward(
        plan, p["h"], di, D, tab(wn), p["cnt"] if norm else None, act, agg, int(norm), p["out"], p["g"], p["gh"], tab(gn),
        ws, nb, st)
    s.bound = lambda lib, plan: lib.rgnn_workspace_bytes(plan, LAYER_RGCN_BACKWARD, di, D, 0)

    def python(pl):
        hd = t(h, dev).requires_grad_(True)
        wd = [t(x, dev).requires_grad_(True) for x in w["edge_weights"]]
        o = G.sparse_rgcn_layer(hd, pl, t(indeg, dev), D, 1, act_name, agg_name, norm, weights={"edge_weights": wd})
        assert torch.equal(o, out)
        o.backward(t(g, dev))
        return {"gh": hd.grad, **{"gw%d" % l: x.grad for l, x in enumerate(wd)}}
    s.python = python

    def oracle(py):
        h64 = torch.as_tensor(h, dtype=torch.float64).requires_grad_(True)
        w64 = [torch.as_tensor(x, dtype=torch.float64).requires_grad_(True) for x in w["edge_weights"]]
        o64 = A.sparse_rgcn_layer(h64, adj, torch.as_tensor(indeg, dtype=torch.float64), 1, act_name, agg_name, norm,
                                  weights={"edge_weights": w64})
        (o64 * torch.as_tensor(g, dtype=torch.float64)).sum().backward()
        errs = {"gh": rel(py["gh"].cpu().numpy(), h64.grad.numpy())}
        errs.update({"gw%d" % l: rel(py["gw%d" % l].cpu().numpy(), x.grad.numpy()) for l, x in enumerate(w64)})
        bad = {n: e for n, e in errs.items() if not e <= TOL}
        assert not bad, "%s: %s" % (c["id"], bad)
        return max(errs.values())
    s.oracle = oracle
    return s


def act64(name, x):
    return {"linear": x, "tanh": np.tanh(x), "relu": np.maximum(x, 0.0)}[name]


def block_setup(c, dev):
    import torch
    from tf_gnn_samples_b200 import ops
    k = c["kind"]
    s = Setup()
    rng = np.random.default_rng(11)
    if k == "dense":
        m, kk, n = c["m"], c["k"], c["n"]
        a = rng.standard_normal((m, kk)).astype(np.float32)
        b = (rng.standard_normal((kk, n)) / np.sqrt(kk)).astype(np.float32)
        bias = rng.standard_normal(n).astype(np.float32)
        s.ins = {"a": t(a, dev), "b": t(b, dev), "bias": t(bias, dev)}
        s.outs = {"c": (m, n)}
        act = get_activation(c["act"])
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_dense_forward(p["a"], m, kk, p["b"], n, p["bias"], act, p["c"],
                                                                             ws, nb, st)
        s.python = lambda pl: {"c": ops.dense(t(a, dev), t(b, dev), t(bias, dev), c["act"])}
        s.oracle = lambda py: assert_parity(py["c"].cpu().numpy(), act64(c["act"], a.astype(np.float64) @ b + bias), c["id"])
        s.bound = lambda lib, plan: lib.rgnn_dense_workspace_bytes(m, kk, n)
    elif k == "dense_backward":
        m, kk, n = c["m"], c["k"], c["n"]
        a = rng.standard_normal((m, kk)).astype(np.float32)
        b = (rng.standard_normal((kk, n)) / np.sqrt(kk)).astype(np.float32)
        gc = rng.standard_normal((m, n)).astype(np.float32)
        s.ins = {"a": t(a, dev), "b": t(b, dev), "gc": t(gc, dev)}
        s.outs = {"ga": (m, kk), "gb": (kk, n)}
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_dense_backward(p["a"], m, kk, p["b"], n, p["gc"], p["ga"], p["gb"],
                                                                              ws, nb, st)

        def python(pl):
            ga, gb = ops.dense_backward(t(a, dev), t(b, dev), t(gc, dev))
            return {"ga": ga, "gb": gb}
        s.python = python

        def oracle(py):
            a64, b64, g64 = a.astype(np.float64), b.astype(np.float64), gc.astype(np.float64)
            if m:
                assert_parity(py["ga"].cpu().numpy(), g64 @ b64.T, c["id"] + " grad_a")
                return assert_parity(py["gb"].cpu().numpy(), a64.T @ g64, c["id"] + " grad_b")
            assert not torch.any(py["gb"]).item(), "%s: grad_b of an empty contraction is not zero" % c["id"]
            return 0.0
        s.oracle = oracle
        s.bound = lambda lib, plan: lib.rgnn_dense_workspace_bytes(m, kk, n)
    elif k == "layer_norm":
        rows, d = c["rows"], c["d"]
        x = (3.0 * rng.standard_normal((rows, d)) + 1.5).astype(np.float32)
        gam = (1.0 + 0.2 * rng.standard_normal(d)).astype(np.float32)
        bet = (0.2 * rng.standard_normal(d)).astype(np.float32)
        s.ins = {"x": t(x, dev), "gamma": t(gam, dev), "beta": t(bet, dev)}
        s.outs = {"out": (rows, d)}
        s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_layer_norm(p["x"], rows, d, p["gamma"], p["beta"], p["out"], st)
        s.python = lambda pl: {"out": ops.layer_norm(t(x, dev), t(gam, dev), t(bet, dev))}
        s.oracle = lambda py: assert_parity(py["out"].cpu().numpy(), R.layer_norm(x.astype(np.float64), gam, bet), c["id"])
    else:                                                    # plan-based building blocks
        adj, indeg, V = graph(c["graph"])
        L, d = len(adj), c["D"]
        s.graph = (adj, V)
        agg_name, norm = c.get("agg", "sum"), c.get("normalize", False)
        agg = get_aggregation_function(agg_name)
        tgt = np.concatenate([a[:, 1] for a in adj]).astype(np.int64)
        src = np.concatenate([a[:, 0] for a in adj]).astype(np.int64)
        typ = np.concatenate([np.full(a.shape[0], l) for l, a in enumerate(adj)])
        if k == "segment":
            data = rng.standard_normal((tgt.size, d)).astype(np.float32)
            s.ins = {"data": t(data, dev)}
            s.outs = {"out": (V, d)}
            s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_segment_aggregate(plan, p["data"], d, agg, p["out"], st)
            s.python = lambda pl: {"out": ops.segment_aggregate(pl, t(data, dev), agg_name)}

            def oracle(py):
                want = R.get_aggregation_function(agg_name)(data.astype(np.float64), tgt, V)
                got = py["out"].cpu().numpy()
                if agg_name == "max":                       # an empty segment is numeric_limits<float>::lowest()
                    empty = np.bincount(tgt, minlength=V) == 0
                    assert empty.any() and np.all(got[empty] == np.finfo(np.float32).min), c["id"]
                    got, want = got[~empty], want[~empty]
                return assert_parity(got, want, c["id"])
            s.oracle = oracle
        else:
            scale = (1.0 / (indeg.astype(np.float64)[typ, tgt] + 1e-7)) if norm else np.ones(tgt.size)
            ins = {"cnt": indeg}
            cnt = lambda p: p["cnt"] if norm else None
            if k == "edge_agg":
                table = rng.standard_normal((V, L, d)).astype(np.float32)
                ins["table"] = table
                s.outs = {"out": (V, d)}
                s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_edge_aggregate_forward(plan, p["table"], d, cnt(p), agg,
                                                                                              p["out"], st)
                s.python = lambda pl: {"out": ops.edge_aggregate(t(table, dev), pl, t(indeg, dev) if norm else None, agg_name)}
                msgs = table.astype(np.float64)[src, typ] * scale[:, None]
                s.oracle = lambda py: assert_parity(py["out"].cpu().numpy(), R.get_aggregation_function(agg_name)(msgs, tgt, V),
                                                    c["id"])
            else:                                            # edge_agg_backward
                g = rng.standard_normal((V, d)).astype(np.float32)
                ins["g"] = g
                s.outs = {"d_table": (V, L, d)}
                s.call = lambda lib, plan, p, tab, ws, nb, st: lib.rgnn_edge_aggregate_backward(plan, p["g"], d, cnt(p), agg,
                                                                                               p["d_table"], st)

                def python(pl):
                    tab_ = torch.zeros((V, L, d), device=dev, requires_grad=True)
                    ops.edge_aggregate(tab_, pl, t(indeg, dev) if norm else None, agg_name).backward(t(g, dev))
                    return {"d_table": tab_.grad}
                s.python = python
                cnt_all = np.bincount(tgt, minlength=V).astype(np.float64)
                div = {"sum": np.ones(V), "mean": np.maximum(cnt_all, 1.0), "sqrt_n": np.sqrt(np.maximum(cnt_all, 1.0))}[agg_name]
                want = np.zeros((V * L, d))
                np.add.at(want, src * L + typ, (g.astype(np.float64) / div[:, None])[tgt] * scale[:, None])
                s.oracle = lambda py: assert_parity(py["d_table"].cpu().numpy(), want.reshape(V, L, d), c["id"])
            s.ins = {n: t(v, dev) for n, v in ins.items()}
    return s


def setup(c, dev):
    if c["kind"] == "rgcn_backward":
        return rgcn_backward_setup(c, dev)
    if c["kind"] in ("dense", "dense_backward", "layer_norm", "segment", "edge_agg", "edge_agg_backward"):
        return block_setup(c, dev)
    return layer_setup(c, dev)


HEAVY = ["seg_reduce_heavy_part_kernel", "seg_reduce_heavy_finish_kernel"]
TN = ["gemm_tn_wgmma_kernel", "gemm_tn_reduce_kernel"]
CASES = [
    # RGCN
    dict(id="rgcn_tiny_d36_to_d100", kind="rgcn", graph=TINY, din=36, D=100, normalize=True, cache=True,
         regime=["small", "isolated", "empty_type"], expect=["seg_reduce_half_kernel"]),
    dict(id="rgcn_both_mean_d36", kind="rgcn", graph=PPI6K, D=36, both=True, agg="mean"),
    dict(id="rgcn_both_max_d100_t2", kind="rgcn", graph=PPI6K, D=100, both=True, agg="max", act="relu", T=2),
    dict(id="rgcn_pair_table_d64", kind="rgcn", graph=QM9_20K, D=64, normalize=True, regime=["pair"], expect=[", true>"]),
    dict(id="rgcn_zipf_heavy_d256", kind="rgcn", graph=ZIPF6K, D=256, normalize=True, regime=["heavy", "isolated"],
         expect=HEAVY),
    dict(id="rgcn_restricted_d64", kind="rgcn", graph=PPI6K_ZIPF, D=64, normalize=True, num_targets=2500),
    # the bench's RGCN stack: PPI-shaped, 3 x 256
    dict(id="rgcn_stack_bench_3x256", kind="rgcn_stack", graph=BENCH, D=256, layers=3, act="relu", normalize=True, cache=True),
    # RGCN backward: the TN weight-gradient GEMM with several splits (one split needs more output tiles than any RGCN shape
    # reaches; dense_backward covers it), heavy reverse segments, gelu's recomputed pre-activation
    dict(id="rgcn_bwd_sum_d64", kind="rgcn_backward", graph=PPI6K, D=64, cache=True, regime=["tn_splits"], expect=TN),
    dict(id="rgcn_bwd_mean_heavy_sources_d36", kind="rgcn_backward", graph=ZIPF_SRC, D=36, agg="mean",
         regime=["heavy_sources"], expect=TN),
    dict(id="rgcn_bwd_gelu_d20", kind="rgcn_backward", graph=TINY, din=12, D=20, act="gelu", expect=TN),
    # GGNN
    dict(id="ggnn_gru_two_slabs_t2_d64", kind="ggnn", graph=QM9_20K, D=64, cell="gru", T=2, cache=True, regime=["two_slabs"]),
    dict(id="ggnn_rnn_d100", kind="ggnn", graph=PPI6K, D=100, cell="rnn"),
    dict(id="ggnn_gru_tiny_d12", kind="ggnn", graph=TINY, D=12, cell="gru"),
    # RGAT
    dict(id="rgat_half_d128_k4", kind="rgat", graph=PPI2K, D=128, heads=4, cache=True, regime=["small"],
         expect=["seg_rgat_half_kernel"]),
    dict(id="rgat_fused_d128_k1", kind="rgat", graph=PPI6K, D=128, heads=1, regime=["large"], expect=["seg_rgat_kernel<1, true>"]),
    dict(id="rgat_unfused_d96_k2", kind="rgat", graph=PPI6K, D=96, heads=2, expect=["rgat_scores_kernel"]),
    # FiLM
    dict(id="film_split_ln_d256", kind="film", graph=PPI2K, D=256, act="relu", normalize=True, cache=True, regime=["small"],
         expect=["layer_norm_kernel"]),
    dict(id="film_whole_row_d384", kind="film", graph=PPI6K, D=384, act="relu", regime=["large"], expect=["seg_reduce_kernel<3, 1,"]),
    dict(id="film_zipf_heavy_d128", kind="film", graph=PPI6K_ZIPF, D=128, normalize=True, regime=["heavy"], expect=HEAVY),
    dict(id="film_max_d36", kind="film", graph=PPI6K, D=36, agg="max", act="relu"),
    dict(id="film_restricted_d64", kind="film", graph=PPI6K_ZIPF, D=64, normalize=True, num_targets=3001),
    # Edge-MLP
    dict(id="edge_mlp_h0_source_d20", kind="edge_mlp", graph=TINY, D=20, hidden=0, use_target=False),
    dict(id="edge_mlp_h0_target_d36", kind="edge_mlp", graph=PPI6K, D=36, hidden=0, use_target=True, normalize=True),
    dict(id="edge_mlp_h1_target_d64", kind="edge_mlp", graph=PPI6K, D=64, hidden=1, use_target=True, cache=True,
         expect=["edge_build_kernel"]),
    dict(id="edge_mlp_h2_source_d100", kind="edge_mlp", graph=QM9_20K, D=100, hidden=2, use_target=False),
    dict(id="edge_mlp_h2_target_d36", kind="edge_mlp", graph=PPI6K, D=36, hidden=2, use_target=True, act="tanh",
         expect=["edge_build_kernel"]),
    # RGIN
    dict(id="rgin_aggr_mlp_d64", kind="rgin", graph=PPI6K_ZIPF, D=64, edge_hidden=1, aggr_hidden=1, use_target=True,
         cache=True, expect=["layer_norm_kernel"]),
    dict(id="rgin_raw_pairs_aggr_d36", kind="rgin", graph=PPI6K, D=36, edge_hidden=None, aggr_hidden=1, use_target=True,
         agg="mean", expect=["edge_build_kernel"]),
    dict(id="rgin_t2_d20", kind="rgin", graph=TINY, D=20, edge_hidden=1, aggr_hidden=None, use_target=False, T=2),
    # RGDCN
    dict(id="rgdcn_full_k4_d64", kind="rgdcn", graph=SMALL_ZIPF, D=64, K=4, full=True, normalize=True, cache=True),
    dict(id="rgdcn_channel_k128_d128", kind="rgdcn", graph=SMALL_ZIPF, D=128, K=128, full=False, tied=True, stddev=0.01),
    dict(id="rgdcn_max_k16_d64", kind="rgdcn", graph=SMALL_ZIPF, D=64, K=16, full=False, agg="max",
         expect=["rgdcn_edge_kernel<1, true>"]),
    dict(id="rgdcn_full_k64_d192", kind="rgdcn", graph=SMALL_ZIPF, D=192, K=64, full=True, stddev=0.01),
    # building blocks
    dict(id="dense_m1_k100_n12", kind="dense", m=1, k=100, n=12, act="tanh", cache=True),
    dict(id="dense_m129_k100_n96", kind="dense", m=129, k=100, n=96, act="relu"),
    dict(id="dense_m40000_k100_n12", kind="dense", m=40000, k=100, n=12, act="linear"),
    dict(id="dense_bwd_m0", kind="dense_backward", m=0, k=100, n=12),
    dict(id="dense_bwd_one_split", kind="dense_backward", m=300, k=1536, n=1536, cache=True, regime=["one_split"], expect=TN),
    dict(id="dense_bwd_splits", kind="dense_backward", m=4000, k=100, n=96, regime=["tn_splits"], expect=TN),
    dict(id="segment_sum_d20", kind="segment", graph=ZIPF6K, D=20, agg="sum"),
    dict(id="segment_mean_d12", kind="segment", graph=ZIPF6K, D=12, agg="mean"),
    dict(id="segment_sqrt_n_d4", kind="segment", graph=ZIPF6K, D=4, agg="sqrt_n"),
    dict(id="segment_max_empty_d36", kind="segment", graph=ZIPF6K, D=36, agg="max", regime=["isolated"]),
    dict(id="edge_agg_sum_norm_heavy_d36", kind="edge_agg", graph=ZIPF6K, D=36, normalize=True, regime=["heavy"],
         expect=["seg_reduce_heavy_kernel<"]),                # no workspace: the one-CTA heavy kernel
    dict(id="edge_agg_bwd_mean_d36", kind="edge_agg_backward", graph=ZIPF6K, D=36, agg="mean", normalize=True,
         regime=["silent_sources"]),
    dict(id="edge_agg_bwd_sum_hub_sources_d20", kind="edge_agg_backward", graph=ZIPF_SRC, D=20, regime=["heavy_sources"]),
] + [dict(id="layer_norm_d%d" % d, kind="layer_norm", rows=rows, d=d) for d, rows in
     ((8, 1001), (12, 333), (100, 4097), (128, 1000), (256, 131), (384, 77), (512, 5283))]
REGIMES = {"small", "large", "isolated", "empty_type", "pair", "heavy", "tn_splits", "one_split", "heavy_sources", "two_slabs",
           "silent_sources"}


def tn_splits(M, N, K):
    """gemm_tn_wgmma.cu tn_shape: split-K count of the weight-gradient GEMM (M x N output tiles of 128, K steps of 32)."""
    tiles = -(-M // 128) * -(-N // 128)
    steps = -(-K // 32)
    want = max(1, min(SMS // tiles, steps))
    per = -(-steps // want)
    return -(-steps // per)


def regime_holds(word, c):
    if word in ("one_split", "tn_splits"):
        if c["kind"] == "rgcn_backward":
            adj, _, V = graph(c["graph"])
            M, N, K = c.get("din", c["D"]), len(adj) * c["D"], V
        else:
            M, N, K = c["k"], c["n"], c["m"]
        return (tn_splits(M, N, K) == 1) == (word == "one_split")
    adj, _, V = graph(c["graph"])
    L, D = len(adj), c["D"]
    deg = in_degrees(adj, V)
    if word == "small":
        return V * -(-D // 128) < SMALL_BATCH
    if word == "large":
        return V * -(-D // 128) >= SMALL_BATCH
    if word == "isolated":
        return bool((deg == 0).any())
    if word == "empty_type":
        return any(a.shape[0] == 0 for a in adj)
    if word == "pair":
        return sum(a.shape[0] for a in adj) < 0.75 * V * L
    if word == "heavy":
        return bool((deg > HEAVY_SEGMENT).any())
    if word == "heavy_sources":
        return bool((segment_sizes(adj, V, "source_type") > HEAVY_SEGMENT).any())
    if word == "silent_sources":
        return bool((segment_sizes(adj, V, "source_type") == 0).any())
    if word == "two_slabs":
        return GRU_SLAB < V < 2 * GRU_SLAB
    raise ValueError(word)


def test_case_regimes():
    """Every case is in the regime it claims; every regime, family, odd row width and the MLP depths are reached."""
    reached = set()
    for c in CASES:
        for word in c.get("regime", []):
            assert regime_holds(word, c), "%s: regime '%s' does not hold" % (c["id"], word)
            reached.add(word)
        if c.get("num_targets") is not None:
            assert 0 < c["num_targets"] < graph(c["graph"])[2]
    assert reached == REGIMES, REGIMES - reached
    kinds = {c["kind"] for c in CASES}
    assert kinds == {"rgcn", "rgcn_stack", "rgcn_backward", "ggnn", "rgat", "film", "edge_mlp", "rgin", "rgdcn", "dense",
                     "dense_backward", "segment", "edge_agg", "edge_agg_backward", "layer_norm"}
    assert {4, 12, 20, 36, 100} <= {c.get("D", c.get("d")) for c in CASES}
    # one weight-cache case per family that takes a workspace
    cached = [c["kind"] for c in CASES if c.get("cache")]
    assert sorted(cached) == sorted(set(cached)) and set(cached) == kinds - {"segment", "edge_agg", "edge_agg_backward",
                                                                            "layer_norm"}
    assert {0, 1, 2} == {c["hidden"] for c in CASES if c["kind"] == "edge_mlp"}
    assert {True, False} == {c["use_target"] for c in CASES if c["kind"] == "edge_mlp"}
    assert {"sum", "mean", "sqrt_n", "max"} == {c["agg"] for c in CASES if c["kind"] == "segment"}
    assert {(1, 12), (129, 96), (40000, 12)} <= {(c["m"], c["n"]) for c in CASES if c["kind"] == "dense"}
    assert {4, 128} <= {c["K"] for c in CASES if c["kind"] == "rgdcn"}
    assert any(c["kind"] == "rgdcn" and c.get("agg") == "max" for c in CASES)
    assert any(c["kind"] == "rgcn_backward" and c.get("act") == "gelu" for c in CASES)
    # the restricted and the undersized checks reach both an RGCN and an MLP-style layer
    assert {"rgcn", "film"} <= {c["kind"] for c in CASES if c.get("num_targets")}


# ---------------------------------------------------------------- the harness --------------------------------------------
def make_plan(lib, adj, V, num_targets, dev, stream):
    import torch
    from tf_gnn_samples_b200.engine import check, ptr_table
    lists = [Guarded.copy_of("adjacency list %d" % l, t(a.astype(np.int32), dev)) for l, a in enumerate(adj)]
    handle = ctypes.c_void_p()
    counts = (ctypes.c_int64 * len(adj))(*[a.shape[0] for a in adj])
    check(lib.rgnn_plan_create(ctypes.byref(handle), V, len(adj), ptr_table([g.payload for g in lists], weights=False),
                               counts, stream))
    if num_targets is not None:
        check(lib.rgnn_plan_set_num_targets(handle, num_targets))
    return handle, lists


@pytest.fixture
def weight_cache_off():
    """The ABI calls bypass the binding's per-address weight tracking: always leave the cache off and empty."""
    from tf_gnn_samples_b200.engine import load_library
    yield
    lib = load_library()
    lib.rgnn_set_weight_cache(0)
    lib.rgnn_weight_cache_clear()


class Harness:
    def __init__(self, case, dev):
        import torch
        from tf_gnn_samples_b200 import GraphPlan
        from tf_gnn_samples_b200.engine import load_library, ptr_table
        self.case, self.dev, self.lib = case, dev, load_library()
        self.stream = torch.cuda.current_stream(dev).cuda_stream
        self.s = s = setup(case, dev)
        self.plan, self.lists, self.pyplan = None, [], None
        if s.graph is not None:
            adj, V = s.graph
            self.plan, self.lists = make_plan(self.lib, adj, V, s.num_targets, dev, self.stream)
            self.pyplan = GraphPlan(adj, V, device=dev)
            if s.num_targets is not None:
                self.pyplan.set_num_targets(s.num_targets)
        self.ins = {n: Guarded.copy_of(n, x) for n, x in s.ins.items()}
        self.saved = {n: g.payload.clone() for n, g in self.ins.items()}
        self.saved_lists = [g.payload.clone() for g in self.lists]
        self.outs = {n: Guarded(n, 4 * int(np.prod(shape)), dev) for n, shape in s.outs.items()}
        self.p = {n: g.ptr for n, g in list(self.ins.items()) + list(self.outs.items())}
        bufs = {**self.ins, **self.outs}
        self.tab = lambda names: ptr_table([bufs[n].payload for n in names], weights=False)

    def call(self, ws_ptr, nbytes):
        return self.s.call(self.lib, self.plan, self.p, self.tab, ws_ptr, nbytes, self.stream)

    def out(self, name):
        return self.outs[name].f32(self.s.outs[name])

    def message(self):
        return self.lib.rgnn_last_error().decode()

    def min_workspace(self):
        """(S_min, bound): bisection on RGNN_E_WORKSPACE over multiples of 256 bytes, in [0, the documented bound]."""
        import torch
        from tf_gnn_samples_b200.engine import check
        bound = int(self.s.bound(self.lib, self.plan))
        big = torch.empty(bound + 256, dtype=torch.uint8, device=self.dev)

        def accepted(nbytes):
            rc = self.call(big.data_ptr(), nbytes)
            if rc == E_WORKSPACE:
                return False
            check(rc)
            return True
        assert accepted(bound), "%s: the documented bound of %d bytes is refused: %s" % (self.case["id"], bound, self.message())
        lo, hi = -1, bound // 256          # refused at lo * 256 (or lo < 0), accepted at hi * 256 or at the bound
        if not accepted(hi * 256):
            hi += 1
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if accepted(mid * 256):
                hi = mid
            else:
                lo = mid
        torch.cuda.synchronize()
        return hi * 256, bound

    def check_intact(self, what):
        """(d) inputs and adjacency lists byte-identical, (e) every guard intact."""
        import torch
        torch.cuda.synchronize()
        for n, g in self.ins.items():
            assert torch.equal(g.payload, self.saved[n]), "%s (%s): input '%s' was modified" % (self.case["id"], what, n)
        for g, sv in zip(self.lists, self.saved_lists):
            assert torch.equal(g.payload, sv), "%s (%s): %s was modified" % (self.case["id"], what, g.name)
        for g in list(self.ins.values()) + list(self.outs.values()) + self.lists:
            g.check_guards()

    def run_poisoned(self, ws, nbytes, py, what):
        """(b) / (f): every workspace x output poison pattern; the result is bit-identical to `py` (rows < num_targets),
        rows >= num_targets keep the poison.  Returns the outputs of the last run."""
        import torch
        from tf_gnn_samples_b200.engine import check
        nt = self.s.num_targets
        for wbits in WS_POISON:
            for obits in OUT_POISON:
                if ws is not None:
                    ws.fill(wbits)
                for g in self.outs.values():
                    g.fill(obits)
                check(self.call(ws.ptr if ws is not None else None, nbytes))
                torch.cuda.synchronize()
                tag = "%s, workspace %08X, output %08X" % (what, wbits, obits)
                for n in self.outs:
                    got, want = self.out(n), py[n]
                    if nt is not None:
                        assert bool(poison_bits(got[nt:], obits).all().item()), "%s (%s): rows >= %d written" % (
                            self.case["id"], tag, nt)
                        got, want = got[:nt], want[:nt]
                    same = got.contiguous().view(torch.int32) == want.contiguous().view(torch.int32)
                    assert bool(same.all().item()), "%s (%s): output '%s' differs from the Python API in %d of %d words" % (
                        self.case["id"], tag, n, int((~same).sum().item()), same.numel())
                self.check_intact(tag)
        return {n: self.out(n).clone() for n in self.outs}

    def close(self):
        if self.plan is not None:
            self.lib.rgnn_plan_destroy(self.plan)
            self.plan = None
        if self.pyplan is not None:
            self.pyplan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_buffer_contract(cuda_device, weight_cache_off, case):
    """(a)-(g) of the module docstring, plus the weight-cache run for the cases marked `cache`."""
    import torch
    from tf_gnn_samples_b200.engine import check
    hs = Harness(case, cuda_device)
    try:
        py = hs.s.python(hs.pyplan)
        torch.cuda.synchronize()
        err = hs.s.oracle(py)                                                 # (c)
        takes_ws = hs.s.bound is not None
        if takes_ws:
            s_min, bound = hs.min_workspace()                                 # (a)
            print("%s: S_min %d bytes, documented bound %d bytes (%.1f%%)" % (case["id"], s_min, bound, 100.0 * s_min / bound))
            assert s_min <= bound
            ws = Guarded("workspace", s_min, cuda_device)
        else:
            s_min, ws = 0, None
        names = launched_kernels(lambda: check(hs.call(ws.ptr if ws else None, s_min)), case.get("expect", ()))
        missing = [k for k in case.get("expect", ()) if not any(k in n for n in names)]
        assert not missing, "%s: kernels %s not launched (got %s)" % (case["id"], missing, sorted(names))
        hs.check_intact("kernel listing")
        got = hs.run_poisoned(ws, s_min, py, "S_min")                        # (b), (d), (e), (f)
        print("%s: bit-identical to the Python API under every poison; vs float64 %.2e" % (case["id"], err))
        if takes_ws:                                                          # (g)
            for nbytes, null in ((s_min - 256, False), (0, False), (0, True)):
                if nbytes < 0:
                    continue
                small = None if null else Guarded("workspace of %d bytes" % nbytes, nbytes, cuda_device)
                if small is not None:
                    small.fill(WS_POISON[0])
                for g in hs.outs.values():
                    g.fill(OUT_POISON[0])
                rc = hs.call(None if null else small.ptr, nbytes)
                what = "NULL workspace" if null else "%d-byte workspace" % nbytes
                assert rc == E_WORKSPACE, "%s: %s returned %d (%s)" % (case["id"], what, rc, hs.message())
                assert "workspace too small" in hs.message(), "%s: %s: %r" % (case["id"], what, hs.message())
                hs.check_intact(what)
                if small is not None:
                    small.check_guards()
                for n in hs.outs:
                    assert bool(poison_bits(hs.out(n), OUT_POISON[0]).all().item()), "%s: %s wrote output '%s'" % (
                        case["id"], what, n)
        if case.get("cache"):
            hs.lib.rgnn_set_weight_cache(1)
            s_cached, _ = hs.min_workspace()
            print("%s: S_min with the weight cache on %d bytes (off: %d)" % (case["id"], s_cached, s_min))
            assert s_cached < s_min
            cached = hs.run_poisoned(Guarded("workspace (cache on)", s_cached, cuda_device), s_cached, got, "weight cache on")
            for n in got:
                assert torch.equal(cached[n].view(torch.int32), got[n].view(torch.int32))
            hs.lib.rgnn_set_weight_cache(0)
    finally:
        hs.close()


WIDE = [
    dict(id="edge_mlp_wide_hidden", kind="edge_mlp", graph=TINY, D=20, hidden=1, use_target=True, width=2 * 40),
    dict(id="rgin_wide_hidden", kind="rgin", graph=TINY, D=20, edge_hidden=1, aggr_hidden=None, use_target=False, width=2 * 40),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", WIDE, ids=[c["id"] for c in WIDE])
def test_mlp_wider_than_workspace_bound_is_refused(cuda_device, case):
    """rgnn_workspace_bytes sizes MLP rows by max(2 d_in, d_out); a hidden layer twice that wide is refused with
    RGNN_E_UNSUPPORTED before anything is enqueued (no launch, no output row written), even with the bound doubled."""
    from tf_gnn_samples_b200.engine import launch_count
    hs = Harness(case, cuda_device)
    try:
        bound = int(hs.s.bound(hs.lib, hs.plan))
        ws = Guarded("workspace", 2 * bound, cuda_device)
        for g in hs.outs.values():
            g.fill(OUT_POISON[0])
        before = launch_count()
        rc = hs.call(ws.ptr, 2 * bound)
        assert rc == E_UNSUPPORTED, "%s: returned %d (%s)" % (case["id"], rc, hs.message())
        assert "limit max(2 * d_in, d_out) = 40" in hs.message(), hs.message()
        assert launch_count() == before
        hs.check_intact("refused")
        ws.check_guards()
        assert bool(poison_bits(hs.out("out"), OUT_POISON[0]).all().item())
    finally:
        hs.close()

"""GPU: training RGDCN through the C ABI alone -- rgnn_rgdcn_backward, the backward of one dynamic-convolution timestep.

The library is called through ctypes with torch-allocated buffers.  The reference for every gradient (d_h and every channel
kernel dF) is float64 autograd of `sparse_rgdcn_autograd` below on the GPU: the reference's op order literally (per channel
and type: gather the [E, K, K] dynamic kernels of the edges' targets, einsum with the source slices, scale, concat, segment
reduce, activation); bench_rgdcn_training.py runs it in float32 as its comparison point.  A CPU test pins its forward to
oracle/ref_layers.sparse_rgdcn_layer.  The criterion is max-norm relative error <= 1e-4.  There is no Python training route
for RGDCN (sparse_rgdcn_layer refuses a gradient), so there is nothing else to compare against.  Covered:

  * every activation x {sum, mean, sqrt_n} x {full state, per channel} x {tied, untied} x normalisation {on, off} at
    K = 4 and K = 16 on a small graph with an empty edge type, isolated targets and duplicate edges;
  * K from 4 to 128, C = 1 (K = D = 128), D = 512 at K = 128 and K = 16, and L C > 64 (the chunked launches);
  * two timesteps as two calls with the weight gradients summed;
  * a Zipf PPI-shaped graph whose hub targets and hub (source, type) segments exceed RGNN_HEAVY_SEGMENT, on an eager and on a
    deferred plan, with a bit-identical repeat; QM9 at the RGDCN model shape (the first committed validation molecules up to
    25,000 nodes, L as the batcher gives it, D = 128, C = 8, K = 16, ELU, sum, normalised), per channel untied and full
    state tied;
  * restricted plans (num_targets < V): the gradient of the loss over the owned rows, halo rows included in d_h;
  * the buffer contract of include/rgnn.h with guard-banded buffers (test_buffer_contract_gpu.Guarded), and every refusal;
  * CUDA-graph capture and replay of forward + backward with new inputs written in place;
  * examples/c_rgdcn_train.c: compiled with -std=c99 -Wall -Wextra -Werror (no GPU needed), then linked and run;
  * sharded training from C calls alone: a 3-layer stack on virtual ranks (world 2 and 4), the INTEGRATION.md section 2c
    loop with rgnn_halo_exchange_backward, against float64 autograd on the whole graph, and a bit-identical repeat.

ReLU, leaky_relu and SELU have a derivative jump at 0, and RGDCN applies the activation twice: to every dynamic kernel's
pre-activation P and to the aggregate.  Where one of them lies within float32 rounding of 0, float32 and float64 take
different branches and no kernel can meet 1e-4.  Kinked activations therefore run on the small graph only, and a CPU test
checks that no nonzero P on a (target, type) row some edge reads, and no nonzero aggregate, lies within KINK_MARGIN of 0 for
the seeded inputs.  The larger graphs have millions of such values, some of them inevitably that close to 0, so they use
ELU (the QM9 default, whose derivative is continuous at 0), tanh or gelu.  Kernels are counted with rgnn_launch_count
deltas."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_autograd as A
from oracle import ref_layers as R
from tf_gnn_samples_b200 import weights as W
from tf_gnn_samples_b200.utils import LAYER_RGDCN, LAYER_RGDCN_BACKWARD, get_activation, get_aggregation_function

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, graph as dispatch_graph
from helpers import node_states, rel, tiny_graph

TOL = 1e-4
KINK_MARGIN = 1e-5
E_INVALID, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTS = ["linear", "tanh", "relu", "leaky_relu", "elu", "selu", "gelu"]
KINKED = ("relu", "leaky_relu", "selu")
AGGS = ["sum", "mean", "sqrt_n"]
VARIANTS = [(full, tied) for full in (True, False) for tied in (True, False)]
SMALL_SEED = 13   # seeds 1 to 12 each put a ReLU-family kink value within 1e-5 of 0 (the closest 1.4e-6); seed 13: 1.2e-5
SMALL_K = {4: 16, 16: 32}   # K -> D of the small-graph cases


# ---------------------------------------------------------------- float64 autograd of the reference ---------------------
def sparse_rgdcn_autograd(h, adjacency_lists, type_to_num_incoming_edges, num_channels=8, channel_dim=16, num_timesteps=1,
                          use_full_state_for_channel_weights=False, tie_channel_weights=False, activation_function="tanh",
                          message_aggregation_function="sum", normalize_by_num_incoming=True, *, weights):
    """gnns/rgdcn.py:116-165 in torch, same arguments as oracle/ref_layers.sparse_rgdcn_layer; tensors stay on their device."""
    import torch
    adj = [torch.as_tensor(a).reshape(-1, 2).long().to(h.device) for a in adjacency_lists]
    act, V = A.get_activation(activation_function), h.shape[0]
    targets = torch.cat([a[:, 1] for a in adj])
    cnt = type_to_num_incoming_edges
    C, K = num_channels, channel_dim
    cur = h
    for _ in range(num_timesteps):                                             # :116
        chunked = cur.reshape(-1, C, K)                                        # :117-118
        new_chunks = []
        for c in range(C):                                                     # :121
            chan = chunked[:, c, :]
            per_type = []
            for l, a in enumerate(adj):                                        # :126
                src, tgt = a[:, 0], a[:, 1]
                inp = cur if use_full_state_for_channel_weights else chan      # :133-136
                kernel = weights["channel_weights"][l][0 if tie_channel_weights else c]
                ew = act(inp @ kernel).reshape(-1, K, K)                       # :139-141 (the Dense carries the activation)
                msgs = torch.einsum("vi,vij->vj", chan[src], ew[tgt])          # :142-146
                if normalize_by_num_incoming:                                  # :147-151
                    msgs = (1.0 / (cnt[l][tgt] + A.SMALL_NUMBER)).unsqueeze(-1) * msgs
                per_type.append(msgs)
            agg = A.segment_reduce(torch.cat(per_type), targets, V, message_aggregation_function)   # :155-159
            new_chunks.append(act(agg))                                        # :160
        cur = torch.cat(new_chunks, dim=1)                                     # :164-165
    return cur


# ---------------------------------------------------------------- graphs -------------------------------------------------
def tiny():
    adj, _ = tiny_graph()
    return adj, 37


def zipf_ppi():
    adj, _, V = dispatch_graph(PPI6K_ZIPF)
    return adj, V


def qm9_rgdcn():
    """The first committed QM9 validation molecules up to 25,000 nodes (RGDCN's max_nodes_in_batch), as the batcher packs them."""
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), max_nodes_per_batch=25000)
    return b.adjacency_lists, b.num_nodes


def in_degrees(adj, V):
    return np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)


def type_counts(adj, V):
    return np.stack([np.bincount(a[:, 1], minlength=V) for a in adj]).astype(np.float32)


def make_weights(L, C, K, full, tied, seed):
    """rgdcn_weights with stddev 1 / sqrt(rows): the dynamic kernels' pre-activations are O(1), so every activation bends."""
    return W.rgdcn_weights(L, C, K, full, tied, seed=seed + 11, stddev=1.0 / math.sqrt(C * K if full else K))


# ---------------------------------------------------------------- one case -----------------------------------------------
class Case:
    """Inputs of one RGDCN layer on the device and the ctypes call of rgnn_rgdcn_backward."""

    def __init__(self, adj, V, D, K, act="elu", agg="sum", full=False, tied=False, normalize=True, seed=SMALL_SEED,
                 num_targets=None, T=1, device=None, deferred=False):
        import torch
        from tf_gnn_samples_b200 import GraphPlan
        self.adj, self.V, self.D, self.K, self.C, self.T = adj, V, D, K, D // K, T
        self.full, self.tied, self.normalize = full, tied, normalize
        self.act_name, self.act = act, get_activation(act)
        self.agg_name, self.agg = agg, get_aggregation_function(agg)
        self.L = len(adj)
        self.dev = device
        self.w = make_weights(self.L, self.C, K, full, tied, seed)
        self.h = node_states(V, D, seed=seed)
        self.cnt = type_counts(adj, V)
        self.plan = GraphPlan(adj, V, device=device, validate=not deferred)   # deferred: heavy counts stay on the device
        self.Vt = V if num_targets is None else num_targets
        if num_targets is not None:
            self.plan.set_num_targets(num_targets)
        self.g = np.random.default_rng(seed + 1).standard_normal((self.Vt, D)).astype(np.float32)
        t = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(device)
        self.th, self.tg, self.tcnt = t(self.h), t(self.g), t(self.cnt)
        self.tw = [[t(k) for k in ks] for ks in self.w["channel_weights"]]
        self.rows = D if full else K

    def table(self, per_type):
        """L x C' tensors -> the host table of L * C pointers (tied: the type's pointer C times)."""
        ptrs = [x if x is None or isinstance(x, int) else x.data_ptr() for ks in per_type for x in (ks * self.C if self.tied else ks)]
        return (ctypes.c_void_p * len(ptrs))(*ptrs)

    @property
    def lib(self):
        from tf_gnn_samples_b200.engine import load_library
        return load_library()

    def ws_bytes(self):
        return int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGDCN_BACKWARD, self.D, self.D, self.K))

    def new_outputs(self):
        import torch
        z = lambda s: torch.empty(s, dtype=torch.float32, device=self.dev)
        return {"gh": z((self.V, self.D)), "gw": [[z((self.rows, self.K * self.K)) for _ in ks] for ks in self.tw]}

    def call(self, outs, h_t=None, g_t=None, ws="own", nbytes=None, stream=None, **over):
        """rgnn_rgdcn_backward; `over` replaces raw arguments (pointers / ints / tables).  ws="own": a workspace of the
        documented size from torch; otherwise the pointer (or None) and nbytes are passed as they are."""
        import torch
        ptr = lambda x: x if x is None or isinstance(x, int) else x.data_ptr()
        if isinstance(ws, str):
            nbytes = self.ws_bytes()
            ws_t = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=self.dev)   # freed stream-ordered after the call
            ws = ws_t.data_ptr()
        if stream is None:
            stream = torch.cuda.current_stream(self.dev).cuda_stream
        a = dict(plan=self.plan.handle, h=ptr(self.th if h_t is None else h_t), d=self.D, C=self.C, w=self.table(self.tw),
                 full=int(self.full), tied=int(self.tied), cnt=ptr(self.tcnt), act=self.act, agg=self.agg,
                 norm=int(self.normalize), g=ptr(self.tg if g_t is None else g_t), gh=ptr(outs.get("gh")),
                 gw=self.table(outs["gw"]) if outs.get("gw") is not None else None)
        a.update(over)
        return self.lib.rgnn_rgdcn_backward(a["plan"], a["h"], a["d"], a["C"], a["w"], a["full"], a["tied"], a["cnt"], a["act"],
                                            a["agg"], a["norm"], a["g"], a["gh"], a["gw"], ws, nbytes, stream)

    def forward(self, h, out=None, ws=None):
        """One timestep through rgnn_rgdcn_forward."""
        import torch
        from tf_gnn_samples_b200.engine import check
        if out is None:
            out = torch.zeros((self.V, self.D), dtype=torch.float32, device=self.dev)
        nb = int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGDCN, self.D, self.D, self.K))
        if ws is None:
            ws = torch.empty(max(nb, 256), dtype=torch.uint8, device=self.dev)
        check(self.lib.rgnn_rgdcn_forward(self.plan.handle, h.data_ptr(), self.D, self.C, self.table(self.tw), int(self.full),
                                          self.tcnt.data_ptr(), self.act, self.agg, int(self.normalize), 1, out.data_ptr(),
                                          ws.data_ptr(), nb, torch.cuda.current_stream(self.dev).cuda_stream))
        return out

    def grads(self):
        """All gradients of the T timesteps through the C ABI: forward per timestep, backward from the last one down."""
        import torch
        from tf_gnn_samples_b200.engine import check
        xs = [self.th]
        for _ in range(self.T - 1):
            xs.append(self.forward(xs[-1]))
        g = self.tg
        res = {}
        for t in reversed(range(self.T)):
            o = self.new_outputs()
            check(self.call(o, h_t=xs[t], g_t=g))
            g = o["gh"]
            for l, ks in enumerate(o["gw"]):
                for c, k in enumerate(ks):
                    key = "d_F%d_%d" % (l, c)
                    res[key] = res.get(key, 0) + k.double()
        res["d_h"] = g
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in res.items()}

    def oracle(self):
        """float64 autograd on the GPU: d/d(h, every kernel) of sum(out[:Vt] * g)."""
        import torch
        f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, device=self.dev, requires_grad=True)
        h = f64(self.h)
        w = {"channel_weights": [[f64(k) for k in ks] for ks in self.w["channel_weights"]]}
        cnt = torch.tensor(self.cnt, dtype=torch.float64, device=self.dev)
        with torch.device(self.dev):
            out = sparse_rgdcn_autograd(h, self.adj, cnt, self.C, self.K, self.T, self.full, self.tied, self.act_name,
                                        self.agg_name, self.normalize, weights=w)
            (out[: self.Vt] * torch.tensor(self.g, dtype=torch.float64)).sum().backward()
        res = {"d_h": h.grad.cpu().numpy()}
        for l, ks in enumerate(w["channel_weights"]):
            for c, k in enumerate(ks):
                res["d_F%d_%d" % (l, c)] = k.grad.cpu().numpy() if k.grad is not None else np.zeros(tuple(k.shape))
        return res


def check_case(c, what):
    got, want = c.grads(), c.oracle()
    errs = {k: rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    print("%s: max rel err vs float64 %.3e (%s)" % (what, errs[worst], worst))
    bad = {k: e for k, e in errs.items() if not e <= TOL}
    assert not bad, "%s: %s" % (what, bad)
    return got


def variant_name(full, tied, normalize):
    return "%s %s %s" % ("full" if full else "channel", "tied" if tied else "untied", "norm" if normalize else "raw")


# ---------------------------------------------------------------- CPU checks ---------------------------------------------
def test_case_regimes():
    """The small graph has an empty edge type, isolated targets and duplicate edges; the Zipf graph has hub targets and hub
    (source, type) segments above the heavy threshold."""
    adj, V = tiny()
    assert any(a.shape[0] == 0 for a in adj)
    assert (in_degrees(adj, V) == 0).any()
    assert any(len(np.unique(a, axis=0)) < len(a) for a in adj if len(a))
    adj, V = zipf_ppi()
    assert in_degrees(adj, V).max() > HEAVY_SEGMENT
    assert max(np.bincount(a[:, 0], minlength=V).max() for a in adj) > HEAVY_SEGMENT


@pytest.mark.parametrize("agg", ["sum", "mean", "sqrt_n", "max"])
@pytest.mark.parametrize("full,tied", VARIANTS, ids=["full_tied", "full_untied", "channel_tied", "channel_untied"])
def test_autograd_oracle_forward_equals_ref_layers(full, tied, agg):
    """The float64 torch restatement computes what oracle/ref_layers.sparse_rgdcn_layer computes, to 1e-12, over two
    timesteps, with and without normalisation."""
    import torch
    adj, V = tiny()
    K, D = 4, 16
    C = D // K
    w = make_weights(len(adj), C, K, full, tied, 3)
    h = node_states(V, D, seed=3)
    cnt = type_counts(adj, V)
    for normalize in (True, False):
        want = R.sparse_rgdcn_layer(h, adj, cnt, C, K, 2, full, tied, "tanh", agg, normalize, weights=w)
        w64 = {"channel_weights": [[torch.tensor(k, dtype=torch.float64) for k in ks] for ks in w["channel_weights"]]}
        got = sparse_rgdcn_autograd(torch.tensor(h, dtype=torch.float64), adj, torch.tensor(cnt, dtype=torch.float64), C, K, 2,
                                    full, tied, "tanh", agg, normalize, weights=w64).numpy()
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), (normalize, np.abs(got - want).max())


@pytest.mark.parametrize("full,tied", VARIANTS, ids=["full_tied", "full_untied", "channel_tied", "channel_untied"])
def test_autograd_oracle_gradcheck(full, tied):
    """torch.autograd.gradcheck of the float64 restatement on a tiny case of each variant (tanh, mean, normalised)."""
    import torch
    adj = [np.array([[0, 1], [2, 1], [3, 0]], np.int32), np.array([[1, 2], [1, 2]], np.int32)]
    V, K, C = 4, 4, 2
    w = make_weights(2, C, K, full, tied, 5)
    cnt = torch.tensor(type_counts(adj, V), dtype=torch.float64)
    h = torch.tensor(node_states(V, C * K, seed=5), dtype=torch.float64, requires_grad=True)
    ks = [torch.tensor(k, dtype=torch.float64, requires_grad=True) for kk in w["channel_weights"] for k in kk]
    per = 1 if tied else C

    def f(h, *flat):
        wt = {"channel_weights": [list(flat[l * per:(l + 1) * per]) for l in range(2)]}
        return sparse_rgdcn_autograd(h, adj, cnt, C, K, 1, full, tied, "tanh", "mean", True, weights=wt)

    assert torch.autograd.gradcheck(f, (h, *ks), eps=1e-6, atol=1e-7)


def kink_values(adj, V, D, K, full, tied, normalize, act, agg, seed, T=1):
    """Every value a kink can act on, float64 in the reference's op order over T timesteps: P = x . F on each (target, type)
    row some edge reads, and the aggregate before the output activation; exact zeros dropped."""
    import torch
    C, L = D // K, len(adj)
    w = make_weights(L, C, K, full, tied, seed)
    f = A.get_activation(act)
    cnt = torch.tensor(type_counts(adj, V), dtype=torch.float64)
    cur = torch.tensor(node_states(V, D, seed=seed), dtype=torch.float64)
    targets = torch.cat([torch.as_tensor(a[:, 1]).long() for a in adj])
    out = []
    for _ in range(T):
        chunked = cur.reshape(-1, C, K)
        new = []
        for c in range(C):
            per_type = []
            for l, a in enumerate(adj):
                src, tgt = torch.as_tensor(a[:, 0]).long(), torch.as_tensor(a[:, 1]).long()
                inp = cur if full else chunked[:, c, :]
                p = inp @ torch.tensor(w["channel_weights"][l][0 if tied else c], dtype=torch.float64)
                out.append(p[torch.unique(tgt)].reshape(-1))
                m = torch.einsum("vi,vij->vj", chunked[:, c, :][src], f(p).reshape(-1, K, K)[tgt])
                if normalize:
                    m = (1.0 / (cnt[l][tgt] + A.SMALL_NUMBER)).unsqueeze(-1) * m
                per_type.append(m)
            agg_v = A.segment_reduce(torch.cat(per_type), targets, V, agg)
            out.append(agg_v.reshape(-1))
            new.append(f(agg_v))
        cur = torch.cat(new, dim=1)
    x = torch.cat(out).numpy()
    return x[x != 0.0]


def kinked_cases():
    """(K, act, agg, full, tied, normalize, T, num_targets) of every GPU case on the small graph with a kinked activation."""
    cases = [(K, act, agg, full, tied, norm, 1) for K in SMALL_K for act in KINKED for agg in AGGS for full, tied in VARIANTS
             for norm in (True, False)]
    cases += [(4, "relu", "sum", full, tied, True, 2) for full, tied in VARIANTS]        # two timesteps
    cases += [(4, "relu", "mean", full, tied, True, 1) for full, tied in VARIANTS]       # restricted plans (same values)
    return cases


def test_no_value_at_a_kink():
    """float64 on the seeded inputs of every small-graph case with a kinked activation: no nonzero dynamic-kernel
    pre-activation on a row some edge reads and no nonzero aggregate lies within KINK_MARGIN of 0."""
    adj, V = tiny()
    closest = np.inf
    for K, act, agg, full, tied, norm, T in kinked_cases():
        x = kink_values(adj, V, SMALL_K[K], K, full, tied, norm, act, agg, SMALL_SEED, T)
        d = float(np.abs(x).min()) if x.size else np.inf
        assert d > KINK_MARGIN, (K, act, agg, full, tied, norm, T, d)
        closest = min(closest, d)
    print("small graph, kinked activations: closest nonzero value to 0 is %.2e" % closest)


def documented_bound(V, Vt, L, d, K):
    """The workspace bound include/rgnn.h states for rgnn_rgdcn_backward, in bytes."""
    C = d // K
    Q = min(L * C, 64) * K * K
    floats = Vt * L * d * K + 2 * V * L * d + Vt * d + Vt * L * K * K + d * Q + 2 * (Q + 128) * (d + 128) + 2163712
    fwd = 2 * (4 * d + 64) * (4 * L * d + 4 * d + 512)
    return (floats + fwd) * 4 + 8192


def test_documented_workspace_bound_has_no_edge_term():
    """The header's formula names V, Vt, L, d and K only; evaluated for equal V and L it is the same for any M."""
    text = open(os.path.join(ROOT, "include", "rgnn.h")).read()
    start = text.index("Workspace: rgnn_workspace_bytes(plan, RGNN_LAYER_RGDCN_BACKWARD")
    formula = text[start:text.index("*/", start)]
    assert "(Vt L d K + 2 V L d + Vt d + Vt L K^2 + d Q + 2 (Q + 128)(d + 128) + 2163712) floats" in formula
    assert " M " not in formula and "M)" not in formula and "num_edges" not in formula
    assert documented_bound(1000, 1000, 4, 128, 16) == documented_bound(1000, 1000, 4, 128, 16)


# ---------------------------------------------------------------- parity -------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", sorted(SMALL_K))
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("act", ACTS)
def test_small_graph_matches_float64_autograd(cuda_device, act, agg, K):
    """Every variant and normalisation of one (activation, aggregation, K) on the small graph."""
    adj, V = tiny()
    for full, tied in VARIANTS:
        for norm in (True, False):
            check_case(Case(adj, V, SMALL_K[K], K, act, agg, full, tied, norm, device=cuda_device),
                       "tiny K=%d %s %s %s" % (K, act, agg, variant_name(full, tied, norm)))


K_SWEEP = [  # (D, K, L, full, tied, act): K from 4 to 128, C = 1, D = 512, L C > 64
    (32, 4, 4, True, False, "tanh"), (64, 8, 4, False, False, "elu"), (128, 32, 4, True, True, "gelu"),
    (128, 64, 4, False, True, "tanh"), (128, 128, 4, False, False, "elu"), (128, 128, 4, True, False, "gelu"),
    (512, 128, 2, False, False, "elu"), (512, 128, 2, True, True, "tanh"), (512, 16, 4, False, False, "gelu"),
    (512, 16, 4, True, False, "elu"), (128, 8, 5, True, False, "tanh"), (128, 8, 5, False, True, "elu")]


def typed_graph(L, V=300, E=900, seed=7):
    """A random multigraph with L edge types (the small graph's edge cases plus many types for L C > 64)."""
    rng = np.random.default_rng(seed)
    return [np.stack([rng.integers(0, V, E // L), rng.integers(0, V - 5, E // L)], 1).astype(np.int32) for _ in range(L)], V


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,L,full,tied,act", K_SWEEP, ids=["D%d_K%d_L%d_%s_%s" % (D, K, L, "full" if f else "channel",
                                                                                       "tied" if t else "untied")
                                                               for D, K, L, f, t, _ in K_SWEEP])
def test_channel_dim_sweep(cuda_device, D, K, L, full, tied, act):
    """K = 4 ... 128 (C = 1 at K = D = 128), D = 512 at K = 128 and K = 16, and L C = 128 and 80 > 64 (two chunks of kernels
    per launch in the full-state case)."""
    adj, V = typed_graph(L)
    if K == 128 and D == 512:
        adj, V = typed_graph(L, V=120, E=360)   # the oracle's [E, K, K] tensors: 360 edges x 128^2 x 8 B per (type, channel)
    check_case(Case(adj, V, D, K, act, "mean", full, tied, True, device=cuda_device),
               "D=%d K=%d L=%d C=%d %s %s" % (D, K, L, D // K, act, variant_name(full, tied, True)))


@pytest.mark.gpu
@pytest.mark.parametrize("full,tied", VARIANTS, ids=["full_tied", "full_untied", "channel_tied", "channel_untied"])
def test_two_timesteps_as_two_calls(cuda_device, full, tied):
    adj, V = tiny()
    check_case(Case(adj, V, 16, 4, "relu", "sum", full, tied, True, T=2, device=cuda_device),
               "tiny two timesteps %s" % variant_name(full, tied, True))


def zipf_case(dev, full, tied, deferred=False, **kw):
    adj, V = zipf_ppi()
    return Case(adj, V, 64, 8, kw.pop("act", "elu"), kw.pop("agg", "mean"), full, tied, True, deferred=deferred, device=dev, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("full,tied", [(False, False), (True, True)], ids=["channel_untied", "full_tied"])
def test_zipf_heavy_targets_and_sources_and_determinism(cuda_device, full, tied):
    """The Zipf PPI-shaped graph at D = 64, K = 8 (the oracle's [E, K, K] tensors stay near 0.5 GB per channel): heavy
    targets and heavy (source, type) segments; two calls are bit-identical."""
    import torch
    from tf_gnn_samples_b200.engine import check, launch_count
    c = zipf_case(cuda_device, full, tied)
    got = check_case(c, "zipf ppi D=64 K=8 elu mean %s" % variant_name(full, tied, True))
    o1, o2 = c.new_outputs(), c.new_outputs()
    before = launch_count()
    check(c.call(o1))
    n1 = launch_count() - before
    check(c.call(o2))
    torch.cuda.synchronize()
    assert n1 == launch_count() - before - n1
    print("zipf ppi %s: %d kernel launches per backward" % (variant_name(full, tied, True), n1))
    assert torch.equal(o1["gh"], o2["gh"])
    assert all(torch.equal(a, b) for ka, kb in zip(o1["gw"], o2["gw"]) for a, b in zip(ka, kb))
    assert np.array_equal(o1["gh"].cpu().numpy(), got["d_h"])


@pytest.mark.gpu
@pytest.mark.parametrize("full,tied", [(False, True), (True, False)], ids=["channel_tied", "full_untied"])
def test_deferred_plan(cuda_device, full, tied):
    """A plan built without a synchronisation (RGNN_PLAN_DEFERRED_CHECK) never read its heavy counts back."""
    check_case(zipf_case(cuda_device, full, tied, deferred=True, act="tanh", agg="sqrt_n"),
               "zipf ppi deferred plan tanh sqrt_n %s" % variant_name(full, tied, True))


@pytest.mark.gpu
@pytest.mark.parametrize("full,tied", [(False, False), (True, True)], ids=["channel_untied", "full_tied"])
def test_qm9_rgdcn_model_shape(cuda_device, full, tied):
    """QM9 at RGDCN's model shape: up to 25,000 nodes of the committed validation molecules, D = 128, C = 8, K = 16, ELU,
    sum, normalised."""
    adj, V = qm9_rgdcn()
    assert 24000 < V <= 25000
    check_case(Case(adj, V, 128, 16, "elu", "sum", full, tied, True, device=cuda_device),
               "qm9 V=%d M=%d L=%d D=128 K=16 %s" % (V, sum(a.shape[0] for a in adj), len(adj), variant_name(full, tied, True)))


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,full,tied", [("tiny", True, False), ("tiny", False, True), ("zipf", False, False),
                                                  ("zipf", True, True)])
def test_restricted_plan(cuda_device, graph_name, full, tied):
    """num_targets < V: the gradient of the loss over the owned rows; the halo rows of d_h receive theirs."""
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    nt = V * 2 // 3
    if graph_name == "tiny":
        c = Case(adj, V, 16, 4, "relu", "mean", full, tied, True, num_targets=nt, device=cuda_device)
    else:
        c = zipf_case(cuda_device, full, tied, num_targets=nt)
    got = check_case(c, "%s %s restricted to %d of %d targets" % (graph_name, variant_name(full, tied, True), nt, V))
    assert np.abs(got["d_h"][nt:]).max() > 0


# ---------------------------------------------------------------- buffer contract ----------------------------------------
def guarded_case(c):
    """Guarded copies of the inputs and guarded outputs; returns (inputs, outputs)."""
    from test_buffer_contract_gpu import Guarded
    ins = {"h": Guarded.copy_of("h", c.th), "g": Guarded.copy_of("g", c.tg), "cnt": Guarded.copy_of("cnt", c.tcnt)}
    ins.update({"w%d_%d" % (l, i): Guarded.copy_of("w%d_%d" % (l, i), x) for l, ks in enumerate(c.tw) for i, x in enumerate(ks)})
    outs = {"gh": Guarded("gh", c.V * c.D * 4, c.dev)}
    outs.update({"gw%d_%d" % (l, i): Guarded("gw%d_%d" % (l, i), c.rows * c.K * c.K * 4, c.dev)
                 for l, ks in enumerate(c.tw) for i, _ in enumerate(ks)})
    return ins, outs


def guarded_call(c, ins, outs, ws_ptr, nbytes, drop=(), **over):
    import torch
    per = 1 if c.tied else c.C
    tab = lambda pre, d: c.table([[d["%s%d_%d" % (pre, l, i)].ptr for i in range(per)] for l in range(c.L)])
    p = dict(h=ins["h"].ptr, g=ins["g"].ptr, cnt=ins["cnt"].ptr, w=tab("w", ins), gh=outs["gh"].ptr, gw=tab("gw", outs))
    for k in drop:
        p[k] = None
    p.update(over)
    return c.call({"gw": None}, ws=ws_ptr, nbytes=nbytes, stream=torch.cuda.current_stream(c.dev).cuda_stream, **p)


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,full,tied", [("tiny", False, False), ("tiny", True, True), ("zipf", True, False),
                                                  ("zipf", False, True)])
def test_buffer_contract(cuda_device, graph_name, full, tied):
    import torch
    from test_buffer_contract_gpu import Guarded, OUT_POISON, WS_POISON, poison_bits
    from tf_gnn_samples_b200.engine import launch_count
    if graph_name == "tiny":
        adj, V = tiny()
        c = Case(adj, V, 16, 4, "tanh", "mean", full, tied, True, device=cuda_device)
    else:
        c = zipf_case(cuda_device, full, tied, act="tanh")
    D = c.D
    ins, outs = guarded_case(c)
    snap = {k: g.payload.clone() for k, g in ins.items()}
    bound = c.ws_bytes()
    assert bound == documented_bound(c.V, c.Vt, c.L, D, c.K)
    big = Guarded("ws", bound, cuda_device)
    # the first call builds the reverse index; then bisect the smallest accepted workspace
    assert guarded_call(c, ins, outs, big.ptr, bound) == 0
    lo, hi = 0, bound
    while lo < hi:
        mid = (lo + hi) // 2
        rc = guarded_call(c, ins, outs, big.ptr, mid)
        assert rc in (0, E_WORKSPACE), rc
        lo, hi = (lo, mid) if rc == 0 else (mid + 1, hi)
    s_min = lo
    what = "%s %s" % (graph_name, variant_name(full, tied, True))
    print("%s: S_min = %d bytes = %.1f%% of the documented bound %d" % (what, s_min, 100.0 * s_min / bound, bound))
    assert 0 < s_min <= bound
    ref = None
    for wp in WS_POISON:
        for op in OUT_POISON:
            ws = Guarded("ws", s_min, cuda_device)
            ws.fill(wp)
            for g in outs.values():
                g.fill(op)
            assert guarded_call(c, ins, outs, ws.ptr, s_min) == 0
            torch.cuda.synchronize()
            got = {k: g.payload.clone() for k, g in outs.items()}
            if ref is None:
                ref = got
                want = c.grads()                          # the same call on torch buffers
                assert np.array_equal(outs["gh"].f32((c.V, D)).cpu().numpy(), want["d_h"])
                assert np.array_equal(outs["gw0_0"].f32((c.rows, c.K * c.K)).cpu().numpy(), want["d_F0_0"].astype(np.float32))
            for k in got:
                assert torch.equal(got[k], ref[k]), "%s differs under poison %x / %x" % (k, wp, op)
            ws.check_guards()
    for k, g in ins.items():
        assert torch.equal(g.payload, snap[k]), "input %s changed" % k
        g.check_guards()
    for g in outs.values():
        g.check_guards()
    # short, empty and NULL workspaces: RGNN_E_WORKSPACE, no output written, nothing enqueued
    for nb, ptr in ((s_min - 256, "ws"), (0, "ws"), (0, None)):
        ws = Guarded("ws", max(s_min - 256, 16), cuda_device)
        for g in outs.values():
            g.fill(OUT_POISON[0])
        before = launch_count()
        assert guarded_call(c, ins, outs, ws.ptr if ptr else None, nb) == E_WORKSPACE
        assert launch_count() == before
        torch.cuda.synchronize()
        for k, g in outs.items():
            assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[0]).all()), "%s written by a refused call" % k
            g.check_guards()
        ws.check_guards()
    # NULL optional outputs are accepted, and what is asked for is unchanged
    ws = Guarded("ws", bound, cuda_device)
    for drop in (("gh",), ("gw",), ("gh", "gw")):
        for g in outs.values():
            g.fill(OUT_POISON[1])
        assert guarded_call(c, ins, outs, ws.ptr, bound, drop=drop) == 0
        torch.cuda.synchronize()
        for k, g in outs.items():
            base = k.rstrip("0123456789_")
            if base in drop:
                assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[1]).all()), k
            else:
                assert torch.equal(g.payload, ref[k]), (drop, k)
    # refusals: each names its argument, enqueues nothing and writes nothing
    n = c.L * c.C
    wtab = lambda ptrs: (ctypes.c_void_p * n)(*ptrs)
    w_ptrs = [ins["w%d_%d" % (i // c.C, 0 if tied else i % c.C)].ptr for i in range(n)]
    gw_ptrs = [outs["gw%d_%d" % (i // c.C, 0 if tied else i % c.C)].ptr for i in range(n)]
    refusals = [("aggregation", dict(agg=1), E_UNSUPPORTED), ("aggregation", dict(agg=9), E_INVALID),
                ("activation", dict(act=99), E_INVALID), ("channel_dim 2", dict(C=D // 2), E_INVALID),
                ("num_channels 3", dict(C=3), E_INVALID), ("state dim d = 516", dict(d=516), E_UNSUPPORTED),
                ("plan", dict(plan=None), E_INVALID), ("node_embeddings", dict(h=None), E_INVALID),
                ("grad_out", dict(g=None), E_INVALID), ("channel_weights", dict(w=None), E_INVALID),
                ("num_incoming", dict(cnt=None), E_INVALID), ("node_embeddings", dict(h=ins["h"].ptr + 4), E_INVALID),
                ("grad_node_embeddings", dict(gh=outs["gh"].ptr + 4), E_INVALID),
                ("grad_node_embeddings must not alias", dict(gh=ins["h"].ptr), E_INVALID),
                ("grad_node_embeddings must not alias", dict(gh=ins["g"].ptr), E_INVALID),
                ("channel weight 0", dict(w=wtab([None] + w_ptrs[1:])), E_INVALID),
                ("channel weight 0", dict(w=wtab([w_ptrs[0] + 4] + w_ptrs[1:])), E_INVALID),
                ("grad channel weight 0", dict(gw=wtab([gw_ptrs[0] + 4] + gw_ptrs[1:])), E_INVALID)]
    if tied:
        refusals += [("tie_channel_weights", dict(w=wtab(w_ptrs[:1] + [ins["h"].ptr] + w_ptrs[2:])), E_INVALID),
                     ("tie_channel_weights", dict(gw=wtab(gw_ptrs[:1] + [outs["gh"].ptr] + gw_ptrs[2:])), E_INVALID),
                     ("grad_channel_weights[0] and grad_channel_weights[%d] alias" % c.C,
                      dict(gw=wtab(gw_ptrs[:c.C] + gw_ptrs[:c.C] + gw_ptrs[2 * c.C:])), E_INVALID)]
    else:
        refusals += [("tie_channel_weights", dict(tied=1), E_INVALID),
                     ("grad_channel_weights[0] and grad_channel_weights[1] alias", dict(gw=wtab(gw_ptrs[:1] * 2 + gw_ptrs[2:])),
                      E_INVALID)]
    for name, over, code in refusals:
        for g in outs.values():
            g.fill(OUT_POISON[0])
        before = launch_count()
        rc = guarded_call(c, ins, outs, ws.ptr, bound, **over)
        msg = c.lib.rgnn_last_error()
        msg = msg.decode() if isinstance(msg, bytes) else str(msg)
        print("refused %-55s %s" % (name, msg))
        assert rc == code, (name, rc, msg)
        assert name in msg, (name, msg)
        assert launch_count() == before, name
        torch.cuda.synchronize()
        for k, g in outs.items():
            assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[0]).all()), (name, k)


@pytest.mark.gpu
def test_workspace_bound_has_no_edge_term(cuda_device):
    """Two graphs with the same V and L and different M: the same bound."""
    from tf_gnn_samples_b200 import GraphPlan
    from tf_gnn_samples_b200.engine import load_library
    lib = load_library()
    a, V = typed_graph(4, V=500, E=800)
    b, _ = typed_graph(4, V=500, E=8000, seed=8)
    plans = [GraphPlan(x, V, device=cuda_device) for x in (a, b)]
    got = [int(lib.rgnn_workspace_bytes(p.handle, LAYER_RGDCN_BACKWARD, 128, 128, 16)) for p in plans]
    assert got[0] == got[1] == documented_bound(V, V, 4, 128, 16)


# ---------------------------------------------------------------- CUDA graph ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("full,tied", [(False, False), (True, True)], ids=["channel_untied", "full_tied"])
def test_cuda_graph_replay_of_forward_and_backward(cuda_device, full, tied):
    import torch
    from tf_gnn_samples_b200.engine import check
    c = zipf_case(cuda_device, full, tied, act="gelu")
    cap = c.new_outputs()
    y_cap = torch.empty((c.V, c.D), dtype=torch.float32, device=cuda_device)
    nb_f = int(c.lib.rgnn_workspace_bytes(c.plan.handle, LAYER_RGDCN, c.D, c.D, c.K))
    ws_f = torch.empty(nb_f, dtype=torch.uint8, device=cuda_device)
    c.forward(c.th, y_cap, ws_f)
    check(c.call(cap))                                    # eager first: builds the reverse index
    nbytes = c.ws_bytes()
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda_device)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.forward(c.th, y_cap, ws_f)
        rc = c.call(cap, ws=ws.data_ptr(), nbytes=nbytes)
    assert rc == 0
    rng = np.random.default_rng(77)
    c.th.copy_(torch.as_tensor(np.tanh(rng.standard_normal(tuple(c.th.shape))).astype(np.float32)))
    c.tg.copy_(torch.as_tensor(rng.standard_normal(tuple(c.tg.shape)).astype(np.float32)))
    for ks in c.tw:
        for x in ks:
            x.mul_(0.75)
    graph.replay()
    torch.cuda.synchronize()
    eager = c.new_outputs()
    y_eager = c.forward(c.th)
    check(c.call(eager))
    torch.cuda.synchronize()
    assert torch.equal(y_cap, y_eager)
    assert torch.equal(cap["gh"], eager["gh"])
    assert all(torch.equal(a, b) for ka, kb in zip(cap["gw"], eager["gw"]) for a, b in zip(ka, kb))
    c.h, c.g = c.th.cpu().numpy(), c.tg.cpu().numpy()
    c.w["channel_weights"] = [[x.cpu().numpy() for x in ks] for ks in c.tw]
    want = c.oracle()
    assert rel(cap["gh"].cpu().numpy(), want["d_h"]) <= TOL
    assert rel(cap["gw"][0][0].cpu().numpy(), want["d_F0_0"]) <= TOL
    # a first backward on a fresh plan refuses under capture, recording nothing
    fresh = zipf_case(cuda_device, full, tied, act="gelu")
    x = torch.zeros(4, device=cuda_device)
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        rc = fresh.call(fresh.new_outputs(), ws=ws.data_ptr(), nbytes=nbytes)
        x.add_(1.0)
    assert rc == E_INVALID
    g2.replay()
    torch.cuda.synchronize()
    assert x[0].item() == 1.0


# ---------------------------------------------------------------- the C host ---------------------------------------------
EXAMPLE = os.path.join(ROOT, "examples", "c_rgdcn_train.c")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def compile_example(out_dir, link):
    gcc = shutil.which("gcc")
    if gcc is None or not os.path.exists(os.path.join(CUDA_HOME, "include", "cuda_runtime.h")):
        pytest.skip("needs gcc and the CUDA runtime headers")
    from tf_gnn_samples_b200 import _build
    cmd = [gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-O2", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(CUDA_HOME, "include"), EXAMPLE]
    if link:
        lib_dir = os.path.dirname(_build.LIB_PATH)
        exe = os.path.join(out_dir, "c_rgdcn_train")
        cmd += ["-o", exe, "-L", lib_dir, "-lrgnn", "-Wl,-rpath," + lib_dir, "-L", os.path.join(CUDA_HOME, "lib64"), "-lcudart",
                "-Wl,-rpath," + os.path.join(CUDA_HOME, "lib64"), "-lm"]
    else:
        exe = os.path.join(out_dir, "c_rgdcn_train.o")
        cmd += ["-c", "-o", exe]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return exe


def test_c_example_compiles_as_c99(tmp_path):
    compile_example(str(tmp_path), link=False)


@pytest.mark.gpu
def test_c_example_trains(tmp_path):
    """The C host's losses decrease."""
    exe = compile_example(str(tmp_path), link=True)
    res = subprocess.run([exe, "6"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    losses = [float(x) for x in res.stdout.split()]
    print("c_rgdcn_train losses:", losses)
    assert len(losses) == 6 and all(b < a for a, b in zip(losses, losses[1:])), losses


# ---------------------------------------------------------------- sharded training from C calls --------------------------
SHARDED = [dict(id="w2_halo_graph", world=2, plan="halo_graph"), dict(id="w4_halo_graph", world=4, plan="halo_graph"),
           dict(id="w2_training_plan", world=2, plan="training_plan")]
SHARDED_D, SHARDED_K, SHARDED_LAYERS, SHARDED_ACT, SHARDED_AGG = 64, 16, 3, "elu", "mean"


def sharded_graph():
    from test_sharded_layers_gpu import TRAIN_ZIPF, graph
    return graph(TRAIN_ZIPF)


def sharded_inputs():
    adj, _, V = sharded_graph()
    L, D, K = len(adj), SHARDED_D, SHARDED_K
    h = node_states(V, D, seed=21)
    ws = [make_weights(L, D // K, K, False, False, 31 + 7 * t) for t in range(SHARDED_LAYERS)]
    proj = np.random.default_rng(22).standard_normal((V, D)).astype(np.float32)
    return h, ws, proj


def sharded_step(sgs, streams, plans, h_own, wt, projs, exchange=True):
    """The loop of INTEGRATION.md section 2c on virtual ranks, every layer call through the C ABI (per channel, untied, no
    normalisation: the local plans need no in-degree table).  Forward per layer: owned rows into state buffer t % 2,
    rgnn_halo_exchange, a copy of the layer's local input (halo rows included: the backward recomputes the forward from it),
    rgnn_rgdcn_forward.  Backward from the last layer down: rgnn_rgdcn_backward on the local graph -> d_local [n_local, D],
    then rgnn_halo_exchange_backward -> d of the owned input rows.  Every phase is enqueued for all ranks before the next.
    exchange=False: no exchange, halo rows zero and their gradients dropped (the warm-up)."""
    import torch
    from tf_gnn_samples_b200.engine import check, load_library
    lib = load_library()
    D, K, R = SHARDED_D, SHARDED_K, len(sgs)
    C = D // K
    act, agg = get_activation(SHARDED_ACT), get_aggregation_function(SHARDED_AGG)
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    wss = []
    for sg, s, pl in zip(sgs, streams, plans):
        with torch.cuda.stream(s):
            nb = max(int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGDCN, D, D, K)),
                     int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGDCN_BACKWARD, D, D, K)))
            wss.append((torch.empty(nb, dtype=torch.uint8, device=sg.device), nb))
    x = list(h_own)
    inputs = [[None] * SHARDED_LAYERS for _ in range(R)]
    for t in range(SHARDED_LAYERS):
        for r, (sg, s) in enumerate(zip(sgs, streams)):
            with torch.cuda.stream(s):
                st = sg.states(t % 2)
                st[: sg.n_own].copy_(x[r])
                if not exchange:
                    st[sg.n_own:].zero_()
        if exchange:
            for sg, s in zip(sgs, streams):
                with torch.cuda.stream(s):
                    sg.exchange(t % 2)
        for r, (sg, s, pl) in enumerate(zip(sgs, streams, plans)):
            with torch.cuda.stream(s):
                inputs[r][t] = sg.states(t % 2).clone()
                y = torch.empty((sg.n_local, D), dtype=torch.float32, device=sg.device)
                check(lib.rgnn_rgdcn_forward(pl.handle, inputs[r][t].data_ptr(), D, C, tab(wt[t]), 0, None, act, agg, 0, 1,
                                             y.data_ptr(), wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
                x[r] = y[: sg.n_own]
    g = list(projs)
    grads = [[None] * SHARDED_LAYERS for _ in range(R)]
    for t in reversed(range(SHARDED_LAYERS)):
        d_local = []
        for r, (sg, s, pl) in enumerate(zip(sgs, streams, plans)):
            with torch.cuda.stream(s):
                z = lambda *shape: torch.empty(shape, dtype=torch.float32, device=sg.device)
                o = {"gh": z(sg.n_local, D), "gw": [z(K, K * K) for _ in wt[t]]}
                check(lib.rgnn_rgdcn_backward(pl.handle, inputs[r][t].data_ptr(), D, C, tab(wt[t]), 0, 0, None, act, agg, 0,
                                              g[r].data_ptr(), o["gh"].data_ptr(), tab(o["gw"]), wss[r][0].data_ptr(),
                                              wss[r][1], s.cuda_stream))
                grads[r][t] = o
                d_local.append(o["gh"])
        for r, (sg, s) in enumerate(zip(sgs, streams)):
            with torch.cuda.stream(s):
                g[r] = sg.exchange_backward(t % 2, d_local[r]) if exchange else d_local[r][: sg.n_own].clone()
    torch.cuda.synchronize()
    return x, g, grads


def run_sharded(case, sgs, streams, h, ws, proj, exchange=True):
    """One step of all ranks from numpy inputs: the owned outputs and d_h concatenated, the weight gradients summed over the
    ranks in float64 (the caller's all-reduce)."""
    import torch
    dev = sgs[0].device
    plans = [sg.plan if case["plan"] == "halo_graph" else sg.training_plan() for sg in sgs]
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(dev)
    wt = [[d(k) for ks in w["channel_weights"] for k in ks] for w in ws]
    h_own = [d(h[sg.lo:sg.hi]) for sg in sgs]
    projs = [d(proj[sg.lo:sg.hi]) for sg in sgs]
    torch.cuda.synchronize()
    x, g, grads = sharded_step(sgs, streams, plans, h_own, wt, projs, exchange)
    res = {"out": np.concatenate([y.cpu().numpy() for y in x]), "d_h": np.concatenate([y.cpu().numpy() for y in g])}
    for t in range(SHARDED_LAYERS):
        for i in range(len(wt[t])):
            res["d_F%d_%d" % (t, i)] = sum(gr[t]["gw"][i].double().cpu().numpy() for gr in grads)
    return res


def sharded_truth(h, ws, proj, device):
    """float64 autograd of the whole-graph stack on the GPU."""
    import torch
    adj, _, _ = sharded_graph()
    D, K = SHARDED_D, SHARDED_K
    with torch.device(device):
        f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
        x = h64 = f64(h)
        w64 = [{"channel_weights": [[f64(k) for k in ks] for ks in w["channel_weights"]]} for w in ws]
        for w in w64:
            x = sparse_rgdcn_autograd(x, adj, None, D // K, K, 1, False, False, SHARDED_ACT, SHARDED_AGG, False, weights=w)
        (x * torch.tensor(proj, dtype=torch.float64)).sum().backward()
    res = {"out": x.detach().cpu().numpy(), "d_h": h64.grad.cpu().numpy()}
    for t, w in enumerate(w64):
        for i, k in enumerate(k for ks in w["channel_weights"] for k in ks):
            res["d_F%d_%d" % (t, i)] = k.grad.cpu().numpy()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARDED, ids=[c["id"] for c in SHARDED])
def test_sharded_training_from_c_calls(cuda_device, case):
    """A 3-layer RGDCN stack (per channel, D = 64, K = 16, ELU, mean) over virtual ranks, every layer forward and backward
    through the C ABI on the rank's local graph (rgnn_halo_plan_graph, or the GraphPlan of training_plan()), halo gradients
    through rgnn_halo_exchange_backward: the owned outputs, d_h and the rank-summed weight gradients equal float64 autograd
    on the whole graph; a repeat is bit identical."""
    import torch
    from tf_gnn_samples_b200 import ShardedGraph
    from tf_gnn_samples_b200.sharded import degree_balanced_cuts
    adj, _, V = sharded_graph()
    cuts = degree_balanced_cuts(adj, V, case["world"])
    sgs = [ShardedGraph(adj, cuts, r, case["world"], device=cuda_device) for r in range(case["world"])]
    ShardedGraph.attach_in_process(sgs, SHARDED_D, training=True)
    streams = [torch.cuda.Stream(device=cuda_device) for _ in sgs]
    torch.cuda.synchronize()
    assert all(sg.n_halo > 0 for sg in sgs)
    h, ws, proj = sharded_inputs()
    run_sharded(case, sgs, streams, h, ws, proj, exchange=False)          # warm-up: loads every kernel but the exchanges
    got = run_sharded(case, sgs, streams, h, ws, proj)
    again = run_sharded(case, sgs, streams, h, ws, proj)
    want = sharded_truth(h, ws, proj, cuda_device)
    errs = {k: rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    print("sharded %s: max rel err vs float64 %.3e (%s)" % (case["id"], errs[worst], worst))
    bad = {k: e for k, e in errs.items() if not e <= TOL}
    assert not bad, bad
    for k in got:
        assert np.array_equal(got[k], again[k]), "%s: repeat differs" % k
    for sg in sgs:
        sg.close()

"""GPU: training RGAT through the C ABI alone -- rgnn_rgat_backward, the backward of one attention timestep.

The library is called through ctypes with torch-allocated buffers.  The reference for every gradient (d_h, every d_W_l and
d_att_l) is float64 autograd of oracle/ref_autograd.sparse_rgat_layer on the GPU; the criterion is max-norm relative error
<= 1e-4.  Each case also checks its difference to the Python training route (sparse_rgat_layer under torch autograd, whose
softmax uses scatter_reduce / index_add) against the same bound.  Covered:

  * every activation on a small graph with an empty edge type and isolated targets; d_in != d_out; head widths
    dh in {4, 12, 16, 32, 80, 128, 256} (butterfly and shared-memory head sums, 1 to 4 float4 per lane); a graph whose
    targets have zero, one or two incoming edges; two timesteps as two calls with the weight gradients summed; a Zipf
    PPI-shaped graph at D = 256 whose hub targets and hub (source, type) segments both exceed RGNN_HEAVY_SEGMENT, on an
    eager and on a deferred plan; BASELINE config 4 at full size;
  * two identical calls are bit-identical;
  * restricted plans (num_targets < V): the gradient of the loss over the owned rows, halo rows included in d_h;
  * the buffer contract of include/rgnn.h with guard-banded buffers at 16 mod 512 (test_buffer_contract_gpu.Guarded), and
    the refusals;
  * CUDA-graph capture and replay of forward + backward with new inputs written in place;
  * examples/c_rgat_train.c: compiled with -std=c99 -Wall -Wextra -Werror (no GPU needed), then linked and run;
  * sharded training from C calls alone: a 3-layer stack on virtual ranks (world 2 and 4), the INTEGRATION.md section 2c
    loop with rgnn_halo_exchange_backward, against float64 autograd on the whole graph, and a bit-identical repeat.

Kernels are counted with rgnn_launch_count deltas (this module asserts nothing from torch.profiler traces)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_autograd as A
from tf_gnn_samples_b200 import weights as W
from tf_gnn_samples_b200.utils import LAYER_RGAT, LAYER_RGAT_BACKWARD, get_activation

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, graph as dispatch_graph
from helpers import node_states, rel, tiny_graph

TOL = 1e-4
E_INVALID, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTS = ["linear", "tanh", "relu", "leaky_relu", "elu", "selu", "gelu"]


def tiny():
    adj, _ = tiny_graph()
    return adj, 37


def sparse_degrees():
    """Targets with no, one and two incoming edges (over all types) beside a few busier ones."""
    adj = [np.array([[0, 1], [2, 3], [4, 3], [5, 6], [7, 6], [8, 6], [1, 9], [3, 9]], np.int32),
           np.array([[6, 9], [9, 6], [2, 10]], np.int32),
           np.zeros((0, 2), np.int32)]
    return adj, 12


def zipf_ppi():
    adj, _, V = dispatch_graph(PPI6K_ZIPF)
    return adj, V


def config4():
    from tf_gnn_samples_b200 import batching
    b = batching.ppi_like_batch()
    return b.adjacency_lists, b.num_nodes


def in_degrees(adj, V):
    return np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)


# leaky_relu' jumps from 0.2 to 1 at a zero logit, so the float64 truth is discontinuous there: a logit within float32
# rounding (~1e-7 here) of zero takes the other branch in float32 and moves that edge's gradient by a factor of 5.  With a
# million logits of spread ~0.15, most seeds of config 4 have one; this seed keeps every logit at least 1e-6 from zero.
CONFIG4_SEED = 12


def min_abs_logit(adj, V, di, D, K, seed):
    """min |x_e,k| in float64 over every edge and head of Case(adj, V, di, D, K, seed=seed)."""
    w = W.rgat_weights(len(adj), di, D, seed + 7)
    h = node_states(V, di, seed=seed).astype(np.float64)
    dh, m = D // K, np.inf
    for l, a in enumerate(adj):
        t = (h @ w["edge_weights"][l].astype(np.float64)).reshape(V, K, dh)
        att = w["attention"][l].astype(np.float64).reshape(K, 2 * dh)
        s_src, s_tgt = np.einsum("vkd,kd->vk", t, att[:, :dh]), np.einsum("vkd,kd->vk", t, att[:, dh:])
        m = min(m, float(np.abs(s_src[a[:, 0]] + s_tgt[a[:, 1]]).min()))
    return m


def test_case_regimes():
    """The small graphs have an empty edge type, isolated targets and single-edge targets; the Zipf graph has hub targets
    and hub (source, type) segments above the heavy threshold."""
    adj, V = tiny()
    assert any(a.shape[0] == 0 for a in adj)
    assert (in_degrees(adj, V) == 0).any()
    adj, V = sparse_degrees()
    deg = in_degrees(adj, V)
    assert (deg == 0).any() and (deg == 1).any() and (deg == 2).any()
    adj, V = zipf_ppi()
    assert in_degrees(adj, V).max() > HEAVY_SEGMENT
    assert max(np.bincount(a[:, 0], minlength=V).max() for a in adj) > HEAVY_SEGMENT
    adj, V = config4()
    assert min_abs_logit(adj, V, 256, 256, 8, CONFIG4_SEED) > 1e-6


# ---------------------------------------------------------------- one case -----------------------------------------------
class Case:
    """Inputs of one timestep on the device and the ctypes call of rgnn_rgat_backward."""

    def __init__(self, adj, V, di, D, K, act="tanh", seed=3, num_targets=None, T=1, device=None, deferred=False):
        import torch
        from tf_gnn_samples_b200 import GraphPlan
        self.adj, self.V, self.di, self.D, self.K, self.T = adj, V, di, D, K, T
        self.act_name, self.act = act, get_activation(act)
        self.L = len(adj)
        self.dev = device
        self.w = W.rgat_weights(self.L, di, D, seed + 7)
        if T > 1:                                        # the recurrence needs d_in == d_out
            assert di == D
        self.h = node_states(V, di, seed=seed)
        self.plan = GraphPlan(adj, V, device=device, validate=not deferred)   # deferred: heavy counts stay on the device
        self.Vt = V if num_targets is None else num_targets
        if num_targets is not None:
            self.plan.set_num_targets(num_targets)
        self.g = np.random.default_rng(seed + 1).standard_normal((self.Vt, D)).astype(np.float32)
        t = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(device)
        self.th, self.tg = t(self.h), t(self.g)
        self.tw = [t(x) for x in self.w["edge_weights"]]
        self.ta = [t(x) for x in self.w["attention"]]

    @property
    def lib(self):
        from tf_gnn_samples_b200.engine import load_library
        return load_library()

    def ws_bytes(self):
        return int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGAT_BACKWARD, self.di, self.D, 0))

    def new_outputs(self):
        import torch
        z = lambda *s: torch.empty(s, dtype=torch.float32, device=self.dev)
        return {"gh": z(self.V, self.di), "gw": [z(self.di, self.D) for _ in range(self.L)],
                "ga": [z(2 * self.D) for _ in range(self.L)]}

    def call(self, outs, h_t=None, g_t=None, ws="own", nbytes=None, stream=None, **over):
        """rgnn_rgat_backward; `over` replaces raw arguments (pointers / ints).  ws="own": a workspace of the documented size
        from torch; otherwise the pointer (or None) and nbytes are passed as they are."""
        import torch
        ptr = lambda x: x if x is None or isinstance(x, int) else x.data_ptr()
        tab = lambda xs: None if xs is None else (ctypes.c_void_p * len(xs))(*[ptr(x) for x in xs])
        if isinstance(ws, str):
            nbytes = self.ws_bytes()
            ws_t = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=self.dev)   # freed stream-ordered after the call
            ws = ws_t.data_ptr()
        if stream is None:
            stream = torch.cuda.current_stream(self.dev).cuda_stream
        a = dict(plan=self.plan.handle, h=ptr(self.th if h_t is None else h_t), di=self.di, D=self.D, w=tab(self.tw),
                 att=tab(self.ta), K=self.K, act=self.act, g=ptr(self.tg if g_t is None else g_t), gh=ptr(outs.get("gh")),
                 gw=tab(outs.get("gw")), ga=tab(outs.get("ga")))
        a.update(over)
        return self.lib.rgnn_rgat_backward(a["plan"], a["h"], a["di"], a["D"], a["w"], a["att"], a["K"], a["act"], a["g"],
                                           a["gh"], a["gw"], a["ga"], ws, nbytes, stream)

    def forward(self, h, out=None, ws=None):
        """One timestep forward through rgnn_rgat_forward (num_timesteps = 1)."""
        import torch
        from tf_gnn_samples_b200.engine import check
        if out is None:
            out = torch.zeros((self.V, self.D), dtype=torch.float32, device=self.dev)
        nb = int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGAT, self.di, self.D, 0))
        if ws is None:
            ws = torch.empty(max(nb, 256), dtype=torch.uint8, device=self.dev)
        tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
        check(self.lib.rgnn_rgat_forward(self.plan.handle, h.data_ptr(), self.di, self.D, tab(self.tw), tab(self.ta), self.K,
                                         self.act, 1, out.data_ptr(), ws.data_ptr(), nb,
                                         torch.cuda.current_stream(self.dev).cuda_stream))
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
            for l in range(self.L):
                res["d_W%d" % l] = res.get("d_W%d" % l, 0) + o["gw"][l].double()
                res["d_att%d" % l] = res.get("d_att%d" % l, 0) + o["ga"][l].double()
        res["d_h"] = g
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in res.items()}

    def oracle(self):
        """float64 autograd of oracle/ref_autograd on the GPU: d/d(everything) of sum(out[:Vt] * g)."""
        import torch
        with torch.device(self.dev):
            f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
            h = f64(self.h)
            w = {"edge_weights": [f64(x) for x in self.w["edge_weights"]], "attention": [f64(x) for x in self.w["attention"]]}
            out = A.sparse_rgat_layer(h, self.adj, self.T, self.K, self.act_name, weights=w)
            (out[: self.Vt] * torch.tensor(self.g, dtype=torch.float64)).sum().backward()
        res = {"d_h": h.grad}
        for l in range(self.L):
            res["d_W%d" % l], res["d_att%d" % l] = w["edge_weights"][l].grad, w["attention"][l].grad
        return {k: v.cpu().numpy() for k, v in res.items()}

    def python_route(self):
        """The Python training route (sparse_rgat_layer under torch autograd: gnns/_train.py)."""
        import tf_gnn_samples_b200 as G
        h = self.th.clone().requires_grad_(True)
        w = {"edge_weights": [x.clone().requires_grad_(True) for x in self.tw],
             "attention": [x.clone().requires_grad_(True) for x in self.ta]}
        out = G.sparse_rgat_layer(h, self.plan, self.D, self.K, self.T, self.act_name, weights=w)
        (out[: self.Vt] * self.tg).sum().backward()
        res = {"d_h": h.grad}
        for l in range(self.L):
            res["d_W%d" % l], res["d_att%d" % l] = w["edge_weights"][l].grad, w["attention"][l].grad
        return {k: v.cpu().numpy() for k, v in res.items()}


def check_case(c, what, python_route=True):
    got, want = c.grads(), c.oracle()
    errs = {k: rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    line = "%s: max rel err vs float64 %.3e (%s)" % (what, errs[worst], worst)
    py_err = None
    if python_route:
        py = c.python_route()
        py_err = max(rel(got[k], py[k]) for k in py)
        line += ", vs the Python route %.3e" % py_err
    print(line)
    bad = {k: e for k, e in errs.items() if not e <= TOL}
    assert not bad, "%s: %s" % (what, bad)
    assert py_err is None or py_err <= TOL, "%s: the Python route differs by %.3e" % (what, py_err)
    return got


# ---------------------------------------------------------------- parity -------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_small_graph_matches_float64_autograd(cuda_device, act):
    adj, V = tiny()
    check_case(Case(adj, V, 16, 16, 4, act, device=cuda_device), "tiny %s" % act)


@pytest.mark.gpu
@pytest.mark.parametrize("di,D,K", [(12, 20, 5), (40, 8, 2)], ids=["12to20", "40to8"])
def test_input_dim_differs_from_state_dim(cuda_device, di, D, K):
    adj, V = tiny()
    check_case(Case(adj, V, di, D, K, "gelu", device=cuda_device), "tiny d_in=%d d_out=%d" % (di, D))


HEAD_WIDTHS = [(16, 4), (96, 8), (128, 8), (256, 8), (320, 4), (256, 2), (512, 2)]   # (D, K): dh = 4, 12, 16, 32, 80, 128, 256


@pytest.mark.gpu
@pytest.mark.parametrize("D,K", HEAD_WIDTHS, ids=["dh%d" % (d // k) for d, k in HEAD_WIDTHS])
def test_head_widths(cuda_device, D, K):
    adj, V = tiny()
    check_case(Case(adj, V, 24, D, K, "tanh", device=cuda_device), "tiny D=%d heads=%d (dh=%d)" % (D, K, D // K))


@pytest.mark.gpu
def test_targets_with_zero_one_and_two_edges(cuda_device):
    adj, V = sparse_degrees()
    check_case(Case(adj, V, 16, 32, 4, "selu", device=cuda_device), "zero / one / two incoming edges")


@pytest.mark.gpu
def test_two_timesteps_as_two_calls(cuda_device):
    adj, V = tiny()
    check_case(Case(adj, V, 16, 16, 2, "tanh", T=2, device=cuda_device), "tiny two timesteps")


@pytest.mark.gpu
def test_zipf_heavy_targets_and_sources_and_determinism(cuda_device):
    """D = 256 on the Zipf PPI-shaped graph: both heavy paths run; two calls are bit-identical."""
    import torch
    from tf_gnn_samples_b200.engine import check, launch_count
    adj, V = zipf_ppi()
    c = Case(adj, V, 256, 256, 8, "gelu", device=cuda_device)
    got = check_case(c, "zipf ppi D=256")
    o1, o2 = c.new_outputs(), c.new_outputs()
    before = launch_count()
    check(c.call(o1))
    n1 = launch_count() - before
    check(c.call(o2))
    torch.cuda.synchronize()
    assert n1 == launch_count() - before - n1
    print("zipf ppi D=256: %d kernel launches per backward" % n1)
    assert torch.equal(o1["gh"], o2["gh"])
    for k in ("gw", "ga"):
        assert all(torch.equal(a, b) for a, b in zip(o1[k], o2[k])), k
    assert np.array_equal(o1["gh"].cpu().numpy(), got["d_h"])


@pytest.mark.gpu
def test_deferred_plan(cuda_device):
    """A plan built without a synchronisation (RGNN_PLAN_DEFERRED_CHECK) never read its heavy-target count back: the
    heavy-target kernel runs as a persistent wave that reads the count on the device."""
    adj, V = zipf_ppi()
    check_case(Case(adj, V, 256, 256, 8, "tanh", deferred=True, device=cuda_device), "zipf ppi deferred plan")


@pytest.mark.gpu
def test_config4_full_size(cuda_device):
    """BASELINE config 4: PPI-shaped, hidden 256, 8 heads, tanh (inputs with no logit at the kink: CONFIG4_SEED)."""
    adj, V = config4()
    check_case(Case(adj, V, 256, 256, 8, "tanh", seed=CONFIG4_SEED, device=cuda_device), "config 4 V=%d M=%d L=%d D=256 K=8"
               % (V, sum(a.shape[0] for a in adj), len(adj)))


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name", ["tiny", "zipf"])
def test_restricted_plan(cuda_device, graph_name):
    """num_targets < V: the gradient of the loss over the owned rows; the halo rows of d_h receive theirs."""
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    D = 16 if graph_name == "tiny" else 64
    nt = V * 2 // 3
    c = Case(adj, V, D, D, 4, "elu", num_targets=nt, device=cuda_device)
    got = check_case(c, "%s restricted to %d of %d targets" % (graph_name, nt, V))
    assert np.abs(got["d_h"][nt:]).max() > 0


# ---------------------------------------------------------------- buffer contract ----------------------------------------
def guarded_case(c):
    """Guarded copies of the inputs and guarded outputs; returns (inputs, outputs)."""
    from test_buffer_contract_gpu import Guarded
    ins = {"h": Guarded.copy_of("h", c.th), "g": Guarded.copy_of("g", c.tg)}
    ins.update({"w%d" % l: Guarded.copy_of("w%d" % l, x) for l, x in enumerate(c.tw)})
    ins.update({"a%d" % l: Guarded.copy_of("a%d" % l, x) for l, x in enumerate(c.ta)})
    outs = {"gh": Guarded("gh", c.V * c.di * 4, c.dev)}
    outs.update({"gw%d" % l: Guarded("gw%d" % l, c.di * c.D * 4, c.dev) for l in range(c.L)})
    outs.update({"ga%d" % l: Guarded("ga%d" % l, 2 * c.D * 4, c.dev) for l in range(c.L)})
    return ins, outs


def guarded_call(c, ins, outs, ws_ptr, nbytes, drop=(), **over):
    import torch
    tab = lambda pre, d: (ctypes.c_void_p * c.L)(*[d["%s%d" % (pre, l)].ptr for l in range(c.L)])
    p = dict(h=ins["h"].ptr, g=ins["g"].ptr, w=tab("w", ins), att=tab("a", ins), gh=outs["gh"].ptr, gw=tab("gw", outs),
             ga=tab("ga", outs))
    for k in drop:
        p[k] = None
    p.update(over)
    return c.call({}, ws=ws_ptr, nbytes=nbytes, stream=torch.cuda.current_stream(c.dev).cuda_stream, **p)


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name", ["tiny", "zipf"])
def test_buffer_contract(cuda_device, graph_name):
    import torch
    from test_buffer_contract_gpu import Guarded, OUT_POISON, WS_POISON, poison_bits
    from tf_gnn_samples_b200.engine import launch_count
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    di, D, K = (12, 20, 5) if graph_name == "tiny" else (64, 96, 8)
    c = Case(adj, V, di, D, K, "tanh", device=cuda_device)
    ins, outs = guarded_case(c)
    snap = {k: g.payload.clone() for k, g in ins.items()}
    bound = c.ws_bytes()
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
    print("%s: S_min = %d bytes = %.1f%% of the documented bound %d" % (graph_name, s_min, 100.0 * s_min / bound, bound))
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
                want = c.grads()                          # the same call on torch buffers, itself checked against float64
                assert np.array_equal(outs["gh"].f32((V, c.di)).cpu().numpy(), want["d_h"])
                assert np.array_equal(outs["gw0"].f32((c.di, c.D)).cpu().numpy(), want["d_W0"].astype(np.float32))
                assert np.array_equal(outs["ga0"].f32((2 * c.D,)).cpu().numpy(), want["d_att0"].astype(np.float32))
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
    for drop in (("gh",), ("gw",), ("ga",), ("gh", "gw", "ga")):
        for g in outs.values():
            g.fill(OUT_POISON[1])
        assert guarded_call(c, ins, outs, ws.ptr, bound, drop=drop) == 0
        torch.cuda.synchronize()
        for k, g in outs.items():
            base = k.rstrip("0123456789")
            if base in drop:
                assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[1]).all()), k
            else:
                assert torch.equal(g.payload, ref[k]), k
    # refusals: each names its argument, enqueues nothing and writes nothing
    misaligned = (ctypes.c_void_p * c.L)(*[ins["a%d" % l].ptr + (4 if l == 0 else 0) for l in range(c.L)])
    refusals = [("d_out", dict(D=516), E_UNSUPPORTED), ("per-head dim", dict(K=D // 2), E_UNSUPPORTED),
                ("num_heads", dict(K=7), E_INVALID), ("num_heads", dict(K=0), E_INVALID),
                ("node_embeddings", dict(h=None), E_INVALID), ("grad_out", dict(g=None), E_INVALID),
                ("edge_weights", dict(w=None), E_INVALID), ("attention", dict(att=None), E_INVALID),
                ("attention vector 0", dict(att=misaligned), E_INVALID), ("activation", dict(act=99), E_INVALID),
                ("d_in", dict(di=6), E_INVALID)]
    for name, over, code in refusals:
        for g in outs.values():
            g.fill(OUT_POISON[0])
        before = launch_count()
        rc = guarded_call(c, ins, outs, ws.ptr, bound, **over)
        msg = c.lib.rgnn_last_error()
        msg = msg.decode() if isinstance(msg, bytes) else str(msg)
        assert rc == code, (over, rc, msg)
        assert name in msg, (name, msg)
        assert launch_count() == before, over
        torch.cuda.synchronize()
        for k, g in outs.items():
            assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[0]).all()), (over, k)


# ---------------------------------------------------------------- CUDA graph ---------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_replay_of_forward_and_backward(cuda_device):
    import torch
    from tf_gnn_samples_b200.engine import check
    adj, V = zipf_ppi()
    c = Case(adj, V, 64, 96, 8, "selu", device=cuda_device)
    cap = c.new_outputs()
    y_cap = torch.empty((V, c.D), dtype=torch.float32, device=cuda_device)
    nb_f = int(c.lib.rgnn_workspace_bytes(c.plan.handle, LAYER_RGAT, c.di, c.D, 0))
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
    for x in c.tw + c.ta:
        x.mul_(0.75)
    graph.replay()
    torch.cuda.synchronize()
    eager = c.new_outputs()
    y_eager = c.forward(c.th)
    check(c.call(eager))
    torch.cuda.synchronize()
    assert torch.equal(y_cap, y_eager)
    assert torch.equal(cap["gh"], eager["gh"])
    for k in ("gw", "ga"):
        assert all(torch.equal(a, b) for a, b in zip(cap[k], eager[k])), k
    c.h, c.g = c.th.cpu().numpy(), c.tg.cpu().numpy()
    c.w["edge_weights"] = [x.cpu().numpy() for x in c.tw]
    c.w["attention"] = [x.cpu().numpy() for x in c.ta]
    want = c.oracle()
    assert rel(cap["gh"].cpu().numpy(), want["d_h"]) <= TOL
    assert rel(cap["ga"][1].cpu().numpy(), want["d_att1"]) <= TOL
    # a first backward on a fresh plan refuses under capture, recording nothing
    fresh = Case(adj, V, 64, 96, 8, "selu", device=cuda_device)
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
EXAMPLE = os.path.join(ROOT, "examples", "c_rgat_train.c")
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
        exe = os.path.join(out_dir, "c_rgat_train")
        cmd += ["-o", exe, "-L", lib_dir, "-lrgnn", "-Wl,-rpath," + lib_dir, "-L", os.path.join(CUDA_HOME, "lib64"), "-lcudart",
                "-Wl,-rpath," + os.path.join(CUDA_HOME, "lib64"), "-lm"]
    else:
        exe = os.path.join(out_dir, "c_rgat_train.o")
        cmd += ["-c", "-o", exe]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return exe


def test_c_example_compiles_as_c99(tmp_path):
    compile_example(str(tmp_path), link=False)


class Lcg:
    """The example's generator: x <- 1664525 x + 1013904223 (mod 2^32), uniform = (x >> 8) / 2^24 in float32."""

    def __init__(self, seed):
        self.x = seed

    def uniform(self):
        self.x = (1664525 * self.x + 1013904223) & 0xFFFFFFFF
        return np.float32(self.x >> 8) * np.float32(1.0 / 16777216.0)


def example_inputs():
    """What examples/c_rgat_train.c builds, drawn in the same order: V = 64, L = 2, 256 edges per type, D = 16, 2 heads."""
    V, L, E, D = 64, 2, 256, 16
    r = Lcg(12345)
    adj = []
    for _ in range(L):
        a = np.zeros((E, 2), np.int32)
        for e in range(E):
            a[e, 0] = int(r.uniform() * np.float32(V))
            a[e, 1] = int(r.uniform() * np.float32(V))
        adj.append(a)
    sym = lambda n, s: np.array([(np.float32(2.0) * r.uniform() - np.float32(1.0)) * np.float32(s) for _ in range(n)], np.float32)
    h = sym(V * D, 1.0).reshape(V, D)
    ws = [sym(D * D, 0.5).reshape(D, D) for _ in range(L)]
    att = [sym(2 * D, 0.5) for _ in range(L)]
    target = sym(V * D, 1.0).reshape(V, D)
    return adj, V, D, h, ws, att, target


@pytest.mark.gpu
def test_c_example_trains(cuda_device, tmp_path):
    """The C host's losses decrease, and its first loss is the same forward through ctypes."""
    import torch
    exe = compile_example(str(tmp_path), link=True)
    res = subprocess.run([exe, "6"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    losses = [float(x) for x in res.stdout.split()]
    print("c_rgat_train losses:", losses)
    assert len(losses) == 6 and all(b < a for a, b in zip(losses, losses[1:])), losses
    adj, V, D, h, ws, att, target = example_inputs()
    c = Case(adj, V, D, D, 2, "tanh", device=cuda_device)
    c.th = torch.as_tensor(h).to(cuda_device)
    c.tw = [torch.as_tensor(x).to(cuda_device) for x in ws]
    c.ta = [torch.as_tensor(x).to(cuda_device) for x in att]
    y = c.forward(c.th).cpu().numpy().astype(np.float64)
    loss = 0.5 * np.sum((y - target) ** 2) / V
    assert abs(loss - losses[0]) <= 1e-5 * max(1.0, abs(loss)), (loss, losses[0])


# ---------------------------------------------------------------- sharded training from C calls --------------------------
SHARDED = [dict(id="w2_halo_graph", world=2, plan="halo_graph"), dict(id="w4_halo_graph", world=4, plan="halo_graph"),
           dict(id="w2_training_plan", world=2, plan="training_plan")]
SHARDED_D, SHARDED_K, SHARDED_LAYERS, SHARDED_ACT = 64, 4, 3, "tanh"


def sharded_graph():
    from test_sharded_layers_gpu import TRAIN_ZIPF, graph
    return graph(TRAIN_ZIPF)


def sharded_inputs():
    adj, _, V = sharded_graph()
    L, D = len(adj), SHARDED_D
    h = node_states(V, D, seed=21)
    ws = [W.rgat_weights(L, D, D, 31 + 7 * t) for t in range(SHARDED_LAYERS)]
    proj = np.random.default_rng(22).standard_normal((V, D)).astype(np.float32)
    return h, ws, proj


def sharded_step(sgs, streams, plans, h_own, wt, projs, exchange=True):
    """The loop of INTEGRATION.md section 2c on virtual ranks, every layer call through the C ABI.  Forward per layer:
    owned rows into state buffer t % 2, rgnn_halo_exchange, a copy of the layer's local input (halo rows included: the
    backward recomputes the forward from it), rgnn_rgat_forward.  Backward from the last layer down: rgnn_rgat_backward on
    the local graph -> d_local [n_local, D], then rgnn_halo_exchange_backward -> d of the owned input rows.  Every phase is
    enqueued for all ranks before the next.  exchange=False: no exchange, halo rows zero and their gradients dropped (the
    warm-up).  Returns per rank the owned output, d_h and the per-layer weight / attention gradients."""
    import torch
    from tf_gnn_samples_b200.engine import check, load_library
    lib = load_library()
    L, D, K, R = len(wt[0]["w"]), SHARDED_D, SHARDED_K, len(sgs)
    act = get_activation(SHARDED_ACT)
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    wss = []
    for sg, s, pl in zip(sgs, streams, plans):
        with torch.cuda.stream(s):
            nb = max(int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGAT, D, D, 0)),
                     int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGAT_BACKWARD, D, D, 0)))
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
                check(lib.rgnn_rgat_forward(pl.handle, inputs[r][t].data_ptr(), D, D, tab(wt[t]["w"]), tab(wt[t]["a"]), K, act,
                                            1, y.data_ptr(), wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
                x[r] = y[: sg.n_own]
    g = list(projs)
    grads = [[None] * SHARDED_LAYERS for _ in range(R)]
    for t in reversed(range(SHARDED_LAYERS)):
        d_local = []
        for r, (sg, s, pl) in enumerate(zip(sgs, streams, plans)):
            with torch.cuda.stream(s):
                z = lambda *shape: torch.empty(shape, dtype=torch.float32, device=sg.device)
                o = {"gh": z(sg.n_local, D), "gw": [z(D, D) for _ in range(L)], "ga": [z(2 * D) for _ in range(L)]}
                check(lib.rgnn_rgat_backward(pl.handle, inputs[r][t].data_ptr(), D, D, tab(wt[t]["w"]), tab(wt[t]["a"]), K, act,
                                             g[r].data_ptr(), o["gh"].data_ptr(), tab(o["gw"]), tab(o["ga"]),
                                             wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
                grads[r][t] = o
                d_local.append(o["gh"])
        for r, (sg, s) in enumerate(zip(sgs, streams)):
            with torch.cuda.stream(s):
                g[r] = sg.exchange_backward(t % 2, d_local[r]) if exchange else d_local[r][: sg.n_own].clone()
    torch.cuda.synchronize()
    return x, g, grads


def run_sharded(case, sgs, streams, h, ws, proj, exchange=True):
    """One step of all ranks from numpy inputs: the owned outputs and d_h concatenated, the weight and attention gradients
    summed over the ranks in float64 (the caller's all-reduce)."""
    import torch
    dev = sgs[0].device
    plans = [sg.plan if case["plan"] == "halo_graph" else sg.training_plan() for sg in sgs]
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(dev)
    wt = [{"w": [d(x) for x in w["edge_weights"]], "a": [d(x) for x in w["attention"]]} for w in ws]
    h_own = [d(h[sg.lo:sg.hi]) for sg in sgs]
    projs = [d(proj[sg.lo:sg.hi]) for sg in sgs]
    torch.cuda.synchronize()
    x, g, grads = sharded_step(sgs, streams, plans, h_own, wt, projs, exchange)
    res = {"out": np.concatenate([y.cpu().numpy() for y in x]), "d_h": np.concatenate([y.cpu().numpy() for y in g])}
    L = len(ws[0]["edge_weights"])
    for t in range(SHARDED_LAYERS):
        for key, name in (("gw", "W"), ("ga", "att")):
            for l in range(L):
                res["d_%s%d_%d" % (name, t, l)] = sum(gr[t][key][l].double().cpu().numpy() for gr in grads)
    return res


def sharded_truth(h, ws, proj, device):
    """float64 autograd of the whole-graph stack on the GPU."""
    import torch
    adj, _, _ = sharded_graph()
    with torch.device(device):
        f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
        x = h64 = f64(h)
        w64 = [{"edge_weights": [f64(a) for a in w["edge_weights"]], "attention": [f64(a) for a in w["attention"]]} for w in ws]
        for w in w64:
            x = A.sparse_rgat_layer(x, adj, 1, SHARDED_K, SHARDED_ACT, weights=w)
        (x * torch.tensor(proj, dtype=torch.float64)).sum().backward()
    res = {"out": x.detach().cpu().numpy(), "d_h": h64.grad.cpu().numpy()}
    for t, w in enumerate(w64):
        for l in range(len(w["edge_weights"])):
            res["d_W%d_%d" % (t, l)] = w["edge_weights"][l].grad.cpu().numpy()
            res["d_att%d_%d" % (t, l)] = w["attention"][l].grad.cpu().numpy()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARDED, ids=[c["id"] for c in SHARDED])
def test_sharded_training_from_c_calls(cuda_device, case):
    """A 3-layer RGAT stack over virtual ranks, every layer forward and backward through the C ABI on the rank's local graph
    (rgnn_halo_plan_graph, or the GraphPlan of training_plan()), halo gradients through rgnn_halo_exchange_backward: the
    owned outputs, d_h and the rank-summed weight and attention gradients equal float64 autograd on the whole graph; a
    repeat is bit identical."""
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

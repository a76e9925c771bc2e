"""GPU: training GGNN through the C ABI alone -- rgnn_ggnn_backward, the backward of one GRU / RNN timestep.

The library is called through ctypes with torch-allocated buffers.  The reference for every gradient (d_h, every d_W_l,
d_K, d_R and d_b) is float64 autograd of oracle/ref_autograd.sparse_ggnn_layer on the GPU; the criterion is max-norm
relative error <= 1e-4.  Each case also prints its difference to the Python training route (sparse_ggnn_layer under torch
autograd: gnns/_train.py).  Covered:

  * every activation x {sum, mean, sqrt_n} x {GRU, RNN} on a small graph with an empty edge type and isolated targets, with
    a random bias; cell weights scaled so that part of the gates saturate; four timesteps as four calls with the weight
    gradients summed; a Zipf PPI-shaped graph whose hub targets and hub (source, type) segments exceed RGNN_HEAVY_SEGMENT,
    on an eager and on a deferred plan; BASELINE config 3 at full size (the real QM9 validation structure, 4 timesteps);
  * two identical calls are bit-identical;
  * restricted plans (num_targets < V): the gradient of the loss over the owned rows, halo rows included in d_h;
  * the buffer contract of include/rgnn.h with guard-banded buffers (test_buffer_contract_gpu.Guarded), and the refusals;
  * CUDA-graph capture and replay of forward + backward with new inputs written in place;
  * examples/c_ggnn_train.c: compiled with -std=c99 -Wall -Wextra -Werror (no GPU needed), then linked and run;
  * sharded training from C calls alone: a 3-layer stack on virtual ranks (world 2 and 4), the INTEGRATION.md section 2c
    loop with rgnn_halo_exchange_backward, against float64 autograd on the whole graph, and a bit-identical repeat.

hard_sigmoid' jumps from 0.2 to 0 at a_z, a_r = +-2.5, so the float64 truth is discontinuous there: a CPU test checks that no
gate pre-activation of the seeded inputs lies within 1e-5 of the kink, and that the saturation case has gates on both
sides of it.  Kernels are counted with rgnn_launch_count deltas (this module asserts nothing from torch.profiler traces)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_autograd as A
from tf_gnn_samples_b200 import weights as W
from tf_gnn_samples_b200.utils import LAYER_GGNN, LAYER_GGNN_BACKWARD, CELL_GRU, CELL_RNN, get_activation, \
    get_aggregation_function

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, graph as dispatch_graph
from helpers import node_states, rel, tiny_graph

TOL = 1e-4
KINK_MARGIN = 1e-5
E_INVALID, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTS = ["linear", "tanh", "relu", "leaky_relu", "elu", "selu", "gelu"]
AGGS = ["sum", "mean", "sqrt_n"]
CELLS = ["gru", "rnn"]
SATURATE = 4.0   # scale of the cell weights in the saturation case


def tiny():
    adj, _ = tiny_graph()
    return adj, 37


def zipf_ppi():
    adj, _, V = dispatch_graph(PPI6K_ZIPF)
    return adj, V


def config3():
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), add_self_loop_edges=False)
    return b.adjacency_lists, b.num_nodes


def in_degrees(adj, V):
    return np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)


def make_weights(L, D, cell, seed, scale=1.0, kernel_scale=1.0):
    """ggnn_weights with a random bias; `scale` multiplies both cell kernels, `kernel_scale` the input kernel K only."""
    w = W.ggnn_weights(L, D, seed + 7, cell=cell, random_bias=True)
    c = w["cell"]
    if scale != 1.0 or kernel_scale != 1.0:
        c["kernel"] = c["kernel"] * np.float32(scale * kernel_scale)
        c["recurrent_kernel"] = c["recurrent_kernel"] * np.float32(scale)
    return w


def gate_preacts(adj, V, D, T, agg, act, seed, scale=1.0, kernel_scale=1.0):
    """Every a_z and a_r (float64, the oracle's op order) of the T timesteps of a GRU case's inputs, flattened."""
    import torch
    w = make_weights(len(adj), D, "gru", seed, scale, kernel_scale)
    f64 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float64)
    cur = f64(node_states(V, D, seed=seed))
    ew = [f64(x) for x in w["edge_weights"]]
    K, R, B = f64(w["cell"]["kernel"]), f64(w["cell"]["recurrent_kernel"]), f64(w["cell"]["bias"])
    adj_t = [torch.as_tensor(a).long() for a in adj]
    targets = torch.cat([a[:, 1] for a in adj_t])
    out = []
    with torch.no_grad():
        for _ in range(T):
            m = A.segment_reduce(torch.cat([cur[a[:, 0]] @ ew[l] for l, a in enumerate(adj_t)]), targets, V, agg)
            azr = m @ K[:, :2 * D] + B[:2 * D] + cur @ R[:, :2 * D]
            out.append(azr.reshape(-1).numpy())
            cur = A.sparse_ggnn_layer(cur, adj, 1, "gru", act, agg,
                                      weights={"edge_weights": ew, "cell": {"kernel": K, "recurrent_kernel": R, "bias": B}})
    return np.concatenate(out)


def kink_distance(a):
    return float(np.abs(np.abs(a) - 2.5).min())


# Config 3 has 185 million gate pre-activations over its 4 timesteps.  With the Glorot cell kernel, 20 to 47 of them lie
# within 1e-5 of +-2.5 for every seed from 1 to 15, where float32 rounding can take the other branch of hard_sigmoid' and move
# a row of d_h by a large fraction.  With the input kernel K halved (the sum over a node's bonds makes m . K the widest term),
# seed 6 keeps every gate at least 1.3e-5 from the kink while 0.013% of the gates still saturate.
CONFIG3_SEED, CONFIG3_KERNEL_SCALE = 6, 0.5


def test_case_regimes():
    """The small graph has an empty edge type and isolated targets; the Zipf graph has hub targets and hub (source, type)
    segments above the heavy threshold."""
    adj, V = tiny()
    assert any(a.shape[0] == 0 for a in adj)
    assert (in_degrees(adj, V) == 0).any()
    adj, V = zipf_ppi()
    assert in_degrees(adj, V).max() > HEAVY_SEGMENT
    assert max(np.bincount(a[:, 0], minlength=V).max() for a in adj) > HEAVY_SEGMENT


def test_no_gate_preactivation_at_the_hard_sigmoid_kink():
    """float64 oracle on the seeded GRU inputs of the small-graph, saturation, multi-timestep and config-3 cases: no a_z / a_r
    lies within 1e-5 of +-2.5, where hard_sigmoid' jumps; the saturation case has gates on both sides of the kink."""
    adj, V = tiny()
    for act in ACTS:
        for agg in AGGS:
            a = gate_preacts(adj, V, 16, 1, agg, act, 3)
            assert kink_distance(a) > KINK_MARGIN, (act, agg, kink_distance(a))
    a = gate_preacts(adj, V, 16, 4, "sum", "tanh", 3)
    assert kink_distance(a) > KINK_MARGIN
    sat = gate_preacts(adj, V, 16, 1, "sum", "tanh", 5, scale=SATURATE)
    print("saturation case: %.1f%% of the gates saturated, closest to the kink %.2e"
          % (100.0 * np.mean(np.abs(sat) > 2.5), kink_distance(sat)))
    assert kink_distance(sat) > KINK_MARGIN
    assert (np.abs(sat) > 2.5).mean() > 0.05 and (np.abs(sat) < 2.5).mean() > 0.05
    adj, V = zipf_ppi()
    for act, agg in (("gelu", "mean"), ("tanh", "sqrt_n"), ("elu", "mean"), ("selu", "mean")):
        a = gate_preacts(adj, V, 64, 1, agg, act, 3)
        assert kink_distance(a) > KINK_MARGIN, (act, agg, kink_distance(a))
    adj, V = config3()
    a = gate_preacts(adj, V, 128, 4, "sum", "tanh", CONFIG3_SEED, kernel_scale=CONFIG3_KERNEL_SCALE)
    print("config 3: closest gate pre-activation to the kink %.2e, max |a| %.2f" % (kink_distance(a), np.abs(a).max()))
    assert kink_distance(a) > KINK_MARGIN


# ---------------------------------------------------------------- one case -----------------------------------------------
class Case:
    """Inputs of one GGNN layer on the device and the ctypes call of rgnn_ggnn_backward."""

    def __init__(self, adj, V, D, cell="gru", act="tanh", agg="sum", seed=3, num_targets=None, T=1, device=None,
                 deferred=False, scale=1.0, kernel_scale=1.0):
        import torch
        from tf_gnn_samples_b200 import GraphPlan
        self.adj, self.V, self.D, self.T = adj, V, D, T
        self.cell_name, self.cell = cell, (CELL_GRU if cell == "gru" else CELL_RNN)
        self.act_name, self.act = act, get_activation(act)
        self.agg_name, self.agg = agg, get_aggregation_function(agg)
        self.L = len(adj)
        self.G = 3 if cell == "gru" else 1
        self.dev = device
        self.w = make_weights(self.L, D, cell, seed, scale, kernel_scale)
        self.h = node_states(V, D, seed=seed)
        self.plan = GraphPlan(adj, V, device=device, validate=not deferred)   # deferred: heavy counts stay on the device
        self.Vt = V if num_targets is None else num_targets
        if num_targets is not None:
            self.plan.set_num_targets(num_targets)
        self.g = np.random.default_rng(seed + 1).standard_normal((self.Vt, D)).astype(np.float32)
        t = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(device)
        self.th, self.tg = t(self.h), t(self.g)
        self.tw = [t(x) for x in self.w["edge_weights"]]
        self.tk, self.tr, self.tb = (t(self.w["cell"][k]) for k in ("kernel", "recurrent_kernel", "bias"))

    @property
    def lib(self):
        from tf_gnn_samples_b200.engine import load_library
        return load_library()

    def ws_bytes(self):
        return int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_GGNN_BACKWARD, self.D, self.D, 0))

    def new_outputs(self):
        import torch
        z = lambda *s: torch.empty(s, dtype=torch.float32, device=self.dev)
        G, D = self.G, self.D
        return {"gh": z(self.V, D), "gw": [z(D, D) for _ in range(self.L)], "gk": z(D, G * D), "gr": z(D, G * D),
                "gb": z(G * D)}

    def call(self, outs, h_t=None, g_t=None, ws="own", nbytes=None, stream=None, **over):
        """rgnn_ggnn_backward; `over` replaces raw arguments (pointers / ints).  ws="own": a workspace of the documented size
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
        a = dict(plan=self.plan.handle, h=ptr(self.th if h_t is None else h_t), D=self.D, w=tab(self.tw), k=ptr(self.tk),
                 r=ptr(self.tr), b=ptr(self.tb), cell=self.cell, act=self.act, agg=self.agg,
                 g=ptr(self.tg if g_t is None else g_t), gh=ptr(outs.get("gh")), gw=tab(outs.get("gw")), gk=ptr(outs.get("gk")),
                 gr=ptr(outs.get("gr")), gb=ptr(outs.get("gb")))
        a.update(over)
        return self.lib.rgnn_ggnn_backward(a["plan"], a["h"], a["D"], a["w"], a["k"], a["r"], a["b"], a["cell"], a["act"],
                                           a["agg"], a["g"], a["gh"], a["gw"], a["gk"], a["gr"], a["gb"], ws, nbytes, stream)

    def forward(self, h, out=None, ws=None):
        """One timestep forward through rgnn_ggnn_forward (num_timesteps = 1)."""
        import torch
        from tf_gnn_samples_b200.engine import check
        if out is None:
            out = torch.zeros((self.V, self.D), dtype=torch.float32, device=self.dev)
        nb = int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_GGNN, self.D, self.D, 0))
        if ws is None:
            ws = torch.empty(max(nb, 256), dtype=torch.uint8, device=self.dev)
        tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
        check(self.lib.rgnn_ggnn_forward(self.plan.handle, h.data_ptr(), self.D, self.D, tab(self.tw), self.tk.data_ptr(),
                                         self.tr.data_ptr(), self.tb.data_ptr(), self.cell, self.act, self.agg, 1, out.data_ptr(),
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
            for l in range(self.L):
                res["d_W%d" % l] = res.get("d_W%d" % l, 0) + o["gw"][l].double()
            for k, name in (("gk", "d_K"), ("gr", "d_R"), ("gb", "d_b")):
                res[name] = res.get(name, 0) + o[k].double()
        res["d_h"] = g
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in res.items()}

    def oracle(self):
        """float64 autograd of oracle/ref_autograd on the GPU: d/d(everything) of sum(out[:Vt] * g)."""
        import torch
        with torch.device(self.dev):
            f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
            h = f64(self.h)
            ew = [f64(x) for x in self.w["edge_weights"]]
            c = {k: f64(self.w["cell"][k]) for k in ("kernel", "recurrent_kernel", "bias")}
            out = A.sparse_ggnn_layer(h, self.adj, self.T, self.cell_name, self.act_name, self.agg_name,
                                      weights={"edge_weights": ew, "cell": c})
            (out[: self.Vt] * torch.tensor(self.g, dtype=torch.float64)).sum().backward()
        res = {"d_h": h.grad, "d_K": c["kernel"].grad, "d_R": c["recurrent_kernel"].grad, "d_b": c["bias"].grad}
        for l in range(self.L):
            res["d_W%d" % l] = ew[l].grad if ew[l].grad is not None else torch.zeros_like(ew[l])
        return {k: v.detach().cpu().numpy() for k, v in res.items()}

    def python_route(self):
        """The Python training route (sparse_ggnn_layer under torch autograd: gnns/_train.py)."""
        import tf_gnn_samples_b200 as G
        h = self.th.clone().requires_grad_(True)
        ew = [x.clone().requires_grad_(True) for x in self.tw]
        c = {k: x.clone().requires_grad_(True) for k, x in zip(("kernel", "recurrent_kernel", "bias"), (self.tk, self.tr, self.tb))}
        out = G.sparse_ggnn_layer(h, self.plan, self.D, self.T, self.cell_name, self.act_name, self.agg_name,
                                  weights={"edge_weights": ew, "cell": c})
        (out[: self.Vt] * self.tg).sum().backward()
        res = {"d_h": h.grad, "d_K": c["kernel"].grad, "d_R": c["recurrent_kernel"].grad, "d_b": c["bias"].grad}
        for l in range(self.L):
            if ew[l].grad is not None:
                res["d_W%d" % l] = ew[l].grad
        return {k: v.cpu().numpy() for k, v in res.items()}


def check_case(c, what, python_route=True):
    got, want = c.grads(), c.oracle()
    errs = {k: rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    line = "%s: max rel err vs float64 %.3e (%s)" % (what, errs[worst], worst)
    if python_route:
        py = c.python_route()
        line += ", vs the Python route %.3e" % max(rel(got[k], py[k]) for k in py)
    print(line)
    bad = {k: e for k, e in errs.items() if not e <= TOL}
    assert not bad, "%s: %s" % (what, bad)
    return got


# ---------------------------------------------------------------- parity -------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("act", ACTS)
def test_small_graph_matches_float64_autograd(cuda_device, act, agg, cell):
    adj, V = tiny()
    check_case(Case(adj, V, 16, cell, act, agg, device=cuda_device), "tiny %s %s %s" % (cell, act, agg))


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_saturated_gates(cuda_device, cell):
    """Cell weights scaled by 4: part of the GRU gates sit in hard_sigmoid's flat tails (none at the kink:
    test_no_gate_preactivation_at_the_hard_sigmoid_kink), and the RNN's tanh saturates."""
    adj, V = tiny()
    check_case(Case(adj, V, 16, cell, "tanh", "sum", seed=5, scale=SATURATE, device=cuda_device), "tiny %s saturated" % cell)


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_four_timesteps_as_four_calls(cuda_device, cell):
    adj, V = tiny()
    check_case(Case(adj, V, 16, cell, "tanh", "sum", T=4, device=cuda_device), "tiny %s four timesteps" % cell)


@pytest.mark.gpu
def test_zipf_heavy_targets_and_sources_and_determinism(cuda_device):
    """The Zipf PPI-shaped graph: heavy targets and heavy (source, type) segments; two calls are bit-identical."""
    import torch
    from tf_gnn_samples_b200.engine import check, launch_count
    adj, V = zipf_ppi()
    c = Case(adj, V, 64, "gru", "gelu", "mean", device=cuda_device)
    got = check_case(c, "zipf ppi D=64 GRU")
    o1, o2 = c.new_outputs(), c.new_outputs()
    before = launch_count()
    check(c.call(o1))
    n1 = launch_count() - before
    check(c.call(o2))
    torch.cuda.synchronize()
    assert n1 == launch_count() - before - n1
    print("zipf ppi D=64 GRU: %d kernel launches per backward" % n1)
    assert torch.equal(o1["gh"], o2["gh"])
    assert all(torch.equal(a, b) for a, b in zip(o1["gw"], o2["gw"]))
    for k in ("gk", "gr", "gb"):
        assert torch.equal(o1[k], o2[k]), k
    assert np.array_equal(o1["gh"].cpu().numpy(), got["d_h"])


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_deferred_plan(cuda_device, cell):
    """A plan built without a synchronisation (RGNN_PLAN_DEFERRED_CHECK) never read its heavy-target count back."""
    adj, V = zipf_ppi()
    check_case(Case(adj, V, 64, cell, "tanh", "sqrt_n", deferred=True, device=cuda_device), "zipf ppi deferred plan %s" % cell)


@pytest.mark.gpu
def test_config3_full_size(cuda_device):
    """BASELINE config 3: the real 10,000 QM9 validation molecules, hidden 128, GRU, tanh, 4 timesteps as 4 calls (inputs
    with no gate at the hard_sigmoid kink: CONFIG3_SEED, CONFIG3_KERNEL_SCALE)."""
    adj, V = config3()
    check_case(Case(adj, V, 128, "gru", "tanh", "sum", seed=CONFIG3_SEED, T=4, kernel_scale=CONFIG3_KERNEL_SCALE,
                    device=cuda_device),
               "config 3 V=%d M=%d L=%d D=128 T=4" % (V, sum(a.shape[0] for a in adj), len(adj)))


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,cell", [("tiny", "gru"), ("tiny", "rnn"), ("zipf", "gru")])
def test_restricted_plan(cuda_device, graph_name, cell):
    """num_targets < V: the gradient of the loss over the owned rows; the halo rows of d_h receive theirs."""
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    D = 16 if graph_name == "tiny" else 64
    nt = V * 2 // 3
    c = Case(adj, V, D, cell, "elu", "mean", num_targets=nt, device=cuda_device)
    got = check_case(c, "%s %s restricted to %d of %d targets" % (graph_name, cell, nt, V), python_route=False)
    assert np.abs(got["d_h"][nt:]).max() > 0


# ---------------------------------------------------------------- buffer contract ----------------------------------------
def guarded_case(c):
    """Guarded copies of the inputs and guarded outputs; returns (inputs, outputs)."""
    from test_buffer_contract_gpu import Guarded
    ins = {"h": Guarded.copy_of("h", c.th), "g": Guarded.copy_of("g", c.tg), "k": Guarded.copy_of("k", c.tk),
           "r": Guarded.copy_of("r", c.tr), "b": Guarded.copy_of("b", c.tb)}
    ins.update({"w%d" % l: Guarded.copy_of("w%d" % l, x) for l, x in enumerate(c.tw)})
    G, D = c.G, c.D
    outs = {"gh": Guarded("gh", c.V * D * 4, c.dev), "gk": Guarded("gk", D * G * D * 4, c.dev),
            "gr": Guarded("gr", D * G * D * 4, c.dev), "gb": Guarded("gb", G * D * 4, c.dev)}
    outs.update({"gw%d" % l: Guarded("gw%d" % l, D * D * 4, c.dev) for l in range(c.L)})
    return ins, outs


def guarded_call(c, ins, outs, ws_ptr, nbytes, drop=(), **over):
    import torch
    tab = lambda pre, d: (ctypes.c_void_p * c.L)(*[d["%s%d" % (pre, l)].ptr for l in range(c.L)])
    p = dict(h=ins["h"].ptr, g=ins["g"].ptr, w=tab("w", ins), k=ins["k"].ptr, r=ins["r"].ptr, b=ins["b"].ptr,
             gh=outs["gh"].ptr, gw=tab("gw", outs), gk=outs["gk"].ptr, gr=outs["gr"].ptr, gb=outs["gb"].ptr)
    for k in drop:
        p[k] = None
    p.update(over)
    return c.call({}, ws=ws_ptr, nbytes=nbytes, stream=torch.cuda.current_stream(c.dev).cuda_stream, **p)


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,cell", [("tiny", "gru"), ("tiny", "rnn"), ("zipf", "gru")])
def test_buffer_contract(cuda_device, graph_name, cell):
    import torch
    from test_buffer_contract_gpu import Guarded, OUT_POISON, WS_POISON, poison_bits
    from tf_gnn_samples_b200.engine import launch_count
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    D = 20 if graph_name == "tiny" else 96
    c = Case(adj, V, D, cell, "tanh", "mean", device=cuda_device)
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
    print("%s %s: S_min = %d bytes = %.1f%% of the documented bound %d" % (graph_name, cell, s_min, 100.0 * s_min / bound, bound))
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
                assert np.array_equal(outs["gh"].f32((V, D)).cpu().numpy(), want["d_h"])
                assert np.array_equal(outs["gw0"].f32((D, D)).cpu().numpy(), want["d_W0"].astype(np.float32))
                assert np.array_equal(outs["gr"].f32((D, c.G * D)).cpu().numpy(), want["d_R"].astype(np.float32))
                assert np.array_equal(outs["gb"].f32((c.G * D,)).cpu().numpy(), want["d_b"].astype(np.float32))
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
    for drop in (("gh",), ("gw",), ("gk",), ("gr",), ("gb",), ("gh", "gw", "gk", "gr", "gb")):
        for g in outs.values():
            g.fill(OUT_POISON[1])
        assert guarded_call(c, ins, outs, ws.ptr, bound, drop=drop) == 0
        torch.cuda.synchronize()
        for k, g in outs.items():
            base = k.rstrip("0123456789")
            if base in drop:
                assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[1]).all()), k
            else:
                assert torch.equal(g.payload, ref[k]), (drop, k)
    # refusals: each names its argument, enqueues nothing and writes nothing
    refusals = [("aggregation", dict(agg=1), E_UNSUPPORTED), ("aggregation", dict(agg=9), E_INVALID),
                ("cell", dict(cell=2), E_INVALID), ("activation", dict(act=99), E_INVALID),
                ("state dim", dict(D=D + 2), E_INVALID), ("plan", dict(plan=None), E_INVALID),
                ("node_embeddings", dict(h=None), E_INVALID), ("grad_out", dict(g=None), E_INVALID),
                ("edge_weights", dict(w=None), E_INVALID), ("cell_kernel", dict(k=None), E_INVALID),
                ("cell_recurrent_kernel", dict(r=None), E_INVALID), ("cell_bias", dict(b=None), E_INVALID),
                ("cell_bias", dict(b=ins["b"].ptr + 4), E_INVALID), ("node_embeddings", dict(h=ins["h"].ptr + 4), E_INVALID),
                ("grad_cell_recurrent_kernel", dict(gr=outs["gr"].ptr + 4), E_INVALID),
                ("alias", dict(gh=ins["h"].ptr), E_INVALID), ("alias", dict(gh=ins["g"].ptr), E_INVALID),
                ("grad edge weight 0", dict(gw=(ctypes.c_void_p * c.L)(*([None] + [outs["gw%d" % l].ptr for l in range(1, c.L)]))),
                 E_INVALID)]
    for name, over, code in refusals:
        for g in outs.values():
            g.fill(OUT_POISON[0])
        before = launch_count()
        rc = guarded_call(c, ins, outs, ws.ptr, bound, **over)
        msg = c.lib.rgnn_last_error()
        msg = msg.decode() if isinstance(msg, bytes) else str(msg)
        assert rc == code, (name, rc, msg)
        assert name in msg, (name, msg)
        assert launch_count() == before, name
        torch.cuda.synchronize()
        for k, g in outs.items():
            assert bool(poison_bits(g.payload.view(torch.float32), OUT_POISON[0]).all()), (name, k)


# ---------------------------------------------------------------- CUDA graph ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_cuda_graph_replay_of_forward_and_backward(cuda_device, cell):
    import torch
    from tf_gnn_samples_b200.engine import check
    adj, V = zipf_ppi()
    c = Case(adj, V, 64, cell, "selu", "mean", device=cuda_device)
    cap = c.new_outputs()
    y_cap = torch.empty((V, c.D), dtype=torch.float32, device=cuda_device)
    nb_f = int(c.lib.rgnn_workspace_bytes(c.plan.handle, LAYER_GGNN, c.D, c.D, 0))
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
    for x in c.tw + [c.tk, c.tr, c.tb]:
        x.mul_(0.75)
    graph.replay()
    torch.cuda.synchronize()
    eager = c.new_outputs()
    y_eager = c.forward(c.th)
    check(c.call(eager))
    torch.cuda.synchronize()
    assert torch.equal(y_cap, y_eager)
    assert all(torch.equal(a, b) for a, b in zip(cap["gw"], eager["gw"]))
    for k in ("gh", "gk", "gr", "gb"):
        assert torch.equal(cap[k], eager[k]), k
    c.h, c.g = c.th.cpu().numpy(), c.tg.cpu().numpy()
    c.w["edge_weights"] = [x.cpu().numpy() for x in c.tw]
    c.w["cell"] = {k: x.cpu().numpy() for k, x in zip(("kernel", "recurrent_kernel", "bias"), (c.tk, c.tr, c.tb))}
    want = c.oracle()
    assert rel(cap["gh"].cpu().numpy(), want["d_h"]) <= TOL
    assert rel(cap["gr"].cpu().numpy(), want["d_R"]) <= TOL
    # a first backward on a fresh plan refuses under capture, recording nothing
    fresh = Case(adj, V, 64, cell, "selu", "mean", device=cuda_device)
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
EXAMPLE = os.path.join(ROOT, "examples", "c_ggnn_train.c")
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
        exe = os.path.join(out_dir, "c_ggnn_train")
        cmd += ["-o", exe, "-L", lib_dir, "-lrgnn", "-Wl,-rpath," + lib_dir, "-L", os.path.join(CUDA_HOME, "lib64"), "-lcudart",
                "-Wl,-rpath," + os.path.join(CUDA_HOME, "lib64"), "-lm"]
    else:
        exe = os.path.join(out_dir, "c_ggnn_train.o")
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
    """What examples/c_ggnn_train.c builds, drawn in the same order: 8 molecules of 9 atoms, L = 4, 40 bonds per type, D = 16."""
    G, ATOMS, L, E, D = 8, 9, 4, 40, 16
    r = Lcg(12345)
    adj = []
    for _ in range(L):
        a = np.zeros((E, 2), np.int32)
        for e in range(E):
            g = int(r.uniform() * np.float32(G))
            a[e, 0] = g * ATOMS + int(r.uniform() * np.float32(ATOMS))
            a[e, 1] = g * ATOMS + int(r.uniform() * np.float32(ATOMS))
        adj.append(a)
    sym = lambda n, s: np.array([(np.float32(2.0) * r.uniform() - np.float32(1.0)) * np.float32(s) for _ in range(n)], np.float32)
    V = G * ATOMS
    h = sym(V * D, 1.0).reshape(V, D)
    ws = [sym(D * D, 0.3).reshape(D, D) for _ in range(L)]
    k = sym(D * 3 * D, 0.3).reshape(D, 3 * D)
    rk = sym(D * 3 * D, 0.3).reshape(D, 3 * D)
    b = sym(3 * D, 0.1)
    target = sym(V * D, 1.0).reshape(V, D)
    return adj, V, D, h, ws, k, rk, b, target


@pytest.mark.gpu
def test_c_example_trains(cuda_device, tmp_path):
    """The C host's losses decrease, and its first loss is the same two forwards through ctypes."""
    import torch
    exe = compile_example(str(tmp_path), link=True)
    res = subprocess.run([exe, "6"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    losses = [float(x) for x in res.stdout.split()]
    print("c_ggnn_train losses:", losses)
    assert len(losses) == 6 and all(b < a for a, b in zip(losses, losses[1:])), losses
    adj, V, D, h, ws, k, rk, b, target = example_inputs()
    c = Case(adj, V, D, "gru", "tanh", "sum", device=cuda_device)
    d = lambda x: torch.as_tensor(x).to(cuda_device)
    c.th, c.tw, c.tk, c.tr, c.tb = d(h), [d(x) for x in ws], d(k), d(rk), d(b)
    y = c.forward(c.forward(c.th)).cpu().numpy().astype(np.float64)
    loss = 0.5 * np.sum((y - target) ** 2) / V
    assert abs(loss - losses[0]) <= 1e-5 * max(1.0, abs(loss)), (loss, losses[0])


# ---------------------------------------------------------------- sharded training from C calls --------------------------
SHARDED = [dict(id="w2_halo_graph", world=2, plan="halo_graph"), dict(id="w4_halo_graph", world=4, plan="halo_graph"),
           dict(id="w2_training_plan", world=2, plan="training_plan")]
SHARDED_D, SHARDED_LAYERS, SHARDED_ACT, SHARDED_AGG = 64, 3, "tanh", "mean"


def sharded_graph():
    from test_sharded_layers_gpu import TRAIN_ZIPF, graph
    return graph(TRAIN_ZIPF)


def sharded_inputs():
    adj, _, V = sharded_graph()
    L, D = len(adj), SHARDED_D
    h = node_states(V, D, seed=21)
    ws = [make_weights(L, D, "gru", 31 + 7 * t) for t in range(SHARDED_LAYERS)]
    proj = np.random.default_rng(22).standard_normal((V, D)).astype(np.float32)
    return h, ws, proj


def sharded_step(sgs, streams, plans, h_own, wt, projs, exchange=True):
    """The loop of INTEGRATION.md section 2c on virtual ranks, every layer call through the C ABI.  Forward per layer:
    owned rows into state buffer t % 2, rgnn_halo_exchange, a copy of the layer's local input (halo rows included: the
    backward recomputes the forward from it), rgnn_ggnn_forward.  Backward from the last layer down: rgnn_ggnn_backward on
    the local graph -> d_local [n_local, D], then rgnn_halo_exchange_backward -> d of the owned input rows.  Every phase is
    enqueued for all ranks before the next.  exchange=False: no exchange, halo rows zero and their gradients dropped (the
    warm-up).  Returns per rank the owned output, d_h and the per-layer weight gradients."""
    import torch
    from tf_gnn_samples_b200.engine import check, load_library
    lib = load_library()
    L, D, R = len(wt[0]["w"]), SHARDED_D, len(sgs)
    act, agg = get_activation(SHARDED_ACT), get_aggregation_function(SHARDED_AGG)
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    wss = []
    for sg, s, pl in zip(sgs, streams, plans):
        with torch.cuda.stream(s):
            nb = max(int(lib.rgnn_workspace_bytes(pl.handle, LAYER_GGNN, D, D, 0)),
                     int(lib.rgnn_workspace_bytes(pl.handle, LAYER_GGNN_BACKWARD, D, D, 0)))
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
                w = wt[t]
                check(lib.rgnn_ggnn_forward(pl.handle, inputs[r][t].data_ptr(), D, D, tab(w["w"]), w["k"].data_ptr(),
                                            w["r"].data_ptr(), w["b"].data_ptr(), CELL_GRU, act, agg, 1, y.data_ptr(),
                                            wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
                x[r] = y[: sg.n_own]
    g = list(projs)
    grads = [[None] * SHARDED_LAYERS for _ in range(R)]
    for t in reversed(range(SHARDED_LAYERS)):
        d_local = []
        for r, (sg, s, pl) in enumerate(zip(sgs, streams, plans)):
            with torch.cuda.stream(s):
                z = lambda *shape: torch.empty(shape, dtype=torch.float32, device=sg.device)
                o = {"gh": z(sg.n_local, D), "gw": [z(D, D) for _ in range(L)], "gk": z(D, 3 * D), "gr": z(D, 3 * D),
                     "gb": z(3 * D)}
                w = wt[t]
                check(lib.rgnn_ggnn_backward(pl.handle, inputs[r][t].data_ptr(), D, tab(w["w"]), w["k"].data_ptr(),
                                             w["r"].data_ptr(), w["b"].data_ptr(), CELL_GRU, act, agg, g[r].data_ptr(),
                                             o["gh"].data_ptr(), tab(o["gw"]), o["gk"].data_ptr(), o["gr"].data_ptr(),
                                             o["gb"].data_ptr(), wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
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
    wt = [{"w": [d(x) for x in w["edge_weights"]], "k": d(w["cell"]["kernel"]), "r": d(w["cell"]["recurrent_kernel"]),
           "b": d(w["cell"]["bias"])} for w in ws]
    h_own = [d(h[sg.lo:sg.hi]) for sg in sgs]
    projs = [d(proj[sg.lo:sg.hi]) for sg in sgs]
    torch.cuda.synchronize()
    x, g, grads = sharded_step(sgs, streams, plans, h_own, wt, projs, exchange)
    res = {"out": np.concatenate([y.cpu().numpy() for y in x]), "d_h": np.concatenate([y.cpu().numpy() for y in g])}
    L = len(ws[0]["edge_weights"])
    for t in range(SHARDED_LAYERS):
        for l in range(L):
            res["d_W%d_%d" % (t, l)] = sum(gr[t]["gw"][l].double().cpu().numpy() for gr in grads)
        for key in ("gk", "gr", "gb"):
            res["d_%s%d" % (key[1].upper(), t)] = sum(gr[t][key].double().cpu().numpy() for gr in grads)
    return res


def sharded_truth(h, ws, proj, device):
    """float64 autograd of the whole-graph stack on the GPU."""
    import torch
    adj, _, _ = sharded_graph()
    with torch.device(device):
        f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
        x = h64 = f64(h)
        w64 = [{"edge_weights": [f64(a) for a in w["edge_weights"]],
                "cell": {k: f64(w["cell"][k]) for k in ("kernel", "recurrent_kernel", "bias")}} for w in ws]
        for w in w64:
            x = A.sparse_ggnn_layer(x, adj, 1, "gru", SHARDED_ACT, SHARDED_AGG, weights=w)
        (x * torch.tensor(proj, dtype=torch.float64)).sum().backward()
    res = {"out": x.detach().cpu().numpy(), "d_h": h64.grad.cpu().numpy()}
    for t, w in enumerate(w64):
        for l in range(len(w["edge_weights"])):
            res["d_W%d_%d" % (t, l)] = w["edge_weights"][l].grad.cpu().numpy()
        for key, name in (("K", "kernel"), ("R", "recurrent_kernel"), ("B", "bias")):
            res["d_%s%d" % (key, t)] = w["cell"][name].grad.cpu().numpy()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARDED, ids=[c["id"] for c in SHARDED])
def test_sharded_training_from_c_calls(cuda_device, case):
    """A 3-layer GGNN stack (GRU, one timestep per layer) over virtual ranks, every layer forward and backward through the
    C ABI on the rank's local graph (rgnn_halo_plan_graph, or the GraphPlan of training_plan()), halo gradients through
    rgnn_halo_exchange_backward: the owned outputs, d_h and the rank-summed weight gradients equal float64 autograd on the
    whole graph; a repeat is bit identical."""
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

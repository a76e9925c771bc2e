"""GPU: training RGIN through the C ABI alone -- rgnn_rgin_backward, the backward of one source-message timestep.

The library is called through ctypes with torch-allocated buffers.  The reference for every gradient (d_h, every edge-MLP
kernel d_E, every aggregation-MLP kernel d_K, d_gamma and d_beta) is float64 autograd of oracle/ref_autograd.sparse_rgin_layer
on the GPU; the criterion is max-norm relative error <= 1e-4.  Each case also prints its difference to the Python training
route (sparse_rgin_layer under torch autograd: gnns/_train.py).  Covered:

  * every activation x {sum, mean, sqrt_n} x edge MLP {None, 0, 1, 2 hidden layers} x aggregation MLP {None, 1 hidden layer}
    on a small graph with an empty edge type, isolated targets and duplicate edges, with random layer-norm parameters;
    d_in != d_out; two timesteps as two calls with the weight gradients summed;
  * a Zipf PPI-shaped graph at D = 256 whose hub targets and hub (source, type) segments exceed RGNN_HEAVY_SEGMENT, on an
    eager and on a deferred plan, with a bit-identical repeat; the QM9 RGIN configuration at full size (the real QM9
    validation structure with self-loop edges, L = 5, D = 128, ELU, sum, one edge-MLP hidden layer);
  * restricted plans (num_targets < V): the gradient of the loss over the owned rows, halo rows included in d_h;
  * the buffer contract of include/rgnn.h with guard-banded buffers (test_buffer_contract_gpu.Guarded), and every refusal;
  * CUDA-graph capture and replay of forward + backward with new inputs written in place;
  * examples/c_rgin_train.c: compiled with -std=c99 -Wall -Wextra -Werror (no GPU needed), then linked and run;
  * sharded training from C calls alone: a 3-layer stack on virtual ranks (world 2 and 4), the INTEGRATION.md section 2c
    loop with rgnn_halo_exchange_backward, against float64 autograd on the whole graph, and a bit-identical repeat.

ReLU, leaky_relu and SELU have a derivative jump at 0, and RGIN applies the activation at every edge-MLP hidden layer, at the
message and at the output.  Where a pre-activation lies within float32 rounding of 0, float32 and float64 take different
branches and no kernel can meet 1e-4.  Kinked activations are therefore run on the small graph only, and a CPU test checks
that no seeded pre-activation of those cases lies within KINK_MARGIN of 0 (exact zeros -- the isolated targets' rows -- are
zero in both precisions and take the same branch).  The large cases use ELU (the QM9 RGIN default, whose derivative is
continuous at 0), tanh or gelu.  Kernels are counted with rgnn_launch_count deltas."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import ref_autograd as A
from tf_gnn_samples_b200 import weights as W
from tf_gnn_samples_b200.utils import LAYER_RGIN, LAYER_RGIN_BACKWARD, get_activation, get_aggregation_function

from dispatch import HEAVY_SEGMENT, PPI6K_ZIPF, graph as dispatch_graph
from helpers import node_states, rel, tiny_graph

TOL = 1e-4
KINK_MARGIN = 1e-5
E_INVALID, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACTS = ["linear", "tanh", "relu", "leaky_relu", "elu", "selu", "gelu"]
KINKED = ("relu", "leaky_relu", "selu")
AGGS = ["sum", "mean", "sqrt_n"]
EDGE_MLPS = [None, 0, 1, 2]      # edge-MLP hidden layers (None: the raw source states are the messages)
AGGR_MLPS = [None, 1]            # aggregation-MLP hidden layers
SMALL_SEED = 4   # seeds 1 to 3 each put a ReLU pre-activation within 1e-5 of 0 (the closest 3.3e-6); seed 4: 3.1e-5


def tiny():
    adj, _ = tiny_graph()
    return adj, 37


def zipf_ppi():
    adj, _, V = dispatch_graph(PPI6K_ZIPF)
    return adj, V


def qm9_rgin():
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), add_self_loop_edges=True)
    return b.adjacency_lists, b.num_nodes


def in_degrees(adj, V):
    return np.bincount(np.concatenate([a[:, 1] for a in adj]), minlength=V)


def make_weights(L, d_in, D, e_hidden, a_hidden, seed, T=1):
    """rgin_weights with random layer-norm parameters (gamma = 1 + 0.2 N(0,1), beta = 0.2 N(0,1)) and Glorot MLP kernels."""
    return W.rgin_weights(L, d_in, D, e_hidden, a_hidden, seed=seed + 11, num_timesteps=T, random_ln=True)


def preacts(adj, V, d_in, D, T, act, agg, e_hidden, a_hidden, seed):
    """Every pre-activation a kink can act on (every edge-MLP layer on the (source, type) rows some edge reads, the last one
    being the message's, every aggregation-MLP layer and the output activation's input), float64 in the oracle's op order,
    over T timesteps; exact zeros dropped."""
    import torch
    w = A.to_torch64(make_weights(len(adj), d_in, D, e_hidden, a_hidden, seed, T), requires_grad=False)
    f = A.get_activation(act)
    cur = torch.as_tensor(node_states(V, d_in, seed=seed), dtype=torch.float64)
    adj_t = [torch.as_tensor(a).long() for a in adj]
    targets = torch.cat([a[:, 1] for a in adj_t])
    out = []
    with torch.no_grad():
        for t in range(T):
            per_type = []
            for l, a in enumerate(adj_t):
                x = cur
                if e_hidden is not None:
                    for k in w["edge_mlps"][l]:
                        x = x @ k
                        out.append(x[torch.unique(a[:, 0])].reshape(-1))
                        x = f(x)
                per_type.append(x[a[:, 0]])
            new = A.segment_reduce(torch.cat(per_type), targets, V, agg)
            if a_hidden is None:
                out.append(new.reshape(-1))
            else:
                for k in w["aggr_mlp"]:
                    new = new @ k
                    out.append(new.reshape(-1))
                    new = f(new)
            cur = A.sparse_rgin_layer(cur, adj, 1, act, agg, weights={**{k: v for k, v in w.items() if k in ("edge_mlps", "aggr_mlp")},
                                                                      "ln_gamma": [w["ln_gamma"][t]], "ln_beta": [w["ln_beta"][t]]})
    x = torch.cat(out).numpy()
    return x[x != 0.0]


def kink_distance(x):
    return float(np.abs(x).min()) if x.size else np.inf


def small_cases():
    """(act, agg, e_hidden, a_hidden) of the small-graph parity test."""
    return [(act, agg, e, a) for act in ACTS for agg in AGGS for e in EDGE_MLPS for a in AGGR_MLPS]


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


def test_no_preactivation_at_a_kink():
    """float64 oracle on the seeded inputs of every small-graph case with a kinked activation (and of the d_in != d_out,
    two-timestep and restricted cases): no nonzero pre-activation lies within KINK_MARGIN of 0."""
    adj, V = tiny()
    closest = np.inf
    for act, agg, e, a in small_cases():
        if act not in KINKED:
            continue
        d = kink_distance(preacts(adj, V, 16, 16, 1, act, agg, e, a, SMALL_SEED))
        assert d > KINK_MARGIN, (act, agg, e, a, d)
        closest = min(closest, d)
    for act in KINKED:
        for e, a in ((1, None), (None, 1), (1, 1)):
            d = kink_distance(preacts(adj, V, 8, 16, 1, act, "mean", e, a, SMALL_SEED))
            assert d > KINK_MARGIN, ("d_in != d_out", act, e, a, d)
            closest = min(closest, d)
        d = kink_distance(preacts(adj, V, 16, 16, 2, act, "sum", 1, 1, SMALL_SEED))
        assert d > KINK_MARGIN, ("two timesteps", act, d)
        closest = min(closest, d)
    print("small graph, kinked activations: closest nonzero pre-activation to 0 is %.2e" % closest)


# ---------------------------------------------------------------- one case -----------------------------------------------
class Case:
    """Inputs of one RGIN layer on the device and the ctypes call of rgnn_rgin_backward."""

    def __init__(self, adj, V, D, act="elu", agg="sum", e_hidden=1, a_hidden=None, d_in=None, seed=SMALL_SEED, num_targets=None,
                 T=1, device=None, deferred=False):
        import torch
        from tf_gnn_samples_b200 import GraphPlan
        self.adj, self.V, self.D, self.T = adj, V, D, T
        self.d_in = D if d_in is None else d_in
        assert T == 1 or self.d_in == D
        self.act_name, self.act = act, get_activation(act)
        self.agg_name, self.agg = agg, get_aggregation_function(agg)
        self.e_hidden, self.a_hidden = e_hidden, a_hidden
        self.n_e = 0 if e_hidden is None else e_hidden + 1
        self.n_a = 0 if a_hidden is None else a_hidden + 1
        self.L = len(adj)
        self.dev = device
        self.w = make_weights(self.L, self.d_in, D, e_hidden, a_hidden, seed, T)
        self.h = node_states(V, self.d_in, seed=seed)
        self.plan = GraphPlan(adj, V, device=device, validate=not deferred)   # deferred: heavy counts stay on the device
        self.Vt = V if num_targets is None else num_targets
        if num_targets is not None:
            self.plan.set_num_targets(num_targets)
        self.g = np.random.default_rng(seed + 1).standard_normal((self.Vt, D)).astype(np.float32)
        t = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(device)
        self.th, self.tg = t(self.h), t(self.g)
        self.te = [t(k) for mlp in self.w.get("edge_mlps", []) for k in mlp]   # type-major
        self.ta = [t(k) for k in self.w.get("aggr_mlp", [])]
        self.tlg = [t(x) for x in self.w["ln_gamma"]]
        self.tlb = [t(x) for x in self.w["ln_beta"]]
        e_dims = [self.d_in] + [int(k.shape[1]) for k in self.w["edge_mlps"][0]] if self.n_e else []
        width = e_dims[-1] if self.n_e else self.d_in
        a_dims = [width] + [int(k.shape[1]) for k in self.w["aggr_mlp"]] if self.n_a else []
        self.e_dims = (ctypes.c_int32 * len(e_dims))(*e_dims) if e_dims else None
        self.a_dims = (ctypes.c_int32 * len(a_dims))(*a_dims) if a_dims else None
        self.e_shapes = [tuple(k.shape) for k in self.te]
        self.a_shapes = [tuple(k.shape) for k in self.ta]

    @property
    def lib(self):
        from tf_gnn_samples_b200.engine import load_library
        return load_library()

    def ws_bytes(self):
        return int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGIN_BACKWARD, self.d_in, self.D, max(self.n_e, self.n_a)))

    def new_outputs(self):
        import torch
        z = lambda s: torch.empty(s, dtype=torch.float32, device=self.dev)
        return {"gh": z((self.V, self.d_in)), "ge": [z(s) for s in self.e_shapes] if self.n_e else None,
                "ga": [z(s) for s in self.a_shapes] if self.n_a else None, "glg": z((self.D,)), "glb": z((self.D,))}

    def call(self, outs, h_t=None, g_t=None, t=0, ws="own", nbytes=None, stream=None, **over):
        """rgnn_rgin_backward for timestep t; `over` replaces raw arguments (pointers / ints).  ws="own": a workspace of the
        documented size from torch; otherwise the pointer (or None) and nbytes are passed as they are."""
        import torch
        ptr = lambda x: x if x is None or isinstance(x, int) else x.data_ptr()
        tab = lambda xs: None if not xs else (ctypes.c_void_p * len(xs))(*[ptr(x) for x in xs])
        if isinstance(ws, str):
            nbytes = self.ws_bytes()
            ws_t = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=self.dev)   # freed stream-ordered after the call
            ws = ws_t.data_ptr()
        if stream is None:
            stream = torch.cuda.current_stream(self.dev).cuda_stream
        a = dict(plan=self.plan.handle, h=ptr(self.th if h_t is None else h_t), d_in=self.d_in, D=self.D, ek=tab(self.te),
                 ed=self.e_dims, eh=-1 if self.e_hidden is None else self.e_hidden, ak=tab(self.ta), ad=self.a_dims,
                 ah=-1 if self.a_hidden is None else self.a_hidden, lg=ptr(self.tlg[t]), lb=ptr(self.tlb[t]), act=self.act,
                 agg=self.agg, ut=0, g=ptr(self.tg if g_t is None else g_t), gh=ptr(outs.get("gh")), ge=tab(outs.get("ge")),
                 ga=tab(outs.get("ga")), glg=ptr(outs.get("glg")), glb=ptr(outs.get("glb")))
        a.update(over)
        return self.lib.rgnn_rgin_backward(a["plan"], a["h"], a["d_in"], a["D"], a["ek"], a["ed"], a["eh"], a["ak"], a["ad"],
                                           a["ah"], a["lg"], a["lb"], a["act"], a["agg"], a["ut"], a["g"], a["gh"], a["ge"],
                                           a["ga"], a["glg"], a["glb"], ws, nbytes, stream)

    def forward(self, h, t=0, out=None, ws=None):
        """Timestep t forward through rgnn_rgin_forward (num_timesteps = 1)."""
        import torch
        from tf_gnn_samples_b200.engine import check
        if out is None:
            out = torch.zeros((self.V, self.D), dtype=torch.float32, device=self.dev)
        nb = int(self.lib.rgnn_workspace_bytes(self.plan.handle, LAYER_RGIN, self.d_in, self.D, max(self.n_e, self.n_a)))
        if ws is None:
            ws = torch.empty(max(nb, 256), dtype=torch.uint8, device=self.dev)
        tab = lambda xs: None if not xs else (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
        check(self.lib.rgnn_rgin_forward(self.plan.handle, h.data_ptr(), self.d_in, self.D, tab(self.te), self.e_dims,
                                         -1 if self.e_hidden is None else self.e_hidden, tab(self.ta), self.a_dims,
                                         -1 if self.a_hidden is None else self.a_hidden, self.tlg[t].data_ptr(),
                                         self.tlb[t].data_ptr(), self.act, self.agg, 0, 1, out.data_ptr(), ws.data_ptr(), nb,
                                         torch.cuda.current_stream(self.dev).cuda_stream))
        return out

    def grads(self):
        """All gradients of the T timesteps through the C ABI: forward per timestep, backward from the last one down."""
        import torch
        from tf_gnn_samples_b200.engine import check
        xs = [self.th]
        for t in range(self.T - 1):
            xs.append(self.forward(xs[-1], t))
        g = self.tg
        res = {}
        for t in reversed(range(self.T)):
            o = self.new_outputs()
            check(self.call(o, h_t=xs[t], g_t=g, t=t))
            g = o["gh"]
            for i in range(self.L * self.n_e):
                key = "d_E%d_%d" % (i // self.n_e, i % self.n_e)
                res[key] = res.get(key, 0) + o["ge"][i].double()
            for k in range(self.n_a):
                res["d_K%d" % k] = res.get("d_K%d" % k, 0) + o["ga"][k].double()
            res["d_gamma%d" % t], res["d_beta%d" % t] = o["glg"], o["glb"]
        res["d_h"] = g
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in res.items()}

    def _named(self, h, w):
        res = {"d_h": h.grad}
        for l, mlp in enumerate(w.get("edge_mlps", [])):
            for j, k in enumerate(mlp):
                res["d_E%d_%d" % (l, j)] = k.grad if k.grad is not None else torch_zeros_like(k)
        for j, k in enumerate(w.get("aggr_mlp", [])):
            res["d_K%d" % j] = k.grad
        for t in range(self.T):
            res["d_gamma%d" % t], res["d_beta%d" % t] = w["ln_gamma"][t].grad, w["ln_beta"][t].grad
        return res

    def oracle(self):
        """float64 autograd of oracle/ref_autograd on the GPU: d/d(everything) of sum(out[:Vt] * g)."""
        import torch
        def leaf(x):
            if isinstance(x, dict):
                return {k: leaf(v) for k, v in x.items()}
            if isinstance(x, (list, tuple)):
                return [leaf(v) for v in x]
            return torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
        with torch.device(self.dev):
            h = leaf(self.h)
            w = leaf(self.w)
            out = A.sparse_rgin_layer(h, self.adj, self.T, self.act_name, self.agg_name, weights=w)
            (out[: self.Vt] * torch.tensor(self.g, dtype=torch.float64)).sum().backward()
        return {k: v.detach().cpu().numpy() for k, v in self._named(h, w).items()}

    def python_route(self):
        """The Python training route (sparse_rgin_layer under torch autograd: gnns/_train.py)."""
        import tf_gnn_samples_b200 as G
        h = self.th.clone().requires_grad_(True)
        w = {"ln_gamma": [x.clone().requires_grad_(True) for x in self.tlg],
             "ln_beta": [x.clone().requires_grad_(True) for x in self.tlb]}
        if self.n_e:
            w["edge_mlps"] = [[self.te[l * self.n_e + j].clone().requires_grad_(True) for j in range(self.n_e)] for l in range(self.L)]
        if self.n_a:
            w["aggr_mlp"] = [x.clone().requires_grad_(True) for x in self.ta]
        out = G.sparse_rgin_layer(h, self.plan, self.D, self.T, self.act_name, self.agg_name, False, self.e_hidden, self.a_hidden,
                                  weights=w)
        (out[: self.Vt] * self.tg).sum().backward()
        return {k: v.detach().cpu().numpy() for k, v in self._named(h, w).items() if v is not None}


def torch_zeros_like(x):
    import torch
    return torch.zeros_like(x)


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
@pytest.mark.parametrize("a_hidden", AGGR_MLPS, ids=["aggr_none", "aggr_1"])
@pytest.mark.parametrize("e_hidden", EDGE_MLPS, ids=["edge_none", "edge_0", "edge_1", "edge_2"])
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("act", ACTS)
def test_small_graph_matches_float64_autograd(cuda_device, act, agg, e_hidden, a_hidden):
    adj, V = tiny()
    check_case(Case(adj, V, 16, act, agg, e_hidden, a_hidden, device=cuda_device),
               "tiny %s %s edge %s aggr %s" % (act, agg, e_hidden, a_hidden))


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["relu", "elu", "gelu"])
@pytest.mark.parametrize("e_hidden,a_hidden", [(1, None), (None, 1), (1, 1)])
def test_d_in_differs_from_d_out(cuda_device, act, e_hidden, a_hidden):
    """d_in = 8, d_out = 16: the edge MLP or the aggregation MLP maps the width."""
    adj, V = tiny()
    check_case(Case(adj, V, 16, act, "mean", e_hidden, a_hidden, d_in=8, device=cuda_device),
               "tiny d_in 8 -> 16 %s edge %s aggr %s" % (act, e_hidden, a_hidden))


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_two_timesteps_as_two_calls(cuda_device, act):
    adj, V = tiny()
    check_case(Case(adj, V, 16, act, "sum", 1, 1, T=2, device=cuda_device), "tiny %s two timesteps" % act)


@pytest.mark.gpu
def test_zipf_heavy_targets_and_sources_and_determinism(cuda_device):
    """The Zipf PPI-shaped graph at D = 256: heavy targets and heavy (source, type) segments; two calls are bit-identical."""
    import torch
    from tf_gnn_samples_b200.engine import check, launch_count
    adj, V = zipf_ppi()
    c = Case(adj, V, 256, "elu", "mean", 1, None, device=cuda_device)
    got = check_case(c, "zipf ppi D=256 elu")
    o1, o2 = c.new_outputs(), c.new_outputs()
    before = launch_count()
    check(c.call(o1))
    n1 = launch_count() - before
    check(c.call(o2))
    torch.cuda.synchronize()
    assert n1 == launch_count() - before - n1
    print("zipf ppi D=256: %d kernel launches per backward" % n1)
    assert torch.equal(o1["gh"], o2["gh"])
    assert all(torch.equal(a, b) for a, b in zip(o1["ge"], o2["ge"]))
    for k in ("glg", "glb"):
        assert torch.equal(o1[k], o2[k]), k
    assert np.array_equal(o1["gh"].cpu().numpy(), got["d_h"])


@pytest.mark.gpu
@pytest.mark.parametrize("e_hidden,a_hidden", [(1, None), (2, 1)])
def test_deferred_plan(cuda_device, e_hidden, a_hidden):
    """A plan built without a synchronisation (RGNN_PLAN_DEFERRED_CHECK) never read its heavy-target count back."""
    adj, V = zipf_ppi()
    check_case(Case(adj, V, 256, "tanh", "sqrt_n", e_hidden, a_hidden, deferred=True, device=cuda_device),
               "zipf ppi deferred plan edge %s aggr %s" % (e_hidden, a_hidden))


@pytest.mark.gpu
def test_qm9_rgin_full_size(cuda_device):
    """The QM9 RGIN configuration: the real 10,000 QM9 validation molecules with self-loop edges (L = 5), D = 128, ELU, sum,
    one edge-MLP hidden layer, no aggregation MLP."""
    adj, V = qm9_rgin()
    assert len(adj) == 5
    check_case(Case(adj, V, 128, "elu", "sum", 1, None, device=cuda_device),
               "qm9 rgin V=%d M=%d L=%d D=128" % (V, sum(a.shape[0] for a in adj), len(adj)))


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,e_hidden,a_hidden", [("tiny", 1, None), ("tiny", None, 1), ("tiny", 2, 1), ("zipf", 1, 1)])
def test_restricted_plan(cuda_device, graph_name, e_hidden, a_hidden):
    """num_targets < V: the gradient of the loss over the owned rows; the halo rows of d_h receive theirs."""
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    D = 16 if graph_name == "tiny" else 256
    act = "relu" if graph_name == "tiny" else "elu"
    nt = V * 2 // 3
    c = Case(adj, V, D, act, "mean", e_hidden, a_hidden, num_targets=nt, device=cuda_device)
    got = check_case(c, "%s edge %s aggr %s restricted to %d of %d targets" % (graph_name, e_hidden, a_hidden, nt, V),
                     python_route=False)
    assert np.abs(got["d_h"][nt:]).max() > 0


# ---------------------------------------------------------------- buffer contract ----------------------------------------
def guarded_case(c):
    """Guarded copies of the inputs and guarded outputs; returns (inputs, outputs)."""
    from test_buffer_contract_gpu import Guarded
    ins = {"h": Guarded.copy_of("h", c.th), "g": Guarded.copy_of("g", c.tg), "lg": Guarded.copy_of("lg", c.tlg[0]),
           "lb": Guarded.copy_of("lb", c.tlb[0])}
    ins.update({"e%d" % i: Guarded.copy_of("e%d" % i, x) for i, x in enumerate(c.te)})
    ins.update({"a%d" % i: Guarded.copy_of("a%d" % i, x) for i, x in enumerate(c.ta)})
    outs = {"gh": Guarded("gh", c.V * c.d_in * 4, c.dev), "glg": Guarded("glg", c.D * 4, c.dev),
            "glb": Guarded("glb", c.D * 4, c.dev)}
    outs.update({"ge%d" % i: Guarded("ge%d" % i, int(np.prod(s)) * 4, c.dev) for i, s in enumerate(c.e_shapes)})
    outs.update({"ga%d" % i: Guarded("ga%d" % i, int(np.prod(s)) * 4, c.dev) for i, s in enumerate(c.a_shapes)})
    return ins, outs


def guarded_call(c, ins, outs, ws_ptr, nbytes, drop=(), **over):
    import torch
    tab = lambda pre, d, n: None if n == 0 else (ctypes.c_void_p * n)(*[d["%s%d" % (pre, i)].ptr for i in range(n)])
    ne, na = c.L * c.n_e, c.n_a
    p = dict(h=ins["h"].ptr, g=ins["g"].ptr, lg=ins["lg"].ptr, lb=ins["lb"].ptr, ek=tab("e", ins, ne), ak=tab("a", ins, na),
             gh=outs["gh"].ptr, ge=tab("ge", outs, ne), ga=tab("ga", outs, na), glg=outs["glg"].ptr, glb=outs["glb"].ptr)
    for k in drop:
        p[k] = None
    p.update(over)
    return c.call({}, ws=ws_ptr, nbytes=nbytes, stream=torch.cuda.current_stream(c.dev).cuda_stream, **p)


CONTRACT = [("tiny", 1, 1), ("tiny", None, None), ("zipf", 2, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("graph_name,e_hidden,a_hidden", CONTRACT)
def test_buffer_contract(cuda_device, graph_name, e_hidden, a_hidden):
    import torch
    from test_buffer_contract_gpu import Guarded, OUT_POISON, WS_POISON, poison_bits
    from tf_gnn_samples_b200.engine import launch_count
    adj, V = tiny() if graph_name == "tiny" else zipf_ppi()
    D = 20 if graph_name == "tiny" else 96
    c = Case(adj, V, D, "tanh", "mean", e_hidden, a_hidden, device=cuda_device)
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
    what = "%s edge %s aggr %s" % (graph_name, e_hidden, a_hidden)
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
                assert np.array_equal(outs["gh"].f32((V, D)).cpu().numpy(), want["d_h"])
                assert np.array_equal(outs["glg"].f32((D,)).cpu().numpy(), want["d_gamma0"])
                if c.n_e:
                    assert np.array_equal(outs["ge0"].f32(c.e_shapes[0]).cpu().numpy(), want["d_E0_0"].astype(np.float32))
                if c.n_a:
                    assert np.array_equal(outs["ga0"].f32(c.a_shapes[0]).cpu().numpy(), want["d_K0"].astype(np.float32))
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
    for drop in (("gh",), ("ge",), ("ga",), ("glg",), ("glb",), ("gh", "ge", "ga", "glg", "glb")):
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
    i32 = lambda xs: (ctypes.c_int32 * len(xs))(*xs)
    refusals = [("use_target_state_as_input", dict(ut=1), E_UNSUPPORTED), ("aggregation", dict(agg=1), E_UNSUPPORTED),
                ("aggregation", dict(agg=9), E_INVALID), ("activation", dict(act=99), E_INVALID),
                ("d_in / d_out", dict(D=D + 2), E_INVALID), ("d_out 516", dict(D=516), E_UNSUPPORTED),
                ("plan", dict(plan=None), E_INVALID), ("node_embeddings", dict(h=None), E_INVALID),
                ("grad_out", dict(g=None), E_INVALID), ("ln_gamma", dict(lg=None), E_INVALID), ("ln_beta", dict(lb=None), E_INVALID),
                ("node_embeddings", dict(h=ins["h"].ptr + 4), E_INVALID), ("ln_beta", dict(lb=ins["lb"].ptr + 4), E_INVALID),
                ("grad_ln_gamma", dict(glg=outs["glg"].ptr + 4), E_INVALID),
                ("grad_node_embeddings", dict(gh=outs["gh"].ptr + 4), E_INVALID),
                ("alias", dict(gh=ins["h"].ptr), E_INVALID), ("alias", dict(gh=ins["g"].ptr), E_INVALID)]
    if c.n_e:
        wide = [D] + [3 * D] * c.n_e
        bad0 = [D + 4] + list(c.e_dims)[1:]
        refusals += [("edge_mlp_kernels", dict(ek=None), E_INVALID), ("edge_mlp_dims", dict(ed=None), E_INVALID),
                     ("edge_mlp_dims[0]", dict(ed=i32(bad0)), E_INVALID),
                     ("edge MLP layer 0", dict(ed=i32(wide), ad=i32([3 * D] + list(c.a_dims)[1:]) if c.n_a else None), E_UNSUPPORTED),
                     ("edge MLP kernel 0", dict(ek=(ctypes.c_void_p * (c.L * c.n_e))(*([None] + [ins["e%d" % i].ptr
                                                                                           for i in range(1, c.L * c.n_e)]))), E_INVALID),
                     ("grad edge MLP kernel 0", dict(ge=(ctypes.c_void_p * (c.L * c.n_e))(*([outs["ge0"].ptr + 4] + [
                         outs["ge%d" % i].ptr for i in range(1, c.L * c.n_e)]))), E_INVALID)]
    if c.n_a:
        refusals += [("aggr_kernels", dict(ak=None), E_INVALID), ("aggr_dims", dict(ad=None), E_INVALID),
                     ("aggr_dims", dict(ad=i32(list(c.a_dims)[:-1] + [D + 4])), E_INVALID),
                     ("grad aggregation MLP kernel 0", dict(ga=(ctypes.c_void_p * c.n_a)(*([None] + [outs["ga%d" % i].ptr
                                                                                               for i in range(1, c.n_a)]))), E_INVALID)]
    else:
        refusals += [("no aggregation MLP maps it", dict(d_in=D - 4, ek=None, ed=None, eh=-1), E_INVALID)]
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
@pytest.mark.parametrize("e_hidden,a_hidden", [(1, None), (None, 1)])
def test_cuda_graph_replay_of_forward_and_backward(cuda_device, e_hidden, a_hidden):
    import torch
    from tf_gnn_samples_b200.engine import check
    adj, V = zipf_ppi()
    c = Case(adj, V, 64, "gelu", "mean", e_hidden, a_hidden, device=cuda_device)
    cap = c.new_outputs()
    y_cap = torch.empty((V, c.D), dtype=torch.float32, device=cuda_device)
    nb_f = int(c.lib.rgnn_workspace_bytes(c.plan.handle, LAYER_RGIN, c.d_in, c.D, max(c.n_e, c.n_a)))
    ws_f = torch.empty(nb_f, dtype=torch.uint8, device=cuda_device)
    c.forward(c.th, 0, y_cap, ws_f)
    check(c.call(cap))                                    # eager first: builds the reverse index
    nbytes = c.ws_bytes()
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda_device)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.forward(c.th, 0, y_cap, ws_f)
        rc = c.call(cap, ws=ws.data_ptr(), nbytes=nbytes)
    assert rc == 0
    rng = np.random.default_rng(77)
    c.th.copy_(torch.as_tensor(np.tanh(rng.standard_normal(tuple(c.th.shape))).astype(np.float32)))
    c.tg.copy_(torch.as_tensor(rng.standard_normal(tuple(c.tg.shape)).astype(np.float32)))
    for x in c.te + c.ta + c.tlg:
        x.mul_(0.75)
    graph.replay()
    torch.cuda.synchronize()
    eager = c.new_outputs()
    y_eager = c.forward(c.th)
    check(c.call(eager))
    torch.cuda.synchronize()
    assert torch.equal(y_cap, y_eager)
    for k in ("ge", "ga"):
        if cap[k] is not None:
            assert all(torch.equal(a, b) for a, b in zip(cap[k], eager[k])), k
    for k in ("gh", "glg", "glb"):
        assert torch.equal(cap[k], eager[k]), k
    c.h, c.g = c.th.cpu().numpy(), c.tg.cpu().numpy()
    if c.n_e:
        c.w["edge_mlps"] = [[c.te[l * c.n_e + j].cpu().numpy() for j in range(c.n_e)] for l in range(c.L)]
    if c.n_a:
        c.w["aggr_mlp"] = [x.cpu().numpy() for x in c.ta]
    c.w["ln_gamma"] = [x.cpu().numpy() for x in c.tlg]
    want = c.oracle()
    assert rel(cap["gh"].cpu().numpy(), want["d_h"]) <= TOL
    assert rel(cap["glg"].cpu().numpy(), want["d_gamma0"]) <= TOL
    # a first backward on a fresh plan refuses under capture, recording nothing
    fresh = Case(adj, V, 64, "gelu", "mean", e_hidden, a_hidden, device=cuda_device)
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
EXAMPLE = os.path.join(ROOT, "examples", "c_rgin_train.c")
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
        exe = os.path.join(out_dir, "c_rgin_train")
        cmd += ["-o", exe, "-L", lib_dir, "-lrgnn", "-Wl,-rpath," + lib_dir, "-L", os.path.join(CUDA_HOME, "lib64"), "-lcudart",
                "-Wl,-rpath," + os.path.join(CUDA_HOME, "lib64"), "-lm"]
    else:
        exe = os.path.join(out_dir, "c_rgin_train.o")
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
    """What examples/c_rgin_train.c builds, drawn in the same order: 8 molecules of 9 atoms, L = 4, 40 bonds per type, D = 16,
    one edge-MLP hidden layer."""
    G, ATOMS, L, E, D, NE = 8, 9, 4, 40, 16, 2
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
    ew = [sym(D * D, 0.5).reshape(D, D) for _ in range(L * NE)]
    gamma = np.array([np.float32(1.0) + np.float32(0.2) * (np.float32(2.0) * r.uniform() - np.float32(1.0)) for _ in range(D)],
                     np.float32)
    beta = sym(D, 0.2)
    target = sym(V * D, 1.0).reshape(V, D)
    return adj, V, D, h, ew, gamma, beta, target


@pytest.mark.gpu
def test_c_example_trains(cuda_device, tmp_path):
    """The C host's losses decrease, and its first loss is the same forward through ctypes."""
    import torch
    exe = compile_example(str(tmp_path), link=True)
    res = subprocess.run([exe, "6"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    losses = [float(x) for x in res.stdout.split()]
    print("c_rgin_train losses:", losses)
    assert len(losses) == 6 and all(b < a for a, b in zip(losses, losses[1:])), losses
    adj, V, D, h, ew, gamma, beta, target = example_inputs()
    c = Case(adj, V, D, "relu", "sum", 1, None, device=cuda_device)
    d = lambda x: torch.as_tensor(x).to(cuda_device)
    c.th, c.te, c.tlg, c.tlb = d(h), [d(x) for x in ew], [d(gamma)], [d(beta)]
    y = c.forward(c.th).cpu().numpy().astype(np.float64)
    loss = 0.5 * np.sum((y - target) ** 2) / V
    assert abs(loss - losses[0]) <= 1e-5 * max(1.0, abs(loss)), (loss, losses[0])


# ---------------------------------------------------------------- sharded training from C calls --------------------------
SHARDED = [dict(id="w2_halo_graph", world=2, plan="halo_graph"), dict(id="w4_halo_graph", world=4, plan="halo_graph"),
           dict(id="w2_training_plan", world=2, plan="training_plan")]
SHARDED_D, SHARDED_LAYERS, SHARDED_ACT, SHARDED_AGG = 64, 3, "elu", "mean"


def sharded_graph():
    from test_sharded_layers_gpu import TRAIN_ZIPF, graph
    return graph(TRAIN_ZIPF)


def sharded_inputs():
    adj, _, V = sharded_graph()
    L, D = len(adj), SHARDED_D
    h = node_states(V, D, seed=21)
    ws = [make_weights(L, D, D, 1, None, 31 + 7 * t) for t in range(SHARDED_LAYERS)]
    proj = np.random.default_rng(22).standard_normal((V, D)).astype(np.float32)
    return h, ws, proj


def sharded_step(sgs, streams, plans, h_own, wt, projs, exchange=True):
    """The loop of INTEGRATION.md section 2c on virtual ranks, every layer call through the C ABI.  Forward per layer:
    owned rows into state buffer t % 2, rgnn_halo_exchange, a copy of the layer's local input (halo rows included: the
    backward recomputes the forward from it), rgnn_rgin_forward.  Backward from the last layer down: rgnn_rgin_backward on
    the local graph -> d_local [n_local, D], then rgnn_halo_exchange_backward -> d of the owned input rows.  Every phase is
    enqueued for all ranks before the next.  exchange=False: no exchange, halo rows zero and their gradients dropped (the
    warm-up).  Returns per rank the owned output, d_h and the per-layer weight gradients."""
    import torch
    from tf_gnn_samples_b200.engine import check, load_library
    lib = load_library()
    L, D, R = len(wt[0]["e"]) // 2, SHARDED_D, len(sgs)
    act, agg = get_activation(SHARDED_ACT), get_aggregation_function(SHARDED_AGG)
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    dims = (ctypes.c_int32 * 3)(D, D, D)
    wss = []
    for sg, s, pl in zip(sgs, streams, plans):
        with torch.cuda.stream(s):
            nb = max(int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGIN, D, D, 2)),
                     int(lib.rgnn_workspace_bytes(pl.handle, LAYER_RGIN_BACKWARD, D, D, 2)))
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
                check(lib.rgnn_rgin_forward(pl.handle, inputs[r][t].data_ptr(), D, D, tab(w["e"]), dims, 1, None, None, -1,
                                            w["lg"].data_ptr(), w["lb"].data_ptr(), act, agg, 0, 1, y.data_ptr(),
                                            wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
                x[r] = y[: sg.n_own]
    g = list(projs)
    grads = [[None] * SHARDED_LAYERS for _ in range(R)]
    for t in reversed(range(SHARDED_LAYERS)):
        d_local = []
        for r, (sg, s, pl) in enumerate(zip(sgs, streams, plans)):
            with torch.cuda.stream(s):
                z = lambda *shape: torch.empty(shape, dtype=torch.float32, device=sg.device)
                o = {"gh": z(sg.n_local, D), "ge": [z(D, D) for _ in range(2 * L)], "glg": z(D), "glb": z(D)}
                w = wt[t]
                check(lib.rgnn_rgin_backward(pl.handle, inputs[r][t].data_ptr(), D, D, tab(w["e"]), dims, 1, None, None, -1,
                                             w["lg"].data_ptr(), w["lb"].data_ptr(), act, agg, 0, g[r].data_ptr(),
                                             o["gh"].data_ptr(), tab(o["ge"]), None, o["glg"].data_ptr(), o["glb"].data_ptr(),
                                             wss[r][0].data_ptr(), wss[r][1], s.cuda_stream))
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
    wt = [{"e": [d(k) for mlp in w["edge_mlps"] for k in mlp], "lg": d(w["ln_gamma"][0]), "lb": d(w["ln_beta"][0])} for w in ws]
    h_own = [d(h[sg.lo:sg.hi]) for sg in sgs]
    projs = [d(proj[sg.lo:sg.hi]) for sg in sgs]
    torch.cuda.synchronize()
    x, g, grads = sharded_step(sgs, streams, plans, h_own, wt, projs, exchange)
    res = {"out": np.concatenate([y.cpu().numpy() for y in x]), "d_h": np.concatenate([y.cpu().numpy() for y in g])}
    L = len(ws[0]["edge_mlps"])
    for t in range(SHARDED_LAYERS):
        for i in range(2 * L):
            res["d_E%d_%d_%d" % (t, i // 2, i % 2)] = sum(gr[t]["ge"][i].double().cpu().numpy() for gr in grads)
        res["d_gamma%d" % t] = sum(gr[t]["glg"].double().cpu().numpy() for gr in grads)
        res["d_beta%d" % t] = sum(gr[t]["glb"].double().cpu().numpy() for gr in grads)
    return res


def sharded_truth(h, ws, proj, device):
    """float64 autograd of the whole-graph stack on the GPU."""
    import torch
    adj, _, _ = sharded_graph()
    with torch.device(device):
        f64 = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=True)
        x = h64 = f64(h)
        w64 = [{"edge_mlps": [[f64(k) for k in mlp] for mlp in w["edge_mlps"]], "ln_gamma": [f64(w["ln_gamma"][0])],
                "ln_beta": [f64(w["ln_beta"][0])]} for w in ws]
        for w in w64:
            x = A.sparse_rgin_layer(x, adj, 1, SHARDED_ACT, SHARDED_AGG, weights=w)
        (x * torch.tensor(proj, dtype=torch.float64)).sum().backward()
    res = {"out": x.detach().cpu().numpy(), "d_h": h64.grad.cpu().numpy()}
    for t, w in enumerate(w64):
        for l, mlp in enumerate(w["edge_mlps"]):
            for j, k in enumerate(mlp):
                res["d_E%d_%d_%d" % (t, l, j)] = k.grad.cpu().numpy()
        res["d_gamma%d" % t] = w["ln_gamma"][0].grad.cpu().numpy()
        res["d_beta%d" % t] = w["ln_beta"][0].grad.cpu().numpy()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHARDED, ids=[c["id"] for c in SHARDED])
def test_sharded_training_from_c_calls(cuda_device, case):
    """A 3-layer RGIN stack (one edge-MLP hidden layer, ELU, one timestep per layer) over virtual ranks, every layer forward
    and backward through the C ABI on the rank's local graph (rgnn_halo_plan_graph, or the GraphPlan of training_plan()),
    halo gradients through rgnn_halo_exchange_backward: the owned outputs, d_h and the rank-summed weight gradients equal
    float64 autograd on the whole graph; a repeat is bit identical."""
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

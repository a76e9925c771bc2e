"""One RGAT training step (forward + the backward of one timestep) two ways, on the same inputs:

  * python: sparse_rgat_layer under torch autograd (the composed training route of gnns/_train.py: per-edge logits, softmax
    statistics from scatter_reduce / index_add);
  * c_abi:  rgnn_rgat_forward + rgnn_rgat_backward through ctypes, with one preallocated workspace.

Workloads: BASELINE config 4 (one PPI-shaped graph, V = 2,245, M = 120,245, L = 3, D = 256, 8 heads, tanh) and a Zipf PPI
shape (V = 6,000, Zipf-skewed targets, so hub targets and hub (source, type) segments run the one-CTA-per-segment kernels).
For each it reports the device time per step with a cold L2 (a 256 MiB buffer is overwritten before every step, outside
the timed events) as the median over `--steps` steps after `--warmup` warm-up steps, torch.cuda.max_memory_allocated during
the timed steps of each route, and the max-norm relative difference between the two routes' gradients.  Prints one JSON
line per workload with the card's name and power limit, read in the same run; writes nothing."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_batching import card  # noqa: E402

FLUSH_BYTES = 256 << 20


def workloads():
    from tf_gnn_samples_b200 import batching
    yield "config4_rgat", batching.ppi_like_batch(), 256, 8, "tanh"
    yield "zipf_ppi_rgat", batching.ppi_like_batch(num_nodes=6000, num_links=24000, seed=45, zipf_targets=True), 256, 8, "tanh"


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / (s if s > 0 else 1.0))


def run(name, b, D, K, act, steps, warmup):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    from tf_gnn_samples_b200.utils import LAYER_RGAT, LAYER_RGAT_BACKWARD, get_activation
    dev = torch.device("cuda", 0)
    lib = load_library()
    V, L = b.num_nodes, len(b.adjacency_lists)
    plan = G.GraphPlan(b.adjacency_lists, V, device=dev)
    rng = np.random.default_rng(0)
    h = torch.as_tensor(np.tanh(rng.standard_normal((V, D))).astype(np.float32)).to(dev)
    g = torch.as_tensor(rng.standard_normal((V, D)).astype(np.float32)).to(dev)
    w = W.to_torch(W.rgat_weights(L, D, D, 7), dev)
    ws, atts = [x.contiguous() for x in w["edge_weights"]], [x.contiguous() for x in w["attention"]]
    stream = torch.cuda.current_stream(dev)
    flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device=dev)

    def timed(step):
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for start, end in ev:
            flush.fill_(1)                                   # evict the step's tables from L2
            start.record()
            step()
            end.record()
        torch.cuda.synchronize()
        return float(np.median([s.elapsed_time(e) for s, e in ev])), torch.cuda.max_memory_allocated(dev)

    # python route
    hp = h.clone().requires_grad_(True)
    wp = {"edge_weights": [x.clone().requires_grad_(True) for x in ws], "attention": [x.clone().requires_grad_(True) for x in atts]}
    leaves = [hp] + wp["edge_weights"] + wp["attention"]

    def py_step():
        for x in leaves:
            x.grad = None
        out = G.sparse_rgat_layer(hp, plan, D, K, 1, act, weights=wp)
        out.backward(g)
    py_ms, py_mem = timed(py_step)
    py_grads = [x.grad.clone() for x in leaves]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # C-ABI route
    nbytes = max(int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGAT, D, D, 0)),
                 int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGAT_BACKWARD, D, D, 0)))
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = torch.empty((V, D), dtype=torch.float32, device=dev)
    gh = torch.empty_like(h)
    gws, gas = [torch.empty_like(x) for x in ws], [torch.empty_like(x) for x in atts]
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    wt, at, gwt, gat = tab(ws), tab(atts), tab(gws), tab(gas)
    a = get_activation(act)

    def c_step():
        check(lib.rgnn_rgat_forward(plan.handle, h.data_ptr(), D, D, wt, at, K, a, 1, out.data_ptr(), work.data_ptr(), nbytes,
                                    stream.cuda_stream))
        check(lib.rgnn_rgat_backward(plan.handle, h.data_ptr(), D, D, wt, at, K, a, g.data_ptr(), gh.data_ptr(), gwt, gat,
                                     work.data_ptr(), nbytes, stream.cuda_stream))
    c_ms, c_mem = timed(c_step)
    c_grads = [gh] + gws + gas
    diff = max(rel(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(c_grads, py_grads))
    m = sum(int(x.shape[0]) for x in b.adjacency_lists)
    return {"workload": name, "V": V, "M": m, "L": L, "D": D, "heads": K, "activation": act, "steps": steps, "warmup": warmup,
            "l2": "cold", "python_ms_per_step": round(py_ms, 4), "c_abi_ms_per_step": round(c_ms, 4),
            "speedup": round(py_ms / c_ms, 3), "python_max_memory_allocated_bytes": int(py_mem),
            "c_abi_max_memory_allocated_bytes": int(c_mem), "max_rel_grad_difference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgat_training.py needs a CUDA device")
    info = card()
    for name, b, D, K, act in workloads():
        res = run(name, b, D, K, act, args.steps, args.warmup)
        res.update(card=info["name"], power_limit=info["power_limit"])
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

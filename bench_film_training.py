"""One GNN-FiLM training step (forward + the backward of one timestep) two ways, on the same inputs:

  * python: sparse_gnn_film_layer under torch autograd (the composed training route of gnns/_train.py);
  * c_abi:  rgnn_film_forward + rgnn_film_backward through ctypes, with one preallocated workspace.

Workloads: BASELINE config 5 (VarMisuse-shaped random graph, V = 50,000, M = 1,000,000, L = 6, D = 128) and the PPI
shape (one graph, V = 2,245, M = 120,245, L = 3, D = 256).  For each it reports the device time per step from CUDA events
over `--steps` steps after `--warmup` warm-up steps, torch.cuda.max_memory_allocated during the timed steps of each route,
and the max-norm relative difference between the two routes' gradients.  Prints one JSON line per workload and the card's
name and power limit, read in the same run; writes nothing."""
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


def workloads():
    from tf_gnn_samples_b200 import batching
    b = batching.varmisuse_like_batch()
    yield "config5_film", b, 128, "tanh"
    b = batching.ppi_like_batch(num_graphs=1, num_nodes=2245, num_links=59000, seed=0)
    yield "ppi_film", b, 256, "tanh"


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / (s if s > 0 else 1.0))


def run(name, b, D, act, steps, warmup):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    from tf_gnn_samples_b200.utils import LAYER_FILM, LAYER_FILM_BACKWARD, get_activation, get_aggregation_function
    dev = torch.device("cuda", 0)
    lib = load_library()
    V, L = b.num_nodes, len(b.adjacency_lists)
    plan = G.GraphPlan(b.adjacency_lists, V, device=dev)
    rng = np.random.default_rng(0)
    h = torch.as_tensor(np.tanh(rng.standard_normal((V, D))).astype(np.float32)).to(dev)
    g = torch.as_tensor(rng.standard_normal((V, D)).astype(np.float32)).to(dev)
    cnt = torch.as_tensor(b.type_to_num_incoming_edges).to(dev)
    w = W.to_torch(W.film_weights(L, D, D, 7, random_ln=True), dev)
    ws, fs = list(w["edge_weights"]), list(w["film_weights"])
    lng, lnb = w["ln_gamma"][0].contiguous(), w["ln_beta"][0].contiguous()
    stream = torch.cuda.current_stream(dev)

    def timed(step):
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(steps):
            step()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / steps, torch.cuda.max_memory_allocated(dev)

    # python route
    hp = h.clone().requires_grad_(True)
    wp = {"edge_weights": [x.clone().requires_grad_(True) for x in ws], "film_weights": [x.clone().requires_grad_(True) for x in fs],
          "ln_gamma": lng.clone().requires_grad_(True), "ln_beta": lnb.clone().requires_grad_(True)}
    leaves = [hp] + wp["edge_weights"] + wp["film_weights"] + [wp["ln_gamma"], wp["ln_beta"]]

    def py_step():
        for x in leaves:
            x.grad = None
        out = G.sparse_gnn_film_layer(hp, plan, cnt, D, 1, act, "sum", True, weights=wp)
        out.backward(g)
    py_ms, py_mem = timed(py_step)
    py_grads = [x.grad.clone() for x in leaves]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # C-ABI route
    nbytes = max(int(lib.rgnn_workspace_bytes(plan.handle, LAYER_FILM, D, D, 0)),
                 int(lib.rgnn_workspace_bytes(plan.handle, LAYER_FILM_BACKWARD, D, D, 0)))
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = torch.empty((V, D), dtype=torch.float32, device=dev)
    gh = torch.empty_like(h)
    gws, gfs = [torch.empty_like(x) for x in ws], [torch.empty_like(x) for x in fs]
    glg, glb = torch.empty_like(lng), torch.empty_like(lnb)
    tab = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    wt, ft, gwt, gft = tab(ws), tab(fs), tab(gws), tab(gfs)
    a, agg = get_activation(act), get_aggregation_function("sum")

    def c_step():
        check(lib.rgnn_film_forward(plan.handle, h.data_ptr(), D, D, wt, ft, cnt.data_ptr(), lng.data_ptr(), lnb.data_ptr(), a, agg,
                                    1, 1, out.data_ptr(), work.data_ptr(), nbytes, stream.cuda_stream))
        check(lib.rgnn_film_backward(plan.handle, h.data_ptr(), D, D, wt, ft, cnt.data_ptr(), lng.data_ptr(), lnb.data_ptr(), a,
                                     agg, 1, g.data_ptr(), gh.data_ptr(), gwt, gft, glg.data_ptr(), glb.data_ptr(),
                                     work.data_ptr(), nbytes, stream.cuda_stream))
    c_ms, c_mem = timed(c_step)
    c_grads = [gh] + gws + gfs + [glg, glb]
    diff = max(rel(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(c_grads, py_grads))
    m = sum(int(x.shape[0]) for x in b.adjacency_lists)
    return {"workload": name, "V": V, "M": m, "L": L, "D": D, "activation": act, "aggregation": "sum", "normalize": True,
            "steps": steps, "warmup": warmup,
            "python_ms_per_step": round(py_ms, 4), "c_abi_ms_per_step": round(c_ms, 4), "speedup": round(py_ms / c_ms, 3),
            "python_max_memory_allocated_bytes": int(py_mem), "c_abi_max_memory_allocated_bytes": int(c_mem),
            "max_rel_grad_difference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_film_training.py needs a CUDA device")
    info = card()
    for name, b, D, act in workloads():
        res = run(name, b, D, act, args.steps, args.warmup)
        res.update(card=info["name"], power_limit=info["power_limit"])
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

"""One RGIN training step (one timestep forward + backward) two ways, on the same inputs:

  * python: sparse_rgin_layer under torch autograd (the composed training route of gnns/_train.py, which keeps the edge MLP's
    intermediates for autograd);
  * c_abi:  rgnn_rgin_forward + rgnn_rgin_backward through ctypes, with one preallocated workspace.

Workloads (source-only messages, one edge-MLP hidden layer, sum aggregation, no aggregation MLP: the reference's RGIN
defaults):
  * qm9_rgin: the real structure of the 10,000 QM9 validation molecules from tests/golden/qm9_valid_structure.npz with
    self-loop edges (L = 5), D = 128, ELU;
  * ppi_rgin: the PPI-shaped batch of batching.ppi_like_batch (L = 3), D = 256, ReLU.
For each it reports the device time per step with a cold L2 (a 256 MiB buffer is overwritten before every step, outside the
timed events) as the median over `--steps` steps after `--warmup` warm-up steps, torch.cuda.max_memory_allocated during the
timed steps of each route, and the max-norm relative difference between the two routes' gradients.  Prints one JSON line
with the card's name and power limit, read in the same run; writes nothing."""
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
SEED = 5


def workloads():
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), add_self_loop_edges=True)
    yield "qm9_rgin", b, 128, "elu"
    yield "ppi_rgin", batching.ppi_like_batch(), 256, "relu"


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / (s if s > 0 else 1.0))


def run(name, b, D, act, steps, warmup):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    from tf_gnn_samples_b200.utils import AGG_SUM, LAYER_RGIN, LAYER_RGIN_BACKWARD, get_activation
    dev = torch.device("cuda", 0)
    lib = load_library()
    V, L = b.num_nodes, len(b.adjacency_lists)
    plan = G.GraphPlan(b.adjacency_lists, V, device=dev)
    h = torch.as_tensor(np.tanh(np.random.default_rng(SEED).standard_normal((V, D))).astype(np.float32)).to(dev)
    g = torch.as_tensor(np.random.default_rng(SEED + 1).standard_normal((V, D)).astype(np.float32)).to(dev)
    w = W.to_torch(W.rgin_weights(L, D, D, 1, None, seed=SEED + 11, random_ln=True), dev)
    ek = [k.contiguous() for mlp in w["edge_mlps"] for k in mlp]     # type-major
    lg, lb = w["ln_gamma"][0].contiguous(), w["ln_beta"][0].contiguous()
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
    wp = {"edge_mlps": [[ek[l * 2 + j].clone().requires_grad_(True) for j in range(2)] for l in range(L)],
          "ln_gamma": [lg.clone().requires_grad_(True)], "ln_beta": [lb.clone().requires_grad_(True)]}
    leaves = [hp] + [k for mlp in wp["edge_mlps"] for k in mlp] + wp["ln_gamma"] + wp["ln_beta"]

    def py_step():
        for x in leaves:
            x.grad = None
        out = G.sparse_rgin_layer(hp, plan, D, 1, act, "sum", False, 1, None, weights=wp)
        out.backward(g)
    py_ms, py_mem = timed(py_step)
    py_grads = [x.grad.clone() for x in leaves]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # C-ABI route
    nbytes = max(int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGIN, D, D, 2)),
                 int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGIN_BACKWARD, D, D, 2)))
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    y = torch.empty_like(h)
    dh = torch.empty_like(h)
    gek = [torch.empty_like(k) for k in ek]
    glg, glb = torch.empty_like(lg), torch.empty_like(lb)
    tab = lambda xs_: (ctypes.c_void_p * len(xs_))(*[x.data_ptr() for x in xs_])
    ekt, gekt = tab(ek), tab(gek)
    dims = (ctypes.c_int32 * 3)(D, D, D)
    a = get_activation(act)

    def c_step():
        check(lib.rgnn_rgin_forward(plan.handle, h.data_ptr(), D, D, ekt, dims, 1, None, None, -1, lg.data_ptr(), lb.data_ptr(),
                                    a, AGG_SUM, 0, 1, y.data_ptr(), work.data_ptr(), nbytes, stream.cuda_stream))
        check(lib.rgnn_rgin_backward(plan.handle, h.data_ptr(), D, D, ekt, dims, 1, None, None, -1, lg.data_ptr(), lb.data_ptr(),
                                     a, AGG_SUM, 0, g.data_ptr(), dh.data_ptr(), gekt, None, glg.data_ptr(), glb.data_ptr(),
                                     work.data_ptr(), nbytes, stream.cuda_stream))
    c_ms, c_mem = timed(c_step)
    c_grads = [dh] + gek + [glg, glb]
    diff = max(rel(x.cpu().numpy(), y_.cpu().numpy()) for x, y_ in zip(c_grads, py_grads))
    m = sum(int(x.shape[0]) for x in b.adjacency_lists)
    plan.close()
    return {"workload": name, "V": V, "M": m, "L": L, "D": D, "activation": act, "edge_mlp_hidden_layers": 1,
            "python_ms_per_step": round(py_ms, 4), "c_abi_ms_per_step": round(c_ms, 4), "speedup": round(py_ms / c_ms, 3),
            "python_max_memory_allocated_bytes": int(py_mem), "c_abi_max_memory_allocated_bytes": int(c_mem),
            "max_rel_grad_difference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgin_training.py needs a CUDA device")
    info = card()
    res = {"steps": args.steps, "warmup": args.warmup, "l2": "cold",
           "workloads": [run(name, b, D, act, args.steps, args.warmup) for name, b, D, act in workloads()],
           "card": info["name"], "power_limit": info["power_limit"]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

"""One GGNN training step (4 GRU timesteps forward + backward) two ways, on the same inputs:

  * python: sparse_ggnn_layer under torch autograd (the composed training route of gnns/_train.py, which keeps every
    timestep's intermediates for autograd);
  * c_abi:  4 x rgnn_ggnn_forward (num_timesteps = 1, keeping each timestep's input) + 4 x rgnn_ggnn_backward from the last
    timestep down through ctypes, with one preallocated workspace; the timesteps' weight gradients are summed on the device.

Workload: BASELINE config 3 at full size (the real structure of the 10,000 QM9 validation molecules from
tests/golden/qm9_valid_structure.npz, L = 4, D = 128, GRU, tanh, 4 timesteps).  It reports the device time per step with a
cold L2 (a 256 MiB buffer is overwritten before every step, outside the timed events) as the median over `--steps` steps
after `--warmup` warm-up steps, torch.cuda.max_memory_allocated during the timed steps of each route, and the max-norm
relative difference between the two routes' gradients.  Prints one JSON line with the card's name and power limit, read in
the same run; writes nothing."""
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
SEED, KERNEL_SCALE = 6, 0.5


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / (s if s > 0 else 1.0))


def config3():
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), add_self_loop_edges=False)
    return b


def run(b, D, T, act, steps, warmup):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    from tf_gnn_samples_b200.utils import AGG_SUM, CELL_GRU, LAYER_GGNN, LAYER_GGNN_BACKWARD, get_activation
    dev = torch.device("cuda", 0)
    lib = load_library()
    V, L = b.num_nodes, len(b.adjacency_lists)
    plan = G.GraphPlan(b.adjacency_lists, V, device=dev)
    # the inputs of tests/test_ggnn_training_through_c_abi_gpu.py::test_config3_full_size: no gate pre-activation within 1e-5
    # of hard_sigmoid's kink at +-2.5, where the two float32 routes could take different branches of hard_sigmoid'
    h = torch.as_tensor(np.tanh(np.random.default_rng(SEED).standard_normal((V, D))).astype(np.float32)).to(dev)
    g = torch.as_tensor(np.random.default_rng(SEED + 1).standard_normal((V, D)).astype(np.float32)).to(dev)
    wn = W.ggnn_weights(L, D, SEED + 7, random_bias=True)
    wn["cell"]["kernel"] = wn["cell"]["kernel"] * np.float32(KERNEL_SCALE)
    w = W.to_torch(wn, dev)
    ws = [x.contiguous() for x in w["edge_weights"]]
    k, r, bias = (w["cell"][n].contiguous() for n in ("kernel", "recurrent_kernel", "bias"))
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
    wp = {"edge_weights": [x.clone().requires_grad_(True) for x in ws],
          "cell": {n: x.clone().requires_grad_(True) for n, x in zip(("kernel", "recurrent_kernel", "bias"), (k, r, bias))}}
    leaves = [hp] + wp["edge_weights"] + [wp["cell"][n] for n in ("kernel", "recurrent_kernel", "bias")]

    def py_step():
        for x in leaves:
            x.grad = None
        out = G.sparse_ggnn_layer(hp, plan, D, T, "gru", act, "sum", weights=wp)
        out.backward(g)
    py_ms, py_mem = timed(py_step)
    py_grads = [x.grad.clone() for x in leaves]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # C-ABI route
    nbytes = max(int(lib.rgnn_workspace_bytes(plan.handle, LAYER_GGNN, D, D, 0)),
                 int(lib.rgnn_workspace_bytes(plan.handle, LAYER_GGNN_BACKWARD, D, D, 0)))
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    xs = [h] + [torch.empty_like(h) for _ in range(T)]          # each timestep's input; xs[T] is the output
    dh = [torch.empty_like(h) for _ in range(2)]
    sums = [torch.zeros_like(x) for x in ws + [k, r, bias]]    # the timesteps' weight gradients, summed
    step_g = [torch.empty_like(x) for x in ws + [k, r, bias]]
    tab = lambda xs_: (ctypes.c_void_p * len(xs_))(*[x.data_ptr() for x in xs_])
    wt, gwt = tab(ws), tab(step_g[:L])
    a = get_activation(act)

    def c_step():
        for t in range(T):
            check(lib.rgnn_ggnn_forward(plan.handle, xs[t].data_ptr(), D, D, wt, k.data_ptr(), r.data_ptr(), bias.data_ptr(),
                                        CELL_GRU, a, AGG_SUM, 1, xs[t + 1].data_ptr(), work.data_ptr(), nbytes, stream.cuda_stream))
        gin = g
        for t in reversed(range(T)):
            gout = dh[t & 1]
            check(lib.rgnn_ggnn_backward(plan.handle, xs[t].data_ptr(), D, wt, k.data_ptr(), r.data_ptr(), bias.data_ptr(),
                                         CELL_GRU, a, AGG_SUM, gin.data_ptr(), gout.data_ptr(), gwt, step_g[L].data_ptr(),
                                         step_g[L + 1].data_ptr(), step_g[L + 2].data_ptr(), work.data_ptr(), nbytes,
                                         stream.cuda_stream))
            for s, x in zip(sums, step_g):
                if t == T - 1:
                    s.copy_(x)
                else:
                    s.add_(x)
            gin = gout
    c_ms, c_mem = timed(c_step)
    c_grads = [dh[0]] + sums
    diff = max(rel(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(c_grads, py_grads))
    m = sum(int(x.shape[0]) for x in b.adjacency_lists)
    plan.close()
    return {"workload": "config3_ggnn", "V": V, "M": m, "L": L, "D": D, "timesteps": T, "cell": "gru", "activation": act,
            "steps": steps, "warmup": warmup, "l2": "cold", "python_ms_per_step": round(py_ms, 4),
            "c_abi_ms_per_step": round(c_ms, 4), "speedup": round(py_ms / c_ms, 3),
            "python_max_memory_allocated_bytes": int(py_mem), "c_abi_max_memory_allocated_bytes": int(c_mem),
            "max_rel_grad_difference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ggnn_training.py needs a CUDA device")
    info = card()
    res = run(config3(), 128, 4, "tanh", args.steps, args.warmup)
    res.update(card=info["name"], power_limit=info["power_limit"])
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

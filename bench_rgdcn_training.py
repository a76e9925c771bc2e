"""One RGDCN training step (one timestep forward + backward) through the C ABI, and the reference's op order in float32 torch
autograd on the same GPU and inputs as the comparison point:

  * c_abi:     rgnn_rgdcn_forward + rgnn_rgdcn_backward through ctypes, with one preallocated workspace;
  * reference: the reference's op order in float32 torch autograd (per channel and type: gather the [E, K, K] dynamic
               kernels, einsum, scale, concat, segment reduce, activation; sparse_rgdcn_autograd of
               tests/test_rgdcn_training_through_c_abi_gpu.py).  The project has no Python training route for RGDCN.

Workloads (the RGDCN model defaults: C = 8 channels of K = 16, per-channel kernel inputs, untied, sum, normalised):
  * qm9_rgdcn: the first molecules of tests/golden/qm9_valid_structure.npz up to 25,000 nodes (RGDCN's max_nodes_in_batch),
    as the batcher packs them, D = 128, ELU;
  * ppi_rgdcn: the PPI-shaped batch of batching.ppi_like_batch, D = 128, tanh.
For each it reports the device time per step with a cold L2 (a 256 MiB buffer is overwritten before every step, outside the
timed events) as the median over `--steps` steps after `--warmup` warm-up steps, torch.cuda.max_memory_allocated during the
timed steps of each route, the bytes the C route's kernels must move (counted from shapes, see algorithmic_bytes) and the
rate that gives, and the max-norm relative difference between the two routes' gradients.  Prints one JSON line with the
card's name and power limit, read in the same run; writes nothing."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_batching import card  # noqa: E402

FLUSH_BYTES = 256 << 20
SEED = 5
C, K = 8, 16


def workloads():
    from tf_gnn_samples_b200 import batching
    struct = os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), max_nodes_per_batch=25000)
    yield "qm9_rgdcn", b.adjacency_lists, b.num_nodes, "elu"
    b = batching.ppi_like_batch()
    yield "ppi_rgdcn", b.adjacency_lists, b.num_nodes, "tanh"


def algorithmic_bytes(V, M, L, D):
    """fp32 traffic of the C route, from shapes.  Forward: the dynamic kernels P [V, L, D K] written by the GEMM and read by
    the edge kernel, the M gathered source rows, h read and the output written, the kernels read.  Backward: P written, read
    twice (the aggregate, then dS / dP) and overwritten by dP, dP read by the d_h GEMM and by the dF GEMM; the M source rows
    gathered again and the M dS rows gathered by the reverse index; dS written, the per-(source, type) sums written and read;
    h, grad_out and d_h, the kernels read and their gradients written."""
    P = V * L * D * K
    w = L * C * K * K * K
    fwd = 2 * P + M * D + 2 * V * D + w
    bwd = 6 * P + 2 * M * D + 3 * V * L * D + 4 * V * D + 2 * w
    return 4 * (fwd + bwd)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / (s if s > 0 else 1.0))


def run(name, adj, V, act, steps, warmup):
    import torch
    import tf_gnn_samples_b200 as G
    from tf_gnn_samples_b200 import weights as W
    from tf_gnn_samples_b200.engine import check, load_library
    from tf_gnn_samples_b200.utils import AGG_SUM, LAYER_RGDCN, LAYER_RGDCN_BACKWARD, get_activation
    from test_rgdcn_training_through_c_abi_gpu import sparse_rgdcn_autograd
    dev = torch.device("cuda", 0)
    lib = load_library()
    D, L = C * K, len(adj)
    plan = G.GraphPlan(adj, V, device=dev)
    h = torch.as_tensor(np.tanh(np.random.default_rng(SEED).standard_normal((V, D))).astype(np.float32)).to(dev)
    g = torch.as_tensor(np.random.default_rng(SEED + 1).standard_normal((V, D)).astype(np.float32)).to(dev)
    cnt = torch.as_tensor(np.stack([np.bincount(a[:, 1], minlength=V) for a in adj]).astype(np.float32)).to(dev)
    w = W.to_torch(W.rgdcn_weights(L, C, K, seed=SEED + 11, stddev=0.25), dev)
    fk = [k.contiguous() for ks in w["channel_weights"] for k in ks]     # type-major
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

    # the reference's op order, float32 torch autograd
    hp = h.clone().requires_grad_(True)
    wp = [[fk[l * C + c].clone().requires_grad_(True) for c in range(C)] for l in range(L)]
    leaves = [hp] + [k for ks in wp for k in ks]
    adj_d = [torch.as_tensor(a).to(dev) for a in adj]

    def ref_step():
        for x in leaves:
            x.grad = None
        with torch.device(dev):
            out = sparse_rgdcn_autograd(hp, adj_d, cnt, C, K, 1, False, False, act, "sum", True, weights={"channel_weights": wp})
            out.backward(g)
    ref_ms, ref_mem = timed(ref_step)
    ref_grads = [x.grad.clone() for x in leaves]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # C-ABI route
    nbytes = max(int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGDCN, D, D, K)),
                 int(lib.rgnn_workspace_bytes(plan.handle, LAYER_RGDCN_BACKWARD, D, D, K)))
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    y = torch.empty_like(h)
    dh = torch.empty_like(h)
    gfk = [torch.empty_like(k) for k in fk]
    tab = lambda xs_: (ctypes.c_void_p * len(xs_))(*[x.data_ptr() for x in xs_])
    fkt, gfkt = tab(fk), tab(gfk)
    a = get_activation(act)

    def c_step():
        check(lib.rgnn_rgdcn_forward(plan.handle, h.data_ptr(), D, C, fkt, 0, cnt.data_ptr(), a, AGG_SUM, 1, 1, y.data_ptr(),
                                     work.data_ptr(), nbytes, stream.cuda_stream))
        check(lib.rgnn_rgdcn_backward(plan.handle, h.data_ptr(), D, C, fkt, 0, 0, cnt.data_ptr(), a, AGG_SUM, 1, g.data_ptr(),
                                      dh.data_ptr(), gfkt, work.data_ptr(), nbytes, stream.cuda_stream))
    c_ms, c_mem = timed(c_step)
    c_grads = [dh] + gfk
    diff = max(rel(x.cpu().numpy(), y_.cpu().numpy()) for x, y_ in zip(c_grads, ref_grads))
    m = sum(int(x.shape[0]) for x in adj)
    nb = algorithmic_bytes(V, m, L, D)
    plan.close()
    return {"workload": name, "V": V, "M": m, "L": L, "D": D, "C": C, "K": K, "activation": act,
            "reference_order_ms_per_step": round(ref_ms, 4), "c_abi_ms_per_step": round(c_ms, 4),
            "reference_order_max_memory_allocated_bytes": int(ref_mem), "c_abi_max_memory_allocated_bytes": int(c_mem),
            "c_abi_algorithmic_bytes": int(nb), "c_abi_achieved_gb_per_s": round(nb / (c_ms * 1e-3) / 1e9, 1),
            "max_rel_grad_difference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgdcn_training.py needs a CUDA device")
    info = card()
    res = {"steps": args.steps, "warmup": args.warmup, "l2": "cold",
           "workloads": [run(name, adj, V, act, args.steps, args.warmup) for name, adj, V, act in workloads()],
           "card": info["name"], "power_limit": info["power_limit"]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

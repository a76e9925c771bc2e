"""Minibatch packing: the host route (pack_batch on pre-converted samples + training.device_args) against the device route
(DeviceGraphSet.pack + GraphPlan(validate=False)), per batch.

For every batch of one shuffled epoch it reports
  * wall clock to "plan and tensors ready": a host clock around the route's work, ending in torch.cuda.synchronize();
  * the device time of the pack kernels alone: CUDA events around one replay of a CUDA graph that holds `--reps` packs of
    the batch back to back, divided by `--reps`.
Workloads: the real config-3 structure (tests/golden/qm9_valid_structure.npz: the reference's 10,000 QM9 validation
molecules, self-loop edges, L = 5) at budgets of 50,000 and 200,000 nodes; five PPI-shaped graphs in one batch (V = 11,225,
M = 601,225, L = 3).  Both routes' outputs are compared bit for bit on every batch.  Prints one JSON line per workload and
the card's name and power limit; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit": "not recorded"}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        if out:
            info["name"], info["power_limit"] = [s.strip() for s in out.split(",")[:2]]
    except (OSError, subprocess.SubprocessError):
        pass
    return info


def same(dev, host):
    import torch
    ok = torch.equal(dev.node_features.cpu(), torch.as_tensor(host.node_features))
    ok &= torch.equal(dev.type_to_num_incoming_edges.cpu(), torch.as_tensor(host.type_to_num_incoming_edges))
    ok &= all(torch.equal(a.cpu(), torch.as_tensor(b)) for a, b in zip(dev.adjacency_lists, host.adjacency_lists))
    return bool(ok)


def run(name, samples, gs, targets_of, order, budget, epochs, reps):
    import torch
    from tf_gnn_samples_b200 import batching, training
    from tf_gnn_samples_b200.engine import GraphPlan
    dev = torch.device("cuda", 0)
    shuffled = [samples[i] for i in order]
    bounds = list(batching.batch_bounds(gs.graph_sizes[order], budget))
    order_host, order_dev = gs.upload_order(order)
    host_ms, dev_ms, equal = [], [], True
    for epoch in range(epochs + 1):                       # epoch 0 warms up every shape
        for start, count in bounds:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b = batching.pack_batch(shuffled[start:start + count])
            gnl = np.repeat(np.arange(b.num_graphs, dtype=np.int32), np.diff(b.graph_node_offsets))
            args = training.device_args(training.TaskBatch(b, targets_of(order[start:start + count], b), gnl), dev)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            d = gs.pack(order_host, order_dev, start, count)
            dargs = d.args()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if epoch > 0:
                host_ms.append(1e3 * (t1 - t0))
                dev_ms.append(1e3 * (t2 - t1))
            else:
                equal &= same(d, b)
            del args, dargs
    # device time of the pack kernels: `reps` packs of the largest batch in one CUDA graph
    start, count = max(bounds, key=lambda b: b[1])
    gs.pack(order_host, order_dev, start, count)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        keep = [gs.pack(order_host, order_dev, start, count) for _ in range(reps)]
    torch.cuda.current_stream(dev).wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kernel_ms = []
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        kernel_ms.append(e0.elapsed_time(e1) / reps)
    big = keep[0]
    del keep, g
    return {"workload": name, "budget": budget, "batches_per_epoch": len(bounds), "epochs_timed": epochs,
            "outputs_bit_identical": equal,
            "host_route_ms_per_batch_median": float(np.median(host_ms)), "device_route_ms_per_batch_median": float(np.median(dev_ms)),
            "host_route_ms_per_epoch": float(np.sum(host_ms) / epochs), "device_route_ms_per_epoch": float(np.sum(dev_ms) / epochs),
            "pack_kernels_us_largest_batch": float(1e3 * np.median(kernel_ms)),
            "largest_batch": {"graphs": big.num_graphs, "nodes": big.num_nodes, "edges": big.num_edges}}


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_batching.py needs a CUDA device")
    from tf_gnn_samples_b200 import batching
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    recs = batching.qm9_records_from_structure(os.path.join(ROOT, "tests", "golden", "qm9_valid_structure.npz"))
    L = batching.qm9_num_edge_types(recs)
    samples = [batching.qm9_graph_to_sample(r, L) for r in recs]
    gs = batching.DeviceGraphSet.from_qm9_records(recs, device=dev)
    targets = np.zeros((1, len(recs)), np.float32)
    order = np.random.default_rng(a.seed).permutation(len(recs))
    for budget in (50000, 200000):
        print(json.dumps(run("qm9_config3_structure", samples, gs, lambda idx, b: targets[:, idx], order, budget, a.epochs,
                             a.reps)), flush=True)
    graphs = [batching.make_ppi_like_graph(seed=i) for i in range(5)]
    labels = [np.zeros((g.node_features.shape[0], 121), np.float32) for g in graphs]
    gs = batching.DeviceGraphSet.from_ppi_fold(graphs, labels, device=dev)
    order = np.random.default_rng(a.seed).permutation(len(graphs))
    print(json.dumps(run("ppi_five_graphs", graphs, gs, lambda idx, b: np.concatenate([labels[i] for i in idx]), order,
                         10 ** 6, max(a.epochs, 10), a.reps)), flush=True)


if __name__ == "__main__":
    main()

"""CPU: host-side logic added in round 2 (no GPU work)."""
import importlib.util
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_degree_balanced_cuts_match_the_torch_distributed_partition():
    from tf_gnn_samples_b200 import batching, degree_balanced_cuts
    from tf_gnn_samples_b200.partition import NodeRangePartition
    g = batching.make_typed_random_graph(500, 6000, (0.5, 0.3, 0.2), 4, seed=3)
    for world in (1, 2, 3, 8):
        cuts = degree_balanced_cuts(g.adjacency_lists, 500, world)
        assert cuts[0] == 0 and cuts[-1] == 500 and np.all(np.diff(cuts) >= 0)
        part = NodeRangePartition(g.adjacency_lists, g.type_to_node_to_num_incoming_edges, 500, 0, world)
        np.testing.assert_array_equal(cuts, part.cuts)
        indeg = g.type_to_node_to_num_incoming_edges.sum(axis=0) + 1
        loads = [indeg[cuts[r]:cuts[r + 1]].sum() for r in range(world)]
        assert max(loads) <= indeg.sum() / world + indeg.max() + 1          # balanced up to one node's weight


def _load_bench():
    spec = importlib.util.spec_from_file_location("bench_module", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_bench_arms_share_one_config_dict():
    """The driver compares the `config` of our arm with the reference arm's: both print bench.CONFIG verbatim."""
    b = _load_bench()
    assert b.CONFIG["workload"] == b.WORKLOAD and b.CONFIG["M"] == 2 * b.NUM_LINKS + b.NUM_NODES
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert src.count('"config": CONFIG') == 2
    assert json.loads(json.dumps(b.CONFIG)) == b.CONFIG
    assert b.algorithmic_bytes_per_layer(2245, 120245, 3, 256) == 129958012        # SURVEY.md 8d: 130.0 MB per layer


def test_big_case_summary_bounds_follow_from_the_elementwise_tolerance():
    """ref_cases.compare_with_summary: an element-wise max-norm error eps implies every returned value <= eps."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import ref_cases as RC
    rng = np.random.default_rng(0)
    for shape in ((1000, 64), (30000, 8)):                                          # the second: thinned rows, block-summed projection
        out = rng.standard_normal(shape)
        z = RC.summarize(out)
        assert ("proj_block" in z) == (shape[0] > RC.PROJ_BLOCK_ABOVE) and len(z["rows"]) <= RC.MAX_SUMMARY_ROWS
        eps = 3e-5
        noisy = out + eps * float(z["maxabs"]) * rng.uniform(-1, 1, size=out.shape)
        assert max(RC.compare_with_summary(noisy, z)) <= eps
        biased = out + eps * float(z["maxabs"])                                     # a systematic bias of eps is still within eps
        assert max(RC.compare_with_summary(biased, z)) <= eps * (1 + 1e-9)
        spoiled = out.copy(); spoiled[501, 7] += 1.0                                # one bad element in an uncommitted row is seen
        assert max(RC.compare_with_summary(spoiled, z)) > 1e-4


def test_tf1_optimizer_update_rules():
    """TF 1.13 RMSProp (ms slot starts at one, epsilon inside the sqrt) and Adam (epsilon-hat form) by hand; a parameter
    without a gradient decays like TF's zero-gradient update."""
    import torch
    from tf_gnn_samples_b200.tf_optimizers import TF1Adam, TF1RMSProp
    w = torch.nn.Parameter(torch.tensor([1.0, -2.0], dtype=torch.float64))
    idle = torch.nn.Parameter(torch.tensor([3.0], dtype=torch.float64))
    opt = TF1RMSProp([w, idle], lr=0.1, decay=0.9, momentum=0.5, epsilon=1e-10)
    g = torch.tensor([0.5, -4.0], dtype=torch.float64)
    ms, mom, val = np.ones(2), np.zeros(2), np.array([1.0, -2.0])
    for _ in range(3):
        w.grad = g.clone(); idle.grad = None
        opt.step()
        ms = 0.9 * ms + 0.1 * g.numpy() ** 2
        mom = 0.5 * mom + 0.1 * g.numpy() / np.sqrt(ms + 1e-10)
        val = val - mom
        np.testing.assert_allclose(w.detach().numpy(), val, rtol=1e-14)
    assert float(idle) == 3.0 and float(opt.state[idle]["ms"]) == 0.9 ** 3          # zero gradient: the slot decays, the variable stays
    first = 0.1 * 0.5 / np.sqrt(0.9 + 0.1 * 0.25)                                   # torch.optim.RMSprop would start from ms = 0: ~3x larger
    assert abs(first - 0.0520) < 1e-3
    v = torch.nn.Parameter(torch.tensor([1.0], dtype=torch.float64))
    adam = TF1Adam([v], lr=0.01, epsilon=1e-8)
    m_, v_, x = 0.0, 0.0, 1.0
    for t in range(1, 4):
        v.grad = torch.tensor([2.0], dtype=torch.float64)
        adam.step()
        m_ = 0.9 * m_ + 0.1 * 2.0; v_ = 0.999 * v_ + 0.001 * 4.0
        x -= 0.01 * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * m_ / (np.sqrt(v_) + 1e-8)
        np.testing.assert_allclose(float(v), x, rtol=1e-14)

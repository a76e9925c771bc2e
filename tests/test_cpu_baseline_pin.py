"""The TIMED CPU baseline (oracle/ref_torch.py: what bench.py's cpu_baseline leg and `--impl reference` execute) computes what
the reference computes: against the committed output of the reference's own gnns/rgcn.py at BASELINE config 2 (float64 and
float32 runs through tests/tf1_shim, tests/golden/ref_config2_rgcn_ppi.npz) and, for the 3-layer stack bench.py times, against
the pinned numpy oracle.  A baseline that timed different arithmetic would make the GPU / CPU ratio meaningless."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import ref_cases as RC                                  # noqa: E402
from oracle import ref_layers as R, ref_torch           # noqa: E402
from tf_gnn_samples_b200 import weights as W            # noqa: E402


def as_torch(h, adj, indeg):
    return (torch.as_tensor(np.asarray(h, np.float32)), [torch.as_tensor(np.asarray(a, np.int64)) for a in adj],
            torch.as_tensor(np.asarray(indeg, np.float32)))


def test_timed_port_equals_the_reference_at_config_2():
    case = RC.CASES["config2_rgcn_ppi"]
    z = np.load(RC.fixture_path("config2_rgcn_ppi"))
    h, adj, indeg = case["graph"]()
    w = case["weights"]()
    ht, at, ct = as_torch(h, adj, indeg)
    out = ref_torch.sparse_rgcn_layer(ht, at, ct, 256, activation_function="ReLU",
                                      weights={"edge_weights": [torch.as_tensor(k) for k in w["edge_weights"]]}).numpy()
    assert out.dtype == np.float32
    err_rows, err_proj, err_col = RC.compare_with_summary(out, z)
    # float32 in the reference's op order: as close to the float64 truth as the reference's own float32 run (err32), BLAS order aside
    bound = 4 * float(z["err32"]) + 1e-6
    assert max(err_rows, err_proj, err_col) <= bound, (err_rows, err_proj, err_col, bound)
    scale = float(z["maxabs"])
    assert np.abs(out[z["rows"]].astype(np.float64) - z["out32_rows"].astype(np.float64)).max() / scale <= 2e-6


def test_the_three_layer_stack_bench_times_is_the_oracles():
    h, adj, indeg = RC.ppi_graph()
    ws = [W.rgcn_weights(3, 256, 256, seed=11 + 7 * i) for i in range(3)]
    ht, at, ct = as_torch(h, adj, indeg)
    got = ref_torch.rgcn_stack(ht, at, ct, [{"edge_weights": [torch.as_tensor(k) for k in w["edge_weights"]]} for w in ws]).numpy()
    want = np.asarray(h, np.float64)
    for w in ws:
        want = R.sparse_rgcn_layer(want, adj, indeg, 256, activation_function="ReLU", weights=w, dtype=np.float64)
    assert R.max_norm_rel_err(got, want) <= 1e-5

"""Generates tests/golden/ref_*.npz by EXECUTING THE REFERENCE'S OWN LAYER CODE.

    python tests/golden/make_ref_fixtures.py [case ...]         (needs the original checkout: TF_GNN_SAMPLES_REFERENCE=<path>)

The unmodified ``/root/reference/gnns/*.py`` + ``utils/utils.py`` are imported with tests/tf1_shim standing in for
``tensorflow`` / ``dpu_utils`` (numpy-backed, eager: only the TF kernel semantics are restated, see the shim's docstring),
fed the seeded inputs and weights of tests/golden/ref_cases.py, and run in float64 ("truth") and float32 ("the reference's
arithmetic").  What is committed per case:
  small cases   h, adjacency, in-degrees, every variable under the TF name the reference created it with, out64, out32
  big cases     BASELINE.json configs: every 97th row of out64, a random projection of all rows, column sums
                (inputs / weights are regenerated from their seeds by ref_cases.py; input checksums are committed)
  err32         max-norm relative error of the float32 run against the float64 run -- the reference path's own rounding
                error, the yardstick of SURVEY.md 8(c)'s second acceptance clause.
tests/golden/make_tf1_fixtures.py writes the same files from a real TensorFlow 1.13.
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import ref_cases as RC                      # noqa: E402
import tf1_shim                             # noqa: E402
from tf1_shim import variables as TV        # noqa: E402


def run_reference(case, h, adj, indeg, weights, dtype):
    """One call of the reference's sparse_<x>_layer under variable scopes graph_model/gnn_layer_0 (as the scaffold
    opens them: models/sparse_graph_model.py:163,177).  Returns (output, {tf variable name: value})."""
    named = TV.flatten(weights, cell_kind=RC.cell_kind(case))
    provider = TV.provider_from(named)
    with tf1_shim.installed(dtype=dtype, provider=provider) as session:
        import gnns   # the reference's package (sys.path[0] is /root/reference inside this block)
        assert os.path.realpath(gnns.__file__).startswith(os.path.realpath(tf1_shim.REFERENCE_ROOT)), gnns.__file__
        fn = getattr(gnns, RC.REFERENCE_FUNCTIONS[case["kind"]])
        tf = session.tf
        args = dict(node_embeddings=np.asarray(h).astype(dtype),
                    adjacency_lists=[np.asarray(a).astype(np.int32) for a in adj])
        if case["indeg"]:
            args["type_to_num_incoming_edges"] = np.asarray(indeg).astype(dtype)
        with tf.variable_scope("graph_model"), tf.variable_scope("gnn_layer_0"):
            out = fn(**args, **case["kw"])
        created = dict(session.variables)
    unused = set(named) - provider.used
    assert not unused, "weights never requested by the reference: %s" % sorted(unused)
    return np.asarray(out), created


def input_checksums(h, adj, indeg):
    return {"h_sum": np.float64(np.asarray(h, np.float64).sum()),
            "adj_sum": np.asarray([int(np.asarray(a, np.int64).sum()) for a in adj], np.int64),
            "adj_len": np.asarray([len(a) for a in adj], np.int64),
            "indeg_sum": np.float64(np.asarray(indeg, np.float64).sum())}


def make_case(name):
    case = RC.CASES[name]
    h, adj, indeg = case["graph"]()
    weights = case["weights"]()
    t0 = time.time()
    out64, created = run_reference(case, h, adj, indeg, weights, np.float64)
    out32, _ = run_reference(case, h, adj, indeg, weights, np.float32)
    assert out32.dtype == np.float32 and out64.dtype == np.float64
    scale = float(np.abs(out64).max())
    err32 = float(np.abs(out32.astype(np.float64) - out64).max() / scale)
    blob = {"err32": np.float64(err32), "variable_names": np.asarray(sorted(created)),
            "meta": np.asarray(json.dumps({"kind": case["kind"], "kw": case["kw"], "source": "reference gnns/*.py via tests/tf1_shim"}))}
    blob.update(input_checksums(h, adj, indeg))
    if case.get("big"):
        blob.update(RC.summarize(out64))
        blob["out32_rows"] = out32[blob["rows"]].astype(np.float32)
    else:
        blob.update({"h": h, "indeg": indeg, "out": out64, "out32": out32})
        for l, a in enumerate(adj):
            blob["adj.%d" % l] = a
        for vname, value in created.items():
            blob["var:" + vname] = value.astype(np.float32)
    np.savez_compressed(RC.fixture_path(name), **blob)
    print("%-28s out %s maxabs %.4f  fp32-vs-fp64 %.2e  %d variables  %.1fs" % (name, out64.shape, scale, err32, len(created),
                                                                               time.time() - t0), flush=True)


def main():
    names = sys.argv[1:] or list(RC.CASES)
    for name in names:
        make_case(name)


if __name__ == "__main__":
    main()

"""The same fixtures as make_ref_fixtures.py, produced by a REAL TensorFlow 1.13 -- for anyone who has one.

    # Python 3.6/3.7 environment with tensorflow==1.13.1 and dpu-utils>=0.1.30, a checkout of
    # microsoft/tf-gnn-samples next to this repository:
    python tests/golden/make_tf1_fixtures.py --reference /path/to/tf-gnn-samples --out /tmp/tf1_fixtures [case ...]
    python tests/golden/make_tf1_fixtures.py --compare /tmp/tf1_fixtures      # against the committed ref_*.npz

This container cannot run it (no TensorFlow for Python 3.12, no network: SURVEY.md 0); it is committed so that the one
remaining assumption of the pin -- that tests/tf1_shim restates the TF 1.13 / Keras / dpu_utils KERNELS faithfully
(SURVEY.md Appendix A) -- can be discharged by anybody with the real stack.  It builds the reference layer in a TF graph under
variable scopes graph_model/gnn_layer_0, assigns the seeded weights of ref_cases.py to the variables BY THE NAMES THE REFERENCE
CREATED (tests/tf1_shim/variables.flatten lists them), runs the forward pass in float32 (the reference's arithmetic) and
writes out32 / out32_rows next to the inputs.  --compare checks those against the committed float32 reference-through-shim
outputs (tolerance 2e-6 max-norm: Eigen vs numpy summation order) and the variable-name lists for equality.
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import ref_cases as RC                      # noqa: E402
from tf1_shim import variables as TV        # noqa: E402


def run_case_tf1(name, reference_root):
    import tensorflow as tf                  # the real one
    if reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    import gnns
    case = RC.CASES[name]
    h, adj, indeg = case["graph"]()
    named = TV.flatten(case["weights"](), cell_kind=RC.cell_kind(case))
    graph = tf.Graph()
    with graph.as_default():
        feeds = {}
        h_ph = tf.placeholder(tf.float32, [None, h.shape[1]], name="node_embeddings")
        feeds[h_ph] = h.astype(np.float32)
        adj_ph = []
        for l, a in enumerate(adj):
            ph = tf.placeholder(tf.int32, [None, 2], name="adjacency_e%d" % l)
            adj_ph.append(ph)
            feeds[ph] = np.asarray(a, np.int32).reshape(-1, 2)
        args = dict(node_embeddings=h_ph, adjacency_lists=adj_ph)
        if case["indeg"]:
            c_ph = tf.placeholder(tf.float32, [len(adj), None], name="type_to_num_incoming_edges")
            args["type_to_num_incoming_edges"] = c_ph
            feeds[c_ph] = np.asarray(indeg, np.float32)
        with tf.variable_scope("graph_model"), tf.variable_scope("gnn_layer_0"):
            out = getattr(gnns, RC.REFERENCE_FUNCTIONS[case["kind"]])(**args, **case["kw"])
        variables = {v.name: v for v in tf.global_variables()}
        missing = sorted(set(variables) - set(named))
        extra = sorted(set(named) - set(variables))
        assert not missing and not extra, "variable names differ: TF created %s; ref_cases provides %s" % (missing, extra)
        with tf.Session(graph=graph) as sess:
            sess.run(tf.global_variables_initializer())
            for vname, var in variables.items():
                var.load(np.asarray(named[vname], np.float32), sess)
            out32 = sess.run(out, feed_dict=feeds)
    return np.asarray(out32, np.float32), sorted(variables)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(HERE, "tf1"))
    ap.add_argument("--compare", default=None, help="directory written by a previous run: compare with the committed fixtures")
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    names = a.cases or list(RC.CASES)
    if a.compare:
        worst = 0.0
        for name in names:
            path = os.path.join(a.compare, "tf1_%s.npz" % name)
            if not os.path.exists(path):
                continue
            got, ref = np.load(path), np.load(RC.fixture_path(name))
            assert [str(s) for s in got["variable_names"]] == [str(s) for s in ref["variable_names"]], name
            want = ref["out32_rows"] if "out32_rows" in ref.files else ref["out32"]
            have = got["out32_rows"] if "out32_rows" in ref.files else got["out32"]
            err = float(np.abs(have.astype(np.float64) - want.astype(np.float64)).max() / np.abs(want).max())
            worst = max(worst, err)
            print("%-28s TF 1.13 float32 vs reference-through-shim float32: %.2e %s" % (name, err, "OK" if err <= 2e-6 else "DIFFERENT"))
        sys.exit(0 if worst <= 2e-6 else 1)
    os.makedirs(a.out, exist_ok=True)
    for name in names:
        out32, var_names = run_case_tf1(name, a.reference)
        blob = {"variable_names": np.asarray(var_names)}
        if RC.CASES[name].get("big"):
            blob["out32_rows"] = out32[np.load(RC.fixture_path(name))["rows"]]
        else:
            blob["out32"] = out32
        np.savez_compressed(os.path.join(a.out, "tf1_%s.npz" % name), **blob)
        print(name, out32.shape)


if __name__ == "__main__":
    main()

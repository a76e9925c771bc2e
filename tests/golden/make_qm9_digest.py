"""Record the reference's single minibatch of all 10,000 QM9 validation molecules (tasks/qm9_task.py loader + batcher run
under tests/tf1_shim on data/qm9/valid.jsonl.gz) as counts + SHA-256 digests of its arrays in ref_qm9_valid_digest.json:

    TF_GNN_SAMPLES_REFERENCE=<checkout> python tests/golden/make_qm9_digest.py <checkout>/data/qm9/valid.jsonl.gz"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC                          # noqa: E402

KEYS = ["graph_nodes_list", "type_to_num_incoming_edges"]


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.tobytes()).hexdigest()


def main(path):
    want, L = BC.reference_qm9_feeds({}, 10 ** 9, path=path)
    f = want[0]
    out = {"num_edge_types": int(L), "num_feeds": len(want),
           "num_graphs": int(f["num_graphs"]), "num_nodes": int(f["num_nodes"]), "num_edges": int(f["num_edges"]),
           "sha256": {k: digest(np.asarray(f[k], np.int32 if k == "graph_nodes_list" else np.float32)) for k in KEYS}}
    for i in range(L):
        out["sha256"]["adjacency_e%d" % i] = digest(np.asarray(f["adjacency_e%d" % i], np.int32))
    with open(os.path.join(HERE, "ref_qm9_valid_digest.json"), "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1])

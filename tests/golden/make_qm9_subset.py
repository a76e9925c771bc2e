"""Regenerates tests/golden/qm9_valid_subset.json.gz: the first 200 records of the reference's data/qm9/valid.jsonl.gz
(graph triples, 15-d node features, 13 targets), re-serialised compactly.  Needs the original checkout (TF_GNN_SAMPLES_REFERENCE);
the committed subset is what the tests read on the GPU box."""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_gnn_samples_b200.batching import load_qm9_jsonl   # noqa: E402

SRC = "/root/reference/data/qm9/valid.jsonl.gz"
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "qm9_valid_subset.json.gz")

records = load_qm9_jsonl(SRC, limit=200)
slim = [{"id": r["id"], "graph": r["graph"], "node_features": r["node_features"], "targets": r["targets"]} for r in records]
with gzip.open(DST, "wt") as f:
    for r in slim:
        f.write(json.dumps(r, separators=(",", ":")) + "\n")
print("wrote", DST, os.path.getsize(DST), "bytes;", sum(len(r["node_features"]) for r in slim), "nodes")

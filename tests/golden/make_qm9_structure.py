"""Regenerates tests/golden/qm9_valid_structure.npz: the GRAPH STRUCTURE (atoms per molecule, bonds as (src, type, dst)) of all
10,000 records of the reference's data/qm9/valid.jsonl.gz -- BASELINE config 3 ("GGNN QM9, 10k-graph batch") on the real
molecules rather than a shape-matched synthetic batch.  Node features and targets are not included (the 200-record subset
in qm9_valid_subset.json.gz carries those for the parity tests).  Needs the original checkout (TF_GNN_SAMPLES_REFERENCE)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_gnn_samples_b200.batching import load_qm9_jsonl   # noqa: E402

SRC = "/root/reference/data/qm9/valid.jsonl.gz"
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "qm9_valid_structure.npz")
recs = load_qm9_jsonl(SRC)
sizes = np.array([len(r["node_features"]) for r in recs], dtype=np.uint8)
nbonds = np.array([len(r["graph"]) for r in recs], dtype=np.uint8)
bonds = np.array([e for r in recs for e in r["graph"]], dtype=np.uint8).reshape(-1, 3)      # (src, bond type, dst), ids local to the molecule
np.savez_compressed(DST, num_atoms=sizes, num_bonds=nbonds, bonds=bonds)
print("wrote", DST, os.path.getsize(DST), "bytes;", len(recs), "graphs,", int(sizes.sum()), "atoms,", bonds.shape[0], "bonds")

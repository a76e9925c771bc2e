"""Writes tests/golden/ref_batcher_feeds.npz by running the REFERENCE's own loaders and batchers (tasks/qm9_task.py,
tasks/ppi_task.py, unmodified, under tests/tf1_shim -- only tf.placeholder as a dict key and dpu_utils RichPath are involved):

    python tests/golden/make_batcher_fixtures.py            (needs the original checkout: TF_GNN_SAMPLES_REFERENCE=<path>)

QM9 cases run on the 200 real validation molecules of qm9_valid_subset.json.gz, PPI cases on a seeded fold in the dgl file
layout (batcher_cases.write_ppi_dir).  Every minibatch feed of every case is stored (keys <case>/b<i>/<placeholder name>);
tests/test_reference_batcher_pin.py compares batching.py against it where the reference is absent."""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC      # noqa: E402


def main():
    blob = {}
    for name, (params, budget) in BC.QM9_CASES.items():
        feeds, L = BC.reference_qm9_feeds(params, budget)
        blob.update({"%s/%s" % (name, k): v for k, v in BC.pack_feeds(feeds).items()})
        blob["%s/num_edge_types" % name] = np.int64(L)
    with tempfile.TemporaryDirectory() as d:
        BC.write_ppi_dir(d, "test")
        for name, (params, budget) in BC.PPI_CASES.items():
            feeds, L = BC.reference_ppi_feeds(params, budget, d)
            blob.update({"%s/%s" % (name, k): v for k, v in BC.pack_feeds(feeds).items()})
            blob["%s/num_edge_types" % name] = np.int64(L)
    out = os.path.join(HERE, "ref_batcher_feeds.npz")
    np.savez_compressed(out, **blob)
    print("wrote %s: %d arrays, %.1f KB" % (out, len(blob), os.path.getsize(out) / 1024))


if __name__ == "__main__":
    main()

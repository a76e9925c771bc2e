"""SURVEY.md 8 rows a12/a13 (the input tensor contract and the task batchers): batching.py against the REFERENCE'S OWN
loaders and minibatch iterators.

tasks/qm9_task.py and tasks/ppi_task.py executed unmodified under tests/tf1_shim (tf.placeholder as a feed_dict key, dpu_utils
RichPath for local files -- nothing numerical is restated) on the 200 real QM9 validation molecules / a seeded PPI fold in the
dgl layout wrote tests/golden/ref_batcher_feeds.npz (make_batcher_fixtures.py); every minibatch feed of batching.py is
compared with it: adjacency lists bit-exact INCLUDING edge order, graph ids, in-degrees, features, targets / labels, counts.
The configurations the reference itself cannot run are pinned as such (the exceptions it raised: ref_batcher_raises.json)."""
import importlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC      # noqa: E402

batching = importlib.import_module("tf_gnn_samples_b200.batching")
FIXTURE = os.path.join(HERE, "golden", "ref_batcher_feeds.npz")


def reference_raised(key):
    import json
    with open(os.path.join(HERE, "golden", "ref_batcher_raises.json")) as f:
        return json.load(f)[key]


@pytest.fixture(scope="module")
def ppi_dir(tmp_path_factory):
    return BC.write_ppi_dir(str(tmp_path_factory.mktemp("ppi")), "test")


@pytest.fixture(scope="module")
def fixture():
    return np.load(FIXTURE)


@pytest.mark.parametrize("case", sorted(BC.QM9_CASES))
def test_qm9_feeds_equal_the_committed_reference_feeds(case, fixture):
    params, budget = BC.QM9_CASES[case]
    got, L = BC.repo_qm9_feeds(params, budget)
    assert L == int(fixture[case + "/num_edge_types"])
    BC.compare_feeds(got, BC.unpack_feeds(fixture, case), case)


@pytest.mark.parametrize("case", sorted(BC.PPI_CASES))
def test_ppi_feeds_equal_the_committed_reference_feeds(case, fixture, ppi_dir):
    params, budget = BC.PPI_CASES[case]
    got, L = BC.repo_ppi_feeds(params, budget, ppi_dir)
    assert L == int(fixture[case + "/num_edge_types"])
    BC.compare_feeds(got, BC.unpack_feeds(fixture, case), case)


@pytest.mark.parametrize("case", sorted(BC.QM9_REFERENCE_RAISES))
def test_untied_qm9_cannot_run_in_the_reference(case):
    """qm9_task.py:139-145 appends to the list it enumerates -> IndexError on the first molecule.  batching.py builds what the
    loop evidently meant (forward types, then their reversals) instead of failing; stated here so the difference is on record."""
    params, budget = BC.QM9_REFERENCE_RAISES[case]
    assert reference_raised("qm9/" + case)[0] == "IndexError"
    feeds, L = BC.repo_qm9_feeds(params, budget)
    half = L // 2
    for f in feeds:
        for t in range(half):
            fwd, bwd = f["adjacency_e%d" % t], f["adjacency_e%d" % (half + t)]
            assert sorted(map(tuple, fwd[:, ::-1].tolist())) == list(map(tuple, bwd.tolist()))


def test_a_linkless_ppi_graph_breaks_the_reference_batcher_only(tmp_path):
    """A graph without links becomes np.array([]) of shape (0,) in ppi_task.py:152; packed next to a graph with links,
    np.concatenate (:247) raises.  batching.py keeps (0, 2) lists and packs it."""
    d = BC.write_ppi_dir(str(tmp_path), "test", linkless_graph=2)
    assert reference_raised("ppi/linkless")[0] == "ValueError"
    feeds, L = BC.repo_ppi_feeds({}, 10 ** 6, d)
    assert len(feeds) == 1 and feeds[0]["num_graphs"] == 5


def test_minibatches_cover_every_graph_once_and_respect_the_budget():
    graphs = batching.make_qm9_like_graphs(300, seed=5)
    seen, budget = 0, 97
    for batch, first in batching.minibatches(graphs, budget):
        assert first == seen and batch.num_graphs >= 1 and batch.num_nodes < budget
        nxt = first + batch.num_graphs
        if nxt < len(graphs):            # the next graph is the one that did not fit (strict '<' of ppi_task.py:220)
            assert not (batch.num_nodes + graphs[nxt].node_features.shape[0] < budget)
        seen = nxt
    assert seen == len(graphs)


def test_minibatches_refuse_a_graph_that_can_never_fit():
    graphs = batching.make_qm9_like_graphs(3, seed=1)
    n = graphs[1].node_features.shape[0]
    with pytest.raises(ValueError, match="does not fit"):
        list(batching.minibatches(graphs, n))       # node_offset + n < n is false even for an empty batch


def test_the_full_qm9_validation_set_is_packed_like_the_reference():
    """BASELINE config 3's batch: all 10,000 validation molecules of data/qm9/valid.jsonl.gz through the reference's loader and
    batcher in ONE minibatch (V = 180,560, M = 554,026, L = 5), recorded as counts + SHA-256 digests of every array
    (tests/golden/make_qm9_digest.py), against batching.py on the structure archive used by the benchmark -- every edge in
    the same position."""
    import hashlib
    import json
    with open(os.path.join(HERE, "golden", "ref_qm9_valid_digest.json")) as f:
        want = json.load(f)
    recs = batching.qm9_records_from_structure(os.path.join(HERE, "golden", "qm9_valid_structure.npz"))
    b, graph_nodes_list, _ = batching.qm9_batch(recs)
    assert (want["num_feeds"], want["num_edge_types"]) == (1, len(b.adjacency_lists)) == (1, 5)
    assert (want["num_graphs"], want["num_nodes"], want["num_edges"]) == (b.num_graphs, b.num_nodes, b.num_edges) == (10000, 180560, 554026)

    def digest(a, dt):
        return hashlib.sha256(np.ascontiguousarray(np.asarray(a, dt)).tobytes()).hexdigest()
    assert digest(graph_nodes_list, np.int32) == want["sha256"]["graph_nodes_list"]
    assert digest(b.type_to_num_incoming_edges, np.float32) == want["sha256"]["type_to_num_incoming_edges"]
    for i, a in enumerate(b.adjacency_lists):
        assert digest(a, np.int32) == want["sha256"]["adjacency_e%d" % i], "edge type %d" % i

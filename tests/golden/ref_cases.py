"""The cases of tests/golden/ref_*.npz: inputs (seeded), weights (seeded), keyword arguments -- shared by the two fixture
generators (make_ref_fixtures.py: the reference's own gnns/*.py through tests/tf1_shim; make_tf1_fixtures.py: the same under
a real TensorFlow 1.13) and by the tests that consume the fixtures.

"small" cases commit the full output; the BASELINE.json configs 2-5 ("big") commit every k-th output row, a seeded
random projection of ALL rows and the column sums (a few hundred KB instead of up to 185 MB per case).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tf_gnn_samples_b200 import batching, weights as W   # noqa: E402
from helpers import node_states, tiny_graph               # noqa: E402

V_SMALL, D_SMALL, EDGES_SMALL = 48, 32, (110, 48, 0, 70)
L_SMALL = len(EDGES_SMALL)


def small_graph():
    adj, indeg = tiny_graph(V_SMALL, EDGES_SMALL, seed=31)
    return node_states(V_SMALL, D_SMALL, seed=32), adj, indeg


def ppi_graph(D=256):
    """BASELINE configs 2 / 4: PPI-shaped, V = 2,245, M = 120,245, L = 3 (SURVEY.md 8d)."""
    b = batching.ppi_like_batch()
    return node_states(b.num_nodes, D, seed=1), b.adjacency_lists, b.type_to_num_incoming_edges


def qm9_graph(add_self_loop_edges=False, D=128):
    """BASELINE config 3: the REAL 10,000 QM9 validation molecules (structure from data/qm9/valid.jsonl.gz via
    tests/golden/make_qm9_structure.py), built like tasks/qm9_task.py:114-147."""
    struct = os.path.join(HERE, "qm9_valid_structure.npz")
    b, _, _ = batching.qm9_batch(batching.qm9_records_from_structure(struct), add_self_loop_edges=add_self_loop_edges)
    return node_states(b.num_nodes, D, seed=1), b.adjacency_lists, b.type_to_num_incoming_edges


def varmisuse_graph(packed_graphs=0, D=128):
    """BASELINE config 5: V = 50,000, M = 1,000,000, L = 6."""
    b = batching.varmisuse_like_batch(packed_graphs=packed_graphs)
    return node_states(b.num_nodes, D, seed=1), b.adjacency_lists, b.type_to_num_incoming_edges


D = D_SMALL
L = L_SMALL
CASES = {
    # ---- small graph: every layer family, the keyword arguments that change the op order ----
    "rgcn_tanh_t2": dict(kind="rgcn", graph=small_graph, indeg=True, weights=lambda: W.rgcn_weights(L, D, D),
                         kw=dict(state_dim=D, num_timesteps=2, activation_function="tanh")),
    "rgcn_both_max": dict(kind="rgcn", graph=small_graph, indeg=True,
                          weights=lambda: W.rgcn_weights(L, D, D, seed=5, use_both_source_and_target=True),
                          kw=dict(state_dim=D, activation_function="ReLU", message_aggregation_function="max",
                                  normalize_by_num_incoming=False, use_both_source_and_target=True)),
    "rgcn_mean_gelu": dict(kind="rgcn", graph=small_graph, indeg=True, weights=lambda: W.rgcn_weights(L, D, D, seed=7),
                           kw=dict(state_dim=D, activation_function="gelu", message_aggregation_function="mean")),
    "rgcn_sqrtn_selu": dict(kind="rgcn", graph=small_graph, indeg=True, weights=lambda: W.rgcn_weights(L, D, D, seed=9),
                            kw=dict(state_dim=D, activation_function="selu", message_aggregation_function="sqrt_n")),
    "ggnn_gru_t3": dict(kind="ggnn", graph=small_graph, indeg=False, weights=lambda: W.ggnn_weights(L, D, random_bias=True),
                        kw=dict(state_dim=D, num_timesteps=3, gated_unit_type="gru", activation_function="tanh")),
    "ggnn_rnn_t2": dict(kind="ggnn", graph=small_graph, indeg=False,
                        weights=lambda: W.ggnn_weights(L, D, seed=4, cell="rnn", random_bias=True),
                        kw=dict(state_dim=D, num_timesteps=2, gated_unit_type="RNN", activation_function="ReLU")),
    "rgat_k4_t2": dict(kind="rgat", graph=small_graph, indeg=False, weights=lambda: W.rgat_weights(L, D, D),
                       kw=dict(state_dim=D, num_timesteps=2, num_heads=4, activation_function="tanh")),
    "film_norm_t2": dict(kind="gnn-film", graph=small_graph, indeg=True,
                         weights=lambda: W.film_weights(L, D, D, num_timesteps=2, random_ln=True),
                         kw=dict(state_dim=D, num_timesteps=2, activation_function="ReLU", normalize_by_num_incoming=True)),
    "film_default": dict(kind="gnn-film", graph=small_graph, indeg=True, weights=lambda: W.film_weights(L, D, D, seed=6),
                         kw=dict(state_dim=D, activation_function="elu")),
    "edge_mlp_h0": dict(kind="gnn-edge-mlp", graph=small_graph, indeg=True,
                        weights=lambda: W.edge_mlp_weights(L, D, D, num_edge_hidden_layers=0, random_ln=True),
                        kw=dict(state_dim=D, activation_function="ReLU", num_edge_hidden_layers=0)),
    "edge_mlp_h1_gelu": dict(kind="gnn-edge-mlp", graph=small_graph, indeg=True,
                             weights=lambda: W.edge_mlp_weights(L, D, D, num_edge_hidden_layers=1, random_ln=True),
                             kw=dict(state_dim=D, activation_function="gelu", num_edge_hidden_layers=1)),
    "edge_mlp_h2_src_norm_t2": dict(kind="gnn-edge-mlp", graph=small_graph, indeg=True,
                                    weights=lambda: W.edge_mlp_weights(L, D, D, num_edge_hidden_layers=2,
                                                                       use_target_state_as_input=False, num_timesteps=2,
                                                                       random_ln=True),
                                    kw=dict(state_dim=D, num_timesteps=2, activation_function="tanh", num_edge_hidden_layers=2,
                                            use_target_state_as_input=False, normalize_by_num_incoming=True,
                                            message_aggregation_function="mean")),
    "rgin_default": dict(kind="rgin", graph=small_graph, indeg=False, weights=lambda: W.rgin_weights(L, D, D, random_ln=True),
                         kw=dict(state_dim=D, activation_function="ReLU")),
    "rgin_aggr1_t2": dict(kind="rgin", graph=small_graph, indeg=False,
                          weights=lambda: W.rgin_weights(L, D, D, num_aggr_MLP_hidden_layers=1, num_timesteps=2, random_ln=True),
                          kw=dict(state_dim=D, num_timesteps=2, activation_function="tanh", num_edge_MLP_hidden_layers=1,
                                  num_aggr_MLP_hidden_layers=1)),
    "rgin_target_noedge_aggr0": dict(kind="rgin", graph=small_graph, indeg=False,
                                     weights=lambda: W.rgin_weights(L, D, D, num_edge_MLP_hidden_layers=None,
                                                                    num_aggr_MLP_hidden_layers=0, use_target_state_as_input=True,
                                                                    random_ln=True),
                                     kw=dict(state_dim=D, activation_function="ReLU", use_target_state_as_input=True,
                                             num_edge_MLP_hidden_layers=None, num_aggr_MLP_hidden_layers=0)),
    "rgdcn_t2": dict(kind="rgdcn", graph=small_graph, indeg=True, weights=lambda: W.rgdcn_weights(L, 4, 8, stddev=0.15),
                     kw=dict(num_channels=4, channel_dim=8, num_timesteps=2, activation_function="tanh")),
    "rgdcn_full_tied": dict(kind="rgdcn", graph=small_graph, indeg=True,
                            weights=lambda: W.rgdcn_weights(L, 4, 8, use_full_state=True, tie_channel_weights=True, stddev=0.15),
                            kw=dict(num_channels=4, channel_dim=8, use_full_state_for_channel_weights=True,
                                    tie_channel_weights=True, activation_function="ReLU",
                                    message_aggregation_function="mean")),
    # ---- BASELINE.json configs (SURVEY.md 8d) ----
    "config2_rgcn_ppi": dict(kind="rgcn", graph=ppi_graph, indeg=True, big=True, weights=lambda: W.rgcn_weights(3, 256, 256),
                             kw=dict(state_dim=256, activation_function="ReLU", message_aggregation_function="sum")),
    "config3_ggnn_qm9": dict(kind="ggnn", graph=qm9_graph, indeg=False, big=True, weights=lambda: W.ggnn_weights(4, 128),
                             kw=dict(state_dim=128, num_timesteps=4, gated_unit_type="gru", activation_function="tanh")),
    "config3_ggnn_qm9_selfloops": dict(kind="ggnn", graph=lambda: qm9_graph(add_self_loop_edges=True), indeg=False, big=True,
                                       weights=lambda: W.ggnn_weights(5, 128),
                                       kw=dict(state_dim=128, num_timesteps=4, gated_unit_type="gru", activation_function="tanh")),
    "config4_rgat_ppi": dict(kind="rgat", graph=ppi_graph, indeg=False, big=True, weights=lambda: W.rgat_weights(3, 256, 256),
                             kw=dict(state_dim=256, num_heads=8, activation_function="tanh")),
    "config5_film_random": dict(kind="gnn-film", graph=varmisuse_graph, indeg=True, big=True,
                                weights=lambda: W.film_weights(6, 128, 128),
                                kw=dict(state_dim=128, activation_function="ReLU", normalize_by_num_incoming=False)),
    "config5_film_packed": dict(kind="gnn-film", graph=lambda: varmisuse_graph(packed_graphs=25), indeg=True, big=True,
                                weights=lambda: W.film_weights(6, 128, 128),
                                kw=dict(state_dim=128, activation_function="ReLU", normalize_by_num_incoming=False)),
    "ppi_edge_mlp1": dict(kind="gnn-edge-mlp", graph=ppi_graph, indeg=True, big=True,
                          weights=lambda: W.edge_mlp_weights(3, 256, 256, num_edge_hidden_layers=1),
                          kw=dict(state_dim=256, activation_function="gelu", num_edge_hidden_layers=1)),
    "ppi_rgin": dict(kind="rgin", graph=ppi_graph, indeg=False, big=True, weights=lambda: W.rgin_weights(3, 256, 256),
                     kw=dict(state_dim=256, activation_function="ReLU")),
}

REFERENCE_FUNCTIONS = {"rgcn": "sparse_rgcn_layer", "ggnn": "sparse_ggnn_layer", "rgat": "sparse_rgat_layer",
                       "gnn-film": "sparse_gnn_film_layer", "gnn-edge-mlp": "sparse_gnn_edge_mlp_layer",
                       "rgin": "sparse_rgin_layer", "rgdcn": "sparse_rgdcn_layer"}
BIG_ROW_STRIDE = 97          # every 97th output row is committed for the big cases
PROJECTION_SEED = 12345


def fixture_path(name):
    return os.path.join(HERE, "ref_%s.npz" % name)


def cell_kind(case):
    return "rnn" if case["kw"].get("gated_unit_type", "gru").lower() == "rnn" else "gru"


def projection_vector(dim):
    return np.random.default_rng(PROJECTION_SEED).standard_normal(dim)


MAX_SUMMARY_ROWS = 256     # keeps every committed file under 1 MB: larger outputs commit every k-th of the stride-97 rows
PROJ_BLOCK_ABOVE = 20000   # ... and, above this many rows, the projection summed over blocks of PROJ_BLOCK rows
PROJ_BLOCK = 16


def summarize(out64):
    """What a big case commits of a [V, D] float64 output."""
    out64 = np.asarray(out64, np.float64)
    return compact_summary({"rows": np.arange(0, out64.shape[0], BIG_ROW_STRIDE), "out_rows": out64[::BIG_ROW_STRIDE].copy(),
                            "proj": out64 @ projection_vector(out64.shape[1]), "colsum": out64.sum(axis=0),
                            "maxabs": np.float64(np.abs(out64).max()), "shape": np.asarray(out64.shape)})


def compact_summary(blob):
    """Thin the committed rows to at most MAX_SUMMARY_ROWS and block-sum the projection of large outputs (out32_rows, when
    present, follows the rows)."""
    blob = dict(blob)
    k = -(-len(blob["rows"]) // MAX_SUMMARY_ROWS)
    for key in ("rows", "out_rows", "out32_rows"):
        if key in blob:
            blob[key] = np.ascontiguousarray(blob[key][::k])
    if int(blob["shape"][0]) > PROJ_BLOCK_ABOVE and "proj_block" not in blob:
        blob["proj"] = np.add.reduceat(blob["proj"], np.arange(0, len(blob["proj"]), PROJ_BLOCK))
        blob["proj_block"] = np.int64(PROJ_BLOCK)
    return blob


def compare_with_summary(got, z, what=""):
    """Errors of a full [V, D] result against a committed big-case summary, each normalised so that an element-wise max-norm
    relative error of eps implies a value <= eps: the committed rows directly; the projection by maxabs * sum|r| and the
    column sums by maxabs * V (|sum_j e_j r_j| <= max|e| * sum|r_j|; a sum of V errors is at most V * max|e|).  The rows
    bound the error itself, the two sums make sure NO row outside the committed sample is badly off (an outlier of size x in
    an uncommitted row moves the projection by ~x)."""
    got = np.asarray(got, np.float64)
    assert tuple(got.shape) == tuple(int(x) for x in z["shape"]), "%s: shape %s vs %s" % (what, got.shape, z["shape"])
    scale = float(z["maxabs"])
    r = projection_vector(got.shape[1])
    err_rows = float(np.abs(got[z["rows"]] - z["out_rows"]).max() / scale)
    proj, block = got @ r, int(z["proj_block"]) if "proj_block" in z else 1
    if block > 1:                                          # a sum of `block` row projections: error bound grows by `block`
        proj = np.add.reduceat(proj, np.arange(0, len(proj), block))
    err_proj = float(np.abs(proj - z["proj"]).max() / (scale * np.abs(r).sum() * block))
    err_col = float(np.abs(got.sum(axis=0) - z["colsum"]).max() / (scale * got.shape[0]))
    return err_rows, err_proj, err_col

"""utils/utils.py's name factories (get_activation, get_aggregation_function, get_gated_unit) and utils/model_utils.py's
name_to_model_class: the names accepted, the exception types and messages raised -- what the REFERENCE's functions did (run
under tests/tf1_shim and recorded in tests/golden/ref_utils_outcomes.json by make_utils_fixtures.py) against the package's."""
import importlib
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

mine = importlib.import_module("tf_gnn_samples_b200.utils")
scaffold = importlib.import_module("tf_gnn_samples_b200.scaffold")

ACTIVATION_NAMES = [None, "linear", "Linear", "tanh", "TANH", "relu", "ReLU", "leaky_relu", "Leaky_ReLU", "elu", "ELU", "selu", "gelu",
                    "GeLU", "sigmoid", "swish", "", "relu ", "leaky-relu"]
AGGREGATION_NAMES = ["sum", "max", "mean", "sqrt_n", "unsorted_segment_sum", "unsorted_segment_max", "unsorted_segment_mean",
                     "unsorted_segment_sqrt_n", "Sum", "MAX", "avg", "", None, "sqrt-n"]
CELL_NAMES = ["rnn", "RNN", "gru", "GRU", "Gru", "lstm", "cnn", ""]
MODEL_NAMES = ["ggnn", "GGNN", "ggnn_model", "gnn_edge_mlp", "gnn-edge-mlp", "GNN-Edge-MLP", "gnn_edge_mlp_model", "gnn_edge_mlp0",
               "gnn-edge-mlp0", "gnn_edge_mlp1", "GNN-Edge-MLP1", "gnn_film", "gnn-film", "GNN-FiLM", "gnn_film_model", "rgat",
               "rgat_model", "rgcn", "RGCN", "rgcn_model", "rgdcn", "rgdcn_model", "rgin", "RGIN", "rgin_model", "gcn", "gat", ""]


def outcome(fn, *args):
    try:
        return ("ok", fn(*args))
    except Exception as e:                                   # noqa: BLE001 -- the exception IS the behaviour under test
        return (type(e).__name__, str(e))


@pytest.fixture(scope="module")
def reference():
    with open(os.path.join(HERE, "golden", "ref_utils_outcomes.json")) as f:
        return json.load(f)


def test_activation_names_and_errors(reference):
    import tf1_shim
    x = np.linspace(-3, 3, 25)
    with tf1_shim.installed(dtype=np.float64) as session:
        tf = session.tf
        values = {mine.ACT_LINEAR: lambda v: v, mine.ACT_TANH: np.tanh, mine.ACT_RELU: lambda v: np.maximum(v, 0),
                  mine.ACT_LEAKY_RELU: lambda v: np.where(v > 0, v, 0.2 * v), mine.ACT_ELU: tf.nn.elu, mine.ACT_SELU: tf.nn.selu,
                  mine.ACT_GELU: lambda v: v * 0.5 * (1.0 + tf.erf(v / np.sqrt(2.0)))}
        for name in ACTIVATION_NAMES:
            ref, got = reference["activations"][repr(name)], outcome(mine.get_activation, name)
            if ref[0] != "ok":
                assert list(got) == ref, (name, got, ref)         # same exception type, same message
                continue
            assert got[0] == "ok", (name, got)
            want = x if ref[1] is None else np.asarray(ref[1])   # None = no activation (rgcn.py:112 etc. guard on it)
            assert np.allclose(values[got[1]](x), want, rtol=0, atol=1e-15), name


def test_aggregation_names_and_errors(reference):
    codes = {mine.AGG_SUM: "sum", mine.AGG_MAX: "max", mine.AGG_MEAN: "mean", mine.AGG_SQRT_N: "sqrt_n"}
    for name in AGGREGATION_NAMES:
        ref, got = reference["aggregations"][repr(name)], outcome(mine.get_aggregation_function, name)
        if ref[0] != "ok":
            assert list(got) == ref, (name, got, ref)
        else:
            assert got[0] == "ok" and codes[got[1]] == ref[1], (name, got, ref)


def test_gated_unit_names_and_errors(reference):
    for name in CELL_NAMES:
        ref, got = reference["cells"][name], outcome(mine.get_gated_unit, 8, name, "tanh")
        if name.lower() == "lstm":                            # constructs in the reference, cannot be CALLED there (ggnn.py:92)
            assert ref == ["ok", "_LSTMCell", "ValueError"] and got[0] == "NotImplementedError"
            continue
        if ref[0] != "ok":
            assert list(got) == ref, (name, got, ref)
        else:
            cell = {"_SimpleRNNCell": mine.CELL_RNN, "_GRUCell": mine.CELL_GRU}[ref[1]]
            assert got == ("ok", (cell, mine.ACT_TANH)), (name, got)
    assert list(outcome(mine.get_gated_unit, 8, "gru", "swish")) == reference["cell_swish"]


def test_model_names_resolve_like_name_to_model_class(reference):
    import test_reference_model_pin as P
    kinds = {v: k for k, v in P.MC.MODEL_CLASSES.items()}
    for name in MODEL_NAMES:
        ref, got = reference["models"][name], outcome(scaffold.model_default_params, name)
        if ref[0] != "ok":
            assert list(got) == ref, (name, got, ref)
            continue
        cls_name, want = ref[1], ref[2]
        assert got[0] == "ok", (name, got)
        for k, v in got[1].items():
            assert want[k] == v, (name, k, want[k], v)
        assert scaffold.resolve_model_name(name)[0] == kinds[cls_name], name


def test_layer_function_signatures_equal_the_references(reference):
    """gnns/__init__.py exports seven sparse_<x>_layer functions; the package's take the same positional / keyword parameters in
    the same order with the same defaults, plus keyword-only extras (weights=, plan=, ...) that the reference cannot know."""
    import inspect
    pkg = importlib.import_module("tf_gnn_samples_b200.gnns")
    names = sorted(reference["signatures"])
    assert names == ["sparse_ggnn_layer", "sparse_gnn_edge_mlp_layer", "sparse_gnn_film_layer", "sparse_rgat_layer",
                     "sparse_rgcn_layer", "sparse_rgdcn_layer", "sparse_rgin_layer"]
    for n in names:
        ref = reference["signatures"][n]
        got = inspect.signature(getattr(pkg, n)).parameters
        shared = [p for p in got.values() if p.kind != inspect.Parameter.KEYWORD_ONLY]
        assert [p.name for p in shared] == [r[0] for r in ref], (n, [p.name for p in shared], ref)
        for p, (_, default) in zip(shared, ref):
            assert repr(p.default) == default, (n, p.name, p.default, default)
        extras = [p.name for p in got.values() if p.kind == inspect.Parameter.KEYWORD_ONLY]
        assert "weights" in extras, (n, extras)
